// Emulation-build stand-ins for the entry points whose kernels are wgmma / TMA code (hardware only): the SAME argument contract
// (shape / alignment checks copied from the real wrappers) over a plain host loop, so that the layers above them -- the op-program
// interpreter of serving_runtime.cu, the engines' launch sequences -- run end to end on the CPU emulation.  Never part of libdeeprec_cuda.so.
#ifndef DR_CUDA_EMU
#error "emulation build only"
#endif
#include "../common.cuh"

namespace {
inline float bf(const __nv_bfloat16* p) { return __bfloat162float(*p); }
}

extern "C" {

// gemm_wgmma.cu::dr_cuda_gemm_tn_ex: out[M,N] = A[M,K](lda) * B[N,K](ldb)^T (+bias)(relu)(*mask); bf16 in / out, fp32 accumulate
int dr_cuda_gemm_tn_ex(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, const float* bias, int relu, const void* mask_src,
                       int64_t ld_mask, int aux_mode, void* out, int64_t ldc, float* out_f32, float* S1, float* S2, int max_ctas, int force_v1, cudaStream_t) {
  (void)max_ctas; (void)force_v1;
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if ((lda % 8) || (ldb % 8) || (ldc % 8) || (N % 8)) return -2;
  if (((uintptr_t)A | (uintptr_t)B | (uintptr_t)out) & 15) return -3;                 // TMA: 16-byte aligned global addresses
  if (lda < K || ldb < K || ldc < N) return -5;
  const bool v2 = !force_v1 && N > 32 && out_f32 == nullptr;
  if (!v2 && (S1 || S2 || aux_mode == 2)) return -4;
  const __nv_bfloat16* a = (const __nv_bfloat16*)A; const __nv_bfloat16* b = (const __nv_bfloat16*)B;
  const __nv_bfloat16* mk = (const __nv_bfloat16*)mask_src;
  __nv_bfloat16* o = (__nv_bfloat16*)out;
  for (int m = 0; m < M; ++m)
    for (int n = 0; n < N; ++n) {
      float acc = 0.f;
      for (int k = 0; k < K; ++k) acc += bf(a + (int64_t)m * lda + k) * bf(b + (int64_t)n * ldb + k);
      if (bias) acc += bias[n];
      if (relu && acc < 0.f) acc = 0.f;
      if (mk && aux_mode == 1 && !(bf(mk + (int64_t)m * ld_mask + n) > 0.f)) acc = 0.f;
      const __nv_bfloat16 r = __float2bfloat16(acc);
      if (o) o[(int64_t)m * ldc + n] = r;
      if (out_f32) out_f32[(int64_t)m * N + n] = acc;
      if (S1) { const float v = __bfloat162float(r); S1[n] += v; if (S2) S2[n] += v * v; }
    }
  return 0;
}

int dr_cuda_gemm_tn(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, const float* bias, int relu, const void* mask_src, int64_t ld_mask,
                    void* out, int64_t ldc, float* out_f32, int max_ctas, cudaStream_t s) {
  return dr_cuda_gemm_tn_ex(A, lda, B, ldb, M, N, K, bias, relu, mask_src, ld_mask, mask_src ? 1 : 0, out, ldc, out_f32, nullptr, nullptr, max_ctas, 0, s);
}

// gemm_wgmma.cu::dr_cuda_gemm_dw: dW[N_out,K_in](ldw, fp32, accumulated into) += dY[batch,N_out](ldy)^T * X[batch,K_in](ldx)
int dr_cuda_gemm_dw(const void* dY, int64_t ldy, const void* X, int64_t ldx, int batch, int N_out, int K_in, float* dW, int64_t ldw, int splits, cudaStream_t) {
  (void)splits;
  if (batch <= 0 || N_out <= 0 || K_in <= 0) return 0;
  if ((ldy % 8) || (ldx % 8)) return -2;
  if (((uintptr_t)dY | (uintptr_t)X) & 15) return -3;
  const __nv_bfloat16* y = (const __nv_bfloat16*)dY; const __nv_bfloat16* x = (const __nv_bfloat16*)X;
  for (int n = 0; n < N_out; ++n)
    for (int k = 0; k < K_in; ++k) {
      float acc = 0.f;
      for (int b = 0; b < batch; ++b) acc += bf(y + (int64_t)b * ldy + n) * bf(x + (int64_t)b * ldx + k);
      dW[(int64_t)n * ldw + k] += acc;
    }
  return 0;
}

// gemm_fp8.cu: the fp8 serving path is not emulated (ModelConfig {"fp8": true} fails to initialise on the emulation, loudly)
int dr_cuda_gemm_fp8_tn(const void*, int64_t, const void*, int64_t, int, int, int, const float*, const float*, int, void*, int64_t, int, float, cudaStream_t) { return -100; }
int dr_cuda_quantize_e4m3(const void*, int, int64_t, int, int64_t, void*, int, float, cudaStream_t) { return -100; }
int dr_cuda_quantize_weights_e4m3(const float*, int, int, int64_t, void*, int, float*, cudaStream_t) { return -100; }
int dr_cuda_absmax_bf16(const void*, int64_t, float*, cudaStream_t) { return -100; }

int64_t dr_cuda_emu_launch_count() { return emu::launch_count().load(); }

}  // extern "C"
