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

// gemm_wgmma.cu::dr_cuda_gemm_tn_ex: out[M,N] = A[M,K](lda) * B[N,K](ldb)^T (+bias)(relu)(*mask); bf16 in / out, fp32 accumulate.
// Same return codes, out_f32 pitch (ldc) and statistics (fp32 epilogue values before the bf16 rounding) as the hardware entry.
int dr_cuda_gemm_tn_ex(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, const float* bias, int relu, const void* mask_src,
                       int64_t ld_mask, int aux_mode, void* out, int64_t ldc, float* out_f32, float* S1, float* S2, int max_ctas, int force_v1, cudaStream_t) {
  (void)max_ctas; (void)force_v1;
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if ((lda % 8) || (ldb % 8) || (ldc % 8) || (N % 8)) return -2;
  if (((uintptr_t)A | (uintptr_t)B | (uintptr_t)out) & 15) return -3;                 // TMA: 16-byte aligned global addresses
  if (lda < K || ldb < K || ldc < N) return -5;
  if ((S2 && !S1) || (aux_mode == 2 && !mask_src)) return -4;
  const __nv_bfloat16* a = (const __nv_bfloat16*)A; const __nv_bfloat16* b = (const __nv_bfloat16*)B;
  const __nv_bfloat16* mk = (const __nv_bfloat16*)mask_src;
  __nv_bfloat16* o = (__nv_bfloat16*)out;
  for (int m = 0; m < M; ++m)
    for (int n = 0; n < N; ++n) {
      float acc = 0.f;
      for (int k = 0; k < K; ++k) acc += bf(a + (int64_t)m * lda + k) * bf(b + (int64_t)n * ldb + k);
      if (bias) acc += bias[n];
      if (relu && acc < 0.f) acc = 0.f;
      const float w = mk ? bf(mk + (int64_t)m * ld_mask + n) : 0.f;
      if (mk && aux_mode == 1 && !(w > 0.f)) acc = 0.f;
      if (o) o[(int64_t)m * ldc + n] = __float2bfloat16(acc);
      if (out_f32) out_f32[(int64_t)m * ldc + n] = acc;
      if (S1) { S1[n] += acc; if (S2) S2[n] += acc * (aux_mode == 2 ? w : acc); }
    }
  return 0;
}

int dr_cuda_gemm_tn(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, const float* bias, int relu, const void* mask_src, int64_t ld_mask,
                    void* out, int64_t ldc, float* out_f32, int max_ctas, cudaStream_t s) {
  return dr_cuda_gemm_tn_ex(A, lda, B, ldb, M, N, K, bias, relu, mask_src, ld_mask, mask_src ? 1 : 0, out, ldc, out_f32, nullptr, nullptr, max_ctas, 0, s);
}

// gemm_wgmma.cu::dr_cuda_gemm_tn_cross: kind 1 out = x0 * (acc + bias) + xl (u_out = acc + bias), kind 2 out = acc + xl; same return codes.
int dr_cuda_gemm_tn_cross(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, const float* bias, int kind, const void* x0,
                          int64_t ld_x0, const void* xl, int64_t ld_xl, void* out, int64_t ldc, void* u_out, int64_t ld_u, int max_ctas, cudaStream_t) {
  (void)max_ctas;
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if ((kind != 1 && kind != 2) || !xl || (kind == 1 && !x0)) return -4;
  if (kind != 1) { x0 = nullptr; u_out = nullptr; }
  if ((lda % 8) || (ldb % 8) || (ldc % 8) || (N % 8) || (ld_xl % 8) || (x0 && ld_x0 % 8) || (u_out && ld_u % 8)) return -2;
  if (((uintptr_t)A | (uintptr_t)B | (uintptr_t)out | (uintptr_t)xl | (uintptr_t)x0 | (uintptr_t)u_out) & 15) return -3;
  if (lda < K || ldb < K || ldc < N || ld_xl < N || (x0 && ld_x0 < N) || (u_out && ld_u < N)) return -5;
  const __nv_bfloat16* a = (const __nv_bfloat16*)A; const __nv_bfloat16* b = (const __nv_bfloat16*)B;
  const __nv_bfloat16* xz = (const __nv_bfloat16*)x0; const __nv_bfloat16* xa = (const __nv_bfloat16*)xl;
  __nv_bfloat16* o = (__nv_bfloat16*)out; __nv_bfloat16* uo = (__nv_bfloat16*)u_out;
  for (int m = 0; m < M; ++m)
    for (int n = 0; n < N; ++n) {
      float acc = 0.f;
      for (int k = 0; k < K; ++k) acc += bf(a + (int64_t)m * lda + k) * bf(b + (int64_t)n * ldb + k);
      if (bias) acc += bias[n];
      const float w = bf(xa + (int64_t)m * ld_xl + n);
      if (kind == 1) {
        if (uo) uo[(int64_t)m * ld_u + n] = __float2bfloat16(acc);
        acc = fmaf(bf(xz + (int64_t)m * ld_x0 + n), acc, w);
      } else {
        acc += w;
      }
      o[(int64_t)m * ldc + n] = __float2bfloat16(acc);
    }
  return 0;
}

// gemm_wgmma.cu::dr_cuda_gemm_tn_ln: h = acc (+ bias), out = relu?(gamma * x^ + beta), x^ = (h - mean) * rstd over each row's N columns
// (two-pass variance), x^ (bf16) and rstd (fp32) optional; same return codes.
int dr_cuda_gemm_tn_ln(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, const float* bias, const float* gamma,
                       const float* beta, float eps, int relu, void* out, int64_t ldc, void* xhat, int64_t ld_xhat, float* rstd, int max_ctas,
                       cudaStream_t) {
  (void)max_ctas;
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if (!gamma || !beta) return -4;
  if ((lda % 8) || (ldb % 8) || (ldc % 8) || (N % 8) || N > 128 || (xhat && ld_xhat % 8)) return -2;
  if (((uintptr_t)A | (uintptr_t)B | (uintptr_t)out | (uintptr_t)xhat) & 15) return -3;
  if (lda < K || ldb < K || ldc < N || (xhat && ld_xhat < N)) return -5;
  const __nv_bfloat16* a = (const __nv_bfloat16*)A; const __nv_bfloat16* b = (const __nv_bfloat16*)B;
  __nv_bfloat16* o = (__nv_bfloat16*)out; __nv_bfloat16* xo = (__nv_bfloat16*)xhat;
  float h[128];
  for (int m = 0; m < M; ++m) {
    float sum = 0.f, sq = 0.f;
    for (int n = 0; n < N; ++n) {
      float acc = 0.f;
      for (int k = 0; k < K; ++k) acc += bf(a + (int64_t)m * lda + k) * bf(b + (int64_t)n * ldb + k);
      h[n] = acc + (bias ? bias[n] : 0.f);
      sum += h[n];
    }
    const float mu = sum / (float)N;
    for (int n = 0; n < N; ++n) sq += (h[n] - mu) * (h[n] - mu);
    const float rs = 1.f / sqrtf(sq / (float)N + eps);
    if (rstd) rstd[m] = rs;
    for (int n = 0; n < N; ++n) {
      const float x = (h[n] - mu) * rs;
      float y = gamma[n] * x + beta[n];
      if (relu && y < 0.f) y = 0.f;
      o[(int64_t)m * ldc + n] = __float2bfloat16(y);
      if (xo) xo[(int64_t)m * ld_xhat + n] = __float2bfloat16(x);
    }
  }
  return 0;
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

// gemm_wgmma.cu::dr_cuda_gemm_tn_grouped / dr_cuda_gemm_dw_grouped: every group checked first (same codes, kMaxGroups = 12), then the
// per-group entries above, so each group's result is the one its own call gives.
int dr_cuda_gemm_tn_grouped(int G, const void* const* A, const int64_t* lda, const void* const* B, const int64_t* ldb, int M, int N, int K,
                            const float* const* bias, int relu, const void* const* mask_src, const int64_t* ld_mask, void* const* out,
                            const int64_t* ldc, float* const* S1, int max_ctas, cudaStream_t s) {
  if (G < 1 || G > 12) return -6;
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  for (int g = 0; g < G; ++g) {
    if ((lda[g] % 8) || (ldb[g] % 8) || (ldc[g] % 8) || (N % 8)) return -2;
    if (((uintptr_t)A[g] | (uintptr_t)B[g] | (uintptr_t)out[g]) & 15) return -3;
    if (lda[g] < K || ldb[g] < K || ldc[g] < N) return -5;
    if (S1 && !S1[g]) return -4;
  }
  for (int g = 0; g < G; ++g) {
    const void* mk = mask_src ? mask_src[g] : nullptr;
    const int rc = dr_cuda_gemm_tn_ex(A[g], lda[g], B[g], ldb[g], M, N, K, bias ? bias[g] : nullptr, relu, mk, mk ? ld_mask[g] : 0, mk ? 1 : 0, out[g],
                                      ldc[g], nullptr, S1 ? S1[g] : nullptr, nullptr, max_ctas, 0, s);
    if (rc) return rc;
  }
  return 0;
}

int dr_cuda_gemm_dw_grouped(int G, const void* const* dY, const int64_t* ldy, const void* const* X, const int64_t* ldx, int batch, int N_out,
                            int K_in, float* const* dW, const int64_t* ldw, int splits, cudaStream_t s) {
  if (G < 1 || G > 12) return -6;
  if (batch <= 0 || N_out <= 0 || K_in <= 0) return 0;
  for (int g = 0; g < G; ++g) {
    if ((ldy[g] % 8) || (ldx[g] % 8)) return -2;
    if (((uintptr_t)dY[g] | (uintptr_t)X[g]) & 15) return -3;
  }
  for (int g = 0; g < G; ++g) {
    const int rc = dr_cuda_gemm_dw(dY[g], ldy[g], X[g], ldx[g], batch, N_out, K_in, dW[g], ldw[g], splits, s);
    if (rc) return rc;
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
