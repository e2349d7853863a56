// FP8 (E4M3) quantisation kernels of the serving MLP: activations per tensor (static scale from calibration), weights per output
// channel, and the abs-max used to calibrate.  The FP8 GEMM that consumes them is dr_cuda_gemm_fp8_tn (gemm_wgmma.cu).
//
// SURVEY §2.9 "tools/low_precision_optimize" (BF16/FP16/INT8 model quantisation incl. EV) is the reference's low-precision
// story -- a graph rewrite that calls library kernels; BASELINE config 5 asks for an fp8 MLP in SessionGroup inference.
#include <cuda_fp8.h>

#include "common.cuh"

using namespace drc;

namespace {

// 4 floats -> 4 packed E4M3 bytes (round-to-nearest, saturate to +-448)
__device__ __forceinline__ uint32_t pack_e4m3x4(float a, float b, float c, float d) {
  uint16_t lo, hi;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(b), "f"(a));
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(d), "f"(c));
  return (uint32_t)lo | ((uint32_t)hi << 16);
}

// x [M, C] (fp32 or bf16) * inv_scale -> e4m3 [M, Cp] (zero padded columns), 16 outputs per thread
template <typename T>
__global__ void k_quantize_e4m3(const T* __restrict__ x, int64_t M, int C, int64_t ldx, uint8_t* __restrict__ y, int Cp, float inv_scale) {
  const int chunks = Cp / 16;
  const int64_t total = M * chunks;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t m = i / chunks; const int c0 = (int)(i % chunks) * 16;
    float v[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = (c0 + j < C) ? (float)x[m * ldx + c0 + j] * inv_scale : 0.f;
    int4 pk;
    pk.x = (int)pack_e4m3x4(v[0], v[1], v[2], v[3]); pk.y = (int)pack_e4m3x4(v[4], v[5], v[6], v[7]);
    pk.z = (int)pack_e4m3x4(v[8], v[9], v[10], v[11]); pk.w = (int)pack_e4m3x4(v[12], v[13], v[14], v[15]);
    *reinterpret_cast<int4*>(y + m * Cp + c0) = pk;
  }
}

// per-row (= per output channel) abs-max of W [N, K] and quantisation to e4m3 [N, Kp]; one warp per row
__global__ void k_quantize_weights_e4m3(const float* __restrict__ w, int N, int K, int64_t ldw, uint8_t* __restrict__ q, int Kp, float* __restrict__ scale) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= N) return;
  float mx = 0.f;
  for (int k = lane; k < K; k += 32) mx = fmaxf(mx, fabsf(w[row * ldw + k]));
#pragma unroll
  for (int off = 16; off; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
  const float sc = mx > 0.f ? mx / 448.f : 1.f;
  if (lane == 0) scale[row] = sc;
  const float inv = 1.f / sc;
  for (int k = lane; k < Kp; k += 32) {
    const float v = k < K ? w[row * ldw + k] * inv : 0.f;
    __nv_fp8_e4m3 f(v);
    q[(int64_t)row * Kp + k] = *reinterpret_cast<uint8_t*>(&f);
  }
}

__global__ void k_absmax(const __nv_bfloat16* __restrict__ x, int64_t n, float* __restrict__ out) {
  float mx = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) mx = fmaxf(mx, fabsf(__bfloat162float(x[i])));
#pragma unroll
  for (int off = 16; off; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
  if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int*>(out), __float_as_int(mx));     // non-negative floats order like ints
}

}  // namespace

extern "C" {

int dr_cuda_quantize_e4m3(const void* x, int is_bf16, int64_t M, int C, int64_t ldx, void* y, int Cp, float inv_scale, cudaStream_t s) {
  if (Cp % 16) return -2;
  const int64_t total = M * (Cp / 16);
  int grid = (int)((total + 255) / 256); if (grid < 1) grid = 1; if (grid > num_sms() * 8) grid = num_sms() * 8;
  if (is_bf16) k_quantize_e4m3<__nv_bfloat16><<<grid, 256, 0, s>>>((const __nv_bfloat16*)x, M, C, ldx, (uint8_t*)y, Cp, inv_scale);
  else k_quantize_e4m3<float><<<grid, 256, 0, s>>>((const float*)x, M, C, ldx, (uint8_t*)y, Cp, inv_scale);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_quantize_weights_e4m3(const float* w, int N, int K, int64_t ldw, void* q, int Kp, float* scale, cudaStream_t s) {
  if (Kp % 16) return -2;
  k_quantize_weights_e4m3<<<(N + 7) / 8, 256, 0, s>>>(w, N, K, ldw, (uint8_t*)q, Kp, scale);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_absmax_bf16(const void* x, int64_t n, float* out, cudaStream_t s) {
  DR_CUDA_CHECK(cudaMemsetAsync(out, 0, 4, s));
  int grid = (int)((n + 255) / 256); if (grid < 1) grid = 1; if (grid > num_sms() * 4) grid = num_sms() * 4;
  k_absmax<<<grid, 256, 0, s>>>((const __nv_bfloat16*)x, n, out);
  DR_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
