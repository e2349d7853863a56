// MXFP8 (block-scaled fp8) quantiser: E4M3 elements with one UE8M0 power-of-two scale per 32 elements along K.  The block-scaled GEMM
// that consumes its output is dr_cuda_gemm_mxfp8_tn (gemm_wgmma.cu: one m64nNk32 wgmma per scale block, scales applied in registers).
#include "common.cuh"

using namespace drc;

namespace {

// ---------------------------------------------------------------------------------------------------------------------------
// Quantiser: x [R, C] (fp32 or bf16, row pitch ldx) -> q [R, Kp] E4M3 (Kp = C rounded up to 128, zero padded) + scale words.
// One warp per (row, 128-wide k block): lane l holds elements 4l .. 4l+3; the 8 lanes of one 32-element scale block reduce their
// abs-max by shuffles; scale = 2^e with e = ceil(log2(amax / 448)) clamped to >= -126 (UE8M0 byte e + 127), q = rn_e4m3(x * 2^-e).
// Scale word of row r, k block kb:  sf[((r / 128) * num_kb + kb) * 128 + (r % 32) * 4 + (r % 128) / 32], byte j = sub-block j.
// Rows R .. 128 * ceil(R / 128) - 1 are never written: the caller zero-fills sf (their operand rows are TMA zero fill).
// ---------------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_e4m3x4_x(float a, float b, float c, float d) {
  uint16_t lo, hi;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(b), "f"(a));
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(d), "f"(c));
  return (uint32_t)lo | ((uint32_t)hi << 16);
}

template <typename T>
__global__ void k_quantize_mxfp8(const T* __restrict__ x, int64_t R, int C, int64_t ldx, uint8_t* __restrict__ q, int Kp, uint32_t* __restrict__ sf) {
  const int num_kb = Kp / 128;
  const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= R * num_kb) return;
  const int64_t r = w / num_kb;
  const int kb = (int)(w % num_kb);
  const int c0 = kb * 128 + lane * 4;
  float v[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) v[j] = (c0 + j < C) ? (float)x[r * ldx + c0 + j] : 0.f;
  float a = fmaxf(fmaxf(fabsf(v[0]), fabsf(v[1])), fmaxf(fabsf(v[2]), fabsf(v[3])));
  a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, 1));
  a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, 2));
  a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, 4));
  const uint32_t bits = __float_as_uint(a * (1.0f / 448.0f));
  int e = (int)((bits >> 23) & 0xffu) - 127 + ((bits & 0x7fffffu) ? 1 : 0);
  e = e < -126 ? -126 : (e > 127 ? 127 : e);
  const float inv = __uint_as_float((uint32_t)(127 - e) << 23);          // 2^-e, exact (e in [-126, 127] -> biased exponent in [0, 253])
  const float inv_s = e == 127 ? 5.877471754111438e-39f : inv;           // 2^-127 is a denormal: not expressible by the exponent field alone
  *reinterpret_cast<uint32_t*>(q + r * (int64_t)Kp + c0) = pack_e4m3x4_x(v[0] * inv_s, v[1] * inv_s, v[2] * inv_s, v[3] * inv_s);
  const uint32_t byte = (uint32_t)(e + 127);
  const uint32_t b0 = __shfl_sync(0xffffffffu, byte, 0), b1 = __shfl_sync(0xffffffffu, byte, 8), b2 = __shfl_sync(0xffffffffu, byte, 16),
                 b3 = __shfl_sync(0xffffffffu, byte, 24);
  if (lane == 0) sf[((r >> 7) * num_kb + kb) * 128 + (r & 31) * 4 + ((r & 127) >> 5)] = b0 | (b1 << 8) | (b2 << 16) | (b3 << 24);
}


}  // namespace

extern "C" {

// q [R, Kp] e4m3 + sf [ceil(R / 128) * (Kp / 128) * 128] uint32 (zero-filled by the caller) from x [R, C]; Kp % 128 == 0, Kp >= C.
int dr_cuda_quantize_mxfp8(const void* x, int is_bf16, int64_t R, int C, int64_t ldx, void* q, int Kp, void* sf, cudaStream_t s) {
  if (R <= 0) return 0;
  if (Kp % 128 || Kp < C) return -2;
  const int64_t warps = R * (Kp / 128);
  const int64_t blocks = (warps * 32 + 255) / 256;
  if (blocks > 0x7fffffff) return -3;
  if (is_bf16)
    k_quantize_mxfp8<__nv_bfloat16><<<(unsigned)blocks, 256, 0, s>>>((const __nv_bfloat16*)x, R, C, ldx, (uint8_t*)q, Kp, (uint32_t*)sf);
  else
    k_quantize_mxfp8<float><<<(unsigned)blocks, 256, 0, s>>>((const float*)x, R, C, ldx, (uint8_t*)q, Kp, (uint32_t*)sf);
  DR_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
