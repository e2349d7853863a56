// Fused element/row-wise ops: LayerNorm, L2-normalize, GELU, Dice (reference: kernels/fused_layer_norm/, kernels/fused_l2_normalize/,
// kernels/gelu_op_gpu.cu.cc, grappler/optimizers/dice_fusion.cc -- AVX512 CPU kernels + graph fusions there; one warp per row here).
#include "common.cuh"

using namespace drc;

namespace {

// y = (x - mean) * rstd * gamma + beta ; saves mean/rstd for the backward
__global__ void __launch_bounds__(256) k_layer_norm_fwd(const float* __restrict__ x, int64_t rows, int cols, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, float eps, float* __restrict__ y, float* __restrict__ mean,
                                                        float* __restrict__ rstd) {
  const int lane = threadIdx.x & 31;
  for (int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; r < rows; r += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const float* xr = x + r * cols;
    float s = 0.f, q = 0.f;
    for (int c = lane; c < cols; c += 32) { float v = xr[c]; s += v; q += v * v; }
    s = warp_sum(s); q = warp_sum(q);
    const float m = s / cols, rs = rsqrtf(fmaxf(q / cols - m * m, 0.f) + eps);
    for (int c = lane; c < cols; c += 32) y[r * cols + c] = (xr[c] - m) * rs * (gamma ? gamma[c] : 1.f) + (beta ? beta[c] : 0.f);
    if (lane == 0) { mean[r] = m; rstd[r] = rs; }
  }
}
// dx = rstd * (g*gamma - mean(g*gamma) - xhat * mean(g*gamma*xhat)); dgamma/dbeta via atomics
__global__ void __launch_bounds__(256) k_layer_norm_bwd(const float* __restrict__ g, const float* __restrict__ x, int64_t rows, int cols,
                                                        const float* __restrict__ gamma, const float* __restrict__ mean, const float* __restrict__ rstd,
                                                        float* __restrict__ dx, float* __restrict__ dgamma, float* __restrict__ dbeta) {
  const int lane = threadIdx.x & 31;
  for (int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; r < rows; r += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const float m = mean[r], rs = rstd[r];
    float a = 0.f, b = 0.f;
    for (int c = lane; c < cols; c += 32) {
      float gg = g[r * cols + c] * (gamma ? gamma[c] : 1.f), xh = (x[r * cols + c] - m) * rs;
      a += gg; b += gg * xh;
    }
    a = warp_sum(a) / cols; b = warp_sum(b) / cols;
    for (int c = lane; c < cols; c += 32) {
      float go = g[r * cols + c], gg = go * (gamma ? gamma[c] : 1.f), xh = (x[r * cols + c] - m) * rs;
      dx[r * cols + c] = rs * (gg - a - xh * b);
      if (dgamma) atomicAdd(&dgamma[c], go * xh);
      if (dbeta) atomicAdd(&dbeta[c], go);
    }
  }
}
// y = x * rsqrt(max(sum x^2, eps))
__global__ void __launch_bounds__(256) k_l2_normalize_fwd(const float* __restrict__ x, int64_t rows, int cols, float eps, float* __restrict__ y,
                                                          float* __restrict__ rnorm) {
  const int lane = threadIdx.x & 31;
  for (int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; r < rows; r += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    float q = 0.f;
    for (int c = lane; c < cols; c += 32) { float v = x[r * cols + c]; q += v * v; }
    q = warp_sum(q);
    const float rn = rsqrtf(fmaxf(q, eps));
    for (int c = lane; c < cols; c += 32) y[r * cols + c] = x[r * cols + c] * rn;
    if (lane == 0) rnorm[r] = rn;
  }
}
// dx = rn * (g - y * sum(g*y))
__global__ void __launch_bounds__(256) k_l2_normalize_bwd(const float* __restrict__ g, const float* __restrict__ y, const float* __restrict__ rnorm,
                                                          int64_t rows, int cols, float* __restrict__ dx) {
  const int lane = threadIdx.x & 31;
  for (int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; r < rows; r += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    float d = 0.f;
    for (int c = lane; c < cols; c += 32) d += g[r * cols + c] * y[r * cols + c];
    d = warp_sum(d);
    for (int c = lane; c < cols; c += 32) dx[r * cols + c] = rnorm[r] * (g[r * cols + c] - y[r * cols + c] * d);
  }
}
__device__ __forceinline__ float gelu_f(float x, int approximate) {
  if (approximate) { float u = 0.7978845608f * (x + 0.044715f * x * x * x); return 0.5f * x * (1.f + tanhf(u)); }
  return 0.5f * x * (1.f + erff(x * 0.70710678f));
}
__global__ void k_gelu_fwd(const float* __restrict__ x, int64_t n, int approximate, float* __restrict__ y) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) y[i] = gelu_f(x[i], approximate);
}
__global__ void k_gelu_bwd(const float* __restrict__ g, const float* __restrict__ x, int64_t n, int approximate, float* __restrict__ dx) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = x[i];
    float d;
    if (approximate) {
      float u = 0.7978845608f * (v + 0.044715f * v * v * v), t = tanhf(u);
      d = 0.5f * (1.f + t) + 0.5f * v * (1.f - t * t) * 0.7978845608f * (1.f + 3.f * 0.044715f * v * v);
    } else {
      d = 0.5f * (1.f + erff(v * 0.70710678f)) + v * 0.3989422804f * __expf(-0.5f * v * v);
    }
    dx[i] = g[i] * d;
  }
}
// Dice: p = sigmoid((x - mean) * rstd); y = p*x + (1-p)*alpha*x   (mean/rstd per column: the BN statistics)
__global__ void k_dice_fwd(const float* __restrict__ x, int64_t rows, int cols, const float* __restrict__ mean, const float* __restrict__ rstd,
                           const float* __restrict__ alpha, float* __restrict__ y) {
  const int64_t n = rows * cols;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % cols);
    const float v = x[i], p = 1.f / (1.f + __expf(-(v - mean[c]) * rstd[c]));
    y[i] = p * v + (1.f - p) * alpha[c] * v;
  }
}

inline int grid_rows(int64_t rows) { int64_t b = (rows + 7) / 8; if (b < 1) b = 1; if (b > num_sms() * 8) b = num_sms() * 8; return (int)b; }
inline int grid_el(int64_t n) { int64_t b = (n + 255) / 256; if (b < 1) b = 1; if (b > num_sms() * 8) b = num_sms() * 8; return (int)b; }

}  // namespace

extern "C" {
int dr_cuda_layer_norm_fwd(const float* x, int64_t rows, int cols, const float* gamma, const float* beta, float eps, float* y, float* mean, float* rstd, cudaStream_t s) {
  k_layer_norm_fwd<<<grid_rows(rows), 256, 0, s>>>(x, rows, cols, gamma, beta, eps, y, mean, rstd); DR_LAUNCH_CHECK(); return 0;
}
int dr_cuda_layer_norm_bwd(const float* g, const float* x, int64_t rows, int cols, const float* gamma, const float* mean, const float* rstd, float* dx,
                           float* dgamma, float* dbeta, cudaStream_t s) {
  k_layer_norm_bwd<<<grid_rows(rows), 256, 0, s>>>(g, x, rows, cols, gamma, mean, rstd, dx, dgamma, dbeta); DR_LAUNCH_CHECK(); return 0;
}
int dr_cuda_l2_normalize_fwd(const float* x, int64_t rows, int cols, float eps, float* y, float* rnorm, cudaStream_t s) {
  k_l2_normalize_fwd<<<grid_rows(rows), 256, 0, s>>>(x, rows, cols, eps, y, rnorm); DR_LAUNCH_CHECK(); return 0;
}
int dr_cuda_l2_normalize_bwd(const float* g, const float* y, const float* rnorm, int64_t rows, int cols, float* dx, cudaStream_t s) {
  k_l2_normalize_bwd<<<grid_rows(rows), 256, 0, s>>>(g, y, rnorm, rows, cols, dx); DR_LAUNCH_CHECK(); return 0;
}
int dr_cuda_gelu_fwd(const float* x, int64_t n, int approximate, float* y, cudaStream_t s) { k_gelu_fwd<<<grid_el(n), 256, 0, s>>>(x, n, approximate, y); DR_LAUNCH_CHECK(); return 0; }
int dr_cuda_gelu_bwd(const float* g, const float* x, int64_t n, int approximate, float* dx, cudaStream_t s) { k_gelu_bwd<<<grid_el(n), 256, 0, s>>>(g, x, n, approximate, dx); DR_LAUNCH_CHECK(); return 0; }
int dr_cuda_dice_fwd(const float* x, int64_t rows, int cols, const float* mean, const float* rstd, const float* alpha, float* y, cudaStream_t s) {
  k_dice_fwd<<<grid_el(rows * cols), 256, 0, s>>>(x, rows, cols, mean, rstd, alpha, y); DR_LAUNCH_CHECK(); return 0;
}
}
