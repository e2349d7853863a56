// Memory-bound dense-path kernels fused as far as data dependencies allow: column statistics
// (BatchNorm forward/backward sums, bias gradients), BatchNorm apply forward/backward (+ReLU mask),
// the logit head (Linear(K->1) + sigmoid + BCE + full backward in one pass), weight packing
// (fp32 master -> bf16 W and W^T for the wgmma GEMMs) and input cast/pad.
//
// Reference equivalents are library/Eigen ops (tf.layers.dense + tf.layers.batch_normalization +
// keras BinaryCrossentropy, modelzoo/dlrm/train.py:163-243); DeepRec ships no CUDA kernel for them.
#include "common.cuh"

using namespace drc;

namespace {

// -------------------------------------------------------------------------------------------------
// Column sums over the batch:  S1[n] += sum_b u[b,n],  S2[n] += sum_b u[b,n] * v[b,n]   (v may be null)
// u, v: bf16 [B, ld].  N multiple of 8.  Each thread owns 8 consecutive columns.
// -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_colstats(const __nv_bfloat16* __restrict__ u, const __nv_bfloat16* __restrict__ v,
                                                  int64_t B, int N, int64_t ldu, int64_t ldv, float* __restrict__ part /* [grid][2N] */,
                                                  int with_s2) {
  pdl_sync();
  const int tpr = N / 8;                         // threads per row
  const int rows_par = blockDim.x / tpr;         // rows processed in parallel by the block
  const int tr = threadIdx.x / tpr, tc = threadIdx.x % tpr;
  float a1[8], a2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) a1[j] = a2[j] = 0.f;
  if (tr < rows_par) {
    for (int64_t b = (int64_t)blockIdx.x * rows_par + tr; b < B; b += (int64_t)gridDim.x * rows_par) {
      int4 ru = ld_nc_v4(u + b * ldu + tc * 8);
      const uint32_t wu[4] = {(uint32_t)ru.x, (uint32_t)ru.y, (uint32_t)ru.z, (uint32_t)ru.w};
      if (v) {
        int4 rv = ld_nc_v4(v + b * ldv + tc * 8);
        const uint32_t wv[4] = {(uint32_t)rv.x, (uint32_t)rv.y, (uint32_t)rv.z, (uint32_t)rv.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float2 fu = unpack_bf16x2(wu[e]), fv = unpack_bf16x2(wv[e]);
          a1[2 * e] += fu.x; a1[2 * e + 1] += fu.y; a2[2 * e] += fu.x * fv.x; a2[2 * e + 1] += fu.y * fv.y;
        }
      } else {
#pragma unroll
        for (int e = 0; e < 4; ++e) { float2 fu = unpack_bf16x2(wu[e]); a1[2 * e] += fu.x; a1[2 * e + 1] += fu.y; }
      }
    }
  }
  // the rows_par row-groups' partials are added in row-group order (no atomics: the sums are the same on every run); the block's
  // partial goes to part[blockIdx.x] and k_det_colsum adds the blocks in order
  extern __shared__ float sh[];                  // [rows_par][2N]
  if (tr < rows_par) {
#pragma unroll
    for (int j = 0; j < 8; ++j) { sh[tr * 2 * N + tc * 8 + j] = a1[j]; sh[tr * 2 * N + N + tc * 8 + j] = a2[j]; }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < (with_s2 ? 2 * N : N); i += blockDim.x) {
    float sum = 0.f;
    for (int r = 0; r < rows_par; ++r) sum += sh[r * 2 * N + i];
    part[(int64_t)blockIdx.x * 2 * N + i] = sum;
  }
}

// BatchNorm forward finalize: sums -> scale/shift (+ running stats), re-zero sums.
__global__ void k_bn_finalize(float* __restrict__ S1, float* __restrict__ S2, int N, float invB, const float* __restrict__ gamma,
                              const float* __restrict__ beta, float eps, float momentum, float* __restrict__ running_mean,
                              float* __restrict__ running_var, float* __restrict__ mean, float* __restrict__ rstd,
                              float* __restrict__ scale, float* __restrict__ shift, int training) {
  pdl_sync();
  int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float m, var;
  if (training) {
    m = S1[n] * invB;
    var = fmaxf(S2[n] * invB - m * m, 0.f);
    running_mean[n] = momentum * running_mean[n] + (1.f - momentum) * m;     // tf.layers BN: moving = m*moving + (1-m)*batch
    running_var[n] = momentum * running_var[n] + (1.f - momentum) * var;
    S1[n] = 0.f; S2[n] = 0.f;
  } else {
    m = running_mean[n]; var = running_var[n];
  }
  float rs = rsqrtf(var + eps);
  mean[n] = m; rstd[n] = rs;
  float sc = gamma[n] * rs;
  scale[n] = sc; shift[n] = beta[n] - m * sc;
}

// y = a * scale + shift   (bf16 in/out, 8 elements per thread)
__global__ void __launch_bounds__(256) k_bn_apply(const __nv_bfloat16* __restrict__ a, int64_t B, int N, int64_t lda,
                                                  const float* __restrict__ scale, const float* __restrict__ shift,
                                                  __nv_bfloat16* __restrict__ y, int64_t ldy) {
  pdl_sync();
  const int tpr = N / 8;
  const int64_t total = B * tpr;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / tpr; const int c = (int)(i % tpr) * 8;
    int4 ra = ld_nc_v4(a + b * lda + c);
    const uint32_t wa[4] = {(uint32_t)ra.x, (uint32_t)ra.y, (uint32_t)ra.z, (uint32_t)ra.w};
    uint32_t o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float2 f = unpack_bf16x2(wa[e]);
      o[e] = pack_bf16x2(f.x * scale[c + 2 * e] + shift[c + 2 * e], f.y * scale[c + 2 * e + 1] + shift[c + 2 * e + 1]);
    }
    *reinterpret_cast<int4*>(y + b * ldy + c) = make_int4((int)o[0], (int)o[1], (int)o[2], (int)o[3]);
  }
}

// BatchNorm backward finalize: S1 = sum dy, S2 = sum dy*a  ->  dgamma, dbeta, c1, c2 ; re-zero sums.
__global__ void k_bn_bwd_finalize(float* __restrict__ S1, float* __restrict__ S2, int N, float invB, const float* __restrict__ mean,
                                  const float* __restrict__ rstd, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                  float* __restrict__ c1, float* __restrict__ c2, float grad_accum_scale) {
  pdl_sync();
  int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float sdy = S1[n], sdya = S2[n];
  float dxhat = rstd[n] * (sdya - mean[n] * sdy);     // sum dy * xhat
  dgamma[n] += grad_accum_scale * dxhat;
  dbeta[n] += grad_accum_scale * sdy;
  c1[n] = sdy * invB; c2[n] = dxhat * invB;
  S1[n] = 0.f; S2[n] = 0.f;
}

// da_pre = relu'(a) * scale * (dy - c1 - xhat * c2),  xhat = (a - mean) * rstd
__global__ void __launch_bounds__(256) k_bn_bwd_apply(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ a, int64_t B,
                                                      int N, int64_t ld, const float* __restrict__ scale, const float* __restrict__ mean,
                                                      const float* __restrict__ rstd, const float* __restrict__ c1,
                                                      const float* __restrict__ c2, __nv_bfloat16* __restrict__ da, int relu_mask) {
  const int tpr = N / 8;
  const int64_t total = B * tpr;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / tpr; const int c = (int)(i % tpr) * 8;
    int4 rdy = ld_nc_v4(dy + b * ld + c), ra = ld_nc_v4(a + b * ld + c);
    const uint32_t wdy[4] = {(uint32_t)rdy.x, (uint32_t)rdy.y, (uint32_t)rdy.z, (uint32_t)rdy.w};
    const uint32_t wa[4] = {(uint32_t)ra.x, (uint32_t)ra.y, (uint32_t)ra.z, (uint32_t)ra.w};
    uint32_t o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float2 fdy = unpack_bf16x2(wdy[e]), fa = unpack_bf16x2(wa[e]);
      float r[2]; const float dys[2] = {fdy.x, fdy.y}; const float as[2] = {fa.x, fa.y};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        int n = c + 2 * e + h;
        float xhat = (as[h] - mean[n]) * rstd[n];
        float g = scale[n] * (dys[h] - c1[n] - xhat * c2[n]);
        r[h] = (relu_mask && !(as[h] > 0.f)) ? 0.f : g;
      }
      o[e] = pack_bf16x2(r[0], r[1]);
    }
    *reinterpret_cast<int4*>(da + b * ld + c) = make_int4((int)o[0], (int)o[1], (int)o[2], (int)o[3]);
  }
}

// -------------------------------------------------------------------------------------------------
// Logit head: z = h.w + b ; p = sigmoid(z) ; loss = BCE(p, y) mean ; dz = (p - y) * inv_batch_global
//   dh_pre[b,:] = dz * w (* relu'(h)) ; dw += sum_b dz*h ; db += sum dz.   One warp per row, K = 8*32*R.
// -------------------------------------------------------------------------------------------------
template <int R>   // K = 256 * R
__global__ void __launch_bounds__(256) k_head(const __nv_bfloat16* __restrict__ h, int64_t ldh, int64_t B, const float* __restrict__ w,
                                              const float* __restrict__ bias, const float* __restrict__ labels, float inv_batch,
                                              float* __restrict__ prob, float* __restrict__ loss_sum, __nv_bfloat16* __restrict__ dh,
                                              float* __restrict__ dw, float* __restrict__ db, int relu_mask, int train,
                                              float* __restrict__ dbias_h /* [K]: sum_b dh[b,:] = bias grad of the layer producing h */,
                                              float* __restrict__ part /* [grid][2K + 2]: dw | dbias_h | loss | db of each block */) {
  pdl_sync();
  constexpr int K = 256 * R;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  float wv[R][8], dwacc[R][8], dhacc[R][8];
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int j = 0; j < 8; ++j) { wv[r][j] = w[r * 256 + lane * 8 + j]; dwacc[r][j] = 0.f; dhacc[r][j] = 0.f; }
  const float b0 = bias[0];
  float dbacc = 0.f, lossacc = 0.f;
  for (int64_t row = (int64_t)blockIdx.x * wpb + warp; row < B; row += (int64_t)gridDim.x * wpb) {
    float hv[R][8];
    float dot = 0.f;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      int4 raw = ld_nc_v4(h + row * ldh + r * 256 + lane * 8);
      const uint32_t ww[4] = {(uint32_t)raw.x, (uint32_t)raw.y, (uint32_t)raw.z, (uint32_t)raw.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) { float2 f = unpack_bf16x2(ww[e]); hv[r][2 * e] = f.x; hv[r][2 * e + 1] = f.y; }
#pragma unroll
      for (int j = 0; j < 8; ++j) dot += hv[r][j] * wv[r][j];
    }
    dot = warp_sum(dot);
    const float z = dot + b0;
    const float p = 1.f / (1.f + __expf(-z));
    const float y = labels[row];
    if (lane == 0) {
      prob[row] = p;
      // numerically stable BCE on the logit: max(z,0) - z*y + log1p(exp(-|z|))
      lossacc += fmaxf(z, 0.f) - z * y + log1pf(__expf(-fabsf(z)));
    }
    if (train) {
      const float dz = (p - y) * inv_batch;
      if (lane == 0) dbacc += dz;
#pragma unroll
      for (int r = 0; r < R; ++r) {
        uint32_t o[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float g0 = dz * wv[r][2 * e], g1 = dz * wv[r][2 * e + 1];
          if (relu_mask) { if (!(hv[r][2 * e] > 0.f)) g0 = 0.f; if (!(hv[r][2 * e + 1] > 0.f)) g1 = 0.f; }
          o[e] = pack_bf16x2(g0, g1);
          dhacc[r][2 * e] += g0; dhacc[r][2 * e + 1] += g1;
          dwacc[r][2 * e] += dz * hv[r][2 * e]; dwacc[r][2 * e + 1] += dz * hv[r][2 * e + 1];
        }
        *reinterpret_cast<int4*>(dh + row * ldh + r * 256 + lane * 8) = make_int4((int)o[0], (int)o[1], (int)o[2], (int)o[3]);
      }
    }
  }
  // per-warp partials -> shared memory -> added in warp order -> part[blockIdx.x]; k_det_colsum adds the blocks in order (no atomics:
  // the loss and the gradients are the same on every run)
  extern __shared__ float sw[];                  // [8 warps][2K + 2]
  constexpr int L = 2 * K + 2;
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int j = 0; j < 8; ++j) { sw[warp * L + r * 256 + lane * 8 + j] = dwacc[r][j]; sw[warp * L + K + r * 256 + lane * 8 + j] = dhacc[r][j]; }
  if (lane == 0) { sw[warp * L + 2 * K] = lossacc * inv_batch; sw[warp * L + 2 * K + 1] = dbacc; }
  __syncthreads();
  for (int i = threadIdx.x; i < L; i += blockDim.x) {
    float sum = 0.f;
    for (int w = 0; w < wpb; ++w) sum += sw[w * L + i];
    part[(int64_t)blockIdx.x * L + i] = sum;
  }
  (void)dw; (void)db; (void)loss_sum; (void)train; (void)dbias_h;
}

// -------------------------------------------------------------------------------------------------
// Weight packing: fp32 master W[N, Kp] -> bf16 W[N, Kp] and bf16 W^T[Kp, Np8]   (32x32 smem tile transpose)
// -------------------------------------------------------------------------------------------------
__global__ void k_pack_weights(const float* __restrict__ w, int N, int Kp, __nv_bfloat16* __restrict__ wb, __nv_bfloat16* __restrict__ wt, int ldt) {
  pdl_sync();
  __shared__ float tile[32][33];
  const int n0 = blockIdx.y * 32, k0 = blockIdx.x * 32;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    int n = n0 + r, k = k0 + threadIdx.x;
    float v = (n < N && k < Kp) ? w[(int64_t)n * Kp + k] : 0.f;
    tile[r][threadIdx.x] = v;
    if (n < N && k < Kp) wb[(int64_t)n * Kp + k] = __float2bfloat16(v);
  }
  __syncthreads();
  if (wt) {
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
      int k = k0 + r, n = n0 + threadIdx.x;
      if (k < Kp && n < ldt) wt[(int64_t)k * ldt + n] = __float2bfloat16(n < N ? tile[threadIdx.x][r] : 0.f);
    }
  }
}

// fp32 [B, C] -> bf16 [B, Cp] zero padded
__global__ void k_cast_pad(const float* __restrict__ x, int64_t B, int C, __nv_bfloat16* __restrict__ y, int Cp) {
  pdl_sync();
  const int64_t total = B * Cp;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t b = i / Cp; int c = (int)(i % Cp);
    y[i] = __float2bfloat16(c < C ? x[b * C + c] : 0.f);
  }
}

__global__ void k_l2_flush(float* __restrict__ buf, int64_t n, float v) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) buf[i] = v;
}


// -------------------------------------------------------------------------------------------------
// BatchNorm folding (forward): finalize the batch statistics of layer l and fold y = s*a + t into layer l+1:
//   W'[n,k] = W[n,k] * s[k]   (bf16, the wgmma B operand)      b'[n] = b[n] + sum_k W[n,k] * t[k]   (fp32)
// so the normalised activation is never materialised (no extra pass over [B, N]).  One block per output row n;
// block 0 also publishes mean/rstd/scale/shift and advances the running statistics.
// -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_bn_fold(const float* __restrict__ S1, const float* __restrict__ S2, int K, float invB,
                                                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float momentum,
                                                 float* __restrict__ running_mean, float* __restrict__ running_var, float* __restrict__ mean,
                                                 float* __restrict__ rstd, float* __restrict__ scale, float* __restrict__ shift, int training,
                                                 const float* __restrict__ Wn, const float* __restrict__ bn, int Kp,
                                                 __nv_bfloat16* __restrict__ Wf, float* __restrict__ bf) {
  pdl_sync();
  const int n = blockIdx.x;
  float part = 0.f;
  for (int k = threadIdx.x; k < Kp; k += blockDim.x) {
    float s = 0.f, t = 0.f;
    if (k < K) {
      float m, var;
      if (training) { m = S1[k] * invB; var = fmaxf(S2[k] * invB - m * m, 0.f); }
      else { m = running_mean[k]; var = running_var[k]; }
      const float rs = rsqrtf(var + eps);
      s = gamma[k] * rs; t = beta[k] - m * s;
      if (n == 0) {
        mean[k] = m; rstd[k] = rs; scale[k] = s; shift[k] = t;
        if (training) {
          running_mean[k] = momentum * running_mean[k] + (1.f - momentum) * m;
          running_var[k] = momentum * running_var[k] + (1.f - momentum) * var;
        }
      }
    }
    const float w = Wn[(int64_t)n * Kp + k];
    Wf[(int64_t)n * Kp + k] = __float2bfloat16(w * s);
    part += w * t;
  }
  __shared__ float red[8];
  part = warp_sum(part);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = part;
  __syncthreads();
  if (threadIdx.x == 0) {
    float tot = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) tot += red[i];
    bf[n] = bn[n] + tot;
  }
}

// dW[n,k] = G[n,k] * s[k] + db[n] * t[k]   (weight gradient of a layer whose input was a folded BatchNorm output)
__global__ void __launch_bounds__(256) k_dw_fixup(float* __restrict__ dW, const float* __restrict__ db, const float* __restrict__ s,
                                                  const float* __restrict__ t, int N, int K, int Kp) {
  pdl_sync();
  const int64_t total = (int64_t)N * Kp;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int n = (int)(i / Kp), k = (int)(i % Kp);
    dW[i] = k < K ? dW[i] * s[k] + db[n] * t[k] : 0.f;
  }
}

// BatchNorm backward apply, v2: each thread owns 8 columns (parameters live in registers) and walks the rows;
// also reduces dbias[n] = sum_b da[b, n] so no separate pass over da is needed.
__global__ void __launch_bounds__(256) k_bn_bwd_apply_v2(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ a, int64_t B,
                                                         int N, int64_t ld, const float* __restrict__ scale, const float* __restrict__ mean,
                                                         const float* __restrict__ rstd, const float* __restrict__ c1,
                                                         const float* __restrict__ c2, __nv_bfloat16* __restrict__ da, int relu_mask,
                                                         float* __restrict__ dbias_part /* [grid][N] or null */) {
  pdl_sync();
  const int tpr = N / 8;
  const int rows_par = blockDim.x / tpr;
  const int tr = threadIdx.x / tpr, tc = threadIdx.x % tpr;
  float sc[8], mu[8], rs[8], k1[8], k2[8], acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (tr < rows_par) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = tc * 8 + j;
      sc[j] = scale[n]; mu[j] = mean[n]; rs[j] = rstd[n]; k1[j] = c1[n]; k2[j] = c2[n]; acc[j] = 0.f;
    }
    const int64_t rstep = (int64_t)gridDim.x * rows_par;
    for (int64_t b = (int64_t)blockIdx.x * rows_par + tr; b < B; b += 2 * rstep) {
      // two rows per iteration: all four 16 B loads are issued before any is consumed (memory-level parallelism)
      const int64_t b2 = b + rstep;
      const bool has2 = b2 < B;
      int4 rdy[2], ra[2];
      rdy[0] = ld_nc_v4(dy + b * ld + tc * 8); ra[0] = ld_nc_v4(a + b * ld + tc * 8);
      if (has2) { rdy[1] = ld_nc_v4(dy + b2 * ld + tc * 8); ra[1] = ld_nc_v4(a + b2 * ld + tc * 8); }
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        if (h2 == 1 && !has2) break;
        const uint32_t wdy[4] = {(uint32_t)rdy[h2].x, (uint32_t)rdy[h2].y, (uint32_t)rdy[h2].z, (uint32_t)rdy[h2].w};
        const uint32_t wa[4] = {(uint32_t)ra[h2].x, (uint32_t)ra[h2].y, (uint32_t)ra[h2].z, (uint32_t)ra[h2].w};
        uint32_t o[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 fdy = unpack_bf16x2(wdy[e]), fa = unpack_bf16x2(wa[e]);
          float g0 = sc[2 * e] * (fdy.x - k1[2 * e] - (fa.x - mu[2 * e]) * rs[2 * e] * k2[2 * e]);
          float g1 = sc[2 * e + 1] * (fdy.y - k1[2 * e + 1] - (fa.y - mu[2 * e + 1]) * rs[2 * e + 1] * k2[2 * e + 1]);
          if (relu_mask) { if (!(fa.x > 0.f)) g0 = 0.f; if (!(fa.y > 0.f)) g1 = 0.f; }
          acc[2 * e] += g0; acc[2 * e + 1] += g1;
          o[e] = pack_bf16x2(g0, g1);
        }
        *reinterpret_cast<int4*>(da + (h2 ? b2 : b) * ld + tc * 8) = make_int4((int)o[0], (int)o[1], (int)o[2], (int)o[3]);
      }
    }
  }
  if (dbias_part) {                               // row-group partials added in order -> part[blockIdx.x] (k_det_colsum adds the blocks)
    extern __shared__ float sh[];                 // [rows_par][N]
    if (tr < rows_par) {
#pragma unroll
      for (int j = 0; j < 8; ++j) sh[tr * N + tc * 8 + j] = acc[j];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
      float sum = 0.f;
      for (int r = 0; r < rows_par; ++r) sum += sh[r * N + i];
      dbias_part[(int64_t)blockIdx.x * N + i] = sum;
    }
  }
}

inline int grid_for(int64_t n, int block, int max_blocks = num_sms() * 8) {
  int64_t b = (n + block - 1) / block;
  if (b < 1) b = 1;
  if (b > max_blocks) b = max_blocks;
  return (int)b;
}

}  // namespace

extern "C" {

int dr_cuda_colstats(const void* u, const void* v, int64_t B, int N, int64_t ldu, int64_t ldv, float* S1, float* S2, cudaStream_t s) {
  if (N % 8 || N / 8 > 256) return -2;
  int tpr = N / 8; int rows_par = 256 / tpr;
  int grid = grid_for((B + rows_par - 1) / rows_par, 2, num_sms() * 4);   // >= 2 row-groups per block
  float* part = dr_workspace(kWsColstats, (size_t)grid * 2 * N, s);
  if (!part) return -5;
  DR_PDL_LAUNCH((k_colstats), grid, 256, rows_par * 2 * N * sizeof(float), s, (const __nv_bfloat16*)u, (const __nv_bfloat16*)v, B, N, ldu, ldv, part,
                S2 ? 1 : 0);
  DR_LAUNCH_CHECK();
  k_det_colsum<<<(N + 127) / 128, 128, 0, s>>>(part, grid, 2 * (int64_t)N, N, S1, S2, 1.f);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_bn_finalize(float* S1, float* S2, int N, int64_t B, const float* gamma, const float* beta, float eps, float momentum,
                        float* running_mean, float* running_var, float* mean, float* rstd, float* scale, float* shift, int training,
                        cudaStream_t s) {
  DR_PDL_LAUNCH((k_bn_finalize), (N + 127) / 128, 128, 0, s, S1, S2, N, 1.0f / (float)B, gamma, beta, eps, momentum, running_mean, running_var, mean, rstd, scale, shift, training);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_bn_apply(const void* a, int64_t B, int N, int64_t lda, const float* scale, const float* shift, void* y, int64_t ldy, cudaStream_t s) {
  if (N % 8) return -2;
  DR_PDL_LAUNCH((k_bn_apply), grid_for(B * (N / 8), 256), 256, 0, s, (const __nv_bfloat16*)a, B, N, lda, scale, shift, (__nv_bfloat16*)y, ldy);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_bn_bwd_finalize(float* S1, float* S2, int N, int64_t B, const float* mean, const float* rstd, float* dgamma, float* dbeta,
                            float* c1, float* c2, float grad_accum_scale, cudaStream_t s) {
  DR_PDL_LAUNCH((k_bn_bwd_finalize), (N + 127) / 128, 128, 0, s, S1, S2, N, 1.0f / (float)B, mean, rstd, dgamma, dbeta, c1, c2, grad_accum_scale);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_bn_bwd_apply(const void* dy, const void* a, int64_t B, int N, int64_t ld, const float* scale, const float* mean, const float* rstd,
                         const float* c1, const float* c2, void* da, int relu_mask, cudaStream_t s) {
  if (N % 8) return -2;
  k_bn_bwd_apply<<<grid_for(B * (N / 8), 256), 256, 0, s>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)a, B, N, ld, scale, mean, rstd, c1, c2,
                                                           (__nv_bfloat16*)da, relu_mask);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_bn_fold(const float* S1, const float* S2, int K, int64_t B, const float* gamma, const float* beta, float eps, float momentum,
                    float* running_mean, float* running_var, float* mean, float* rstd, float* scale, float* shift, int training,
                    const float* Wn, const float* bn, int Nn, int Kp, void* Wf, float* bf, cudaStream_t s) {
  DR_PDL_LAUNCH((k_bn_fold), Nn, 256, 0, s, S1, S2, K, 1.0f / (float)B, gamma, beta, eps, momentum, running_mean, running_var, mean, rstd, scale, shift,
                              training, Wn, bn, Kp, (__nv_bfloat16*)Wf, bf);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_dw_fixup(float* dW, const float* db, const float* scale, const float* shift, int N, int K, int Kp, cudaStream_t s) {
  DR_PDL_LAUNCH((k_dw_fixup), grid_for((int64_t)N * Kp, 256), 256, 0, s, dW, db, scale, shift, N, K, Kp);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_bn_bwd_apply_v2(const void* dy, const void* a, int64_t B, int N, int64_t ld, const float* scale, const float* mean,
                            const float* rstd, const float* c1, const float* c2, void* da, int relu_mask, float* dbias, cudaStream_t s) {
  if (N % 8 || N / 8 > 256) return -2;
  int tpr = N / 8; int rows_par = 256 / tpr;
  int grid = grid_for((B + rows_par - 1) / rows_par, 2, num_sms() * 8);
  float* part = nullptr;
  if (dbias) {
    part = dr_workspace(kWsBnBwd, (size_t)grid * N, s);
    if (!part) return -5;
  }
  DR_PDL_LAUNCH((k_bn_bwd_apply_v2), grid, 256, rows_par * N * sizeof(float), s, (const __nv_bfloat16*)dy, (const __nv_bfloat16*)a, B, N, ld, scale, mean, rstd,
                c1, c2, (__nv_bfloat16*)da, relu_mask, part);
  DR_LAUNCH_CHECK();
  if (dbias) {
    k_det_colsum<<<(N + 127) / 128, 128, 0, s>>>(part, grid, (int64_t)N, N, dbias, nullptr, 1.f);
    DR_LAUNCH_CHECK();
  }
  return 0;
}

int dr_cuda_head(const void* h, int64_t ldh, int64_t B, int K, const float* w, const float* bias, const float* labels, float inv_batch,
                 float* prob, float* loss_sum, void* dh, float* dw, float* db, int relu_mask, int train, float* dbias_h, cudaStream_t s) {
  int grid = grid_for((B + 7) / 8, 1, num_sms() * 4);
  if (K != 256 && K != 512 && K != 1024) return -2;
  float* part = dr_workspace(kWsHead, (size_t)grid * (2 * K + 2), s);
  if (!part) return -5;
  const size_t smem = 8 * (2 * K + 2) * sizeof(float);
#define HEAD(R)                                                                                                                     \
  do {                                                                                                                              \
    static DrPerDeviceOnce attr_once; bool& attr = attr_once();                                                                     \
    if (!attr) { DR_CUDA_CHECK(cudaFuncSetAttribute(k_head<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = true; } \
    DR_PDL_LAUNCH((k_head<R>), grid, 256, smem, s, (const __nv_bfloat16*)h, ldh, B, w, bias, labels, inv_batch, prob, loss_sum, (__nv_bfloat16*)dh, dw, db, \
                  relu_mask, train, dbias_h, part);                                                                                 \
  } while (0)
  if (K == 256) HEAD(1); else if (K == 512) HEAD(2); else HEAD(4);
#undef HEAD
  DR_LAUNCH_CHECK();
  const int64_t L = 2 * (int64_t)K + 2;
  if (train) {
    k_det_colsum<<<(K + 127) / 128, 128, 0, s>>>(part, grid, L, K, dw, nullptr, 1.f);
    if (dbias_h) k_det_colsum<<<(K + 127) / 128, 128, 0, s>>>(part + K, grid, L, K, dbias_h, nullptr, 1.f);
  }
  k_det_colsum<<<1, 1, 0, s>>>(part + 2 * K, grid, L, 1, loss_sum, train ? db : nullptr, 1.f);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_pack_weights(const float* w, int N, int Kp, void* wb, void* wt, int ldt, cudaStream_t s) {
  dim3 grid((Kp + 31) / 32, ((wt ? max(N, ldt) : N) + 31) / 32), block(32, 8);
  DR_PDL_LAUNCH((k_pack_weights), grid, block, 0, s, w, N, Kp, (__nv_bfloat16*)wb, (__nv_bfloat16*)wt, ldt);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_cast_pad(const float* x, int64_t B, int C, void* y, int Cp, cudaStream_t s) {
  DR_PDL_LAUNCH((k_cast_pad), grid_for(B * Cp, 256), 256, 0, s, x, B, C, (__nv_bfloat16*)y, Cp);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_l2_flush(float* buf, int64_t n, float v, cudaStream_t s) {
  k_l2_flush<<<num_sms() * 4, 256, 0, s>>>(buf, n, v);
  DR_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
