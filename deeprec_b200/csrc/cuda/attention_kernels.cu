// Fused DIN attention unit (forward, inference / no-grad path).
//
// Reference model (modelzoo/din/train.py:143-188): per sample, for every history position t
//     f_t = concat[q, k_t, q - k_t, q * k_t]  ->  Dense(H1)+sigmoid -> Dense(H2)+sigmoid -> Dense(1)   = s_t
//     w   = masked softmax(s) ,  out = sum_t w_t k_t
// which the reference runs as ~12 separate ops materialising a [B, L, 4D] tensor (210 MB at B=8192, L=50, D=32).
// Here one persistent block per SM keeps all attention weights in shared memory and processes a sample at a time:
//   * algebra: W1 [q | k | q-k | q*k] = (W1q + W1d) q  +  (W1k - W1d) k  +  W1p (q*k): the q term is computed ONCE per sample,
//     the per-position work is a [L, 2D] x [2D, H1] product -- half the first-layer FLOPs, and the concat never exists;
//   * register tiling: each thread produces kRT history positions of one hidden unit, so a weight read from shared memory is
//     reused kRT times and the k reads are warp-wide broadcasts;
//   * sigmoid / masked softmax / weighted sum fused behind the three layers; nothing but q, k, mask is read and only
//     out [B, D] is written.
// The training path keeps the composite autograd implementation (ops/attention.py decides).
#include "common.cuh"

using namespace drc;

namespace {

constexpr int kThreads = 256;
constexpr int kRT = 4;               // history positions per thread in the layer-1 / layer-2 tiles

__device__ __forceinline__ float sigmoidf_fast(float x) { return 1.f / (1.f + __expf(-x)); }

struct DinShape { int L, D, H1, H2; };

// shared-memory carve-up (floats), shared by the host (size) and the kernel (offsets)
struct DinSmem {
  int wq, wk, wp, b1, w2, b2, w3, q, k, hq, h1, h2, s, total;
  __host__ __device__ explicit DinSmem(const DinShape& p) {
    const int Lp = (p.L + kRT - 1) / kRT * kRT;      // rows padded to the register tile
    int o = 0;
    wq = o; o += p.D * p.H1;
    wk = o; o += p.D * p.H1;
    wp = o; o += p.D * p.H1;
    b1 = o; o += p.H1;
    w2 = o; o += p.H1 * p.H2;
    b2 = o; o += p.H2;
    w3 = o; o += p.H2;
    q = o; o += p.D;
    k = o; o += Lp * p.D;
    hq = o; o += p.H1;
    h1 = o; o += Lp * p.H1;
    h2 = o; o += Lp * p.H2;
    s = o; o += Lp;
    total = o;
  }
};

__global__ void __launch_bounds__(kThreads) k_din_attention_fwd(const float* __restrict__ q, const float* __restrict__ k, const uint8_t* __restrict__ mask, int64_t B,
                                                                DinShape p, const float* __restrict__ W1, const float* __restrict__ b1,
                                                                const float* __restrict__ W2, const float* __restrict__ b2, const float* __restrict__ w3, float b3,
                                                                float* __restrict__ out, float* __restrict__ weights_out) {
  extern __shared__ float sm[];
  const DinSmem o(p);
  const int L = p.L, D = p.D, H1 = p.H1, H2 = p.H2, tid = threadIdx.x;
  const int Lp = (L + kRT - 1) / kRT * kRT;
  float *sWq = sm + o.wq, *sWk = sm + o.wk, *sWp = sm + o.wp, *sB1 = sm + o.b1, *sW2 = sm + o.w2, *sB2 = sm + o.b2, *sW3 = sm + o.w3;
  float *sQ = sm + o.q, *sK = sm + o.k, *sHq = sm + o.hq, *sH1 = sm + o.h1, *sH2 = sm + o.h2, *sS = sm + o.s;

  // ---- weights -> shared memory, transposed to [in][out] so that consecutive threads (consecutive outputs) are conflict-free
  for (int i = tid; i < D * H1; i += kThreads) {
    const int d = i / H1, j = i % H1;
    const float* w = W1 + (size_t)j * 4 * D;           // row j of the [H1, 4D] weight
    const float wqv = w[d], wkv = w[D + d], wdv = w[2 * D + d], wpv = w[3 * D + d];
    sWq[i] = wqv + wdv; sWk[i] = wkv - wdv; sWp[i] = wpv;
  }
  for (int i = tid; i < H1 * H2; i += kThreads) { const int j = i / H2, m = i % H2; sW2[i] = W2[(size_t)m * H1 + j]; }
  for (int i = tid; i < H1; i += kThreads) sB1[i] = b1[i];
  for (int i = tid; i < H2; i += kThreads) { sB2[i] = b2[i]; sW3[i] = w3[i]; }
  __syncthreads();

  for (int64_t b = blockIdx.x; b < B; b += gridDim.x) {
    // ---- stage q, masked k (padding rows zero)
    for (int i = tid; i < D; i += kThreads) sQ[i] = q[b * D + i];
    for (int i = tid; i < Lp * D; i += kThreads) {
      const int t = i / D;
      sK[i] = (t < L && mask[b * L + t]) ? k[(b * L + t) * (int64_t)D + (i - t * D)] : 0.f;
    }
    __syncthreads();
    // ---- q part of layer 1 (once per sample)
    for (int j = tid; j < H1; j += kThreads) {
      float a = sB1[j];
      for (int d = 0; d < D; ++d) a = fmaf(sWq[d * H1 + j], sQ[d], a);
      sHq[j] = a;
    }
    __syncthreads();
    // ---- layer 1: h1[t][j] = sigmoid(hq[j] + sum_d (Wk[d][j] + Wp[d][j] q[d]) k[t][d]),  kRT positions per thread
    for (int idx = tid; idx < (Lp / kRT) * H1; idx += kThreads) {
      const int tg = idx / H1, j = idx - tg * H1, t0 = tg * kRT;
      float acc[kRT];
#pragma unroll
      for (int r = 0; r < kRT; ++r) acc[r] = sHq[j];
      for (int d = 0; d < D; ++d) {
        const float w = fmaf(sWp[d * H1 + j], sQ[d], sWk[d * H1 + j]);
#pragma unroll
        for (int r = 0; r < kRT; ++r) acc[r] = fmaf(w, sK[(t0 + r) * D + d], acc[r]);
      }
#pragma unroll
      for (int r = 0; r < kRT; ++r) sH1[(t0 + r) * H1 + j] = sigmoidf_fast(acc[r]);
    }
    __syncthreads();
    // ---- layer 2: h2[t][m] = sigmoid(b2[m] + sum_j W2[j][m] h1[t][j])
    for (int idx = tid; idx < (Lp / kRT) * H2; idx += kThreads) {
      const int tg = idx / H2, m = idx - tg * H2, t0 = tg * kRT;
      float acc[kRT];
#pragma unroll
      for (int r = 0; r < kRT; ++r) acc[r] = sB2[m];
      for (int j = 0; j < H1; ++j) {
        const float w = sW2[j * H2 + m];
#pragma unroll
        for (int r = 0; r < kRT; ++r) acc[r] = fmaf(w, sH1[(t0 + r) * H1 + j], acc[r]);
      }
#pragma unroll
      for (int r = 0; r < kRT; ++r) sH2[(t0 + r) * H2 + m] = sigmoidf_fast(acc[r]);
    }
    __syncthreads();
    // ---- layer 3 -> scores
    for (int t = tid; t < L; t += kThreads) {
      float a = b3;
      for (int m = 0; m < H2; ++m) a = fmaf(sW3[m], sH2[t * H2 + m], a);
      sS[t] = a;
    }
    __syncthreads();
    // ---- masked softmax over the history (warp 0), weights written back into sS
    if (tid < 32) {
      float mx = -INFINITY;
      for (int t = tid; t < L; t += 32) if (mask[b * L + t]) mx = fmaxf(mx, sS[t]);
#pragma unroll
      for (int s = 16; s > 0; s >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, s));
      float sum = 0.f;
      for (int t = tid; t < L; t += 32) {
        const float e = mask[b * L + t] ? __expf(sS[t] - mx) : 0.f;
        sS[t] = e; sum += e;
      }
      sum = warp_sum(sum);
      const float inv = sum > 0.f ? 1.f / sum : 0.f;        // no valid position -> zero output (softmax * mask.any())
      for (int t = tid; t < L; t += 32) sS[t] *= inv;
      // DIEN reads the weights themselves: softmax(masked_fill(s, -2^31)) is UNIFORM when no position is valid
      if (weights_out) for (int t = tid; t < L; t += 32) weights_out[b * L + t] = sum > 0.f ? sS[t] : 1.f / (float)L;
    }
    __syncthreads();
    // ---- weighted sum of the keys
    for (int d = tid; d < D; d += kThreads) {
      float a = 0.f;
      for (int t = 0; t < L; ++t) a = fmaf(sS[t], sK[t * D + d], a);
      out[b * D + d] = a;
    }
    __syncthreads();                                         // sK / sS are overwritten by the next sample
  }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Backward of the same unit (training path): per sample the forward activations are RECOMPUTED in shared memory (they were never written
// to HBM), then
//     dw_t = g . k_t,  ds_t = w_t (dw_t - sum_u w_u dw_u)                    softmax over the valid positions
//     layer 3 / 2 / 1 backward through the two sigmoids                       dz2 = ds w3 h2 (1 - h2),  dz1 = (dz2 W2^T) h1 (1 - h1)
//     dq, dk written per sample; weight gradients accumulated in shared memory across the samples of a block and flushed with atomics once.
// With W1 [q | k | q - k | q * k] = Wq q + Wk k + Wp (q * k):  A[d][j] = sum_t dz1[t][j] k[t][d],  dhq[j] = sum_t dz1[t][j]
//     dWk = A,  dWp = q (x) A,  dWq = q (x) dhq,  db1 = dhq;   dW1 = [dWq | dWk | dWq - dWk | dWp]
//     dq = Wq dhq + sum_j Wp[:, j] A[:, j],   dk_t = w_t g + (Wk + Wp diag(q)) dz1_t
// Plain thread-per-output loops (no register tiling): the training path is GEMM-bound elsewhere; this kernel removes the [B, L, 4D] concat, the
// two [B * L, H] activations and their gradients from HBM.  Verified against autograd in tests (and the algebra in numpy, DESIGN §6b).
struct DinBwdSmem {
  int g, ds, dz1, A, dhq, gWq, gWk, gWp, gW2, gb1, gb2, gw3, gb3, total;
  __host__ __device__ DinBwdSmem(const DinShape& p, int base) {
    const int Lp = (p.L + kRT - 1) / kRT * kRT;
    int o = base;
    g = o; o += p.D;
    ds = o; o += Lp;
    dz1 = o; o += Lp * p.H1;
    A = o; o += p.D * p.H1;
    dhq = o; o += p.H1;
    gWq = o; o += p.D * p.H1;
    gWk = o; o += p.D * p.H1;
    gWp = o; o += p.D * p.H1;
    gW2 = o; o += p.H1 * p.H2;
    gb1 = o; o += p.H1;
    gb2 = o; o += p.H2;
    gw3 = o; o += p.H2;
    gb3 = o; o += 1;
    total = o;
  }
};

__global__ void __launch_bounds__(kThreads) k_din_attention_bwd(const float* __restrict__ q, const float* __restrict__ k, const uint8_t* __restrict__ mask,
                                                                const float* __restrict__ gout, int64_t B, DinShape p, const float* __restrict__ W1,
                                                                const float* __restrict__ b1, const float* __restrict__ W2, const float* __restrict__ b2,
                                                                const float* __restrict__ w3, float b3, float* __restrict__ dq, float* __restrict__ dk,
                                                                float* __restrict__ dW1, float* __restrict__ db1, float* __restrict__ dW2,
                                                                float* __restrict__ db2, float* __restrict__ dw3, float* __restrict__ db3) {
  extern __shared__ float sm[];
  const DinSmem o(p);
  const DinBwdSmem ob(p, o.total);
  const int L = p.L, D = p.D, H1 = p.H1, H2 = p.H2, tid = threadIdx.x;
  const int Lp = (L + kRT - 1) / kRT * kRT;
  float *sWq = sm + o.wq, *sWk = sm + o.wk, *sWp = sm + o.wp, *sB1 = sm + o.b1, *sW2 = sm + o.w2, *sB2 = sm + o.b2, *sW3 = sm + o.w3;
  float *sQ = sm + o.q, *sK = sm + o.k, *sHq = sm + o.hq, *sH1 = sm + o.h1, *sH2 = sm + o.h2, *sS = sm + o.s;
  float *sG = sm + ob.g, *sDs = sm + ob.ds, *sDz1 = sm + ob.dz1, *sA = sm + ob.A, *sDhq = sm + ob.dhq;
  float *gWq = sm + ob.gWq, *gWk = sm + ob.gWk, *gWp = sm + ob.gWp, *gW2 = sm + ob.gW2, *gB1 = sm + ob.gb1, *gB2 = sm + ob.gb2, *gW3 = sm + ob.gw3, *gB3 = sm + ob.gb3;

  for (int i = tid; i < D * H1; i += kThreads) {
    const int d = i / H1, j = i % H1;
    const float* w = W1 + (size_t)j * 4 * D;
    const float wqv = w[d], wkv = w[D + d], wdv = w[2 * D + d], wpv = w[3 * D + d];
    sWq[i] = wqv + wdv; sWk[i] = wkv - wdv; sWp[i] = wpv;
    gWq[i] = 0.f; gWk[i] = 0.f; gWp[i] = 0.f;
  }
  for (int i = tid; i < H1 * H2; i += kThreads) { const int j = i / H2, m = i % H2; sW2[i] = W2[(size_t)m * H1 + j]; gW2[i] = 0.f; }
  for (int i = tid; i < H1; i += kThreads) { sB1[i] = b1[i]; gB1[i] = 0.f; }
  for (int i = tid; i < H2; i += kThreads) { sB2[i] = b2[i]; sW3[i] = w3[i]; gB2[i] = 0.f; gW3[i] = 0.f; }
  if (tid == 0) gB3[0] = 0.f;
  __syncthreads();

  for (int64_t b = blockIdx.x; b < B; b += gridDim.x) {
    // ---- stage q, masked k, upstream gradient
    for (int i = tid; i < D; i += kThreads) { sQ[i] = q[b * D + i]; sG[i] = gout[b * D + i]; }
    for (int i = tid; i < Lp * D; i += kThreads) {
      const int t = i / D;
      sK[i] = (t < L && mask[b * L + t]) ? k[(b * L + t) * (int64_t)D + (i - t * D)] : 0.f;
    }
    __syncthreads();
    // ---- forward, recomputed: hq, h1, h2, scores, softmax weights (sS)
    for (int j = tid; j < H1; j += kThreads) {
      float a = sB1[j];
      for (int d = 0; d < D; ++d) a = fmaf(sWq[d * H1 + j], sQ[d], a);
      sHq[j] = a;
    }
    __syncthreads();
    for (int idx = tid; idx < L * H1; idx += kThreads) {
      const int t = idx / H1, j = idx - t * H1;
      float a = sHq[j];
      for (int d = 0; d < D; ++d) a = fmaf(fmaf(sWp[d * H1 + j], sQ[d], sWk[d * H1 + j]), sK[t * D + d], a);
      sH1[t * H1 + j] = sigmoidf_fast(a);
    }
    __syncthreads();
    for (int idx = tid; idx < L * H2; idx += kThreads) {
      const int t = idx / H2, m = idx - t * H2;
      float a = sB2[m];
      for (int j = 0; j < H1; ++j) a = fmaf(sW2[j * H2 + m], sH1[t * H1 + j], a);
      sH2[t * H2 + m] = sigmoidf_fast(a);
    }
    __syncthreads();
    for (int t = tid; t < L; t += kThreads) {
      float a = b3;
      for (int m = 0; m < H2; ++m) a = fmaf(sW3[m], sH2[t * H2 + m], a);
      sS[t] = a;
    }
    __syncthreads();
    if (tid < 32) {
      float mx = -INFINITY;
      for (int t = tid; t < L; t += 32) if (mask[b * L + t]) mx = fmaxf(mx, sS[t]);
#pragma unroll
      for (int s = 16; s > 0; s >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, s));
      float sum = 0.f;
      for (int t = tid; t < L; t += 32) { const float e = mask[b * L + t] ? __expf(sS[t] - mx) : 0.f; sS[t] = e; sum += e; }
      sum = warp_sum(sum);
      const float inv = sum > 0.f ? 1.f / sum : 0.f;
      for (int t = tid; t < L; t += 32) sS[t] *= inv;                       // sS = softmax weights w_t (0 on masked positions)
      __syncwarp();
      // ---- ds_t = w_t (g . k_t - sum_u w_u g . k_u)
      float c = 0.f;
      for (int t = tid; t < L; t += 32) {
        float dw = 0.f;
        for (int d = 0; d < D; ++d) dw = fmaf(sG[d], sK[t * D + d], dw);
        sDs[t] = dw; c = fmaf(sS[t], dw, c);
      }
      c = warp_sum(c);
      float dsum = 0.f;
      for (int t = tid; t < L; t += 32) { const float v = sS[t] * (sDs[t] - c); sDs[t] = v; dsum += v; }
      dsum = warp_sum(dsum);
      if (tid == 0) gB3[0] += dsum;
    }
    __syncthreads();
    // ---- layer 3: dw3[m] += sum_t ds_t h2[t][m]
    for (int m = tid; m < H2; m += kThreads) {
      float a = 0.f;
      for (int t = 0; t < L; ++t) a = fmaf(sDs[t], sH2[t * H2 + m], a);
      gW3[m] += a;
    }
    __syncthreads();
    // dz2 (in place of h2) = ds_t w3[m] h2 (1 - h2)
    for (int idx = tid; idx < L * H2; idx += kThreads) {
      const int t = idx / H2, m = idx - t * H2;
      const float h = sH2[idx];
      sH2[idx] = sDs[t] * sW3[m] * h * (1.f - h);
    }
    __syncthreads();
    // ---- layer 2: db2, dW2 (accumulators), dz1 = (dz2 W2^T) h1 (1 - h1)
    for (int m = tid; m < H2; m += kThreads) {
      float a = 0.f;
      for (int t = 0; t < L; ++t) a += sH2[t * H2 + m];
      gB2[m] += a;
    }
    for (int idx = tid; idx < H1 * H2; idx += kThreads) {
      const int j = idx / H2, m = idx - j * H2;
      float a = 0.f;
      for (int t = 0; t < L; ++t) a = fmaf(sH1[t * H1 + j], sH2[t * H2 + m], a);
      gW2[idx] += a;
    }
    for (int idx = tid; idx < L * H1; idx += kThreads) {
      const int t = idx / H1, j = idx - t * H1;
      float a = 0.f;
      for (int m = 0; m < H2; ++m) a = fmaf(sW2[j * H2 + m], sH2[t * H2 + m], a);
      const float h = sH1[idx];
      sDz1[idx] = a * h * (1.f - h);
    }
    __syncthreads();
    // ---- layer 1: dhq, A = K^T dz1
    for (int j = tid; j < H1; j += kThreads) {
      float a = 0.f;
      for (int t = 0; t < L; ++t) a += sDz1[t * H1 + j];
      sDhq[j] = a; gB1[j] += a;
    }
    for (int idx = tid; idx < D * H1; idx += kThreads) {
      const int d = idx / H1, j = idx - d * H1;
      float a = 0.f;
      for (int t = 0; t < L; ++t) a = fmaf(sK[t * D + d], sDz1[t * H1 + j], a);
      sA[idx] = a;
    }
    __syncthreads();
    for (int idx = tid; idx < D * H1; idx += kThreads) {
      const int d = idx / H1, j = idx - d * H1;
      gWq[idx] = fmaf(sQ[d], sDhq[j], gWq[idx]);
      gWk[idx] += sA[idx];
      gWp[idx] = fmaf(sQ[d], sA[idx], gWp[idx]);
    }
    // dq[d] = sum_j Wq[d][j] dhq[j] + Wp[d][j] A[d][j]
    for (int d = tid; d < D; d += kThreads) {
      float a = 0.f;
      for (int j = 0; j < H1; ++j) a = fmaf(sWq[d * H1 + j], sDhq[j], fmaf(sWp[d * H1 + j], sA[d * H1 + j], a));
      dq[b * D + d] = a;
    }
    // dk[t][d] = w_t g[d] + sum_j (Wk[d][j] + Wp[d][j] q[d]) dz1[t][j]   (0 on masked positions)
    for (int idx = tid; idx < L * D; idx += kThreads) {
      const int t = idx / D, d = idx - t * D;
      float a = 0.f;
      if (mask[b * L + t]) {
        a = sS[t] * sG[d];
        const float qd = sQ[d];
        for (int j = 0; j < H1; ++j) a = fmaf(fmaf(sWp[d * H1 + j], qd, sWk[d * H1 + j]), sDz1[t * H1 + j], a);
      }
      dk[(b * L + t) * (int64_t)D + d] = a;
    }
    __syncthreads();                                         // every staging buffer is overwritten by the next sample
  }
  // ---- flush the block's weight-gradient accumulators
  for (int i = tid; i < D * H1; i += kThreads) {
    const int d = i / H1, j = i % H1;
    float* w = dW1 + (size_t)j * 4 * D;
    atomicAdd(w + d, gWq[i]); atomicAdd(w + D + d, gWk[i]); atomicAdd(w + 2 * D + d, gWq[i] - gWk[i]); atomicAdd(w + 3 * D + d, gWp[i]);
  }
  for (int i = tid; i < H1 * H2; i += kThreads) { const int j = i / H2, m = i % H2; atomicAdd(dW2 + (size_t)m * H1 + j, gW2[i]); }
  for (int i = tid; i < H1; i += kThreads) atomicAdd(db1 + i, gB1[i]);
  for (int i = tid; i < H2; i += kThreads) { atomicAdd(db2 + i, gB2[i]); atomicAdd(dw3 + i, gW3[i]); }
  if (tid == 0) atomicAdd(db3, gB3[0]);
}

}  // namespace

extern "C" {

// q [B, D], k [B, L, D], mask [B, L] (uint8), W1 [H1, 4D], W2 [H2, H1], w3 [H2] (PyTorch Linear layouts) -> out [B, D].
// Returns 0, a CUDA error code, or -1 when the shape does not fit in shared memory.
int dr_cuda_din_attention_fwd_w(const float* q, const float* k, const uint8_t* mask, int64_t B, int L, int D, const float* W1, const float* b1, int H1,
                                const float* W2, const float* b2, int H2, const float* w3, float b3, float* out, float* weights_out, cudaStream_t s) {
  if (B <= 0) return 0;
  const DinShape p{L, D, H1, H2};
  const size_t bytes = (size_t)DinSmem(p).total * sizeof(float);
  if (L <= 0 || D <= 0 || H1 <= 0 || H2 <= 0 || bytes > 200 * 1024) return -1;
  DR_CUDA_CHECK(cudaFuncSetAttribute(k_din_attention_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  const int per_sm = bytes <= 100 * 1024 ? 2 : 1;
  const int grid = (int)(B < (int64_t)num_sms() * per_sm ? B : (int64_t)num_sms() * per_sm);
  k_din_attention_fwd<<<grid, kThreads, bytes, s>>>(q, k, mask, B, p, W1, b1, W2, b2, w3, b3, out, weights_out);
  DR_LAUNCH_CHECK();
  return 0;
}
// weights_out [B, L] (optional): the softmax weights themselves (uniform for a row without a valid position) -- the DIEN op program
int dr_cuda_din_attention_fwd(const float* q, const float* k, const uint8_t* mask, int64_t B, int L, int D, const float* W1, const float* b1, int H1,
                              const float* W2, const float* b2, int H2, const float* w3, float b3, float* out, cudaStream_t s) {
  return dr_cuda_din_attention_fwd_w(q, k, mask, B, L, D, W1, b1, H1, W2, b2, H2, w3, b3, out, nullptr, s);
}

// Gradients of dr_cuda_din_attention_fwd.  dq [B, D] and dk [B, L, D] are written; dW1 [H1, 4D], db1 [H1], dW2 [H2, H1], db2 [H2], dw3 [H2],
// db3 [1] are ACCUMULATED (the caller zeroes them).  Returns -1 when the shape does not fit in shared memory.
int dr_cuda_din_attention_bwd(const float* q, const float* k, const uint8_t* mask, const float* gout, int64_t B, int L, int D, const float* W1, const float* b1,
                              int H1, const float* W2, const float* b2, int H2, const float* w3, float b3, float* dq, float* dk, float* dW1, float* db1,
                              float* dW2, float* db2, float* dw3, float* db3, cudaStream_t s) {
  if (B <= 0) return 0;
  const DinShape p{L, D, H1, H2};
  const size_t bytes = (size_t)DinBwdSmem(p, DinSmem(p).total).total * sizeof(float);
  if (L <= 0 || D <= 0 || H1 <= 0 || H2 <= 0 || bytes > 220 * 1024) return -1;
  DR_CUDA_CHECK(cudaFuncSetAttribute(k_din_attention_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  const int grid = (int)(B < (int64_t)num_sms() ? B : (int64_t)num_sms());
  k_din_attention_bwd<<<grid, kThreads, bytes, s>>>(q, k, mask, gout, B, p, W1, b1, W2, b2, w3, b3, dq, dk, dW1, db1, dW2, db2, dw3, db3);
  DR_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
