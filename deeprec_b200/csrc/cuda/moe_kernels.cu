// Expert-mixture gate kernels (MMoE, PLE; nn.fused_moe_mix) -- SIMT, also compiled into the CPU emulation.
//
// One launch handles one mixture layer: T gates over one packed expert buffer X [M, E_total H] (bf16, expert i in columns [i H, i H + H)).
// Gate t reads its input x_t [M, K_t] (bf16), its fp32 weight W_t [E_t, K_t] and bias b_t [E_t], and the E_t experts sel_t[0..E_t):
//   k_moe_mix_fwd   l = x_t W_t^T + b_t (fp32),  g_t = softmax(l) (fp32, saved),  mix_t = sum_e g_t,e X[:, sel_t[e]] (fp32, one bf16 rounding)
//   k_moe_mix_bwd   dX_i = sum over the gates t that read expert i, in gate order, of g_t,e dmix_t   (each element has one owner thread)
//                   dg_t,e = <dmix_t, X_sel_t[e]>,  dl_t = g_t (dg_t - sum_e g_t,e dg_t,e),  dx_t = dl_t W_t
//                   [dW_t | db_t] partials of the block's rows (dl_t^T x_t | sum dl_t), added in block order by k_det_colsum
// No floating-point atomics anywhere, so every output is bitwise repeatable.  One warp per row: lane l owns the 8-column chunks l and l + 32
// of the H columns (H <= 512), and lane e the gate column e (E_t <= 32); dot products are lane partials added by the warp's butterfly.
#include <algorithm>

#include "common.cuh"

using namespace drc;

namespace {

constexpr int kMoeMaxGates = 8;       // gates of one mixture layer
constexpr int kMoeMaxExperts = 32;    // experts one gate reads, and experts in the packed buffer
constexpr int kMoeMaxH = 512;
constexpr int kMoeThreads = 256;
constexpr int kMoeWarps = kMoeThreads / 32;
constexpr int kMoeBwdRows = 64;       // rows of one backward block: its partial is one workspace row

struct MoeGate {
  const __nv_bfloat16* x;             // [M, K] (pitch ldx)
  const float* W;                     // [E, K] fp32, row pitch K
  const float* b;                     // [E] or null
  __nv_bfloat16* mix;                 // forward: [M, H] (pitch ldmix)
  float* g;                           // [M, E] softmax weights: written by the forward, read by the backward
  const __nv_bfloat16* dmix;          // backward: [M, H] (pitch ldmix)
  __nv_bfloat16* dx;                  // backward: [M, K] (pitch lddx) or null
  int64_t ldx, ldmix, lddx;
  int64_t ws_col;                     // backward: first workspace column of this gate's [dW (E K) | db (E)] partials
  int K, E;
  uint8_t sel[kMoeMaxExperts];        // packed-buffer expert of gate column e
};

struct MoeLayer {
  MoeGate gate[kMoeMaxGates];
  const __nv_bfloat16* X;             // packed experts [M, E_total H] (pitch ldX)
  __nv_bfloat16* dX;                  // backward: their gradient (pitch lddX)
  float* dl;                          // backward: dl_t of every row [M][sum_t E_t] (gate t from column dl_col[t])
  float* part;                        // backward: [blocks][ws_ld] partials
  int64_t ldX, lddX, ws_ld;
  int T, E_total, H, dl_ld;
  int dl_col[kMoeMaxGates];
  uint8_t nread[kMoeMaxExperts];      // gates reading expert i, and (t, e) of each, in gate order
  uint8_t read_t[kMoeMaxExperts][kMoeMaxGates];
  uint8_t read_e[kMoeMaxExperts][kMoeMaxGates];
};

__device__ __forceinline__ void load_chunk(float (&v)[8], const __nv_bfloat16* p) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) { const float2 f = unpack_bf16x2(w[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
}
__device__ __forceinline__ void store_chunk(__nv_bfloat16* p, const float (&v)[8]) {
  *reinterpret_cast<uint4*>(p) = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
}

// logit of gate column `lane` (lanes >= E: -inf) of row r
__device__ __forceinline__ float gate_logit(const MoeGate& G, int64_t r, int lane) {
  const __nv_bfloat16* xr = G.x + r * G.ldx;
  float mine = -INFINITY;
  for (int e = 0; e < G.E; ++e) {
    const float* w = G.W + (int64_t)e * G.K;
    float p = 0.f;
    for (int k = lane; k < G.K; k += 32) p = fmaf(__bfloat162float(xr[k]), w[k], p);
    p = warp_sum(p);
    if (lane == e) mine = p + (G.b ? G.b[e] : 0.f);
  }
  return mine;
}

__global__ void __launch_bounds__(kMoeThreads) k_moe_mix_fwd(const __grid_constant__ MoeLayer p, int64_t M) {
  pdl_sync();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nch = p.H / 8;
  for (int64_t r = (int64_t)blockIdx.x * kMoeWarps + warp; r < M; r += (int64_t)gridDim.x * kMoeWarps) {
    for (int t = 0; t < p.T; ++t) {
      const MoeGate& G = p.gate[t];
      const float l = gate_logit(G, r, lane);
      float mx = l;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      const float ex = lane < G.E ? __expf(l - mx) : 0.f;
      const float g = ex / warp_sum(ex);
      if (lane < G.E) G.g[r * G.E + lane] = g;
      float acc[2][8];
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
      for (int e = 0; e < G.E; ++e) {
        const float ge = __shfl_sync(0xffffffffu, g, e);
        const __nv_bfloat16* xe = p.X + r * p.ldX + (int64_t)G.sel[e] * p.H;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int c = lane + 32 * i;
          if (c < nch) {
            float v[8];
            load_chunk(v, xe + 8 * c);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(ge, v[j], acc[i][j]);
          }
        }
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int c = lane + 32 * i;
        if (c < nch) store_chunk(G.mix + r * G.ldmix + 8 * c, acc[i]);
      }
    }
  }
}

// Block b owns rows [64 b, 64 b + 64): warp w takes rows w, w + 8, ...; after a block barrier its threads add the dW / db partials of those
// rows in row order into workspace row b.
__global__ void __launch_bounds__(kMoeThreads) k_moe_mix_bwd(const __grid_constant__ MoeLayer p, int64_t M) {
  pdl_sync();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nch = p.H / 8;
  const int64_t r0 = (int64_t)blockIdx.x * kMoeBwdRows;
  const int64_t r1 = r0 + kMoeBwdRows < M ? r0 + kMoeBwdRows : M;
  for (int64_t r = r0 + warp; r < r1; r += kMoeWarps) {
    for (int t = 0; t < p.T; ++t) {
      const MoeGate& G = p.gate[t];
      float dm[2][8];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int c = lane + 32 * i;
        if (c < nch) load_chunk(dm[i], G.dmix + r * G.ldmix + 8 * c);
      }
      float dg = 0.f;
      for (int e = 0; e < G.E; ++e) {
        const __nv_bfloat16* xe = p.X + r * p.ldX + (int64_t)G.sel[e] * p.H;
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int c = lane + 32 * i;
          if (c < nch) {
            float v[8];
            load_chunk(v, xe + 8 * c);
#pragma unroll
            for (int j = 0; j < 8; ++j) s = fmaf(dm[i][j], v[j], s);
          }
        }
        s = warp_sum(s);
        if (lane == e) dg = s;
      }
      const float g = lane < G.E ? G.g[r * G.E + lane] : 0.f;
      const float dl = g * (dg - warp_sum(g * dg));
      if (lane < G.E) p.dl[r * p.dl_ld + p.dl_col[t] + lane] = dl;
      if (G.dx) {
        for (int k0 = 0; k0 < G.K; k0 += 32) {             // whole-warp iterations: every lane takes part in the shuffles
          const int k = k0 + lane;
          float v = 0.f;
          for (int e = 0; e < G.E; ++e) {
            const float d = __shfl_sync(0xffffffffu, dl, e);
            if (k < G.K) v = fmaf(d, G.W[(int64_t)e * G.K + k], v);
          }
          if (k < G.K) G.dx[r * G.lddx + k] = __float2bfloat16(v);
        }
      }
    }
    for (int i = 0; i < p.E_total; ++i) {                // dX_i: its readers' g dmix in gate order
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int c = lane + 32 * h;
        if (c >= nch) continue;
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
        for (int q = 0; q < p.nread[i]; ++q) {
          const MoeGate& G = p.gate[p.read_t[i][q]];
          const float ge = G.g[r * G.E + p.read_e[i][q]];
          float v[8];
          load_chunk(v, G.dmix + r * G.ldmix + 8 * c);
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] = fmaf(ge, v[j], acc[j]);
        }
        store_chunk(p.dX + r * p.lddX + (int64_t)i * p.H + 8 * c, acc);
      }
    }
  }
  __syncthreads();                                       // this block's dl rows are written
  for (int64_t col = threadIdx.x; col < p.ws_ld; col += kMoeThreads) {
    int t = 0;
    while (t + 1 < p.T && col >= p.gate[t + 1].ws_col) ++t;
    const MoeGate& G = p.gate[t];
    const int64_t c = col - G.ws_col;
    const int e = c < (int64_t)G.E * G.K ? (int)(c / G.K) : (int)(c - (int64_t)G.E * G.K);
    const int k = c < (int64_t)G.E * G.K ? (int)(c % G.K) : -1;   // -1: the bias column of e
    float s = 0.f;
    for (int64_t r = r0; r < r1; ++r) {
      const float d = p.dl[r * p.dl_ld + p.dl_col[t] + e];
      s = k < 0 ? s + d : fmaf(d, __bfloat162float(G.x[r * G.ldx + k]), s);
    }
    p.part[(int64_t)blockIdx.x * p.ws_ld + col] = s;
  }
}

// Fills the layer description shared by both entry points.  Returns 0 or the entry points' error code.
int moe_layer(MoeLayer& L, const void* X, int64_t ldX, int64_t M, int E_total, int H, int T, const void* const* x, const int64_t* ldx, const int* K,
              const int* E, const float* const* W, const float* const* b, const int* sel) {
  L = MoeLayer{};
  if (T < 1 || T > kMoeMaxGates || E_total < 1 || E_total > kMoeMaxExperts || H <= 0 || H % 8 || H > kMoeMaxH || (ldX % 8) || ldX < (int64_t)E_total * H)
    return -2;
  if (!X || !x || !ldx || !K || !E || !W || !sel) return -4;
  if ((uintptr_t)X & 15) return -3;
  L.X = (const __nv_bfloat16*)X; L.ldX = ldX; L.T = T; L.E_total = E_total; L.H = H;
  int dl = 0;
  for (int t = 0; t < T; ++t) {
    MoeGate& G = L.gate[t];
    if (E[t] < 1 || E[t] > kMoeMaxExperts || K[t] < 1 || ldx[t] < K[t]) return -2;
    if (!x[t] || !W[t]) return -4;
    G.x = (const __nv_bfloat16*)x[t]; G.ldx = ldx[t]; G.K = K[t]; G.E = E[t]; G.W = W[t]; G.b = b ? b[t] : nullptr;
    for (int e = 0; e < E[t]; ++e) {
      const int i = sel[t * kMoeMaxExperts + e];
      if (i < 0 || i >= E_total) return -2;
      G.sel[e] = (uint8_t)i;
      L.read_t[i][L.nread[i]] = (uint8_t)t;
      L.read_e[i][L.nread[i]] = (uint8_t)e;
      ++L.nread[i];
    }
    L.dl_col[t] = dl;
    dl += E[t];
  }
  L.dl_ld = dl;
  return 0;
}

}  // namespace

extern "C" {

// Forward of one mixture layer (k_moe_mix_fwd): for each gate t < T, g_t [M, E_t] (fp32, contiguous) = softmax(x_t W_t^T + b_t) and
// mix_t [M, H] (bf16, pitch ldmix[t]) = sum_e g_t,e X[:, sel[t * 32 + e]].  X: the packed experts [M, E_total H] (bf16, pitch ldX); b may be
// null, or any b[t].  Limits: T <= 8, E_t and E_total <= 32, H a multiple of 8 and <= 512, any K_t.
// -2  a limit, a pitch below its width, ldX or ldmix not a multiple of 8, or an expert index outside [0, E_total);  -3  X or a mix_t not
// 16-byte aligned;  -4  a missing operand.
int dr_cuda_moe_mix_fwd(const void* X, int64_t ldX, int64_t M, int E_total, int H, int T, const void* const* x, const int64_t* ldx, const int* K,
                        const int* E, const float* const* W, const float* const* b, const int* sel, void* const* mix, const int64_t* ldmix,
                        float* const* g, cudaStream_t s) {
  if (M <= 0) return 0;
  MoeLayer L;
  int rc = moe_layer(L, X, ldX, M, E_total, H, T, x, ldx, K, E, W, b, sel);
  if (rc) return rc;
  if (!mix || !ldmix || !g) return -4;
  for (int t = 0; t < T; ++t) {
    if (!mix[t] || !g[t]) return -4;
    if ((ldmix[t] % 8) || ldmix[t] < H) return -2;
    if ((uintptr_t)mix[t] & 15) return -3;
    L.gate[t].mix = (__nv_bfloat16*)mix[t]; L.gate[t].ldmix = ldmix[t]; L.gate[t].g = g[t];
  }
  const int grid = (int)std::min<int64_t>((M + 4 * kMoeWarps - 1) / (4 * kMoeWarps), num_sms() * 8);   // >= 4 rows per warp
  DR_PDL_LAUNCH((k_moe_mix_fwd), grid, kMoeThreads, 0, s, L, M);
  DR_LAUNCH_CHECK();
  return 0;
}

// Backward of dr_cuda_moe_mix_fwd (k_moe_mix_bwd) from dmix_t (bf16, pitch lddmix[t]) and the forward's g_t:
//   dX [M, E_total H] (bf16, pitch lddX) = for expert i the sum, in gate order, of g_t,e dmix_t over the gates reading it (0 if none does);
//   dx_t [M, K_t] (bf16, pitch lddx[t]) = dl_t W_t, skipped where dx[t] is null;
//   dWb_t (fp32 [E_t K_t + E_t], accumulated into) += [dl_t^T x_t (row-major [E_t, K_t]) | sum_rows dl_t], summed in block order.
// Same limits and codes as the forward, for dmix_t / dX in place of mix_t, and -5 when the workspace cannot be had.
int dr_cuda_moe_mix_bwd(const void* X, int64_t ldX, int64_t M, int E_total, int H, int T, const void* const* x, const int64_t* ldx, const int* K,
                        const int* E, const float* const* W, const int* sel, float* const* g, const void* const* dmix, const int64_t* lddmix,
                        void* dX, int64_t lddX, void* const* dx, const int64_t* lddx, float* const* dWb, cudaStream_t s) {
  if (M <= 0) return 0;
  MoeLayer L;
  int rc = moe_layer(L, X, ldX, M, E_total, H, T, x, ldx, K, E, W, nullptr, sel);
  if (rc) return rc;
  if (!g || !dmix || !lddmix || !dX || !dWb) return -4;
  if ((lddX % 8) || lddX < (int64_t)E_total * H) return -2;
  if ((uintptr_t)dX & 15) return -3;
  int64_t ws_ld = 0;
  for (int t = 0; t < T; ++t) {
    MoeGate& G = L.gate[t];
    if (!g[t] || !dmix[t] || !dWb[t]) return -4;
    if ((lddmix[t] % 8) || lddmix[t] < H) return -2;
    if ((uintptr_t)dmix[t] & 15) return -3;
    G.g = g[t]; G.dmix = (const __nv_bfloat16*)dmix[t]; G.ldmix = lddmix[t];
    if (dx && dx[t]) {
      if (!lddx || lddx[t] < G.K) return -2;
      G.dx = (__nv_bfloat16*)dx[t]; G.lddx = lddx[t];
    }
    G.ws_col = ws_ld;
    ws_ld += (int64_t)G.E * G.K + G.E;
  }
  L.dX = (__nv_bfloat16*)dX; L.lddX = lddX; L.ws_ld = ws_ld;
  const int blocks = (int)((M + kMoeBwdRows - 1) / kMoeBwdRows);
  float* ws = dr_workspace(kWsMoe, (size_t)M * L.dl_ld + (size_t)blocks * ws_ld, s);
  if (!ws) return -5;
  L.dl = ws; L.part = ws + (size_t)M * L.dl_ld;
  DR_PDL_LAUNCH((k_moe_mix_bwd), blocks, kMoeThreads, 0, s, L, M);
  DR_LAUNCH_CHECK();
  for (int t = 0; t < T; t += kDetColsumMaxRanges) {     // [dW | db] of up to four gates per k_det_colsum launch
    DetColsumRange r[kDetColsumMaxRanges] = {};
    for (int j = 0; j < kDetColsumMaxRanges && t + j < T; ++j) {
      const MoeGate& G = L.gate[t + j];
      r[j] = DetColsumRange{G.ws_col, G.E * G.K + G.E, dWb[t + j]};
    }
    det_colsum(L.part, blocks, ws_ld, r, s);
    DR_LAUNCH_CHECK();
  }
  return 0;
}

}  // extern "C"
