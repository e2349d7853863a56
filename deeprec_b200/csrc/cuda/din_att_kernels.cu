// DIN attention unit for training (DIN's history attention, DIEN's attention over the interest states), forward and backward:
//
//   s_t = w3 . sig(W2 sig(W1 [q, k_t, q - k_t, q * k_t] + b1) + b2) + b3,   w = softmax(s | mask)   (t < L, per sample)
//   mode 0 (sum, DIN):      out[b] = sum_t w_t k_t  fp32 [B][D];  a sample with no valid position gives out = 0
//   mode 1 (weights, DIEN): out = w                fp32 [B][L];  a sample with no valid position gives w = 1 / L everywhere
//
// Algebra.  W1 [q, k, q - k, q * k] = Wq q + Wk k + Wp (q * k) with Wq = Wa + Wc, Wk = Wb - Wc, Wp = Wd (W1 = [Wa | Wb | Wc | Wd]).  The q
// term hq = Wq q + b1 is computed once per sample in fp32; the per-position first layer is one [L, 2D] x [2D, H1] product over the bf16
// operand X = [k | q * k].  b3 is never read: shifting every score by the same b3 does not change the softmax, so no output depends on it,
// and its gradient is exactly 0.  No host read of a parameter, so the op can be captured into a CUDA graph.
//
// One warp owns one sample and walks its positions in m16 row tiles.  The weights are converted from the fp32 masters to bf16 as the block
// stages them in shared memory (row-major for the forward products, transposed for the backward's).  Per tile, all on mma.sync m16n8k16
// (bf16 operands, fp32 accumulators): z1 = X Wkp^T + hq (the accumulators start at hq), h1 = sig(z1); two adjacent n8 accumulator tiles of
// h1 rounded to bf16 are the m16k16 A fragment of z2 = h1 W2^T + b2, h2 = sig(z2); s = h2 . w3 is a lane-local dot plus a 4-lane butterfly.
// The scores of the sample go to shared memory and the warp takes the masked softmax in fp32 (max, __expf, sum, one reciprocal).
//
// Backward.  It recomputes the forward with the same instructions on the same operands, so h1, h2, s and w are bit-identical to the
// forward's; the op saves only q, k and the mask.  ds_t = w_t (g_t - sum_u w_u g_u) with g_t = dout . k_t (sum mode) or dw_t (weights
// mode); ds is exactly 0 at a masked position and on a sample with no valid position (masked_fill zeroes those gradients in autograd), so
// such positions pass no gradient to dk, dq or any weight.  Then, per tile: dz2 = ds w3 h2 (1 - h2), dh1 = bf16(dz2) W2 (mma.sync),
// dz1 = dh1 h1 (1 - h1), dX = bf16(dz1) [Wk | Wp] (mma.sync), dk = dX_k + q * dX_p (+ w_t dout in sum mode), dq = Wq^T sum_t dz1_t +
// sum_t k_t * dX_p,t.  The kernel writes X, bf16(h1), bf16(dz1) and bf16(dz2) row for row; [dWk | dWp] = bf16(dz1)^T X and dW2 =
// bf16(dz2)^T bf16(h1) are the split-K weight-gradient GEMM (dr_cuda_gemm_dw), so the kernel keeps no [H1, 2D] accumulators per block.
// The per-sample sums (dhq = sum_t dz1_t, sum_t dz2_t, sum_t ds_t h2_t) are reduced in a fixed shuffle order; a block owns a static,
// contiguous range of samples, folds its warps' samples in warp order into fp32 block accumulators (dWq += dhq q^T, db1, db2, dw3) and
// writes them as one workspace row, which k_det_colsum adds in block order.  No floating-point atomics: two runs and a graph replay give
// the same bits.  dW1 = [dWq | dWk | dWq - dWk | dWp], as the SIMT kernel's flush maps it.
//
// Limits: D in {16, 32, 48, 64}; H1 a multiple of 16 up to 128; H2 a multiple of 8 up to 64; 1 <= L <= 128; B >= 1 with B L < 2^31.
#include "common.cuh"
#include "mma_sync.cuh"

using namespace drc;

namespace {

constexpr int kDinWarps = 4;          // warps per block, one sample per warp at a time
constexpr int kDinMaxH1 = 128, kDinMaxH2 = 64, kDinMaxL = 128;
constexpr int kDinCtaTarget = 256;    // blocks the batch is split into (a function of B only, so the partial sums do not depend on the device)

// bf16 row pitch for n columns (n a multiple of 8): n / 2 = 4 mod 8 words, so the 8 rows x 4 words of an mma fragment load hit 32 banks
__host__ __device__ constexpr int bf_pitch(int n) { return (n / 2) % 8 == 4 ? n : n + 8; }

// Shared memory of one block, in bytes from the start; the same function on the host (launch size) and the device.
struct DinLayout {
  int D, H1, H2, H2P, P1, PH1, PH2;     // H2P = H2 rounded up to 16; pitches of [*][2D], [*][H1], [*][H2P]
  int wkp, wkpt, w2, w2t, wq, b1, b2, w3, acc, warp, warp_bytes, bytes;
  __host__ __device__ DinLayout(int D_, int H1_, int H2_, bool bwd) : D(D_), H1(H1_), H2(H2_) {
    H2P = (H2 + 15) / 16 * 16;
    P1 = bf_pitch(2 * D); PH1 = bf_pitch(H1); PH2 = bf_pitch(H2P);
    int o = 0;
    wkp = o;  o += H1 * P1 * 2;                             // [Wk | Wp]    bf16 [H1][P1]
    w2 = o;   o += H2 * PH1 * 2;                            // W2           bf16 [H2][PH1]
    wkpt = o; if (bwd) o += 2 * D * PH1 * 2;                // [Wk | Wp]^T  bf16 [2D][PH1]
    w2t = o;  if (bwd) o += H1 * PH2 * 2;                   // W2^T         bf16 [H1][PH2], columns H2.. zero
    o = (o + 15) / 16 * 16;
    wq = o;   o += H1 * D * 4;                              // Wq fp32 [H1][D]
    b1 = o;   o += H1 * 4;
    b2 = o;   o += H2 * 4;
    w3 = o;   o += H2 * 4;
    acc = o;  if (bwd) o += (H1 * D + H1 + 2 * H2) * 4;     // block accumulators [dWq | db1 | db2 | dw3]
    o = (o + 15) / 16 * 16;
    warp = o;
    // per warp: s / w [128], ds [128], q [64], dout [64], dq partial [64], hq [128], dhq [128], db2 [64], dw3 [64], h1 fp32 [16][H1 + 8]
    warp_bytes = (2 * kDinMaxL + 3 * 64 + 2 * kDinMaxH1 + 2 * kDinMaxH2 + (bwd ? 16 * (H1 + 8) : 0)) * 4;
    bytes = warp + kDinWarps * warp_bytes;
  }
};

struct DinWarpSmem {
  float *s, *ds, *q, *gd, *dqp, *hq, *dhq, *db2, *dw3, *h1;
};
__device__ __forceinline__ DinWarpSmem warp_smem(unsigned char* base) {
  float* p = reinterpret_cast<float*>(base);
  DinWarpSmem w;
  w.s = p; w.ds = p + kDinMaxL; w.q = w.ds + kDinMaxL; w.gd = w.q + 64; w.dqp = w.gd + 64; w.hq = w.dqp + 64; w.dhq = w.hq + kDinMaxH1;
  w.db2 = w.dhq + kDinMaxH1; w.dw3 = w.db2 + kDinMaxH2; w.h1 = w.dw3 + kDinMaxH2;
  return w;
}

__device__ __forceinline__ float din_sigmoid(float x) { return __frcp_rn(__fadd_rn(1.f, __expf(-x))); }
__device__ __forceinline__ uint32_t ld_u32s(const uint16_t* p) { return *reinterpret_cast<const uint32_t*>(p); }
__device__ __forceinline__ uint16_t bf_bits(float x) { return __bfloat16_as_ushort(__float2bfloat16_rn(x)); }

template <typename KT> __device__ __forceinline__ float2 ld2(const KT* p);
template <> __device__ __forceinline__ float2 ld2<__nv_bfloat16>(const __nv_bfloat16* p) { return unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p)); }
template <> __device__ __forceinline__ float2 ld2<float>(const float* p) { return *reinterpret_cast<const float2*>(p); }
template <typename KT> __device__ __forceinline__ float ld1(const KT* p);
template <> __device__ __forceinline__ float ld1<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <> __device__ __forceinline__ float ld1<float>(const float* p) { return *p; }
template <typename KT> __device__ __forceinline__ void st2(KT* p, float a, float b);
template <> __device__ __forceinline__ void st2<__nv_bfloat16>(__nv_bfloat16* p, float a, float b) { *reinterpret_cast<uint32_t*>(p) = pack_bf16x2(a, b); }
template <> __device__ __forceinline__ void st2<float>(float* p, float a, float b) { *reinterpret_cast<float2*>(p) = make_float2(a, b); }

// sum over the 8 row groups g of a lane's value (xor 4, 8, 16: a fixed order)
__device__ __forceinline__ float rows_sum(float v) {
#pragma unroll
  for (int o = 4; o < 32; o <<= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Stage the weights of the unit into shared memory: [Wk | Wp] (and its transpose), W2 (and its transpose) as bf16, Wq, b1, b2, w3 as fp32.
__device__ __forceinline__ void stage_weights(const DinLayout& ly, unsigned char* sm, const float* __restrict__ W1, const float* __restrict__ b1,
                                              const float* __restrict__ W2, const float* __restrict__ b2, const float* __restrict__ w3, bool bwd) {
  const int D = ly.D, H1 = ly.H1, H2 = ly.H2;
  uint16_t* sWkp = reinterpret_cast<uint16_t*>(sm + ly.wkp);
  uint16_t* sWkpT = reinterpret_cast<uint16_t*>(sm + ly.wkpt);
  uint16_t* sW2 = reinterpret_cast<uint16_t*>(sm + ly.w2);
  uint16_t* sW2T = reinterpret_cast<uint16_t*>(sm + ly.w2t);
  float* sWq = reinterpret_cast<float*>(sm + ly.wq);
  for (int e = threadIdx.x; e < H1 * 2 * D; e += blockDim.x) {
    const int h = e / (2 * D), c = e % (2 * D);
    const float* row = W1 + (int64_t)h * 4 * D;
    const float v = c < D ? __fsub_rn(row[D + c], row[2 * D + c]) : row[2 * D + c];    // Wk = Wb - Wc | Wp = Wd
    const uint16_t bits = bf_bits(v);
    sWkp[h * ly.P1 + c] = bits;
    if (bwd) sWkpT[c * ly.PH1 + h] = bits;
  }
  for (int e = threadIdx.x; e < H1 * D; e += blockDim.x) {
    const float* row = W1 + (int64_t)(e / D) * 4 * D;
    sWq[e] = __fadd_rn(row[e % D], row[2 * D + e % D]);                                 // Wq = Wa + Wc
  }
  for (int e = threadIdx.x; e < H2 * H1; e += blockDim.x) {
    const int j = e / H1, h = e % H1;
    const uint16_t bits = bf_bits(W2[e]);
    sW2[j * ly.PH1 + h] = bits;
    if (bwd) sW2T[h * ly.PH2 + j] = bits;
  }
  if (bwd)
    for (int e = threadIdx.x; e < H1 * (ly.H2P - H2); e += blockDim.x) sW2T[(e / (ly.H2P - H2)) * ly.PH2 + H2 + e % (ly.H2P - H2)] = 0;
  float* sB1 = reinterpret_cast<float*>(sm + ly.b1);
  float* sB2 = reinterpret_cast<float*>(sm + ly.b2);
  float* sW3 = reinterpret_cast<float*>(sm + ly.w3);
  for (int e = threadIdx.x; e < H1; e += blockDim.x) sB1[e] = b1[e];
  for (int e = threadIdx.x; e < H2; e += blockDim.x) { sB2[e] = b2[e]; sW3[e] = w3[e]; }
}

// q of the sample into ws.q and hq = Wq q + b1 (fp32, sequential over d) into ws.hq
template <int D>
__device__ __forceinline__ void sample_q(const DinLayout& ly, const unsigned char* sm, const DinWarpSmem& ws, const float* __restrict__ qb, int lane) {
  const float* sWq = reinterpret_cast<const float*>(sm + ly.wq);
  const float* sB1 = reinterpret_cast<const float*>(sm + ly.b1);
  for (int d = lane; d < D; d += 32) ws.q[d] = qb[d];
  __syncwarp();
  for (int h = lane; h < ly.H1; h += 32) {
    float a = sB1[h];
#pragma unroll 8
    for (int d = 0; d < D; ++d) a = __fmaf_rn(sWq[h * D + d], ws.q[d], a);
    ws.hq[h] = a;
  }
  __syncwarp();
}

// The forward of one m16 tile of positions r0 .. r0 + 15 (rows g and g + 8 of this lane).  Positions at or past L and masked positions get
// X = 0.  Returns the scores of rows g and g + 8 (in every lane) and leaves h1 (bf16 A fragments) and h2 (fp32 accumulators) in registers;
// with xh (backward) it also writes X and bf16(h1) rows below L to xh / h1g and the fp32 h1 tile to ws.h1.
template <int D, typename KT>
__device__ __forceinline__ void tile_forward(const DinLayout& ly, const unsigned char* sm, const DinWarpSmem& ws, const KT* __restrict__ kb,
                                             bool v0, bool v1, bool in0, bool in1, int r0, int g, int t, uint32_t (&h1a)[kDinMaxH1 / 16][4],
                                             float (&h2)[kDinMaxH2 / 8][4], float& s0, float& s1, __nv_bfloat16* xh, __nv_bfloat16* h1g) {
  constexpr int XC = 2 * D / 16;      // k16 chunks of X
  const uint16_t* sWkp = reinterpret_cast<const uint16_t*>(sm + ly.wkp);
  const uint16_t* sW2 = reinterpret_cast<const uint16_t*>(sm + ly.w2);
  const float* sB2 = reinterpret_cast<const float*>(sm + ly.b2);
  const float* sW3 = reinterpret_cast<const float*>(sm + ly.w3);
  uint32_t xa[XC][4];
#pragma unroll
  for (int c = 0; c < XC; ++c) {
    const bool kpart = 16 * c < D;
    const int col0 = kpart ? 16 * c : 16 * c - D;
#pragma unroll
    for (int i = 0; i < 4; ++i) {      // a[0]: row g, cols 2t; a[1]: row g + 8; a[2]: row g, cols 8 + 2t; a[3]: row g + 8, cols 8 + 2t
      const int row = r0 + g + 8 * (i & 1), col = col0 + 8 * (i >> 1) + 2 * t;
      const bool v = (i & 1) ? v1 : v0;
      float2 x = v ? ld2<KT>(kb + (int64_t)row * D + col) : make_float2(0.f, 0.f);
      if (!kpart) x = make_float2(__fmul_rn(x.x, ws.q[col]), __fmul_rn(x.y, ws.q[col + 1]));
      xa[c][i] = pack_bf16x2(x.x, x.y);
    }
    if (xh) {
      if (in0) *reinterpret_cast<uint32_t*>(xh + (int64_t)(r0 + g) * 2 * D + 16 * c + 2 * t) = xa[c][0];
      if (in1) *reinterpret_cast<uint32_t*>(xh + (int64_t)(r0 + g + 8) * 2 * D + 16 * c + 2 * t) = xa[c][1];
      if (in0) *reinterpret_cast<uint32_t*>(xh + (int64_t)(r0 + g) * 2 * D + 16 * c + 8 + 2 * t) = xa[c][2];
      if (in1) *reinterpret_cast<uint32_t*>(xh + (int64_t)(r0 + g + 8) * 2 * D + 16 * c + 8 + 2 * t) = xa[c][3];
    }
  }
  // layer 1, one k16 chunk of H1 (two n8 tiles) at a time
#pragma unroll
  for (int kc = 0; kc < kDinMaxH1 / 16; ++kc) {
    if (16 * kc < ly.H1) {
      float z[2][4];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int col = 16 * kc + 8 * i + 2 * t;
        z[i][0] = z[i][2] = ws.hq[col];
        z[i][1] = z[i][3] = ws.hq[col + 1];
        const uint16_t* wrow = sWkp + (16 * kc + 8 * i + g) * ly.P1 + 2 * t;
#pragma unroll
        for (int c = 0; c < XC; ++c) mma_bf16_16816(z[i], xa[c], ld_u32s(wrow + 16 * c), ld_u32s(wrow + 16 * c + 8));
#pragma unroll
        for (int e = 0; e < 4; ++e) z[i][e] = din_sigmoid(z[i][e]);
        if (xh) {
          *reinterpret_cast<float2*>(ws.h1 + g * (ly.H1 + 8) + col) = make_float2(z[i][0], z[i][1]);
          *reinterpret_cast<float2*>(ws.h1 + (g + 8) * (ly.H1 + 8) + col) = make_float2(z[i][2], z[i][3]);
        }
      }
      h1a[kc][0] = pack_bf16x2(z[0][0], z[0][1]);
      h1a[kc][1] = pack_bf16x2(z[0][2], z[0][3]);
      h1a[kc][2] = pack_bf16x2(z[1][0], z[1][1]);
      h1a[kc][3] = pack_bf16x2(z[1][2], z[1][3]);
      if (h1g) {
        if (in0) *reinterpret_cast<uint32_t*>(h1g + (int64_t)(r0 + g) * ly.H1 + 16 * kc + 2 * t) = h1a[kc][0];
        if (in1) *reinterpret_cast<uint32_t*>(h1g + (int64_t)(r0 + g + 8) * ly.H1 + 16 * kc + 2 * t) = h1a[kc][1];
        if (in0) *reinterpret_cast<uint32_t*>(h1g + (int64_t)(r0 + g) * ly.H1 + 16 * kc + 8 + 2 * t) = h1a[kc][2];
        if (in1) *reinterpret_cast<uint32_t*>(h1g + (int64_t)(r0 + g + 8) * ly.H1 + 16 * kc + 8 + 2 * t) = h1a[kc][3];
      }
    }
  }
  // layer 2 and the score
  float p0 = 0.f, p1 = 0.f;
#pragma unroll
  for (int j = 0; j < kDinMaxH2 / 8; ++j) {
    if (8 * j < ly.H2) {
      const int col = 8 * j + 2 * t;
      h2[j][0] = h2[j][2] = sB2[col];
      h2[j][1] = h2[j][3] = sB2[col + 1];
      const uint16_t* wrow = sW2 + (8 * j + g) * ly.PH1 + 2 * t;
#pragma unroll
      for (int kc = 0; kc < kDinMaxH1 / 16; ++kc)
        if (16 * kc < ly.H1) mma_bf16_16816(h2[j], h1a[kc], ld_u32s(wrow + 16 * kc), ld_u32s(wrow + 16 * kc + 8));
#pragma unroll
      for (int e = 0; e < 4; ++e) h2[j][e] = din_sigmoid(h2[j][e]);
      p0 = __fmaf_rn(sW3[col + 1], h2[j][1], __fmaf_rn(sW3[col], h2[j][0], p0));
      p1 = __fmaf_rn(sW3[col + 1], h2[j][3], __fmaf_rn(sW3[col], h2[j][2], p1));
    }
  }
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    p0 = __fadd_rn(p0, __shfl_xor_sync(0xffffffffu, p0, o));
    p1 = __fadd_rn(p1, __shfl_xor_sync(0xffffffffu, p1, o));
  }
  s0 = p0;
  s1 = p1;
}

// Scores of every position of the sample into ws.s, then the masked softmax in place: ws.s[t] = w_t (t < L).  Returns whether the sample has
// a valid position.  mode 0: a sample without one gets w = 0; mode 1: w = 1 / L.
template <int D, typename KT>
__device__ __forceinline__ bool sample_weights(const DinLayout& ly, const unsigned char* sm, const DinWarpSmem& ws, const KT* __restrict__ kb,
                                               const uint8_t* __restrict__ mb, int L, int mode, int lane) {
  const int g = lane >> 2, t = lane & 3;
  for (int r0 = 0; r0 < L; r0 += 16) {
    uint32_t h1a[kDinMaxH1 / 16][4];
    float h2[kDinMaxH2 / 8][4];
    float s0, s1;
    const bool in0 = r0 + g < L, in1 = r0 + g + 8 < L;
    tile_forward<D, KT>(ly, sm, ws, kb, in0 && mb[r0 + g], in1 && mb[r0 + g + 8], in0, in1, r0, g, t, h1a, h2, s0, s1, nullptr, nullptr);
    if (t == 0) {
      if (in0) ws.s[r0 + g] = s0;
      if (in1) ws.s[r0 + g + 8] = s1;
    }
  }
  __syncwarp();
  float sv[kDinMaxL / 32];
  bool vv[kDinMaxL / 32];
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < kDinMaxL / 32; ++i) {
    const int p = lane + 32 * i;
    vv[i] = p < L && mb[p];
    sv[i] = vv[i] ? ws.s[p] : 0.f;
    if (vv[i]) m = fmaxf(m, sv[i]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  const bool any = m != -INFINITY;
  float l = 0.f;
#pragma unroll
  for (int i = 0; i < kDinMaxL / 32; ++i) {
    sv[i] = vv[i] ? __expf(__fsub_rn(sv[i], m)) : 0.f;
    l = __fadd_rn(l, sv[i]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) l = __fadd_rn(l, __shfl_xor_sync(0xffffffffu, l, o));
  const float r = any ? __frcp_rn(l) : 0.f;
  const float empty = mode == 1 ? __frcp_rn((float)L) : 0.f;
  __syncwarp();
#pragma unroll
  for (int i = 0; i < kDinMaxL / 32; ++i) {
    const int p = lane + 32 * i;
    if (p < L) ws.s[p] = any ? __fmul_rn(sv[i], r) : empty;
  }
  __syncwarp();
  return any;
}

// samples per block: a multiple of the warp count, from B alone
__host__ __device__ inline int din_spc(int B) {
  const int per = (B + kDinCtaTarget - 1) / kDinCtaTarget;
  return (per + kDinWarps - 1) / kDinWarps * kDinWarps;
}

template <int D, typename KT>
__global__ void __launch_bounds__(32 * kDinWarps, 1) k_din_att_fwd(const float* __restrict__ q, const KT* __restrict__ k, const uint8_t* __restrict__ mask,
                                                                int B, int L, int H1, int H2, const float* __restrict__ W1, const float* __restrict__ b1,
                                                                const float* __restrict__ W2, const float* __restrict__ b2,
                                                                const float* __restrict__ w3, int mode, float* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char din_smem[];
  const DinLayout ly(D, H1, H2, false);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  pdl_sync();
  stage_weights(ly, din_smem, W1, b1, W2, b2, w3, false);
  __syncthreads();
  const DinWarpSmem ws = warp_smem(din_smem + ly.warp + warp * ly.warp_bytes);
  const int spc = din_spc(B);
  const int64_t first = (int64_t)blockIdx.x * spc, last = min((int64_t)B, first + spc);
  for (int64_t b = first + warp; b < last; b += kDinWarps) {
    const KT* kb = k + b * L * D;
    const uint8_t* mb = mask + b * L;
    sample_q<D>(ly, din_smem, ws, q + b * D, lane);
    const bool any = sample_weights<D, KT>(ly, din_smem, ws, kb, mb, L, mode, lane);
    if (mode == 1) {
      for (int p = lane; p < L; p += 32) out[b * L + p] = ws.s[p];
    } else {
      for (int d = lane; d < D; d += 32) {
        float a = 0.f;
        if (any)
          for (int p = 0; p < L; ++p)
            if (mb[p]) a = __fmaf_rn(ws.s[p], ld1<KT>(kb + (int64_t)p * D + d), a);
        out[b * D + d] = a;
      }
    }
    __syncwarp();
  }
}

template <int D, typename KT>
__global__ void __launch_bounds__(32 * kDinWarps, 1) k_din_att_bwd(const float* __restrict__ q, const KT* __restrict__ k, const uint8_t* __restrict__ mask,
                                                                const float* __restrict__ gout, int B, int L, int H1, int H2,
                                                                const float* __restrict__ W1, const float* __restrict__ b1,
                                                                const float* __restrict__ W2, const float* __restrict__ b2,
                                                                const float* __restrict__ w3, int mode, float* __restrict__ dq, KT* __restrict__ dk,
                                                                __nv_bfloat16* __restrict__ xh, __nv_bfloat16* __restrict__ h1h,
                                                                __nv_bfloat16* __restrict__ dz1h, __nv_bfloat16* __restrict__ dz2h,
                                                                float* __restrict__ part) {
  extern __shared__ __align__(16) unsigned char din_smem[];
  const DinLayout ly(D, H1, H2, true);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  pdl_sync();
  stage_weights(ly, din_smem, W1, b1, W2, b2, w3, true);
  float* acc = reinterpret_cast<float*>(din_smem + ly.acc);
  const int nacc = H1 * D + H1 + 2 * H2;
  for (int e = threadIdx.x; e < nacc; e += blockDim.x) acc[e] = 0.f;
  __syncthreads();
  const uint16_t* sWkpT = reinterpret_cast<const uint16_t*>(din_smem + ly.wkpt);
  const uint16_t* sW2T = reinterpret_cast<const uint16_t*>(din_smem + ly.w2t);
  const float* sWq = reinterpret_cast<const float*>(din_smem + ly.wq);
  const float* sW3 = reinterpret_cast<const float*>(din_smem + ly.w3);
  const DinWarpSmem ws = warp_smem(din_smem + ly.warp + warp * ly.warp_bytes);
  const int spc = din_spc(B);
  const int64_t first = (int64_t)blockIdx.x * spc, last = min((int64_t)B, first + spc);
  for (int64_t base = first; base < last; base += kDinWarps) {
    const int64_t b = base + warp;
    if (b < last) {
      const KT* kb = k + b * L * D;
      const uint8_t* mb = mask + b * L;
      sample_q<D>(ly, din_smem, ws, q + b * D, lane);
      for (int h = lane; h < kDinMaxH1; h += 32) ws.dhq[h] = 0.f;
      for (int j = lane; j < kDinMaxH2; j += 32) ws.db2[j] = ws.dw3[j] = ws.dqp[j] = 0.f;
      const bool any = sample_weights<D, KT>(ly, din_smem, ws, kb, mb, L, mode, lane);
      // ds_t = w_t (g_t - sum_u w_u g_u) at valid positions of a sample with one; 0 elsewhere
      if (mode == 0)
        for (int d = lane; d < D; d += 32) ws.gd[d] = gout[b * D + d];
      __syncwarp();
      float gv[kDinMaxL / 32], c = 0.f;
#pragma unroll
      for (int i = 0; i < kDinMaxL / 32; ++i) {
        const int p = lane + 32 * i;
        gv[i] = 0.f;
        if (p < L && any && mb[p]) {
          if (mode == 1) {
            gv[i] = gout[b * L + p];
          } else {
            float a = 0.f;
            for (int d = 0; d < D; ++d) a = __fmaf_rn(ws.gd[d], ld1<KT>(kb + (int64_t)p * D + d), a);
            gv[i] = a;
          }
          c = __fmaf_rn(ws.s[p], gv[i], c);
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) c = __fadd_rn(c, __shfl_xor_sync(0xffffffffu, c, o));
#pragma unroll
      for (int i = 0; i < kDinMaxL / 32; ++i) {
        const int p = lane + 32 * i;
        if (p < L) ws.ds[p] = (any && mb[p]) ? __fmul_rn(ws.s[p], __fsub_rn(gv[i], c)) : 0.f;
      }
      __syncwarp();
      const int64_t row0 = b * L;
      for (int r0 = 0; r0 < L; r0 += 16) {
        const bool in0 = r0 + g < L, in1 = r0 + g + 8 < L;
        const bool v0 = in0 && mb[r0 + g], v1 = in1 && mb[r0 + g + 8];
        uint32_t h1a[kDinMaxH1 / 16][4];
        float h2[kDinMaxH2 / 8][4];
        float s0, s1;
        tile_forward<D, KT>(ly, din_smem, ws, kb, v0, v1, in0, in1, r0, g, t, h1a, h2, s0, s1, xh + row0 * 2 * D, h1h + row0 * H1);
        const float ds0 = in0 ? ws.ds[r0 + g] : 0.f, ds1 = in1 ? ws.ds[r0 + g + 8] : 0.f;
        // dz2 = ds w3 h2 (1 - h2); column sums of dz2 and ds h2
        uint32_t dz2a[kDinMaxH2 / 16][4];
#pragma unroll
        for (int j = 0; j < kDinMaxH2 / 8; ++j) {
          float z[4] = {0.f, 0.f, 0.f, 0.f};
          if (8 * j < H2) {
            const int col = 8 * j + 2 * t;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float ds = e < 2 ? ds0 : ds1, h = h2[j][e];
              z[e] = __fmul_rn(__fmul_rn(ds, sW3[col + (e & 1)]), __fmul_rn(h, __fsub_rn(1.f, h)));
            }
#pragma unroll
            for (int cc = 0; cc < 2; ++cc) {
              const float sz = rows_sum(__fadd_rn(z[cc], z[2 + cc]));
              const float sh = rows_sum(__fadd_rn(__fmul_rn(ds0, h2[j][cc]), __fmul_rn(ds1, h2[j][2 + cc])));
              if (g == 0) { ws.db2[col + cc] = __fadd_rn(ws.db2[col + cc], sz); ws.dw3[col + cc] = __fadd_rn(ws.dw3[col + cc], sh); }
            }
            const uint32_t lo = pack_bf16x2(z[0], z[1]), hi = pack_bf16x2(z[2], z[3]);
            __nv_bfloat16* zr = dz2h + (row0 + r0 + g) * H2 + col;
            if (in0) *reinterpret_cast<uint32_t*>(zr) = lo;
            if (in1) *reinterpret_cast<uint32_t*>(zr + 8 * H2) = hi;
          }
          // two n8 tiles of dz2 are one m16k16 A fragment (an odd last tile pairs with zeros)
          dz2a[j / 2][2 * (j & 1)] = pack_bf16x2(z[0], z[1]);
          dz2a[j / 2][2 * (j & 1) + 1] = pack_bf16x2(z[2], z[3]);
        }
        __syncwarp();
        // dh1 = bf16(dz2) W2, dz1 = dh1 h1 (1 - h1); column sums of dz1 into dhq
        uint32_t dz1a[kDinMaxH1 / 16][4];
#pragma unroll
        for (int kc = 0; kc < kDinMaxH1 / 16; ++kc) {
          if (16 * kc < H1) {
            float z[2][4];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const int col = 16 * kc + 8 * i + 2 * t;
              z[i][0] = z[i][1] = z[i][2] = z[i][3] = 0.f;
              const uint16_t* wrow = sW2T + (16 * kc + 8 * i + g) * ly.PH2 + 2 * t;
#pragma unroll
              for (int c2 = 0; c2 < kDinMaxH2 / 16; ++c2)
                if (16 * c2 < ly.H2P) mma_bf16_16816(z[i], dz2a[c2], ld_u32s(wrow + 16 * c2), ld_u32s(wrow + 16 * c2 + 8));
              const float2 ha = *reinterpret_cast<const float2*>(ws.h1 + g * (H1 + 8) + col);
              const float2 hb = *reinterpret_cast<const float2*>(ws.h1 + (g + 8) * (H1 + 8) + col);
              z[i][0] = v0 ? __fmul_rn(z[i][0], __fmul_rn(ha.x, __fsub_rn(1.f, ha.x))) : 0.f;
              z[i][1] = v0 ? __fmul_rn(z[i][1], __fmul_rn(ha.y, __fsub_rn(1.f, ha.y))) : 0.f;
              z[i][2] = v1 ? __fmul_rn(z[i][2], __fmul_rn(hb.x, __fsub_rn(1.f, hb.x))) : 0.f;
              z[i][3] = v1 ? __fmul_rn(z[i][3], __fmul_rn(hb.y, __fsub_rn(1.f, hb.y))) : 0.f;
#pragma unroll
              for (int cc = 0; cc < 2; ++cc) {
                const float sz = rows_sum(__fadd_rn(z[i][cc], z[i][2 + cc]));
                if (g == 0) ws.dhq[col + cc] = __fadd_rn(ws.dhq[col + cc], sz);
              }
            }
            dz1a[kc][0] = pack_bf16x2(z[0][0], z[0][1]);
            dz1a[kc][1] = pack_bf16x2(z[0][2], z[0][3]);
            dz1a[kc][2] = pack_bf16x2(z[1][0], z[1][1]);
            dz1a[kc][3] = pack_bf16x2(z[1][2], z[1][3]);
            __nv_bfloat16* zr = dz1h + (row0 + r0 + g) * H1 + 16 * kc + 2 * t;
            if (in0) { *reinterpret_cast<uint32_t*>(zr) = dz1a[kc][0]; *reinterpret_cast<uint32_t*>(zr + 8) = dz1a[kc][2]; }
            if (in1) { *reinterpret_cast<uint32_t*>(zr + 8 * H1) = dz1a[kc][1]; *reinterpret_cast<uint32_t*>(zr + 8 * H1 + 8) = dz1a[kc][3]; }
          }
        }
        // dX = bf16(dz1) [Wk | Wp]: dk = dX_k + q dX_p (+ w dout), dq += k dX_p
#pragma unroll 1
        for (int j = 0; j < D / 8; ++j) {
          float ak[4] = {0.f, 0.f, 0.f, 0.f}, ap[4] = {0.f, 0.f, 0.f, 0.f};
          const uint16_t* wk = sWkpT + (8 * j + g) * ly.PH1 + 2 * t;
          const uint16_t* wp = sWkpT + (D + 8 * j + g) * ly.PH1 + 2 * t;
#pragma unroll
          for (int kc = 0; kc < kDinMaxH1 / 16; ++kc)
            if (16 * kc < H1) {
              mma_bf16_16816(ak, dz1a[kc], ld_u32s(wk + 16 * kc), ld_u32s(wk + 16 * kc + 8));
              mma_bf16_16816(ap, dz1a[kc], ld_u32s(wp + 16 * kc), ld_u32s(wp + 16 * kc + 8));
            }
          const int col = 8 * j + 2 * t;
          float dqp[2] = {0.f, 0.f};
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const bool in = rr ? in1 : in0, v = rr ? v1 : v0;
            const int row = r0 + g + 8 * rr;
            if (!in) continue;
            float o[2] = {0.f, 0.f};
            if (v) {
              const float2 kv = ld2<KT>(kb + (int64_t)row * D + col);
#pragma unroll
              for (int cc = 0; cc < 2; ++cc) {
                const float dxp = ap[2 * rr + cc];
                o[cc] = __fmaf_rn(ws.q[col + cc], dxp, ak[2 * rr + cc]);
                if (mode == 0) o[cc] = __fmaf_rn(ws.s[row], ws.gd[col + cc], o[cc]);     // + w_t dout (ws.gd holds dout in mode 0 only)
                dqp[cc] = __fmaf_rn(cc ? kv.y : kv.x, dxp, dqp[cc]);
              }
            }
            st2<KT>(dk + (row0 + row) * D + col, o[0], o[1]);
          }
#pragma unroll
          for (int cc = 0; cc < 2; ++cc) {
            const float v = rows_sum(dqp[cc]);
            if (g == 0) ws.dqp[col + cc] = __fadd_rn(ws.dqp[col + cc], v);
          }
        }
      }
      // dq = Wq^T dhq + sum_t k_t dX_p,t
      __syncwarp();
      for (int d = lane; d < D; d += 32) {
        float a = 0.f;
        for (int h = 0; h < H1; ++h) a = __fmaf_rn(sWq[h * D + d], ws.dhq[h], a);
        dq[b * D + d] = __fadd_rn(a, ws.dqp[d]);
      }
    }
    // fold the warps' samples into the block accumulators in warp order
    __syncthreads();
    const int nw = (int)min((int64_t)kDinWarps, last - base);
    for (int e = threadIdx.x; e < nacc; e += blockDim.x) {
      float a = acc[e];
      for (int w = 0; w < nw; ++w) {
        const DinWarpSmem o = warp_smem(din_smem + ly.warp + w * ly.warp_bytes);
        if (e < H1 * D) a = __fmaf_rn(o.dhq[e / D], o.q[e % D], a);
        else if (e < H1 * D + H1) a = __fadd_rn(a, o.dhq[e - H1 * D]);
        else if (e < H1 * D + H1 + H2) a = __fadd_rn(a, o.db2[e - H1 * D - H1]);
        else a = __fadd_rn(a, o.dw3[e - H1 * D - H1 - H2]);
      }
      acc[e] = a;
    }
    __syncthreads();
  }
  for (int e = threadIdx.x; e < nacc; e += blockDim.x) part[(int64_t)blockIdx.x * nacc + e] = acc[e];
}

// dW1 [H1][4D] = [dWq | dWk | dWq - dWk | dWp] from dWq [H1][D] and [dWk | dWp] [H1][2D]
__global__ void k_din_att_dw1(const float* __restrict__ dwq, const float* __restrict__ dwkp, int H1, int D, float* __restrict__ dW1) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (int64_t)H1 * D) return;
  const int h = (int)(e / D), d = (int)(e % D);
  const float wq = dwq[e], wk = dwkp[(int64_t)h * 2 * D + d], wp = dwkp[(int64_t)h * 2 * D + D + d];
  float* row = dW1 + (int64_t)h * 4 * D;
  row[d] = wq;
  row[D + d] = wk;
  row[2 * D + d] = __fsub_rn(wq, wk);
  row[3 * D + d] = wp;
}

template <typename K>
int din_set_smem(K kernel, int bytes, DrPerDeviceOnce& once) {
  if (bytes > 48 * 1024 && !once()) {
    DR_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    once() = true;
  }
  return 0;
}

struct DinArgs {
  const float* q; const void* k; const uint8_t* mask; const float* g; int B, L, D, H1, H2;
  const float *W1, *b1, *W2, *b2, *w3; int mode;
};

template <int D, typename KT>
int din_fwd(const DinArgs& a, float* out, cudaStream_t s) {
  const DinLayout ly(D, a.H1, a.H2, false);
  static DrPerDeviceOnce once;                      // one per instantiation
  if (int rc = din_set_smem(k_din_att_fwd<D, KT>, ly.bytes, once)) return rc;
  const int grid = (a.B + din_spc(a.B) - 1) / din_spc(a.B);
  DR_PDL_LAUNCH((k_din_att_fwd<D, KT>), grid, 32 * kDinWarps, ly.bytes, s, a.q, (const KT*)a.k, a.mask, a.B, a.L, a.H1, a.H2, a.W1, a.b1, a.W2,
                a.b2, a.w3, a.mode, out);
  DR_LAUNCH_CHECK();
  return 0;
}

template <int D, typename KT>
int din_bwd(const DinArgs& a, float* dq, void* dk, __nv_bfloat16* scratch, float* part, cudaStream_t s) {
  const DinLayout ly(D, a.H1, a.H2, true);
  static DrPerDeviceOnce once;                      // one per instantiation
  if (int rc = din_set_smem(k_din_att_bwd<D, KT>, ly.bytes, once)) return rc;
  const int grid = (a.B + din_spc(a.B) - 1) / din_spc(a.B);
  const int64_t M = (int64_t)a.B * a.L;
  __nv_bfloat16* xh = scratch;
  __nv_bfloat16* h1h = xh + M * 2 * D;
  __nv_bfloat16* dz1h = h1h + M * a.H1;
  __nv_bfloat16* dz2h = dz1h + M * a.H1;
  DR_PDL_LAUNCH((k_din_att_bwd<D, KT>), grid, 32 * kDinWarps, ly.bytes, s, a.q, (const KT*)a.k, a.mask, a.g, a.B, a.L, a.H1, a.H2, a.W1, a.b1,
                a.W2, a.b2, a.w3, a.mode, dq, (KT*)dk, xh, h1h, dz1h, dz2h, part);
  DR_LAUNCH_CHECK();
  return 0;
}

template <typename KT>
int din_fwd_d(const DinArgs& a, float* out, cudaStream_t s) {
  switch (a.D) {
    case 16: return din_fwd<16, KT>(a, out, s);
    case 32: return din_fwd<32, KT>(a, out, s);
    case 48: return din_fwd<48, KT>(a, out, s);
    default: return din_fwd<64, KT>(a, out, s);
  }
}

template <typename KT>
int din_bwd_d(const DinArgs& a, float* dq, void* dk, __nv_bfloat16* scratch, float* part, cudaStream_t s) {
  switch (a.D) {
    case 16: return din_bwd<16, KT>(a, dq, dk, scratch, part, s);
    case 32: return din_bwd<32, KT>(a, dq, dk, scratch, part, s);
    case 48: return din_bwd<48, KT>(a, dq, dk, scratch, part, s);
    default: return din_bwd<64, KT>(a, dq, dk, scratch, part, s);
  }
}

int din_check(const DinArgs& a, int k_bf16) {
  if (!a.q || !a.k || !a.mask || !a.W1 || !a.b1 || !a.W2 || !a.b2 || !a.w3) return -1;
  if (a.D != 16 && a.D != 32 && a.D != 48 && a.D != 64) return -2;
  if (a.H1 < 16 || a.H1 > kDinMaxH1 || a.H1 % 16 || a.H2 < 8 || a.H2 > kDinMaxH2 || a.H2 % 8) return -2;
  if (a.L < 1 || a.L > kDinMaxL || a.B < 1 || (int64_t)a.B * a.L > INT32_MAX) return -2;
  if ((a.mode != 0 && a.mode != 1) || (k_bf16 != 0 && k_bf16 != 1)) return -2;
  if (((uintptr_t)a.q | (uintptr_t)a.k) & 15) return -4;
  return 0;
}

}  // namespace

extern "C" {

int dr_cuda_gemm_dw(const void* dY, int64_t ldy, const void* X, int64_t ldx, int batch, int N_out, int K_in, float* dW, int64_t ldw, int splits,
                    cudaStream_t s);                                                                          // gemm_wgmma.cu

// Forward of the DIN attention unit.  q fp32 [B][D]; k [B][L][D], bf16 (k_bf16 = 1) or fp32; mask uint8 / bool [B][L] (nonzero = valid);
// W1 fp32 [H1][4D], b1 [H1], W2 [H2][H1], b2 [H2], w3 [H2] (the last layer's bias is not needed).  mode 0: out fp32 [B][D] = sum_t w_t k_t;
// mode 1: out fp32 [B][L] = w.  Codes: -1 a null pointer; -2 a shape outside the limits above, or a bad mode / k_bf16; -4 q or k not 16-byte
// aligned.
int dr_cuda_din_att_fwd(const float* q, const void* k, int k_bf16, const uint8_t* mask, int B, int L, int D, const float* W1, const float* b1,
                        int H1, const float* W2, const float* b2, int H2, const float* w3, int mode, float* out, cudaStream_t s) {
  const DinArgs a{q, k, mask, nullptr, B, L, D, H1, H2, W1, b1, W2, b2, w3, mode};
  if (int rc = din_check(a, k_bf16)) return rc;
  if (!out) return -1;
  return k_bf16 ? din_fwd_d<__nv_bfloat16>(a, out, s) : din_fwd_d<float>(a, out, s);
}

// Backward of dr_cuda_din_att_fwd for the same inputs; g fp32 is dL/dout ([B][D] in mode 0, [B][L] in mode 1).  Writes dq fp32 [B][D], dk
// [B][L][D] in k's dtype (exactly 0 at masked positions), dW1 fp32 [H1][4D], db1 [H1], dW2 [H2][H1], db2 [H2], dw3 [H2] and db3 = 0 (one float).
// scratch: bf16, B L (2D + 2 H1 + H2) elements, 16-byte aligned (X, h1, dz1 and dz2 rows for the weight-gradient GEMMs).
int dr_cuda_din_att_bwd(const float* q, const void* k, int k_bf16, const uint8_t* mask, const float* g, int B, int L, int D, const float* W1,
                        const float* b1, int H1, const float* W2, const float* b2, int H2, const float* w3, int mode, float* dq, void* dk,
                        float* dW1, float* db1, float* dW2, float* db2, float* dw3, float* db3, void* scratch, cudaStream_t s) {
  const DinArgs a{q, k, mask, g, B, L, D, H1, H2, W1, b1, W2, b2, w3, mode};
  if (int rc = din_check(a, k_bf16)) return rc;
  if (!g || !dq || !dk || !dW1 || !db1 || !dW2 || !db2 || !dw3 || !db3 || !scratch) return -1;
  if (((uintptr_t)dk | (uintptr_t)scratch) & 15) return -4;
  const int grid = (B + din_spc(B) - 1) / din_spc(B);
  const int nacc = H1 * D + H1 + 2 * H2;
  // workspace: the blocks' partial rows [grid][nacc], then dWq [H1][D] and [dWk | dWp] [H1][2D]
  float* ws = dr_workspace(kWsDinAtt, (size_t)grid * nacc + 3 * (size_t)H1 * D, s);
  if (!ws) return -5;
  float* dwq = ws + (size_t)grid * nacc;
  float* dwkp = dwq + (size_t)H1 * D;
  DR_CUDA_CHECK(cudaMemsetAsync(dwq, 0, 3 * (size_t)H1 * D * sizeof(float), s));
  DR_CUDA_CHECK(cudaMemsetAsync(dW2, 0, (size_t)H2 * H1 * sizeof(float), s));
  DR_CUDA_CHECK(cudaMemsetAsync(db1, 0, (size_t)H1 * sizeof(float), s));
  DR_CUDA_CHECK(cudaMemsetAsync(db2, 0, (size_t)H2 * sizeof(float), s));
  DR_CUDA_CHECK(cudaMemsetAsync(dw3, 0, (size_t)H2 * sizeof(float), s));
  DR_CUDA_CHECK(cudaMemsetAsync(db3, 0, sizeof(float), s));
  __nv_bfloat16* sc = (__nv_bfloat16*)scratch;
  int rc = k_bf16 ? din_bwd_d<__nv_bfloat16>(a, dq, dk, sc, ws, s) : din_bwd_d<float>(a, dq, dk, sc, ws, s);
  if (rc) return rc;
  det_colsum(ws, grid, (int64_t)nacc, {{0, H1 * D, dwq}, {(int64_t)H1 * D, H1, db1}, {(int64_t)H1 * D + H1, H2, db2},
                                       {(int64_t)H1 * D + H1 + H2, H2, dw3}}, s);
  const int M = B * L;
  const __nv_bfloat16* xh = sc;
  const __nv_bfloat16* h1h = xh + (int64_t)M * 2 * D;
  const __nv_bfloat16* dz1h = h1h + (int64_t)M * H1;
  const __nv_bfloat16* dz2h = dz1h + (int64_t)M * H1;
  rc = dr_cuda_gemm_dw(dz1h, H1, xh, 2 * D, M, H1, 2 * D, dwkp, 2 * D, 0, s);     // [dWk | dWp] = bf16(dz1)^T X
  if (rc) return rc;
  rc = dr_cuda_gemm_dw(dz2h, H2, h1h, H1, M, H2, H1, dW2, H1, 0, s);            // dW2 = bf16(dz2)^T bf16(h1)
  if (rc) return rc;
  k_din_att_dw1<<<(H1 * D + 255) / 256, 256, 0, s>>>(dwq, dwkp, H1, D, dW1);
  DR_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
