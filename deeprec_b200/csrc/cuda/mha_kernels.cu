// Multi-head self-attention core for training: softmax(Q K^T / sqrt(dh) + key mask) V per (sample, head), forward and backward, as
// nn.MultiheadAttention computes it between its in_proj and out_proj (the same layout as the serving kernel k_prog_mha):
//
//   qkv   bf16 [B S][3E], [q | k | v] per token, head h in columns h dh .. (h + 1) dh of each part (the in_proj GEMM's output)
//   valid uint8 [B][S], a KEY-padding mask: key j of sample b takes part iff valid[b][j] != 0 (at any position, not only a tail)
//   o     bf16 [B S][E] (the out_proj GEMM's input),  do bf16 [B S][E],  dqkv bf16 [B S][3E] (the in_proj GEMM's dY)
//
// Semantics.  Every query row is computed, padded ones included (they attend to the valid keys, as PyTorch does).  A masked key gets a
// probability of exactly 0, so its dK and dV rows are exactly 0.  A sample with no valid key gives o = 0 and dq = 0 (PyTorch gives NaN).
//
// One warp owns one (sample, head) and walks its query tiles of 16 rows.  K and V are staged once in shared memory (bf16, zero rows past
// S), row-major and transposed, so every mma.sync fragment is one 32-bit shared load; the whole key row of a query tile (S padded to SP, a
// multiple of 16, <= 128) stays in registers, so the softmax needs no online rescaling.  Q K^T and dP = dO V^T contract over dh
// (m16n8k8 at dh = 8, m16n8k16 otherwise); P V, dQ = dS K contract over the keys, with the score accumulator tiles rounded to bf16 as the
// A fragment; dV = P^T dO and dK = dS^T Q contract over the 16 queries of the tile, with P^T, dS^T, dO^T and Q^T staged in shared memory.
// dK and dV accumulate over the query tiles in fp32 in shared memory (in registers they would take 2 SP dh / 32 = 256 per lane at
// SP = 128, dh = 32), each element by one lane in query-tile order: there are no atomics and every sum has a fixed order.
//
// Rounding points (tests/mha_cases.py mirrors them):
//   s  = fp32(mma(bf16 q, bf16 k)) * scale, scale = fp32(1 / sqrt(dh));  masked keys: -inf
//   m  = max_j s,  p_j = __expf(s_j - m),  l = sum_j p_j (fp32, lane-sequential over j then a 4-lane butterfly),  P = p * rcp(l)
//   o  = bf16(mma(bf16(P), bf16 v))
//   D  = sum_d do * o (fp32, from the bf16 do and o),  dP = mma(bf16 do, bf16 v),  dS = P (dP - D) * scale (fp32)
//   dq = bf16(mma(bf16(dS), k)),  dk = bf16(sum over tiles of mma(bf16(dS)^T, q)),  dv = bf16(sum over tiles of mma(bf16(P)^T, do))
// The backward recomputes P with the same function on the same operands, so its P is bit-identical to the forward's; it saves nothing
// beyond qkv, o and valid.
#include "common.cuh"
#include "mma_sync.cuh"

using namespace drc;

namespace {

constexpr int kMhaWarps = 4;                // warps per block (fewer where one warp's shared memory is large)
constexpr int kMhaSmemCap = 200 * 1024;     // dynamic shared memory per block we size the block against
constexpr int kQS = 24;                     // row pitch (bf16) of the [*][16] per-tile arrays: conflict-free fragment loads

template <int DH, int SP>
struct MhaShape {
  static constexpr int NT = SP / 8;         // n8 tiles of the keys (score columns)
  static constexpr int KT = SP / 16;        // k16 tiles of the keys
  static constexpr int DC = DH / 8;         // k8 chunks / n8 tiles of dh
  static constexpr int KS = (DH / 2) % 8 == 4 ? DH : DH + 8;   // row pitch (bf16) of [key][dh]: 4 mod 8 words, conflict-free
  static constexpr int TS = SP + 8;         // row pitch (bf16) of [dh][key]
  static constexpr int kFwdBytes = SP * KS * 2 + DH * TS * 2;                                       // K, V^T
  static constexpr int kBwdBytes = 2 * SP * DH * 4 + 2 * SP * KS * 2 + DH * TS * 2 + 2 * DH * kQS * 2 + 2 * SP * kQS * 2;
  // dK, dV (fp32), K, V, K^T, Q^T, dO^T, P^T, dS^T
};

__device__ __forceinline__ uint32_t ld_u32(const uint16_t* p) { return *reinterpret_cast<const uint32_t*>(p); }

// c += a b over dh: a[c] = A fragment of dh chunk c (rows g, g + 8), b[c] = B fragment of chunk c
template <int DH>
__device__ __forceinline__ void mma_dh(float (&c)[4], const uint32_t (&a)[DH / 8][2], const uint32_t (&b)[DH / 8]) {
  if constexpr (DH == 8) {
    mma_bf16_1688(c, a[0][0], a[0][1], b[0]);
  } else {
#pragma unroll
    for (int k = 0; k < DH / 16; ++k) {
      const uint32_t aa[4] = {a[2 * k][0], a[2 * k][1], a[2 * k + 1][0], a[2 * k + 1][1]};
      mma_bf16_16816(c, aa, b[2 * k], b[2 * k + 1]);
    }
  }
}

// A fragments over dh of rows r0 + g and r0 + g + 8 of one [rows][ld] bf16 operand (rows at or past S read as 0)
template <int DH>
__device__ __forceinline__ void load_rows_dh(const __nv_bfloat16* __restrict__ p, int64_t ld, int r0, int S, int g, int t, uint32_t (&a)[DH / 8][2]) {
#pragma unroll
  for (int c = 0; c < DH / 8; ++c) {
    a[c][0] = r0 + g < S ? *reinterpret_cast<const uint32_t*>(p + (int64_t)(r0 + g) * ld + 8 * c + 2 * t) : 0u;
    a[c][1] = r0 + g + 8 < S ? *reinterpret_cast<const uint32_t*>(p + (int64_t)(r0 + g + 8) * ld + 8 * c + 2 * t) : 0u;
  }
}

// rows 0..SP-1 of one head's [S][dh] slice (ld = 3E) into sRow [key][KS] and, if given, sT [dh][TS]; zero past S
template <int DH, int SP>
__device__ __forceinline__ void stage_keys(const __nv_bfloat16* __restrict__ p, int64_t ld, int S, int lane, uint16_t* sRow, uint16_t* sT) {
  using Sh = MhaShape<DH, SP>;
  for (int i = lane; i < SP * DH / 2; i += 32) {
    const int r = i / (DH / 2), c = 2 * (i % (DH / 2));
    const uint32_t v = r < S ? *reinterpret_cast<const uint32_t*>(p + (int64_t)r * ld + c) : 0u;
    if (sRow) *reinterpret_cast<uint32_t*>(sRow + r * Sh::KS + c) = v;
    if (sT) { sT[c * Sh::TS + r] = (uint16_t)(v & 0xffffu); sT[(c + 1) * Sh::TS + r] = (uint16_t)(v >> 16); }
  }
}

// bit 2 j + c: key 8 j + 2 t + c (this lane's score columns) is below S and valid
template <int SP>
__device__ __forceinline__ uint32_t key_bits(const uint8_t* __restrict__ valid, int S, int t) {
  uint32_t m = 0;
#pragma unroll
  for (int j = 0; j < SP / 8; ++j)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int key = 8 * j + 2 * t + c;
      if (key < S && valid[key]) m |= 1u << (2 * j + c);
    }
  return m;
}

// P [16 x SP] of one query tile in the accumulator layout (s[j][0..1]: row g, keys 8 j + 2 t + {0, 1}; s[j][2..3]: row g + 8).  Shared by
// the forward and the backward: the same instructions on the same operands give the same bits.  Masked keys, rows at or past S and rows
// with no valid key get P = 0.
template <int DH, int SP>
__device__ __forceinline__ void mha_probs(const uint32_t (&qa)[DH / 8][2], const uint16_t* sK, uint32_t kbits, float scale, bool live0,
                                          bool live1, int g, int t, float (&s)[SP / 8][4]) {
  using Sh = MhaShape<DH, SP>;
#pragma unroll
  for (int j = 0; j < Sh::NT; ++j) {
    uint32_t kb[Sh::DC];
#pragma unroll
    for (int c = 0; c < Sh::DC; ++c) kb[c] = ld_u32(sK + (8 * j + g) * Sh::KS + 8 * c + 2 * t);
    s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
    mma_dh<DH>(s[j], qa, kb);
  }
  float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
  for (int j = 0; j < Sh::NT; ++j)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      // + 0 for a valid key, + -inf (0xff800000) for a masked one: integer ops, no predicates to keep live
      const float bias = __uint_as_float((((kbits >> (2 * j + c)) & 1u) - 1u) & 0xff800000u);
      s[j][c] = __fadd_rn(__fmul_rn(s[j][c], scale), bias);
      s[j][2 + c] = __fadd_rn(__fmul_rn(s[j][2 + c], scale), bias);
      m0 = fmaxf(m0, s[j][c]);
      m1 = fmaxf(m1, s[j][2 + c]);
    }
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, o));
    m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, o));
  }
  // a row with no valid key: every s is -inf, and exp(-inf - 0) = 0
  m0 = m0 == -INFINITY ? 0.f : m0;
  m1 = m1 == -INFINITY ? 0.f : m1;
  float l0 = 0.f, l1 = 0.f;
#pragma unroll
  for (int j = 0; j < Sh::NT; ++j)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      s[j][c] = __expf(__fsub_rn(s[j][c], m0));            // masked keys: exp(-inf) = +0
      s[j][2 + c] = __expf(__fsub_rn(s[j][2 + c], m1));
      l0 = __fadd_rn(l0, s[j][c]);
      l1 = __fadd_rn(l1, s[j][2 + c]);
    }
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    l0 = __fadd_rn(l0, __shfl_xor_sync(0xffffffffu, l0, o));
    l1 = __fadd_rn(l1, __shfl_xor_sync(0xffffffffu, l1, o));
  }
  const float r0 = live0 && l0 > 0.f ? __frcp_rn(l0) : 0.f, r1 = live1 && l1 > 0.f ? __frcp_rn(l1) : 0.f;
#pragma unroll
  for (int j = 0; j < Sh::NT; ++j) {
    s[j][0] = __fmul_rn(s[j][0], r0); s[j][1] = __fmul_rn(s[j][1], r0);
    s[j][2] = __fmul_rn(s[j][2], r1); s[j][3] = __fmul_rn(s[j][3], r1);
  }
}

// k16 tile kt of a [16 x SP] accumulator-layout matrix, rounded to bf16, as an m16k16 A fragment
template <int SP>
__device__ __forceinline__ void acc_to_a(const float (&s)[SP / 8][4], int kt, uint32_t (&a)[4]) {
  a[0] = pack_bf16x2(s[2 * kt][0], s[2 * kt][1]);
  a[1] = pack_bf16x2(s[2 * kt][2], s[2 * kt][3]);
  a[2] = pack_bf16x2(s[2 * kt + 1][0], s[2 * kt + 1][1]);
  a[3] = pack_bf16x2(s[2 * kt + 1][2], s[2 * kt + 1][3]);
}

// out[16 x DH] = bf16(s) [16 x SP] X [SP x DH], X given transposed in shared memory (sT [dh][TS])
template <int DH, int SP>
__device__ __forceinline__ void acc_times_keys(const float (&s)[SP / 8][4], const uint16_t* sT, int g, int t, float (&out)[DH / 8][4]) {
  using Sh = MhaShape<DH, SP>;
#pragma unroll
  for (int d = 0; d < Sh::DC; ++d) out[d][0] = out[d][1] = out[d][2] = out[d][3] = 0.f;
#pragma unroll
  for (int kt = 0; kt < Sh::KT; ++kt) {
    uint32_t a[4];
    acc_to_a<SP>(s, kt, a);
#pragma unroll
    for (int d = 0; d < Sh::DC; ++d) {
      const uint16_t* p = sT + (8 * d + g) * Sh::TS + 16 * kt + 2 * t;
      mma_bf16_16816(out[d], a, ld_u32(p), ld_u32(p + 8));
    }
  }
}

// rows r0 + g, r0 + g + 8 (those below S) of a [16 x DH] accumulator, rounded to bf16, into dst (row pitch ld)
template <int DH>
__device__ __forceinline__ void store_rows(const float (&acc)[DH / 8][4], __nv_bfloat16* __restrict__ dst, int64_t ld, int r0, int S, int g, int t) {
#pragma unroll
  for (int d = 0; d < DH / 8; ++d) {
    if (r0 + g < S) *reinterpret_cast<uint32_t*>(dst + (int64_t)(r0 + g) * ld + 8 * d + 2 * t) = pack_bf16x2(acc[d][0], acc[d][1]);
    if (r0 + g + 8 < S) *reinterpret_cast<uint32_t*>(dst + (int64_t)(r0 + g + 8) * ld + 8 * d + 2 * t) = pack_bf16x2(acc[d][2], acc[d][3]);
  }
}

template <int DH, int SP>
__global__ void __launch_bounds__(32 * kMhaWarps, 1) k_mha_fwd(const __nv_bfloat16* __restrict__ qkv, const uint8_t* __restrict__ valid, int B, int S,
                                                            int E, int heads, float scale, __nv_bfloat16* __restrict__ o) {
  using Sh = MhaShape<DH, SP>;
  extern __shared__ __align__(16) unsigned char mha_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  uint16_t* sK = reinterpret_cast<uint16_t*>(mha_smem + warp * Sh::kFwdBytes);
  uint16_t* sVt = sK + SP * Sh::KS;
  pdl_sync();
  const int64_t pair = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
  if (pair >= (int64_t)B * heads) return;
  const int64_t b = pair / heads;
  const int h = (int)(pair % heads);
  const int64_t ld = 3 * (int64_t)E;
  const __nv_bfloat16* q = qkv + b * S * ld + h * DH;
  stage_keys<DH, SP>(q + E, ld, S, lane, sK, nullptr);
  stage_keys<DH, SP>(q + 2 * E, ld, S, lane, nullptr, sVt);
  const uint32_t kbits = key_bits<SP>(valid + b * S, S, t);
  __syncwarp();
  __nv_bfloat16* out = o + b * S * E + h * DH;
  for (int r0 = 0; r0 < S; r0 += 16) {
    uint32_t qa[Sh::DC][2];
    load_rows_dh<DH>(q, ld, r0, S, g, t, qa);
    float s[Sh::NT][4];
    mha_probs<DH, SP>(qa, sK, kbits, scale, r0 + g < S, r0 + g + 8 < S, g, t, s);
    float acc[Sh::DC][4];
    acc_times_keys<DH, SP>(s, sVt, g, t, acc);               // o = bf16(P) V
    store_rows<DH>(acc, out, E, r0, S, g, t);
  }
}

template <int DH, int SP>
__global__ void __launch_bounds__(32 * kMhaWarps, 1) k_mha_bwd(const __nv_bfloat16* __restrict__ qkv, const uint8_t* __restrict__ valid,
                                                            const __nv_bfloat16* __restrict__ o, const __nv_bfloat16* __restrict__ dout, int B,
                                                            int S, int E, int heads, float scale, __nv_bfloat16* __restrict__ dqkv) {
  using Sh = MhaShape<DH, SP>;
  extern __shared__ __align__(16) unsigned char mha_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  float4* sdK = reinterpret_cast<float4*>(mha_smem + warp * Sh::kBwdBytes);   // [(mt DC + d) 32 + lane]: accumulator tiles of dK
  float4* sdV = sdK + SP * DH / 4;
  uint16_t* sK = reinterpret_cast<uint16_t*>(sdV + SP * DH / 4);               // [key][KS]
  uint16_t* sV = sK + SP * Sh::KS;                                            // [key][KS]
  uint16_t* sKt = sV + SP * Sh::KS;                                           // [d][TS]
  uint16_t* sQt = sKt + DH * Sh::TS;                                          // [d][kQS]: Q^T of the tile
  uint16_t* sdOt = sQt + DH * kQS;                                            // [d][kQS]: dO^T of the tile
  uint16_t* sPt = sdOt + DH * kQS;                                            // [key][kQS]: bf16(P)^T of the tile
  uint16_t* sdSt = sPt + SP * kQS;                                            // [key][kQS]: bf16(dS)^T of the tile
  pdl_sync();
  const int64_t pair = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
  if (pair >= (int64_t)B * heads) return;
  const int64_t b = pair / heads;
  const int h = (int)(pair % heads);
  const int64_t ld = 3 * (int64_t)E;
  const __nv_bfloat16* q = qkv + b * S * ld + h * DH;
  const __nv_bfloat16* ob = o + b * S * E + h * DH;
  const __nv_bfloat16* dob = dout + b * S * E + h * DH;
  __nv_bfloat16* dq = dqkv + b * S * ld + h * DH;
  stage_keys<DH, SP>(q + E, ld, S, lane, sK, sKt);
  stage_keys<DH, SP>(q + 2 * E, ld, S, lane, sV, nullptr);
  for (int i = lane; i < SP * DH / 4; i += 32) sdK[i] = sdV[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  const uint32_t kbits = key_bits<SP>(valid + b * S, S, t);
  __syncwarp();
  for (int r0 = 0; r0 < S; r0 += 16) {
    uint32_t qa[Sh::DC][2], da[Sh::DC][2], oa[Sh::DC][2];
    load_rows_dh<DH>(q, ld, r0, S, g, t, qa);
    load_rows_dh<DH>(dob, E, r0, S, g, t, da);
    load_rows_dh<DH>(ob, E, r0, S, g, t, oa);
    // Q^T and dO^T of the tile; D = rowsum(dO (.) O)
    float D0 = 0.f, D1 = 0.f;
#pragma unroll
    for (int c = 0; c < Sh::DC; ++c) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int col = 8 * c + 2 * t, row = g + 8 * i;
        sQt[col * kQS + row] = (uint16_t)(qa[c][i] & 0xffffu); sQt[(col + 1) * kQS + row] = (uint16_t)(qa[c][i] >> 16);
        sdOt[col * kQS + row] = (uint16_t)(da[c][i] & 0xffffu); sdOt[(col + 1) * kQS + row] = (uint16_t)(da[c][i] >> 16);
      }
      const float2 d0 = unpack_bf16x2(da[c][0]), o0 = unpack_bf16x2(oa[c][0]), d1 = unpack_bf16x2(da[c][1]), o1 = unpack_bf16x2(oa[c][1]);
      D0 = __fmaf_rn(d0.y, o0.y, __fmaf_rn(d0.x, o0.x, D0));
      D1 = __fmaf_rn(d1.y, o1.y, __fmaf_rn(d1.x, o1.x, D1));
    }
#pragma unroll
    for (int s_ = 1; s_ <= 2; s_ <<= 1) {
      D0 = __fadd_rn(D0, __shfl_xor_sync(0xffffffffu, D0, s_));
      D1 = __fadd_rn(D1, __shfl_xor_sync(0xffffffffu, D1, s_));
    }
    float s[Sh::NT][4];
    mha_probs<DH, SP>(qa, sK, kbits, scale, r0 + g < S, r0 + g + 8 < S, g, t, s);
#pragma unroll
    for (int j = 0; j < Sh::NT; ++j) {
      // P^T into shared memory, then dS = P (dP - D) scale in place of P, dP = dO V^T
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int key = 8 * j + 2 * t + c;
        sPt[key * kQS + g] = __bfloat16_as_ushort(__float2bfloat16_rn(s[j][c]));
        sPt[key * kQS + g + 8] = __bfloat16_as_ushort(__float2bfloat16_rn(s[j][2 + c]));
      }
      uint32_t vb[Sh::DC];
#pragma unroll
      for (int c = 0; c < Sh::DC; ++c) vb[c] = ld_u32(sV + (8 * j + g) * Sh::KS + 8 * c + 2 * t);
      float dp[4] = {0.f, 0.f, 0.f, 0.f};
      mma_dh<DH>(dp, da, vb);
      s[j][0] = __fmul_rn(__fmul_rn(s[j][0], __fsub_rn(dp[0], D0)), scale);
      s[j][1] = __fmul_rn(__fmul_rn(s[j][1], __fsub_rn(dp[1], D0)), scale);
      s[j][2] = __fmul_rn(__fmul_rn(s[j][2], __fsub_rn(dp[2], D1)), scale);
      s[j][3] = __fmul_rn(__fmul_rn(s[j][3], __fsub_rn(dp[3], D1)), scale);
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int key = 8 * j + 2 * t + c;
        sdSt[key * kQS + g] = __bfloat16_as_ushort(__float2bfloat16_rn(s[j][c]));
        sdSt[key * kQS + g + 8] = __bfloat16_as_ushort(__float2bfloat16_rn(s[j][2 + c]));
      }
    }
    float acc[Sh::DC][4];
    acc_times_keys<DH, SP>(s, sKt, g, t, acc);               // dq = bf16(dS) K
    store_rows<DH>(acc, dq, ld, r0, S, g, t);
    __syncwarp();
    // dV += bf16(P)^T dO, dK += bf16(dS)^T Q over the 16 queries of the tile
#pragma unroll
    for (int mt = 0; mt < Sh::KT; ++mt) {
      const uint16_t* pp = sPt + (16 * mt + g) * kQS + 2 * t;
      const uint16_t* ps = sdSt + (16 * mt + g) * kQS + 2 * t;
      const uint32_t ap[4] = {ld_u32(pp), ld_u32(pp + 8 * kQS), ld_u32(pp + 8), ld_u32(pp + 8 * kQS + 8)};
      const uint32_t as[4] = {ld_u32(ps), ld_u32(ps + 8 * kQS), ld_u32(ps + 8), ld_u32(ps + 8 * kQS + 8)};
#pragma unroll
      for (int d = 0; d < Sh::DC; ++d) {
        const uint16_t* bo = sdOt + (8 * d + g) * kQS + 2 * t;
        const uint16_t* bq = sQt + (8 * d + g) * kQS + 2 * t;
        const int i = (mt * Sh::DC + d) * 32 + lane;
        float4 v = sdV[i], k = sdK[i];
        float cv[4] = {v.x, v.y, v.z, v.w}, ck[4] = {k.x, k.y, k.z, k.w};
        mma_bf16_16816(cv, ap, ld_u32(bo), ld_u32(bo + 8));
        mma_bf16_16816(ck, as, ld_u32(bq), ld_u32(bq + 8));
        sdV[i] = make_float4(cv[0], cv[1], cv[2], cv[3]);
        sdK[i] = make_float4(ck[0], ck[1], ck[2], ck[3]);
      }
    }
    __syncwarp();
  }
  // dK, dV rows below S
#pragma unroll
  for (int mt = 0; mt < Sh::KT; ++mt) {
    float ak[Sh::DC][4], av[Sh::DC][4];
#pragma unroll
    for (int d = 0; d < Sh::DC; ++d) {
      const float4 k = sdK[(mt * Sh::DC + d) * 32 + lane], v = sdV[(mt * Sh::DC + d) * 32 + lane];
      ak[d][0] = k.x; ak[d][1] = k.y; ak[d][2] = k.z; ak[d][3] = k.w;
      av[d][0] = v.x; av[d][1] = v.y; av[d][2] = v.z; av[d][3] = v.w;
    }
    store_rows<DH>(ak, dq + E, ld, 16 * mt, S, g, t);
    store_rows<DH>(av, dq + 2 * E, ld, 16 * mt, S, g, t);
  }
}

// warps per block: kMhaWarps, halved while one block's shared memory exceeds kMhaSmemCap
inline int mha_warps(int per_warp) {
  int w = kMhaWarps;
  while (w > 1 && w * per_warp > kMhaSmemCap) w >>= 1;
  return w;
}

template <typename K>
int mha_set_smem(K kernel, int bytes, DrPerDeviceOnce& once) {
  if (bytes > 48 * 1024 && !once()) {
    DR_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    once() = true;
  }
  return 0;
}

template <int DH, int SP>
int mha_fwd(const void* qkv, const uint8_t* valid, int B, int S, int E, int heads, float scale, void* o, cudaStream_t s) {
  const int per = MhaShape<DH, SP>::kFwdBytes, w = mha_warps(per);
  static DrPerDeviceOnce once;
  if (int rc = mha_set_smem(k_mha_fwd<DH, SP>, w * per, once)) return rc;
  const int64_t grid = ((int64_t)B * heads + w - 1) / w;
  DR_PDL_LAUNCH((k_mha_fwd<DH, SP>), (unsigned)grid, 32 * w, w * per, s, (const __nv_bfloat16*)qkv, valid, B, S, E, heads, scale,
                (__nv_bfloat16*)o);
  DR_LAUNCH_CHECK();
  return 0;
}

template <int DH, int SP>
int mha_bwd(const void* qkv, const uint8_t* valid, const void* o, const void* dout, int B, int S, int E, int heads, float scale, void* dqkv,
            cudaStream_t s) {
  const int per = MhaShape<DH, SP>::kBwdBytes, w = mha_warps(per);
  static DrPerDeviceOnce once;
  if (int rc = mha_set_smem(k_mha_bwd<DH, SP>, w * per, once)) return rc;
  const int64_t grid = ((int64_t)B * heads + w - 1) / w;
  DR_PDL_LAUNCH((k_mha_bwd<DH, SP>), (unsigned)grid, 32 * w, w * per, s, (const __nv_bfloat16*)qkv, valid, (const __nv_bfloat16*)o,
                (const __nv_bfloat16*)dout, B, S, E, heads, scale, (__nv_bfloat16*)dqkv);
  DR_LAUNCH_CHECK();
  return 0;
}

// one instantiation per (dh, S rounded up to 16)
template <int DH, template <int, int> class F, typename... A>
int mha_dispatch_sp(int S, A... args) {
  switch ((S + 15) / 16) {
    case 1: return F<DH, 16>::run(args...);
    case 2: return F<DH, 32>::run(args...);
    case 3: return F<DH, 48>::run(args...);
    case 4: return F<DH, 64>::run(args...);
    case 5: return F<DH, 80>::run(args...);
    case 6: return F<DH, 96>::run(args...);
    case 7: return F<DH, 112>::run(args...);
    default: return F<DH, 128>::run(args...);
  }
}

template <int DH, int SP>
struct FwdOp {
  static int run(const void* qkv, const uint8_t* valid, int B, int S, int E, int heads, float scale, void* o, cudaStream_t s) {
    return mha_fwd<DH, SP>(qkv, valid, B, S, E, heads, scale, o, s);
  }
};

template <int DH, int SP>
struct BwdOp {
  static int run(const void* qkv, const uint8_t* valid, const void* o, const void* dout, int B, int S, int E, int heads, float scale, void* dqkv,
                 cudaStream_t s) {
    return mha_bwd<DH, SP>(qkv, valid, o, dout, B, S, E, heads, scale, dqkv, s);
  }
};

int mha_check(const void* qkv, const void* valid, int B, int S, int E, int heads, const void* a, const void* b) {
  if (!qkv || !valid || !a || !b) return -1;
  if (heads < 1 || E < 1 || E % heads) return -2;
  const int dh = E / heads;
  if ((dh != 8 && dh != 16 && dh != 32) || S < 1 || S > 128) return -2;
  if (B < 1 || (int64_t)B * S > INT32_MAX) return -3;
  if (((uintptr_t)qkv | (uintptr_t)a | (uintptr_t)b) & 15) return -4;
  return 0;
}

}  // namespace

extern "C" {

// o = softmax(q k^T / sqrt(dh) + key mask) v per (sample, head).  qkv bf16 [B S][3E] ([q | k | v] per token), valid uint8 [B][S] (key mask),
// o bf16 [B S][E].  dh = E / heads in {8, 16, 32}, 1 <= S <= 128; -2 otherwise.
int dr_cuda_mha_fwd(const void* qkv, const uint8_t* valid, int B, int S, int E, int heads, void* o, cudaStream_t s) {
  int rc = mha_check(qkv, valid, B, S, E, heads, o, o);
  if (rc) return rc;
  const int dh = E / heads;
  const float scale = 1.0f / sqrtf((float)dh);
  if (dh == 8) return mha_dispatch_sp<8, FwdOp>(S, qkv, valid, B, S, E, heads, scale, o, s);
  if (dh == 16) return mha_dispatch_sp<16, FwdOp>(S, qkv, valid, B, S, E, heads, scale, o, s);
  return mha_dispatch_sp<32, FwdOp>(S, qkv, valid, B, S, E, heads, scale, o, s);
}

// Backward of dr_cuda_mha_fwd for the same qkv, valid and its o; do bf16 [B S][E].  Writes dqkv bf16 [B S][3E] ([dq | dk | dv]).
int dr_cuda_mha_bwd(const void* qkv, const uint8_t* valid, const void* o, const void* dout, int B, int S, int E, int heads, void* dqkv, cudaStream_t s) {
  int rc = mha_check(qkv, valid, B, S, E, heads, o, dqkv);
  if (rc) return rc;
  if (!dout) return -1;
  if ((uintptr_t)dout & 15) return -4;
  const int dh = E / heads;
  const float scale = 1.0f / sqrtf((float)dh);
  if (dh == 8) return mha_dispatch_sp<8, BwdOp>(S, qkv, valid, o, dout, B, S, E, heads, scale, dqkv, s);
  if (dh == 16) return mha_dispatch_sp<16, BwdOp>(S, qkv, valid, o, dout, B, S, E, heads, scale, dqkv, s);
  return mha_dispatch_sp<32, BwdOp>(S, qkv, valid, o, dout, B, S, E, heads, scale, dqkv, s);
}

}  // extern "C"
