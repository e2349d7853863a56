// GRU recurrence for training: PyTorch's single-layer GRU (gate order r, z, n; h_0 = 0) over tail-padded sequences.
//
//   r = sigmoid(gi_r + W_hr h + b_hr),  z = sigmoid(gi_z + W_hz h + b_hz),  n = tanh(gi_n + r * (W_hn h + b_hn)),  h' = (1 - z) n + z h
//
// The input projection gi = x W_ih^T + b_ih is one GEMM over all B L rows (nn.FusedMLP's wgmma kernel, whose backward gives dx, dW_ih and
// db_ih); these kernels run the sequential part.  Sample b runs len[b] steps: y[b, t] = h_t for t < len[b] and exactly 0 past it, as
// tf.nn.dynamic_rnn(..., sequence_length=) gives (reference modelzoo/dien/train.py:491-534).
//
// One warp owns 16 samples and computes h W_hh^T [16 x 3H x H] with mma.sync.m16n8k16 (bf16 operands, fp32 accumulators).  Because H is a
// multiple of 8, gate columns j, H + j and 2H + j of the accumulator tiles sit in the same lane and register slot, so the gate math is
// lane-local; and two adjacent n8 accumulator tiles of h, rounded to bf16, are exactly the m16k16 A fragment of the next step's product.
// A forward step therefore needs no shared memory traffic beyond the W_hh fragments, no shuffles and no barriers.  The state stays fp32;
// it is rounded to bf16 only as a matmul operand.
//
// Saved for the backward: y itself (fp32 h_t, 4 H bytes per sample-step).  The backward reads h_{t-1} from it and recomputes the gates with
// the same instructions on the same operands, so they are bit-identical to the forward's.  It runs through time in reverse with the carry
//   dh_{t-1} = dgh_t W_hh + z (.) dh_t,   dgh = [da_r, da_z, da_n (.) r],   dgi = [da_r, da_z, da_n]
// (the product again on mma.sync, dgh rounded to bf16 as its operand), and writes dgi, dgh and bf16(h_{t-1}) row for row.  dW_hh and db_hh
// are then the split-K weight-gradient GEMM dgh^T bf16(h_{t-1}) and the column sums of dgh (dr_cuda_gemm_dw / dr_cuda_colstats): every sum
// has a fixed order, so two runs and a graph replay give the same bits.
#include "common.cuh"
#include "mma_sync.cuh"

using namespace drc;

namespace {

constexpr int kGruWarps = 4;        // warps per block, 16 samples per warp

__device__ __forceinline__ float gru_sigmoid(float x) { return __frcp_rn(__fadd_rn(1.f, __expf(-x))); }
// 1 - 2 / (1 + e^2x): absolute error a few fp32 ulps (tanh.approx, what tanhf becomes under --use_fast_math, is good to about 2^-11 only)
__device__ __forceinline__ float gru_tanh(float x) { return __fsub_rn(1.f, __fmul_rn(2.f, __frcp_rn(__fadd_rn(1.f, __expf(2.f * x))))); }

// the gates from gi (bf16 -> fp32) and gh = W_hh h + b_hh; shared by the forward and the backward's recomputation
__device__ __forceinline__ void gru_gates(float gir, float giz, float gin, float ghr, float ghz, float ghn, float& r, float& z, float& n) {
  r = gru_sigmoid(__fadd_rn(gir, ghr));
  z = gru_sigmoid(__fadd_rn(giz, ghz));
  n = gru_tanh(__fmaf_rn(r, ghn, gin));
}

template <int H>
struct GruShape {
  static constexpr int NT = 3 * H / 8;   // n8 tiles of the 3H gate columns
  static constexpr int KT = H / 16;      // k16 tiles of h
  static constexpr int JT = H / 8;       // n8 tiles of h
  static constexpr int GT = 3 * H / 16;  // k16 tiles of the 3H gate columns
};

// W_hh (fp32 [3H][H]) -> bf16 B fragments in shared memory, one uint2 per lane and tile:
//   sWf[(nt KT + kt) 32 + lane]: B[k][n] = W_hh[n][k] for h W_hh^T (k over h, n over the gate columns)
//   sWb[(jt GT + kt) 32 + lane]: B[k][n] = W_hh[k][n] for dgh W_hh   (k over the gate columns, n over h)
template <int H>
__device__ void gru_load_frags(const float* __restrict__ W, uint2* sWf, uint2* sWb) {
  using S = GruShape<H>;
  for (int i = threadIdx.x; i < S::NT * S::KT * 32; i += blockDim.x) {
    const int lane = i & 31, f = i >> 5, nt = f / S::KT, kt = f % S::KT;
    const int n = 8 * nt + (lane >> 2), k = 16 * kt + 2 * (lane & 3);
    const float* w = W + (int64_t)n * H + k;
    sWf[i] = make_uint2(pack_bf16x2(w[0], w[1]), pack_bf16x2(w[8], w[9]));
  }
  if (sWb) {
    for (int i = threadIdx.x; i < S::JT * S::GT * 32; i += blockDim.x) {
      const int lane = i & 31, f = i >> 5, jt = f / S::GT, kt = f % S::GT;
      const int n = 8 * jt + (lane >> 2), k = 16 * kt + 2 * (lane & 3);
      const float* w = W + (int64_t)k * H + n;
      sWb[i] = make_uint2(pack_bf16x2(w[0], w[H]), pack_bf16x2(w[8 * H], w[9 * H]));
    }
  }
}

// gh[nt] = b_hh + bf16(h) W_hh^T for the warp's 16 rows; h[jt][e] is the C-fragment layout of the state
template <int H>
__device__ __forceinline__ void gru_gh(const float (&h)[H / 8][4], const float (&bias)[3 * H / 8][2], const uint2* __restrict__ sWf, int lane,
                                       float (&gh)[3 * H / 8][4]) {
  using S = GruShape<H>;
  uint32_t a[S::KT][4];
#pragma unroll
  for (int kt = 0; kt < S::KT; ++kt) {
    a[kt][0] = pack_bf16x2(h[2 * kt][0], h[2 * kt][1]);
    a[kt][1] = pack_bf16x2(h[2 * kt][2], h[2 * kt][3]);
    a[kt][2] = pack_bf16x2(h[2 * kt + 1][0], h[2 * kt + 1][1]);
    a[kt][3] = pack_bf16x2(h[2 * kt + 1][2], h[2 * kt + 1][3]);
  }
#pragma unroll
  for (int nt = 0; nt < S::NT; ++nt) {
    gh[nt][0] = gh[nt][2] = bias[nt][0];
    gh[nt][1] = gh[nt][3] = bias[nt][1];
#pragma unroll
    for (int kt = 0; kt < S::KT; ++kt) {
      const uint2 b = sWf[(nt * S::KT + kt) * 32 + lane];
      mma_bf16_16816(gh[nt], a[kt], b.x, b.y);
    }
  }
}

// the warp's 16 samples: row (g, g + 8) of the fragments; rows at or past B have length 0.  Returns the longest length of the warp.
__device__ __forceinline__ int gru_rows(const int32_t* __restrict__ len, int64_t b0, int B, int L, int g, int64_t (&row)[2], int (&lr)[2]) {
  int lw = 0;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    row[i] = b0 + g + 8 * i;
    lr[i] = row[i] < B ? min(max(len[row[i]], 0), L) : 0;
    lw = max(lw, lr[i]);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) lw = max(lw, __shfl_xor_sync(0xffffffffu, lw, o));
  return lw;
}

template <int H>
__global__ void __launch_bounds__(32 * kGruWarps) k_gru_fwd(const __nv_bfloat16* __restrict__ gi, const float* __restrict__ w_hh,
                                                            const float* __restrict__ b_hh, const int32_t* __restrict__ len, int B, int L,
                                                            float* __restrict__ y) {
  using S = GruShape<H>;
  __shared__ uint2 sWf[S::NT * S::KT * 32];
  pdl_sync();
  gru_load_frags<H>(w_hh, sWf, nullptr);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tq = lane & 3;
  const int64_t b0 = ((int64_t)blockIdx.x * kGruWarps + warp) * 16;
  if (b0 >= B) return;
  int64_t row[2]; int lr[2];
  const int lw = gru_rows(len, b0, B, L, g, row, lr);
  float bias[S::NT][2];
#pragma unroll
  for (int nt = 0; nt < S::NT; ++nt) { bias[nt][0] = b_hh[8 * nt + 2 * tq]; bias[nt][1] = b_hh[8 * nt + 2 * tq + 1]; }
  float h[S::JT][4];
#pragma unroll
  for (int jt = 0; jt < S::JT; ++jt) h[jt][0] = h[jt][1] = h[jt][2] = h[jt][3] = 0.f;
  for (int t = 0; t < lw; ++t) {
    uint32_t x[2][S::JT][3];                          // gi (r, z, n) at the lane's two columns of each h tile, both rows
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const __nv_bfloat16* p = gi + (row[i] * L + t) * (3 * H) + 2 * tq;
#pragma unroll
      for (int jt = 0; jt < S::JT; ++jt)
#pragma unroll
        for (int q = 0; q < 3; ++q) x[i][jt][q] = t < lr[i] ? *reinterpret_cast<const uint32_t*>(p + q * H + 8 * jt) : 0u;
    }
    float gh[S::NT][4];
    gru_gh<H>(h, bias, sWf, lane, gh);
#pragma unroll
    for (int jt = 0; jt < S::JT; ++jt) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float2 xr = unpack_bf16x2(x[i][jt][0]), xz = unpack_bf16x2(x[i][jt][1]), xn = unpack_bf16x2(x[i][jt][2]);
        float out[2];
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int e = 2 * i + c;
          float r, z, n;
          gru_gates(c ? xr.y : xr.x, c ? xz.y : xz.x, c ? xn.y : xn.x, gh[jt][e], gh[S::JT + jt][e], gh[2 * S::JT + jt][e], r, z, n);
          if (t < lr[i]) h[jt][e] = __fmaf_rn(z, __fsub_rn(h[jt][e], n), n);     // (1 - z) n + z h; a finished sample keeps its state
          out[c] = t < lr[i] ? h[jt][e] : 0.f;
        }
        if (row[i] < B) *reinterpret_cast<float2*>(y + (row[i] * L + t) * H + 8 * jt + 2 * tq) = make_float2(out[0], out[1]);
      }
    }
  }
  // steps past the warp's longest sample: zeros
  const int nrow = B - b0 < 16 ? (int)(B - b0) : 16, per_row = (L - lw) * H / 4;
  for (int i = lane; i < nrow * per_row; i += 32) {
    const int r = i / per_row, c = i % per_row;
    reinterpret_cast<float4*>(y + ((b0 + r) * L + lw) * H)[c] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

template <int H>
__global__ void __launch_bounds__(32 * kGruWarps) k_gru_bwd(const __nv_bfloat16* __restrict__ gi, const float* __restrict__ w_hh,
                                                            const float* __restrict__ b_hh, const int32_t* __restrict__ len,
                                                            const float* __restrict__ y, const float* __restrict__ dy, int B, int L,
                                                            __nv_bfloat16* __restrict__ dgi, __nv_bfloat16* __restrict__ dgh,
                                                            __nv_bfloat16* __restrict__ hprev) {
  using S = GruShape<H>;
  __shared__ uint2 sWf[S::NT * S::KT * 32];
  __shared__ uint2 sWb[S::JT * S::GT * 32];
  pdl_sync();
  gru_load_frags<H>(w_hh, sWf, sWb);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tq = lane & 3;
  const int64_t b0 = ((int64_t)blockIdx.x * kGruWarps + warp) * 16;
  if (b0 >= B) return;
  int64_t row[2]; int lr[2];
  const int lw = gru_rows(len, b0, B, L, g, row, lr);
  {
    // steps past the warp's longest sample: zero rows of dgi, dgh and h_{t-1}
    const int nrow = B - b0 < 16 ? (int)(B - b0) : 16, per_row = (L - lw) * (3 * H) / 8, per_rowh = (L - lw) * H / 8;
    const int4 z4 = make_int4(0, 0, 0, 0);
    for (int i = lane; i < nrow * per_row; i += 32) {
      const int r = i / per_row, c = i % per_row;
      reinterpret_cast<int4*>(dgi + ((b0 + r) * L + lw) * (3 * H))[c] = z4;
      reinterpret_cast<int4*>(dgh + ((b0 + r) * L + lw) * (3 * H))[c] = z4;
    }
    for (int i = lane; i < nrow * per_rowh; i += 32) {
      const int r = i / per_rowh, c = i % per_rowh;
      reinterpret_cast<int4*>(hprev + ((b0 + r) * L + lw) * H)[c] = z4;
    }
  }
  float bias[S::NT][2];
#pragma unroll
  for (int nt = 0; nt < S::NT; ++nt) { bias[nt][0] = b_hh[8 * nt + 2 * tq]; bias[nt][1] = b_hh[8 * nt + 2 * tq + 1]; }
  float dh[S::JT][4];                                   // dL/dh_t: dy[t] plus the carry from step t + 1
#pragma unroll
  for (int jt = 0; jt < S::JT; ++jt) dh[jt][0] = dh[jt][1] = dh[jt][2] = dh[jt][3] = 0.f;
  for (int t = lw - 1; t >= 0; --t) {
    float h[S::JT][4];
    uint32_t x[2][S::JT][3];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const bool live = t < lr[i];
      const int64_t o = row[i] * L + t;
#pragma unroll
      for (int jt = 0; jt < S::JT; ++jt) {
        const int col = 8 * jt + 2 * tq;
        const float2 hp = live && t > 0 ? *reinterpret_cast<const float2*>(y + (o - 1) * H + col) : make_float2(0.f, 0.f);
        const float2 d = live ? *reinterpret_cast<const float2*>(dy + o * H + col) : make_float2(0.f, 0.f);
        h[jt][2 * i] = hp.x; h[jt][2 * i + 1] = hp.y;
        dh[jt][2 * i] = live ? __fadd_rn(dh[jt][2 * i], d.x) : 0.f;
        dh[jt][2 * i + 1] = live ? __fadd_rn(dh[jt][2 * i + 1], d.y) : 0.f;
#pragma unroll
        for (int q = 0; q < 3; ++q) x[i][jt][q] = live ? *reinterpret_cast<const uint32_t*>(gi + o * (3 * H) + q * H + col) : 0u;
      }
    }
    float gh[S::NT][4];
    gru_gh<H>(h, bias, sWf, lane, gh);
    float da[S::NT][4];                                 // dgh as it enters the carry product: [da_r, da_z, da_n r]
#pragma unroll
    for (int jt = 0; jt < S::JT; ++jt) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float2 xr = unpack_bf16x2(x[i][jt][0]), xz = unpack_bf16x2(x[i][jt][1]), xn = unpack_bf16x2(x[i][jt][2]);
        float ar[2], az[2], an[2];
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int e = 2 * i + c;
          float r, z, n;
          const float ghn = gh[2 * S::JT + jt][e];
          gru_gates(c ? xr.y : xr.x, c ? xz.y : xz.x, c ? xn.y : xn.x, gh[jt][e], gh[S::JT + jt][e], ghn, r, z, n);
          const float d = dh[jt][e];
          const float dn = __fmul_rn(d, __fsub_rn(1.f, z));
          const float dz = __fmul_rn(d, __fsub_rn(h[jt][e], n));
          an[c] = __fmul_rn(dn, __fsub_rn(1.f, __fmul_rn(n, n)));
          az[c] = __fmul_rn(dz, __fmul_rn(z, __fsub_rn(1.f, z)));
          ar[c] = __fmul_rn(__fmul_rn(an[c], ghn), __fmul_rn(r, __fsub_rn(1.f, r)));
          da[jt][e] = ar[c]; da[S::JT + jt][e] = az[c]; da[2 * S::JT + jt][e] = __fmul_rn(an[c], r);
          dh[jt][e] = __fmul_rn(z, d);                  // the direct term of the carry; the product is added below
        }
        if (row[i] < B) {
          const int64_t o = row[i] * L + t;
          const int col = 8 * jt + 2 * tq;
          const bool live = t < lr[i];
          uint32_t* pi = reinterpret_cast<uint32_t*>(dgi + o * (3 * H) + col);
          uint32_t* ph = reinterpret_cast<uint32_t*>(dgh + o * (3 * H) + col);
          const uint32_t vr = live ? pack_bf16x2(ar[0], ar[1]) : 0u, vz = live ? pack_bf16x2(az[0], az[1]) : 0u;
          pi[0] = vr; pi[H / 2] = vz; pi[H] = live ? pack_bf16x2(an[0], an[1]) : 0u;
          ph[0] = vr; ph[H / 2] = vz; ph[H] = live ? pack_bf16x2(da[2 * S::JT + jt][2 * i], da[2 * S::JT + jt][2 * i + 1]) : 0u;
          *reinterpret_cast<uint32_t*>(hprev + o * H + col) = live ? pack_bf16x2(h[jt][2 * i], h[jt][2 * i + 1]) : 0u;
        }
      }
    }
    // dh_{t-1} = bf16(dgh) W_hh + z dh_t
    uint32_t a[S::GT][4];
#pragma unroll
    for (int kt = 0; kt < S::GT; ++kt) {
      a[kt][0] = pack_bf16x2(da[2 * kt][0], da[2 * kt][1]);
      a[kt][1] = pack_bf16x2(da[2 * kt][2], da[2 * kt][3]);
      a[kt][2] = pack_bf16x2(da[2 * kt + 1][0], da[2 * kt + 1][1]);
      a[kt][3] = pack_bf16x2(da[2 * kt + 1][2], da[2 * kt + 1][3]);
    }
#pragma unroll
    for (int jt = 0; jt < S::JT; ++jt) {
      float c[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int kt = 0; kt < S::GT; ++kt) {
        const uint2 b = sWb[(jt * S::GT + kt) * 32 + lane];
        mma_bf16_16816(c, a[kt], b.x, b.y);
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) dh[jt][e] = __fadd_rn(c[e], dh[jt][e]);
    }
  }
}

template <int H>
int gru_fwd(const void* gi, const float* w_hh, const float* b_hh, const int32_t* len, int B, int L, float* y, cudaStream_t s) {
  const int grid = (B + 16 * kGruWarps - 1) / (16 * kGruWarps);
  DR_PDL_LAUNCH((k_gru_fwd<H>), grid, 32 * kGruWarps, 0, s, (const __nv_bfloat16*)gi, w_hh, b_hh, len, B, L, y);
  DR_LAUNCH_CHECK();
  return 0;
}

template <int H>
int gru_bwd(const void* gi, const float* w_hh, const float* b_hh, const int32_t* len, const float* y, const float* dy, int B, int L, void* dgi,
            void* dgh, void* hprev, cudaStream_t s) {
  const int grid = (B + 16 * kGruWarps - 1) / (16 * kGruWarps);
  DR_PDL_LAUNCH((k_gru_bwd<H>), grid, 32 * kGruWarps, 0, s, (const __nv_bfloat16*)gi, w_hh, b_hh, len, y, dy, B, L, (__nv_bfloat16*)dgi,
                (__nv_bfloat16*)dgh, (__nv_bfloat16*)hprev);
  DR_LAUNCH_CHECK();
  return 0;
}

int gru_check(const void* gi, const float* w_hh, const float* b_hh, const int32_t* len, int B, int L, int H, const void* a, const void* b) {
  if (!gi || !w_hh || !b_hh || !len || !a || !b) return -1;
  if (H != 16 && H != 32 && H != 48 && H != 64) return -2;
  if (B < 1 || L < 1 || (int64_t)B * L > INT32_MAX) return -3;
  if (((uintptr_t)gi | (uintptr_t)a | (uintptr_t)b) & 15) return -4;
  return 0;
}

}  // namespace

extern "C" {

int dr_cuda_gemm_dw(const void* dY, int64_t ldy, const void* X, int64_t ldx, int batch, int N_out, int K_in, float* dW, int64_t ldw, int splits,
                    cudaStream_t s);                                                                          // gemm_wgmma.cu
int dr_cuda_colstats(const void* u, const void* v, int64_t B, int N, int64_t ldu, int64_t ldv, float* S1, float* S2, cudaStream_t s);   // dense_kernels.cu

// gi: bf16 [B L][3H] (x W_ih^T + b_ih); w_hh fp32 [3H][H], b_hh fp32 [3H]; len int32 [B] on the device (clamped to 0..L).
// y: fp32 [B][L][H], h_t for t < len[b] and 0 past it.  H in {16, 32, 48, 64}.
int dr_cuda_gru_fwd(const void* gi, const float* w_hh, const float* b_hh, const int32_t* len, int B, int L, int H, float* y, cudaStream_t s) {
  int rc = gru_check(gi, w_hh, b_hh, len, B, L, H, y, y);
  if (rc) return rc;
  switch (H) {
    case 16: return gru_fwd<16>(gi, w_hh, b_hh, len, B, L, y, s);
    case 32: return gru_fwd<32>(gi, w_hh, b_hh, len, B, L, y, s);
    case 48: return gru_fwd<48>(gi, w_hh, b_hh, len, B, L, y, s);
    default: return gru_fwd<64>(gi, w_hh, b_hh, len, B, L, y, s);
  }
}

// Backward of dr_cuda_gru_fwd for the same gi, w_hh, b_hh, len and its y; dy fp32 [B][L][H].
// Writes dgi bf16 [B L][3H] (0 past the length) and, as scratch, dgh bf16 [B L][3H] and hprev bf16 [B L][H]; adds the weight gradients into
// dw_hh fp32 [3H][H] and db_hh fp32 [3H].
int dr_cuda_gru_bwd(const void* gi, const float* w_hh, const float* b_hh, const int32_t* len, const float* y, const float* dy, int B, int L, int H,
                    void* dgi, void* dgh, void* hprev, float* dw_hh, float* db_hh, cudaStream_t s) {
  int rc = gru_check(gi, w_hh, b_hh, len, B, L, H, dgi, dgh);
  if (rc) return rc;
  if (!y || !dy || !hprev || !dw_hh || !db_hh) return -1;
  if (((uintptr_t)y | (uintptr_t)dy | (uintptr_t)hprev) & 15) return -4;
  switch (H) {
    case 16: rc = gru_bwd<16>(gi, w_hh, b_hh, len, y, dy, B, L, dgi, dgh, hprev, s); break;
    case 32: rc = gru_bwd<32>(gi, w_hh, b_hh, len, y, dy, B, L, dgi, dgh, hprev, s); break;
    case 48: rc = gru_bwd<48>(gi, w_hh, b_hh, len, y, dy, B, L, dgi, dgh, hprev, s); break;
    default: rc = gru_bwd<64>(gi, w_hh, b_hh, len, y, dy, B, L, dgi, dgh, hprev, s); break;
  }
  if (rc) return rc;
  const int M = B * L;
  rc = dr_cuda_gemm_dw(dgh, 3 * H, hprev, H, M, 3 * H, H, dw_hh, H, 0, s);      // dW_hh += dgh^T bf16(h_{t-1})
  if (rc) return rc;
  return dr_cuda_colstats(dgh, nullptr, M, 3 * H, 3 * H, 3 * H, db_hh, nullptr, s);
}

}  // extern "C"
