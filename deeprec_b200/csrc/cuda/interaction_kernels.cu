// Feature-interaction kernels: DLRM pairwise dot (strict lower triangle of F F^T, concatenated with the
// dense vector), DeepFM second-order FM term, DIN attention pooling.  One warp per sample; lane i owns
// feature row i in registers, rows are broadcast through shared memory.
//
// Reference: modelzoo/dlrm/train.py:121-133 (_dot_op: matmul + boolean_mask), modelzoo/deepfm/train.py:178-187,
// modelzoo/din/train.py:143-188.  The interaction is a batch of 27x16 Gram matrices -- 23 kFLOP per sample
// against 1.6 kB of traffic -- so it is HBM-bound by two orders of magnitude; it reads the embedding rows
// exactly once, straight from the (peer-written) feature-major receive buffer, and emits the padded bf16
// activation the wgmma top-MLP GEMM consumes through TMA.
#include "sp_sync.cuh"

using namespace drc;

namespace {

template <int D>
__device__ __forceinline__ void load_row_bf16(const __nv_bfloat16* p, float (&f)[D]) {
#pragma unroll
  for (int c = 0; c < D; c += 8) {
    int4 raw = ld_nc_v4(p + c);
    const uint32_t w[4] = {(uint32_t)raw.x, (uint32_t)raw.y, (uint32_t)raw.z, (uint32_t)raw.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) { float2 v = unpack_bf16x2(w[e]); f[c + 2 * e] = v.x; f[c + 2 * e + 1] = v.y; }
  }
}
template <int D>
__device__ __forceinline__ void store_row_bf16(__nv_bfloat16* p, const float (&f)[D]) {
#pragma unroll
  for (int c = 0; c < D; c += 8) {
    int4 pk;
    pk.x = (int)pack_bf16x2(f[c], f[c + 1]); pk.y = (int)pack_bf16x2(f[c + 2], f[c + 3]);
    pk.z = (int)pack_bf16x2(f[c + 4], f[c + 5]); pk.w = (int)pack_bf16x2(f[c + 6], f[c + 7]);
    *reinterpret_cast<int4*>(p + c) = pk;
  }
}

// Z[b] = [ x[b] (D) | { <F_i, F_j> : 0 <= j < i < F } | 0-pad ],  F_0 = x[b], F_t = emb[t-1][b]
template <int D>
__global__ void __launch_bounds__(256) k_dot_fwd(const __nv_bfloat16* __restrict__ x, int64_t ldx, const __nv_bfloat16* __restrict__ emb,
                                                 int64_t emb_stride_t, int64_t emb_stride_b, int T, int64_t B,
                                                 __nv_bfloat16* __restrict__ Z, int64_t ldz) {
  constexpr int WPB = 8;
  __shared__ __align__(16) float sF[WPB][32][D];
  __shared__ __align__(16) __nv_bfloat16 sZ[WPB][512];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int F = T + 1;
  for (int64_t b = (int64_t)blockIdx.x * WPB + warp; b < B; b += (int64_t)gridDim.x * WPB) {
    float f[D];
    if (lane < F) {
      const __nv_bfloat16* src = lane == 0 ? x + b * ldx : emb + (int64_t)(lane - 1) * emb_stride_t + b * emb_stride_b;
      load_row_bf16<D>(src, f);
#pragma unroll
      for (int c = 0; c < D; c += 4) *reinterpret_cast<float4*>(&sF[warp][lane][c]) = make_float4(f[c], f[c + 1], f[c + 2], f[c + 3]);
      if (lane == 0) {
#pragma unroll
        for (int c = 0; c < D; ++c) sZ[warp][c] = __float2bfloat16(f[c]);
      }
    }
    __syncwarp();
    const int base = D + lane * (lane - 1) / 2;
    for (int j = 0; j < F - 1; ++j) {
      float g = 0.f;
#pragma unroll
      for (int c = 0; c < D; c += 4) {
        float4 v = *reinterpret_cast<const float4*>(&sF[warp][j][c]);
        g += f[c] * v.x + f[c + 1] * v.y + f[c + 2] * v.z + f[c + 3] * v.w;
      }
      if (lane < F && j < lane) sZ[warp][base + j] = __float2bfloat16(g);
    }
    const int used = D + F * (F - 1) / 2;
    for (int c = used + lane; c < ldz; c += 32) sZ[warp][c] = __float2bfloat16(0.f);
    __syncwarp();
    for (int c = lane * 8; c < ldz; c += 256)
      *reinterpret_cast<int4*>(Z + b * ldz + c) = *reinterpret_cast<const int4*>(&sZ[warp][c]);
    __syncwarp();
  }
}

// dF_i = sum_{j != i} S_ij F_j (+ dZ[0:D] for i = 0),  S symmetric from the lower-triangle grads.
template <int D>
__global__ void __launch_bounds__(256) k_dot_bwd(const __nv_bfloat16* __restrict__ dZ, int64_t ldz, const __nv_bfloat16* __restrict__ x,
                                                 int64_t ldx, const __nv_bfloat16* __restrict__ emb, int64_t emb_stride_t,
                                                 int64_t emb_stride_b, int T, int64_t B, __nv_bfloat16* __restrict__ dx, int64_t lddx,
                                                 __nv_bfloat16* __restrict__ demb, int64_t demb_stride_t, int64_t demb_stride_b) {
  constexpr int WPB = 8;
  __shared__ __align__(16) float sF[WPB][32][D];
  __shared__ __align__(16) float sG[WPB][512];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int F = T + 1;
  const int used = D + F * (F - 1) / 2;
  for (int64_t b = (int64_t)blockIdx.x * WPB + warp; b < B; b += (int64_t)gridDim.x * WPB) {
    float f[D];
    if (lane < F) {
      const __nv_bfloat16* src = lane == 0 ? x + b * ldx : emb + (int64_t)(lane - 1) * emb_stride_t + b * emb_stride_b;
      load_row_bf16<D>(src, f);
#pragma unroll
      for (int c = 0; c < D; c += 4) *reinterpret_cast<float4*>(&sF[warp][lane][c]) = make_float4(f[c], f[c + 1], f[c + 2], f[c + 3]);
    }
    for (int c = lane * 8; c < ldz; c += 256) {
      int4 raw = ld_nc_v4(dZ + b * ldz + c);
      const uint32_t w[4] = {(uint32_t)raw.x, (uint32_t)raw.y, (uint32_t)raw.z, (uint32_t)raw.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) { float2 v = unpack_bf16x2(w[e]); sG[warp][c + 2 * e] = v.x; sG[warp][c + 2 * e + 1] = v.y; }
    }
    __syncwarp();
    float acc[D];
#pragma unroll
    for (int c = 0; c < D; ++c) acc[c] = (lane == 0) ? sG[warp][c] : 0.f;
    const int mybase = D + lane * (lane - 1) / 2;
    for (int j = 0; j < F; ++j) {
      float s = 0.f;
      if (lane < F) {
        if (j < lane) s = sG[warp][mybase + j];
        else if (j > lane) s = sG[warp][D + j * (j - 1) / 2 + lane];
      }
#pragma unroll
      for (int c = 0; c < D; c += 4) {
        float4 v = *reinterpret_cast<const float4*>(&sF[warp][j][c]);
        acc[c] += s * v.x; acc[c + 1] += s * v.y; acc[c + 2] += s * v.z; acc[c + 3] += s * v.w;
      }
    }
    (void)used;
    if (lane == 0) store_row_bf16<D>(dx + b * lddx, acc);
    else if (lane < F) store_row_bf16<D>(demb + (int64_t)(lane - 1) * demb_stride_t + b * demb_stride_b, acc);
    __syncwarp();
  }
}

// -------------------------------------------------------------------------------------------------
// DeepFM second-order term: fm[b, :] = 0.5 * ((sum_t e_t)^2 - sum_t e_t^2)  and its backward
//   d e_t = dfm * (sum_t e - e_t).   emb: [T][B][D] bf16 (strided), out fp32/bf16 [B, D].
// -------------------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(256) k_fm_fwd(const __nv_bfloat16* __restrict__ emb, int64_t st, int64_t sb, int T, int64_t B,
                                                __nv_bfloat16* __restrict__ out, int64_t ldo, float* __restrict__ sum_out) {
  constexpr int LPR = D / 8;                 // lanes per sample (8 elements per lane)
  const int lane = threadIdx.x % LPR;
  const int64_t gid = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / LPR;
  const int64_t gstride = (int64_t)gridDim.x * blockDim.x / LPR;
  for (int64_t b = gid; b < B; b += gstride) {
    float s[8], q[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] = q[j] = 0.f;
    for (int t = 0; t < T; ++t) {
      float f[8];
      load_row_bf16<8>(emb + t * st + b * sb + lane * 8, f);
#pragma unroll
      for (int j = 0; j < 8; ++j) { s[j] += f[j]; q[j] += f[j] * f[j]; }
    }
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = 0.5f * (s[j] * s[j] - q[j]);
    store_row_bf16<8>(out + b * ldo + lane * 8, o);
    if (sum_out) {
#pragma unroll
      for (int j = 0; j < 8; ++j) sum_out[b * D + lane * 8 + j] = s[j];
    }
  }
}
template <int D>
__global__ void __launch_bounds__(256) k_fm_bwd(const __nv_bfloat16* __restrict__ dfm, int64_t ldd, const __nv_bfloat16* __restrict__ emb,
                                                int64_t st, int64_t sb, const float* __restrict__ sum_in, int T, int64_t B,
                                                __nv_bfloat16* __restrict__ demb, int64_t dst, int64_t dsb, int accumulate) {
  constexpr int LPR = D / 8;
  const int lane = threadIdx.x % LPR;
  const int64_t gid = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / LPR;
  const int64_t gstride = (int64_t)gridDim.x * blockDim.x / LPR;
  for (int64_t b = gid; b < B; b += gstride) {
    float g[8], s[8];
    load_row_bf16<8>(dfm + b * ldd + lane * 8, g);
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] = sum_in[b * D + lane * 8 + j];
    for (int t = 0; t < T; ++t) {
      float f[8], o[8];
      load_row_bf16<8>(emb + t * st + b * sb + lane * 8, f);
      if (accumulate) load_row_bf16<8>(demb + t * dst + b * dsb + lane * 8, o);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (accumulate ? o[j] : 0.f) + g[j] * (s[j] - f[j]);
      store_row_bf16<8>(demb + t * dst + b * dsb + lane * 8, o);
    }
  }
}


#ifndef DR_CUDA_EMU   // warp-level tensor-core MMA: hardware only (the emulation build runs the SIMT kernels above for every shape)
// =================================================================================================
// Tensor-core versions (D = 16, T + 1 <= 32): one warp per sample, the sample's 32 (padded) feature rows staged in shared memory.
//   forward :  G = F F^T [32 x 32 x 16] with six mma.sync.m16n8k16 (the 16 x 8 tiles on or below the diagonal); every lane scatters
//              the strict lower-triangle elements of its accumulator fragments into the sample's Z row.
//   backward:  dF = S F [32 x 16 x 32] with S the symmetric 32 x 32 gradient matrix of the sample (eight mma.sync.m16n8k16);
//              lane i then owns dF_i.
// The SIMT kernels above remain as the general-shape fallback.
// =================================================================================================
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// INDIRECT: `emb` is the requester-side unique-row buffer urow[gs][16] (written by the owners over NVLink) and feature t of sample b
// is row inv[b][t] of it (-1 = padding -> zeros); the kernel first waits for every owner's ROWS flag (sp_sync.cuh).
template <bool INDIRECT>
__global__ void __launch_bounds__(128) k_dot_fwd_tc(const __nv_bfloat16* __restrict__ x, int64_t ldx, const __nv_bfloat16* __restrict__ emb,
                                                    int64_t emb_stride_t, int64_t emb_stride_b, int T, int64_t B,
                                                    __nv_bfloat16* __restrict__ Z, int64_t ldz, const int32_t* __restrict__ inv, int ldinv,
                                                    DrSpSync sync) {
  pdl_sync();
  if (INDIRECT) sp_wait_all(sync, SP_CH_ROWS);
  constexpr int D = 16;
  __shared__ __align__(16) uint8_t sF[4][32 * 32];           // per warp: [32 feature rows][16 bf16]
  __shared__ __align__(16) __nv_bfloat16 sZ[4][512];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gI = lane >> 2, tI = lane & 3;                    // mma.sync fragment coordinates
  const int F = T + 1;
  uint8_t* myF = sF[warp];
  const int64_t stride = (int64_t)gridDim.x * 4;
  // software pipeline: the row of sample b + stride is fetched into registers while sample b is in the tensor core / epilogue
  int4 c0 = make_int4(0, 0, 0, 0), c1 = c0;
  int32_t gsn = -1;                                   // INDIRECT: row index of my feature for the NEXT sample to fetch
  auto fetch_idx = [&](int64_t bb) {
    gsn = (lane >= 1 && lane < F && bb < B) ? inv[bb * ldinv + lane - 1] : -1;
  };
  auto fetch = [&](int64_t bb, int4& r0, int4& r1) {
    r0 = r1 = make_int4(0, 0, 0, 0);
    if (lane < F && bb < B) {
      if (INDIRECT) {
        if (lane == 0) { r0 = ld_nc_v4(x + bb * ldx); r1 = ld_nc_v4(x + bb * ldx + 8); }
        else if (gsn >= 0) { const __nv_bfloat16* src = emb + (int64_t)gsn * D; r0 = ld_v4_volatile(src); r1 = ld_v4_volatile(src + 8); }
      } else {
        const __nv_bfloat16* src = lane == 0 ? x + bb * ldx : emb + (int64_t)(lane - 1) * emb_stride_t + bb * emb_stride_b;
        r0 = ld_nc_v4(src); r1 = ld_nc_v4(src + 8);
      }
    }
    if (INDIRECT) {
      fetch_idx(bb + stride);                         // index of the sample after this one: in flight for a whole iteration
    } else {
      // two more samples ahead: L2 prefetch only (one sample of register loads per warp cannot cover the DRAM latency)
      const int64_t pb = bb + 2 * stride;
      if (lane < F && pb < B) prefetch_l2(lane == 0 ? x + pb * ldx : emb + (int64_t)(lane - 1) * emb_stride_t + pb * emb_stride_b);
    }
  };
  const int64_t first = (int64_t)blockIdx.x * 4 + warp;
  if (INDIRECT) fetch_idx(first);
  fetch(first, c0, c1);
  for (int64_t b = first; b < B; b += stride) {
    *reinterpret_cast<int4*>(myF + lane * 32) = c0;
    *reinterpret_cast<int4*>(myF + lane * 32 + 16) = c1;
    if (lane == 0) { *reinterpret_cast<int4*>(&sZ[warp][0]) = c0; *reinterpret_cast<int4*>(&sZ[warp][8]) = c1; }
    fetch(b + stride, c0, c1);
    __syncwarp();
    uint32_t af[2][4], bf[4][2];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi) {
      const uint8_t* r0 = myF + (16 * mi + gI) * 32 + 4 * tI;
      af[mi][0] = *reinterpret_cast<const uint32_t*>(r0);
      af[mi][1] = *reinterpret_cast<const uint32_t*>(r0 + 8 * 32);
      af[mi][2] = *reinterpret_cast<const uint32_t*>(r0 + 16);
      af[mi][3] = *reinterpret_cast<const uint32_t*>(r0 + 8 * 32 + 16);
    }
#pragma unroll
    for (int ni = 0; ni < 4; ++ni) {
      const uint8_t* r0 = myF + (8 * ni + gI) * 32 + 4 * tI;
      bf[ni][0] = *reinterpret_cast<const uint32_t*>(r0);
      bf[ni][1] = *reinterpret_cast<const uint32_t*>(r0 + 16);
    }
#pragma unroll
    for (int mi = 0; mi < 2; ++mi) {
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) {
        if (8 * ni > 16 * mi + 15) continue;            // tile entirely above the diagonal (compile-time)
        float c[4] = {0.f, 0.f, 0.f, 0.f};
        mma_bf16_16816(c, af[mi], bf[ni][0], bf[ni][1]);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int fi = 16 * mi + gI + 8 * (e >> 1), j = 8 * ni + 2 * tI + (e & 1);
          if (j < fi && fi < F) sZ[warp][D + fi * (fi - 1) / 2 + j] = __float2bfloat16(c[e]);
        }
      }
    }
    const int used = D + F * (F - 1) / 2;
    for (int c = used + lane; c < ldz; c += 32) sZ[warp][c] = __float2bfloat16(0.f);
    __syncwarp();
    for (int c = lane * 8; c < ldz; c += 256)
      *reinterpret_cast<int4*>(Z + b * ldz + c) = *reinterpret_cast<const int4*>(&sZ[warp][c]);
    __syncwarp();                                      // the staging tiles are rewritten by the next sample
  }
}

// INDIRECT: features come from urow[inv[b][t]] (unique-first pipeline); the per-sample gradient rows still go to the feature-major
// demb buffer, which k_sp_segsum (sparse_pipeline.cu) pre-reduces per distinct key on the side stream.
template <bool INDIRECT>
__global__ void __launch_bounds__(128) k_dot_bwd_tc(const __nv_bfloat16* __restrict__ dZ, int64_t ldz, const __nv_bfloat16* __restrict__ x,
                                                    int64_t ldx, const __nv_bfloat16* __restrict__ emb, int64_t emb_stride_t,
                                                    int64_t emb_stride_b, int T, int64_t B, __nv_bfloat16* __restrict__ dx, int64_t lddx,
                                                    __nv_bfloat16* __restrict__ demb, int64_t demb_stride_t, int64_t demb_stride_b,
                                                    const int32_t* __restrict__ inv, int ldinv) {
  pdl_sync();
  constexpr int D = 16;
  __shared__ __align__(16) __nv_bfloat16 sG[4][512];         // per warp: the sample's dZ row
  __shared__ __align__(16) __nv_bfloat16 sS[4][32 * 32];     // per warp: S row-major [i][j]
  __shared__ __align__(16) __nv_bfloat16 sFt[4][16 * 32];    // per warp: F^T [d][j]
  __shared__ __align__(16) float sO[4][32 * 17];             // per warp: dF [i][d] (padded rows)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gI = lane >> 2, tI = lane & 3;
  const int F = T + 1;
  __nv_bfloat16* myG = sG[warp];
  const int64_t stride = (int64_t)gridDim.x * 4;
  // software pipeline: dZ chunks + the feature row of sample b + stride are fetched while sample b is being processed
  int4 pz0 = make_int4(0, 0, 0, 0), pz1 = pz0, pf0 = pz0, pf1 = pz0;
  int32_t gsn = -1;                                   // INDIRECT: row index of my feature for the NEXT sample to fetch
  auto fetch_idx = [&](int64_t bb) {
    gsn = (lane >= 1 && lane < F && bb < B) ? inv[bb * ldinv + lane - 1] : -1;
  };
  auto fetch = [&](int64_t bb) {
    pz0 = pz1 = pf0 = pf1 = make_int4(0, 0, 0, 0);
    if (bb < B) {
      if (lane * 8 < ldz) pz0 = ld_nc_v4(dZ + bb * ldz + lane * 8);
      if (lane * 8 + 256 < ldz) pz1 = ld_nc_v4(dZ + bb * ldz + lane * 8 + 256);
      if (lane < F) {
        if (INDIRECT) {
          if (lane == 0) { pf0 = ld_nc_v4(x + bb * ldx); pf1 = ld_nc_v4(x + bb * ldx + 8); }
          else if (gsn >= 0) {
            const __nv_bfloat16* src = emb + (int64_t)gsn * D;
            pf0 = ld_nc_v4(src); pf1 = ld_nc_v4(src + 8);
          }
        } else {
          const __nv_bfloat16* src = lane == 0 ? x + bb * ldx : emb + (int64_t)(lane - 1) * emb_stride_t + bb * emb_stride_b;
          pf0 = ld_nc_v4(src); pf1 = ld_nc_v4(src + 8);
        }
      }
    }
    if (INDIRECT) fetch_idx(bb + stride);
    // two more samples ahead: L2 prefetch only (one sample of register loads per warp cannot cover the DRAM latency)
    const int64_t pb = bb + 2 * stride;
    if (pb < B) {
      if (lane * 8 < ldz) prefetch_l2(dZ + pb * ldz + lane * 8);
      if (lane * 8 + 256 < ldz) prefetch_l2(dZ + pb * ldz + lane * 8 + 256);
      if (!INDIRECT && lane < F) prefetch_l2(lane == 0 ? x + pb * ldx : emb + (int64_t)(lane - 1) * emb_stride_t + pb * emb_stride_b);
    }
  };
  const int64_t first = (int64_t)blockIdx.x * 4 + warp;
  if (INDIRECT) fetch_idx(first);
  fetch(first);
  for (int64_t b = first; b < B; b += stride) {
    // ---- stage the dZ row and F^T from the prefetched registers (lanes >= F hold zeros)
    if (lane * 8 < ldz) *reinterpret_cast<int4*>(myG + lane * 8) = pz0;
    if (lane * 8 + 256 < ldz) *reinterpret_cast<int4*>(myG + lane * 8 + 256) = pz1;
    {
      const int4 c0 = pf0, c1 = pf1;
      const uint32_t w[8] = {(uint32_t)c0.x, (uint32_t)c0.y, (uint32_t)c0.z, (uint32_t)c0.w, (uint32_t)c1.x, (uint32_t)c1.y, (uint32_t)c1.z, (uint32_t)c1.w};
      uint16_t* ft = reinterpret_cast<uint16_t*>(sFt[warp]);
#pragma unroll
      for (int d = 0; d < 16; ++d) ft[d * 32 + lane] = (d & 1) ? (uint16_t)(w[d >> 1] >> 16) : (uint16_t)(w[d >> 1] & 0xFFFF);
    }
    fetch(b + stride);
    __syncwarp();
    // ---- my row of S: S[i][j] = dG[max][min], zero on the diagonal / padding
    {
      uint32_t packed[16];
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        uint32_t lo = 0, hi = 0;
        const int j0 = 2 * jj, j1 = 2 * jj + 1;
        if (lane < F) {
          if (j0 < F && j0 != lane) { const int hiI = max(lane, j0), loI = min(lane, j0); lo = *reinterpret_cast<const uint16_t*>(myG + D + hiI * (hiI - 1) / 2 + loI); }
          if (j1 < F && j1 != lane) { const int hiI = max(lane, j1), loI = min(lane, j1); hi = *reinterpret_cast<const uint16_t*>(myG + D + hiI * (hiI - 1) / 2 + loI); }
        }
        packed[jj] = lo | (hi << 16);
      }
      int4* row = reinterpret_cast<int4*>(sS[warp] + lane * 32);
#pragma unroll
      for (int c = 0; c < 4; ++c) row[c] = make_int4((int)packed[4 * c], (int)packed[4 * c + 1], (int)packed[4 * c + 2], (int)packed[4 * c + 3]);
    }
    __syncwarp();
    // ---- dF = S F on the tensor cores
    const uint8_t* S8 = reinterpret_cast<const uint8_t*>(sS[warp]);
    const uint8_t* Ft8 = reinterpret_cast<const uint8_t*>(sFt[warp]);
#pragma unroll
    for (int mi = 0; mi < 2; ++mi) {
#pragma unroll
      for (int ni = 0; ni < 2; ++ni) {
        float c[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int ki = 0; ki < 2; ++ki) {
          const uint8_t* a0 = S8 + (16 * mi + gI) * 64 + 32 * ki + 4 * tI;
          const uint32_t a[4] = {*reinterpret_cast<const uint32_t*>(a0), *reinterpret_cast<const uint32_t*>(a0 + 8 * 64),
                                 *reinterpret_cast<const uint32_t*>(a0 + 16), *reinterpret_cast<const uint32_t*>(a0 + 8 * 64 + 16)};
          const uint8_t* b0 = Ft8 + (8 * ni + gI) * 64 + 32 * ki + 4 * tI;
          mma_bf16_16816(c, a, *reinterpret_cast<const uint32_t*>(b0), *reinterpret_cast<const uint32_t*>(b0 + 16));
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) sO[warp][(16 * mi + gI + 8 * (e >> 1)) * 17 + 8 * ni + 2 * tI + (e & 1)] = c[e];
      }
    }
    __syncwarp();
    if (b < B && lane < F) {
      float acc[16];
#pragma unroll
      for (int d = 0; d < 16; ++d) acc[d] = sO[warp][lane * 17 + d];
      if (lane == 0) {
#pragma unroll
        for (int d = 0; d < 16; ++d) acc[d] += __bfloat162float(myG[d]);
        store_row_bf16<16>(dx + b * lddx, acc);
      } else {
        store_row_bf16<16>(demb + (int64_t)(lane - 1) * demb_stride_t + b * demb_stride_b, acc);
      }
    }
    __syncwarp();                                      // the staging tiles are rewritten by the next sample
  }
}

#endif  // DR_CUDA_EMU

inline int grid_for(int64_t n, int block, int max_blocks = num_sms() * 8) {
  int64_t b = (n + block - 1) / block;
  if (b < 1) b = 1;
  if (b > max_blocks) b = max_blocks;
  return (int)b;
}

}  // namespace

#ifdef DR_CUDA_EMU
static int& dot_force_simt() { static int v = 1; return v; }
#else
static int& dot_force_simt() { static int v = 0; return v; }
#endif

extern "C" {

int dr_cuda_dot_set_simt(int v) { dot_force_simt() = v; return 0; }

// unique-first pipeline variants: features gathered from urow through inv (fwd), gradients pre-reduced into ugrad (bwd)
int dr_cuda_dot_interaction_fwd_u(const void* x, int64_t ldx, const void* urow, const int32_t* inv, int ldinv, int T, int D, int64_t B, void* Z,
                                  int64_t ldz, const DrSpSync* sync, cudaStream_t s) {
  if (T + 1 > 32 || ldz > 512 || ldz % 8 || D + (T + 1) * T / 2 > ldz || D != 16) return -2;
#ifdef DR_CUDA_EMU
  return -100;
#else
  int g = grid_for((B + 3) / 4, 1, num_sms() * 4);
  DR_PDL_LAUNCH((k_dot_fwd_tc<true>), g, 128, 0, s, (const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)urow, 0, 0, T, B, (__nv_bfloat16*)Z, ldz, inv, ldinv, *sync);
  DR_LAUNCH_CHECK();
  return 0;
#endif
}

int dr_cuda_dot_interaction_bwd_u(const void* dZ, int64_t ldz, const void* x, int64_t ldx, const void* urow, const int32_t* inv, int ldinv,
                                  int T, int D, int64_t B, void* dx, int64_t lddx, void* demb, int64_t demb_stride_t, int64_t demb_stride_b,
                                  cudaStream_t s) {
  if (T + 1 > 32 || ldz > 512 || ldz % 8 || D != 16) return -2;
#ifdef DR_CUDA_EMU
  return -100;
#else
  int g = grid_for((B + 3) / 4, 1, num_sms() * 4);
  DR_PDL_LAUNCH((k_dot_bwd_tc<true>), g, 128, 0, s, (const __nv_bfloat16*)dZ, ldz, (const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)urow, 0, 0, T, B,
                (__nv_bfloat16*)dx, lddx, (__nv_bfloat16*)demb, demb_stride_t, demb_stride_b, inv, ldinv);
  DR_LAUNCH_CHECK();
  return 0;
#endif
}

int dr_cuda_dot_interaction_fwd(const void* x, int64_t ldx, const void* emb, int64_t emb_stride_t, int64_t emb_stride_b, int T, int D,
                                int64_t B, void* Z, int64_t ldz, cudaStream_t s) {
  if (T + 1 > 32 || ldz > 512 || ldz % 8 || D + (T + 1) * T / 2 > ldz) return -2;
#ifndef DR_CUDA_EMU
  if (D == 16 && !dot_force_simt()) {
    int g = grid_for((B + 3) / 4, 1, num_sms() * 4);
    DR_PDL_LAUNCH((k_dot_fwd_tc<false>), g, 128, 0, s, (const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)emb, emb_stride_t, emb_stride_b, T, B, (__nv_bfloat16*)Z, ldz,
                  (const int32_t*)nullptr, 0, DrSpSync{});
    DR_LAUNCH_CHECK();
    return 0;
  }
#endif
  int grid = grid_for((B + 7) / 8, 1, num_sms() * 6);
  switch (D) {
    case 8: k_dot_fwd<8><<<grid, 256, 0, s>>>((const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)emb, emb_stride_t, emb_stride_b, T, B, (__nv_bfloat16*)Z, ldz); break;
    case 16: k_dot_fwd<16><<<grid, 256, 0, s>>>((const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)emb, emb_stride_t, emb_stride_b, T, B, (__nv_bfloat16*)Z, ldz); break;
    case 32: k_dot_fwd<32><<<grid, 256, 0, s>>>((const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)emb, emb_stride_t, emb_stride_b, T, B, (__nv_bfloat16*)Z, ldz); break;
    default: return -3;
  }
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_dot_interaction_bwd(const void* dZ, int64_t ldz, const void* x, int64_t ldx, const void* emb, int64_t emb_stride_t,
                                int64_t emb_stride_b, int T, int D, int64_t B, void* dx, int64_t lddx, void* demb, int64_t demb_stride_t,
                                int64_t demb_stride_b, cudaStream_t s) {
  if (T + 1 > 32 || ldz > 512 || ldz % 8) return -2;
#ifndef DR_CUDA_EMU
  if (D == 16 && !dot_force_simt()) {
    int g = grid_for((B + 3) / 4, 1, num_sms() * 4);
    DR_PDL_LAUNCH((k_dot_bwd_tc<false>), g, 128, 0, s, (const __nv_bfloat16*)dZ, ldz, (const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)emb, emb_stride_t, emb_stride_b, T, B,
                                       (__nv_bfloat16*)dx, lddx, (__nv_bfloat16*)demb, demb_stride_t, demb_stride_b, (const int32_t*)nullptr, 0);
    DR_LAUNCH_CHECK();
    return 0;
  }
#endif
  int grid = grid_for((B + 7) / 8, 1, num_sms() * 6);
#define BWD(DD) k_dot_bwd<DD><<<grid, 256, 0, s>>>((const __nv_bfloat16*)dZ, ldz, (const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)emb, emb_stride_t, emb_stride_b, T, B, (__nv_bfloat16*)dx, lddx, (__nv_bfloat16*)demb, demb_stride_t, demb_stride_b)
  switch (D) { case 8: BWD(8); break; case 16: BWD(16); break; case 32: BWD(32); break; default: return -3; }
#undef BWD
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_fm_fwd(const void* emb, int64_t st, int64_t sb, int T, int D, int64_t B, void* out, int64_t ldo, float* sum_out, cudaStream_t s) {
  int grid = grid_for(B * (D / 8), 256);
  switch (D) {
    case 8: k_fm_fwd<8><<<grid, 256, 0, s>>>((const __nv_bfloat16*)emb, st, sb, T, B, (__nv_bfloat16*)out, ldo, sum_out); break;
    case 16: k_fm_fwd<16><<<grid, 256, 0, s>>>((const __nv_bfloat16*)emb, st, sb, T, B, (__nv_bfloat16*)out, ldo, sum_out); break;
    case 32: k_fm_fwd<32><<<grid, 256, 0, s>>>((const __nv_bfloat16*)emb, st, sb, T, B, (__nv_bfloat16*)out, ldo, sum_out); break;
    case 64: k_fm_fwd<64><<<grid, 256, 0, s>>>((const __nv_bfloat16*)emb, st, sb, T, B, (__nv_bfloat16*)out, ldo, sum_out); break;
    default: return -3;
  }
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_fm_bwd(const void* dfm, int64_t ldd, const void* emb, int64_t st, int64_t sb, const float* sum_in, int T, int D, int64_t B,
                   void* demb, int64_t dst, int64_t dsb, int accumulate, cudaStream_t s) {
  int grid = grid_for(B * (D / 8), 256);
#define FMB(DD) k_fm_bwd<DD><<<grid, 256, 0, s>>>((const __nv_bfloat16*)dfm, ldd, (const __nv_bfloat16*)emb, st, sb, sum_in, T, B, (__nv_bfloat16*)demb, dst, dsb, accumulate)
  switch (D) { case 8: FMB(8); break; case 16: FMB(16); break; case 32: FMB(32); break; case 64: FMB(64); break; default: return -3; }
#undef FMB
  DR_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
