// Warpgroup-MMA / TMA GEMM kernels for the dense (MLP) path -- hand-written for sm_90a.
//
//   k_gemm_tn      D[M,N] = A[M,K] * B[N,K]^T (+bias)(ReLU)(* relu-mask)(column statistics)   bf16 in, fp32 register accumulate,
//                  bf16 out (optional fp32 copy); the same kernel with FP8 = true multiplies E4M3 operands and applies a per-column
//                  scale (serving MLP, dr_cuda_gemm_fp8_tn).
//                  Persistent and warp-specialised: warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = consumers that
//                  each own 64 rows of a 128-row tile, issue wgmma.mma_async straight from the 128B-swizzled K-major smem tiles and
//                  run the fused epilogue from their accumulator registers.  A 4-stage smem ring of mbarrier-guarded stages keeps
//                  the loads of the next tile in flight while the consumers finish the current one.
//                  Variants: BRES (B-resident: a CTA keeps one [BLOCK_N, K] weight slab in smem for its whole life and streams only
//                  A) and CL2 (thread-block cluster of 2 CTAs on vertically adjacent tiles: each CTA loads half of the B tile and
//                  multicasts it to both, halving the B traffic from L2).
//                  Used for: Linear forward (A = activations, B = W[N,K]) and dX (A = dY, B = W^T[K,N]).
//   k_gemm_nt_splitk  dW[N_out,K_in] += dY[b,N_out]^T * X[b,K_in]     both operands MN-major straight from the row-major activations
//                  (wgmma transpose bits: no transposes materialised), split over the batch; every split writes its partial dW
//                  and k_dw_reduce adds the splits in order, so the result does not depend on which split finishes first.
//
// The reference has no tensor-core kernel of its own: its MLP GEMMs are cuBLAS/cuBLASLt calls
// (stream_executor/cuda/cuda_blas.cc:431-455, kernels/matmul_op_fused.cc) -- SURVEY §2.14 row L1.
#include <cuda.h>

#include <algorithm>

#include "common.cuh"
#include "wgmma.cuh"

using namespace drc;

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;          // 64 bf16 = 128 B = one swizzle-128B row (128 fp8 elements on the FP8 path)
constexpr int kStages = 4;
constexpr int kGemmThreads = 384;    // 3 warpgroups: TMA producer, 2 x 64-row consumers
constexpr int kMaxKbRes = 8;         // B-resident variant: K <= 512

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeTiled)p;
  }
  return fn;
}

// 2-D tensor map: dims {inner, outer}, row pitch in bytes, box {box_inner, box_outer}, 128B swizzle; out-of-bounds elements read as 0.
int make_tmap(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer, uint64_t pitch_bytes, uint32_t box_inner, uint32_t box_outer,
              CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return -100;
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {pitch_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -101 - (int)r;
}

struct Epilogue {
  const float* bias;              // [N] or null
  const __nv_bfloat16* mask_src;  // aux tile [M, ld_mask] or null
  void* out;                      // bf16 [M, ldc] (or e4m3 on the FP8 path with out_fp8)
  float* out_f32;                 // optional fp32 copy of the output (or null)
  int64_t ldc, ld_mask;
  int relu;
  int aux_mode;                   // 1: out *= (aux > 0) (ReLU backward)   2: aux only feeds S2 (S2 += out * aux)
  float* S1;                      // optional column sums over M:  S1[n] += sum_m out[m, n]
  float* S2;                      // optional:  S2[n] += sum_m out[m,n] * (aux_mode == 2 ? aux[m,n] : out[m,n])
  float* stat_ws;                 // [m_tiles][2N] per-tile column statistics, summed in tile order by k_det_colsum (with S1)
  const float* col_scale;         // FP8 path: out = acc * col_scale[n] + bias[n]
  int out_fp8;                    // FP8 path: E4M3 output, re-quantised with out_inv_scale
  float out_inv_scale;
  const uint32_t* sfa;            // MX path: UE8M0 scale words of A / B (layout of k_quantize_mxfp8, gemm_mxfp8.cu)
  const uint32_t* sfb;
};

// UE8M0 scale byte -> 2^(b - 127)  (b = 0 is the denormal 2^-127)
__device__ __forceinline__ float ue8m0(uint32_t b) { return b ? __uint_as_float(b << 23) : 5.877471754111438e-39f; }
// scale word of row r, 128-wide k block kb (k_quantize_mxfp8 layout); byte j = 32-element sub-block j
__device__ __forceinline__ uint32_t mx_word(const uint32_t* sf, int r, int num_kb, int kb) {
  return __ldg(sf + ((int64_t)(r >> 7) * num_kb + kb) * 128 + (r & 31) * 4 + ((r & 127) >> 5));
}

template <int BLOCK_N, bool BRES>
struct SmemLayoutTN {
  static constexpr int kABytes = BLOCK_M * 128;
  static constexpr int kBBytes = BLOCK_N * 128;
  static constexpr int kSt = BRES ? 3 : kStages;
  static constexpr int kStageBytes = BRES ? kABytes : kABytes + kBBytes;
  static constexpr int kBResBytes = BRES ? kMaxKbRes * kBBytes : 0;
  static constexpr int kStatBytes = 2 * 8 * BLOCK_N * 4;      // [S1 | S2][consumer warp][column]
  static constexpr int kTotal = kBResBytes + kSt * kStageBytes + kStatBytes + 256 /*barriers*/ + 1024 /*align slack*/;
};

__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// TMA load delivered to the same smem offset (and completing on the same barrier offset) in every CTA of `mask`
__device__ __forceinline__ void tma_load_2d_mc(void* smem_dst, const void* desc, uint64_t* bar, int c0, int c1, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(desc), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask) : "memory");
}
// arrive on the barrier at this offset in cluster CTA `rank`
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t}"
      ::"r"(smem_u32(bar)), "r"(rank) : "memory");
}
__device__ __forceinline__ void consumer_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

__device__ __forceinline__ uint16_t pack_e4m3x2(float a, float b) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(b), "f"(a));
  return r;
}

template <int BLOCK_N, bool BRES, bool CL2, bool FP8, bool MX = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
k_gemm_tn(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, int M, int N, int K, Epilogue ep) {
  using L = SmemLayoutTN<BLOCK_N, BRES>;
  constexpr int kSt = L::kSt;
  constexpr int kAcc = BLOCK_N / 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem_al = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* bres_base = smem_al;                                  // [kMaxKbRes][BLOCK_N x 128 B] resident weight slab (BRES only)
  uint8_t* ring = smem_al + L::kBResBytes;
  float* sS1 = reinterpret_cast<float*>(ring + kSt * L::kStageBytes);
  float* sS2 = sS1 + 8 * BLOCK_N;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sS2 + 8 * BLOCK_N);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kSt;
  uint64_t* bfull_bar = bars + 2 * kSt;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t rank = CL2 ? cluster_ctarank() : 0;
  const int m_tiles = (M + BLOCK_M - 1) / BLOCK_M;
  const int n_tiles = (N + BLOCK_N - 1) / BLOCK_N;
  constexpr int kKElems = FP8 ? 128 : BLOCK_K;           // elements per 128 B smem row
  const int num_kb = (K + kKElems - 1) / kKElems;
  // tile schedule.  streaming: round-robin over (m, n) tiles; B-resident: fixed n block, strided m blocks; cluster: both CTAs of a pair
  // walk the same (m pair, n) tiles, CTA r taking the 128 rows r of the pair's 256.
  const int m_units = CL2 ? (m_tiles + 1) / 2 : m_tiles;
  const int unit0 = CL2 ? (int)blockIdx.x / 2 : BRES ? (int)blockIdx.x / n_tiles : (int)blockIdx.x;
  const int unit_step = CL2 ? (int)gridDim.x / 2 : BRES ? (int)gridDim.x / n_tiles : (int)gridDim.x;
  const int num_units = BRES ? m_units : m_units * n_tiles;
  auto tile_m = [&](int u) { return (BRES ? u : u / n_tiles) * (CL2 ? 2 : 1) + (int)rank; };
  auto tile_n = [&](int u) { return BRES ? (int)blockIdx.x % n_tiles : u % n_tiles; };

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < kSt; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], CL2 ? 16 : 8); }
    mbar_init(bfull_bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if constexpr (CL2) cluster_sync_all();     // the peer's barriers are initialised before any multicast lands on them
  pdl_sync();      // everything above overlapped the previous kernel's tail; nothing before this touched global memory

  if (warp == 0) {
    // ================= TMA producer =================
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      if constexpr (BRES) {
        if (unit0 < num_units) {          // the whole [BLOCK_N, K] weight slab, once
          mbar_expect_tx(bfull_bar, (uint32_t)(num_kb * L::kBBytes));
          for (int kb = 0; kb < num_kb; ++kb) tma_load_2d(bres_base + kb * L::kBBytes, &tmB, bfull_bar, kb * 64, tile_n(0) * BLOCK_N);
        }
      }
      for (int u = unit0; u < num_units; u += unit_step) {
        const int m_blk = tile_m(u), n_blk = tile_n(u);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = ring + stage * L::kStageBytes;
          mbar_expect_tx(&full_bar[stage], L::kStageBytes);
          tma_load_2d(sa, &tmA, &full_bar[stage], kb * kKElems, m_blk * BLOCK_M);
          if constexpr (!BRES) {
            uint8_t* sb = sa + L::kABytes;
            if constexpr (CL2) {          // my half of the B tile, into both CTAs
              tma_load_2d_mc(sb + rank * (L::kBBytes / 2), &tmB, &full_bar[stage], kb * 64, n_blk * BLOCK_N + (int)rank * (BLOCK_N / 2), 3);
            } else {
              tma_load_2d(sb, &tmB, &full_bar[stage], kb * kKElems, n_blk * BLOCK_N);
            }
          }
          if (++stage == kSt) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    // ================= consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of every tile =================
    // (warps 1-3 of the producer warpgroup have no role: wgmma is issued by whole warpgroups only)
    const int wg = (warp >> 2) - 1;
    const int wl = warp & 3;
    const int ct = threadIdx.x - 128;                   // 0..255
    int stage = 0; uint32_t phase = 0;
    if constexpr (BRES) { if (unit0 < num_units) mbar_wait(bfull_bar, 0); }
    for (int u = unit0; u < num_units; u += unit_step) {
      const int m_blk = tile_m(u), n_blk = tile_n(u);
      float acc[kAcc];
#pragma unroll
      for (int i = 0; i < kAcc; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(ring + stage * L::kStageBytes) + wg * 64 * 128;
        const uint32_t sb = BRES ? smem_u32(bres_base + kb * L::kBBytes) : smem_u32(ring + stage * L::kStageBytes) + L::kABytes;
        const uint64_t adesc = gmma_desc_sw128(sa, 16, 1024);
        const uint64_t bdesc = gmma_desc_sw128(sb, 16, 1024);
        if constexpr (MX) {
          // block-scaled fp8: one m64nNk32 wgmma covers exactly one 32-element scale block; its fresh product is promoted into the fp32
          // accumulator with the two scales:  acc[m, n] += sa[m, k32] * sb[n, k32] * (A_q B_q^T)[m, n]
          const int r0 = m_blk * BLOCK_M + wg * 64 + wl * 16 + (lane >> 2);
          const uint32_t wa0 = mx_word(ep.sfa, r0, num_kb, kb), wa1 = mx_word(ep.sfa, r0 + 8, num_kb, kb);
          uint32_t wb[BLOCK_N / 4];
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j)
#pragma unroll
            for (int c = 0; c < 2; ++c) wb[2 * j + c] = mx_word(ep.sfb, n_blk * BLOCK_N + 8 * j + 2 * (lane & 3) + c, num_kb, kb);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            float part[kAcc];
            wgmma_fence();
            wgmma_e4m3<BLOCK_N>(part, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), 0);
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_acc(part);
            const float sa0 = ue8m0((wa0 >> (8 * k)) & 0xffu), sa1 = ue8m0((wa1 >> (8 * k)) & 0xffu);
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j)
#pragma unroll
              for (int c = 0; c < 2; ++c) {
                const float sb = ue8m0((wb[2 * j + c] >> (8 * k)) & 0xffu);
                acc[4 * j + c] = fmaf(part[4 * j + c], sa0 * sb, acc[4 * j + c]);
                acc[4 * j + 2 + c] = fmaf(part[4 * j + 2 + c], sa1 * sb, acc[4 * j + 2 + c]);
              }
          }
        } else {
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) {   // 32 B (16 bf16 / 32 fp8) per step inside the 128B swizzle atom: +2 in the (addr >> 4) field
            if constexpr (FP8) wgmma_e4m3<BLOCK_N>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), 1);
            else wgmma_bf16<BLOCK_N, 0, 0>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), 1);
          }
          wgmma_commit();
        }
        wgmma_wait<1>();                                  // the previous stage's MMAs have retired: hand it back to the producer
        if (prev >= 0 && lane == 0) {
          mbar_arrive(&empty_bar[prev]);
          if constexpr (CL2) mbar_arrive_cluster(&empty_bar[prev], rank ^ 1);
        }
        prev = stage;
        if (++stage == kSt) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if (lane == 0) {
        mbar_arrive(&empty_bar[prev]);
        if constexpr (CL2) mbar_arrive_cluster(&empty_bar[prev], rank ^ 1);
      }

      // ---- fused epilogue straight from the accumulator registers
      const int row0 = m_blk * BLOCK_M + wg * 64 + wl * 16 + (lane >> 2);
      const bool stats = !FP8 && ep.S1 != nullptr;
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int col = n_blk * BLOCK_N + 8 * j + 2 * (lane & 3);
        const bool col_ok = col < N;                      // N is even: col + 1 < N too
        float b0 = 0.f, b1 = 0.f, s0 = 1.f, s1 = 1.f;
        if (col_ok && ep.bias) { b0 = __ldg(ep.bias + col); b1 = __ldg(ep.bias + col + 1); }
        if (FP8 && !MX && col_ok) { s0 = __ldg(ep.col_scale + col); s1 = __ldg(ep.col_scale + col + 1); }
        float p1[2] = {0.f, 0.f}, p2[2] = {0.f, 0.f};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = row0 + 8 * h;
          const bool ok = col_ok && row < M;
          float v0 = FP8 && !MX ? fmaf(acc[4 * j + 2 * h], s0, b0) : acc[4 * j + 2 * h] + b0;
          float v1 = FP8 && !MX ? fmaf(acc[4 * j + 2 * h + 1], s1, b1) : acc[4 * j + 2 * h + 1] + b1;
          if (ep.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
          float w0 = 0.f, w1 = 0.f;
          if (!FP8 && ep.mask_src && ok) {
            const __nv_bfloat16* ms = ep.mask_src + (int64_t)row * ep.ld_mask + col;
            w0 = __bfloat162float(ms[0]); w1 = __bfloat162float(ms[1]);
            if (ep.aux_mode == 1) { if (!(w0 > 0.f)) v0 = 0.f; if (!(w1 > 0.f)) v1 = 0.f; }
          }
          if (ok) {
            if (FP8 && !MX && ep.out_fp8) {
              *reinterpret_cast<uint16_t*>(reinterpret_cast<uint8_t*>(ep.out) + (int64_t)row * ep.ldc + col) =
                  pack_e4m3x2(v0 * ep.out_inv_scale, v1 * ep.out_inv_scale);
            } else {
              *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(ep.out) + (int64_t)row * ep.ldc + col) = pack_bf16x2(v0, v1);
            }
            if (ep.out_f32) *reinterpret_cast<float2*>(ep.out_f32 + (int64_t)row * ep.ldc + col) = make_float2(v0, v1);
            if (stats) {
              p1[0] += v0; p1[1] += v1;
              const float a0 = ep.aux_mode == 2 ? w0 : v0, a1 = ep.aux_mode == 2 ? w1 : v1;
              p2[0] += v0 * a0; p2[1] += v1 * a1;
            }
          }
        }
        if (stats) {                                      // column sums of the warp's 16 rows -> lanes 0..3 -> the warp's smem row
#pragma unroll
          for (int c = 0; c < 2; ++c) {
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) {
              p1[c] += __shfl_xor_sync(0xffffffffu, p1[c], o);
              p2[c] += __shfl_xor_sync(0xffffffffu, p2[c], o);
            }
          }
          if (lane < 4) {
            float* r1 = sS1 + (warp - 4) * BLOCK_N + 8 * j + 2 * lane;
            float* r2 = sS2 + (warp - 4) * BLOCK_N + 8 * j + 2 * lane;
            r1[0] = p1[0]; r1[1] = p1[1]; r2[0] = p2[0]; r2[1] = p2[1];
          }
        }
      }
      if (!FP8 && ep.S1) {                                // the tile's column sums, warps added in row order -> workspace row m_blk
        consumer_bar_sync();
        if (m_blk < m_tiles) {
          for (int i = ct; i < BLOCK_N; i += 256) {
            const int col = n_blk * BLOCK_N + i;
            if (col < N) {
              float a1 = 0.f, a2 = 0.f;
#pragma unroll
              for (int w = 0; w < 8; ++w) { a1 += sS1[w * BLOCK_N + i]; a2 += sS2[w * BLOCK_N + i]; }
              ep.stat_ws[(int64_t)m_blk * 2 * N + col] = a1;
              ep.stat_ws[(int64_t)m_blk * 2 * N + N + col] = a2;
            }
          }
        }
        consumer_bar_sync();
      }
    }
  }
  if constexpr (CL2) {
    __syncwarp();
    cluster_sync_all();   // no CTA leaves while its peer may still multicast into it or arrive on its barriers
  }
}

// -------------------------------------------------------------------------------------------------
// dW[N_out, K_in] += sum_b dY[b, N_out] * X[b, K_in]   (split over b; fp32 atomics epilogue)
//   A operand = dY^T  : M = N_out, MN-major (tensor map over dY: inner = N_out, outer = batch)
//   B operand = X^T   : N = K_in , MN-major (tensor map over X : inner = K_in , outer = batch)
// smem per stage: A = 2 chunks [BLOCK_KB rows][64 elems] (one per consumer warpgroup); B = BLOCK_N/64 such chunks.
// -------------------------------------------------------------------------------------------------
constexpr int BLOCK_KB = 64;            // batch rows (reduction) per pipeline stage
constexpr int kChunkBytes = BLOCK_KB * 128;

template <int BLOCK_N>
struct SmemLayoutNT {
  static constexpr int kAChunks = BLOCK_M / 64;
  static constexpr int kBChunks = BLOCK_N / 64;
  static constexpr int kStageBytes = (kAChunks + kBChunks) * kChunkBytes;
  static constexpr int kTotal = kStages * kStageBytes + 1024 + 256;
};

template <int BLOCK_N>
__global__ void __launch_bounds__(kGemmThreads, 1)
k_gemm_nt_splitk(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, int Mo /*N_out*/, int No /*K_in*/,
                 int batch, int rows_per_split, float* __restrict__ part /* [splits][Mo][No] */) {
  using L = SmemLayoutNT<BLOCK_N>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * L::kStageBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_blk = blockIdx.x, n_blk = blockIdx.y, split = blockIdx.z;
  const int b0 = split * rows_per_split;
  const int b1 = min(batch, b0 + rows_per_split);
  const int num_kb = (b1 - b0 + BLOCK_KB - 1) / BLOCK_KB;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA); tma_prefetch_desc(&tmB);
    for (int i = 0; i < kStages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_sync();      // everything above overlapped the previous kernel's tail
  if (num_kb <= 0) return;

  if (warp == 0) {
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sa = smem + stage * L::kStageBytes;
        uint8_t* sb = sa + L::kAChunks * kChunkBytes;
        mbar_expect_tx(&full_bar[stage], L::kStageBytes);
        const int brow = b0 + kb * BLOCK_KB;   // rows_per_split is a multiple of BLOCK_KB: a stage never crosses into the next split;
                                               // rows beyond `batch` are zero-filled by TMA
#pragma unroll
        for (int c = 0; c < L::kAChunks; ++c) tma_load_2d(sa + c * kChunkBytes, &tmA, &full_bar[stage], m_blk * BLOCK_M + c * 64, brow);
#pragma unroll
        for (int c = 0; c < L::kBChunks; ++c) tma_load_2d(sb + c * kChunkBytes, &tmB, &full_bar[stage], n_blk * BLOCK_N + c * 64, brow);
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {                            // whole consumer warpgroups only (wgmma is warpgroup-wide)
    const int wg = (warp >> 2) - 1, wl = warp & 3;
    float acc[BLOCK_N / 2];
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
    int stage = 0; uint32_t phase = 0, prev = 0;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * L::kStageBytes) + wg * kChunkBytes;   // my 64 output rows = one MN chunk
      const uint32_t sb = smem_u32(smem + stage * L::kStageBytes) + L::kAChunks * kChunkBytes;
      // MN-major SW128: LBO = distance between 64-element MN chunks, SBO = 8 k-rows (1024 B)
      const uint64_t adesc = gmma_desc_sw128(sa, kChunkBytes, 1024);
      const uint64_t bdesc = gmma_desc_sw128(sb, kChunkBytes, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_KB / 16; ++k)       // 16 k-rows = 2048 B  -> +128 in the (addr >> 4) field
        wgmma_bf16<BLOCK_N, 1, 1>(acc, adesc + (uint64_t)(k * 128), bdesc + (uint64_t)(k * 128), 1);
      wgmma_commit();
      wgmma_wait<1>();
      if (kb > 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    const int row0 = m_blk * BLOCK_M + wg * 64 + wl * 16 + (lane >> 2);     // N_out index
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      const int col = n_blk * BLOCK_N + 8 * j + 2 * (lane & 3);              // K_in index
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = row0 + 8 * h;
        if (row >= Mo) continue;
        float* dst = part + ((int64_t)split * Mo + row) * No + col;
        if (col < No) dst[0] = acc[4 * j + 2 * h];
        if (col + 1 < No) dst[1] = acc[4 * j + 2 * h + 1];
      }
    }
  }
}

// dW[r, c] += sum over splits of part[split][r][c], splits added in order
__global__ void k_dw_reduce(const float* __restrict__ part, int splits, int Mo, int No, float* __restrict__ dW, int64_t ldw) {
  const int64_t n = (int64_t)Mo * No;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float sum = 0.f;
    for (int k = 0; k < splits; ++k) sum += part[k * n + i];
    dW[(i / No) * ldw + i % No] += sum;
  }
}

template <int BN, bool BRES, bool CL2, bool FP8, bool MX = false>
int launch_tn(const CUtensorMap& ta, const void* B, int M, int N, int K, int64_t ldb, const Epilogue& ep, int max_ctas, cudaStream_t s) {
  CUtensorMap tb;
  const uint32_t box_rows = CL2 ? BN / 2 : BN;
  int rc = FP8 ? make_tmap(&tb, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb, 128, box_rows, CU_TENSOR_MAP_DATA_TYPE_UINT8)
               : make_tmap(&tb, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb * 2, BLOCK_K, box_rows);
  if (rc) return rc;
  using L = SmemLayoutTN<BN, BRES>;
  static_assert(L::kTotal <= 227 * 1024, "shared-memory budget");
  auto kern = k_gemm_tn<BN, BRES, CL2, FP8, MX>;
  static DrPerDeviceOnce attr_once; bool& attr_set = attr_once();
  if (!attr_set) {
    DR_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal));
    attr_set = true;
  }
  const int m_tiles = (M + BLOCK_M - 1) / BLOCK_M, n_tiles = (N + BN - 1) / BN;
  int grid = m_tiles * n_tiles;
  if (grid > max_ctas) grid = max_ctas;
  if (BRES) grid = grid / n_tiles * n_tiles;        // every CTA owns one n block: the grid is a whole number of n-block groups
  if (CL2) {
    const int pairs_needed = (m_tiles + 1) / 2 * n_tiles;
    int pairs = grid / 2 < 1 ? 1 : grid / 2;
    if (pairs > pairs_needed) pairs = pairs_needed;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(2 * pairs); cfg.blockDim = dim3(kGemmThreads); cfg.dynamicSmemBytes = L::kTotal; cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    DR_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, ta, tb, M, N, K, ep));
  } else {
    DR_PDL_LAUNCH(kern, grid, kGemmThreads, L::kTotal, s, ta, tb, M, N, K, ep);
  }
  DR_LAUNCH_CHECK();
  return 0;
}

// DEEPREC_GEMM_BRES=1 selects the B-resident (weight-stationary) kernel where it applies (K <= 512, enough CTAs for one per n block).
inline int& gemm_bres_enabled() { static int v = [] { const char* e = getenv("DEEPREC_GEMM_BRES"); return (e && e[0] == '1') ? 1 : 0; }(); return v; }
// DEEPREC_GEMM_2CTA=1 routes the shapes with N >= 64 to the cluster-of-2 kernel (B tile multicast to both CTAs).
inline int& gemm_2cta_enabled() { static int v = [] { const char* e = getenv("DEEPREC_GEMM_2CTA"); return (e && e[0] == '1') ? 1 : 0; }(); return v; }

template <int BN>
int launch_nt(const CUtensorMap& ta, const CUtensorMap& tb, int Mo, int No, int batch, int splits, float* dW, int64_t ldw, cudaStream_t s) {
  using L = SmemLayoutNT<BN>;
  static DrPerDeviceOnce attr_once; bool& attr_set = attr_once();
  if (!attr_set) {
    DR_CUDA_CHECK(cudaFuncSetAttribute(k_gemm_nt_splitk<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal));
    attr_set = true;
  }
  int rows_per_split = ((batch + splits - 1) / splits + BLOCK_KB - 1) / BLOCK_KB * BLOCK_KB;
  splits = (batch + rows_per_split - 1) / rows_per_split;
  float* part = dr_workspace(kWsGemmDw, (size_t)splits * Mo * No, s);
  if (!part) return -5;
  dim3 grid((Mo + BLOCK_M - 1) / BLOCK_M, (No + BN - 1) / BN, splits);
  DR_PDL_LAUNCH((k_gemm_nt_splitk<BN>), grid, kGemmThreads, L::kTotal, s, ta, tb, Mo, No, batch, rows_per_split, part);
  DR_LAUNCH_CHECK();
  const int64_t n = (int64_t)Mo * No;
  k_dw_reduce<<<(int)std::min<int64_t>((n + 255) / 256, num_sms() * 8), 256, 0, s>>>(part, splits, Mo, No, dW, ldw);
  DR_LAUNCH_CHECK();
  return 0;
}

template <int BN>
int launch_tn_sel(const CUtensorMap& ta, const void* B, int M, int N, int K, int64_t ldb, const Epilogue& ep, int max_ctas, cudaStream_t s) {
  if (BN >= 64 && gemm_2cta_enabled()) return launch_tn<BN, false, true, false>(ta, B, M, N, K, ldb, ep, max_ctas, s);
  if (gemm_bres_enabled() && (K + BLOCK_K - 1) / BLOCK_K <= kMaxKbRes && (N + BN - 1) / BN <= max_ctas)
    return launch_tn<BN, true, false, false>(ta, B, M, N, K, ldb, ep, max_ctas, s);
  return launch_tn<BN, false, false, false>(ta, B, M, N, K, ldb, ep, max_ctas, s);
}

}  // namespace

extern "C" {

int dr_cuda_gemm_tn_ex(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, const float* bias, int relu,
                       const void* mask_src, int64_t ld_mask, int aux_mode, void* out, int64_t ldc, float* out_f32, float* S1, float* S2,
                       int max_ctas, int force_v1, cudaStream_t s);

// out[M,N] = A[M,K](lda) * B[N,K](ldb)^T (+bias)(relu)(*mask).  Requirements: bf16, K-major, lda/ldb/ldc multiples of 8,
// N multiple of 8, pointers 16B-aligned.  out_f32 optional.
int dr_cuda_gemm_tn(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, const float* bias, int relu,
                    const void* mask_src, int64_t ld_mask, void* out, int64_t ldc, float* out_f32, int max_ctas, cudaStream_t s) {
  return dr_cuda_gemm_tn_ex(A, lda, B, ldb, M, N, K, bias, relu, mask_src, ld_mask, mask_src ? 1 : 0, out, ldc, out_f32, nullptr, nullptr,
                            max_ctas, 0, s);
}

// Extended entry: aux_mode 1 = ReLU-backward mask, 2 = statistics partner; S1/S2 = fused column statistics.  force_v1 is accepted for
// callers that select the unfused-statistics path; every shape runs the same kernel.
int dr_cuda_gemm_tn_ex(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, const float* bias, int relu,
                       const void* mask_src, int64_t ld_mask, int aux_mode, void* out, int64_t ldc, float* out_f32, float* S1, float* S2,
                       int max_ctas, int force_v1, cudaStream_t s) {
  (void)force_v1;
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if ((lda % 8) || (ldb % 8) || (ldc % 8) || (N % 8)) return -2;
  if (max_ctas <= 0) max_ctas = num_sms();
  CUtensorMap ta;
  int rc = make_tmap(&ta, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda * 2, BLOCK_K, BLOCK_M);
  if (rc) return rc;
  if (S2 && !S1) return -4;
  const int m_tiles = (M + BLOCK_M - 1) / BLOCK_M;
  float* ws = nullptr;
  if (S1) {
    ws = dr_workspace(kWsGemmStats, (size_t)m_tiles * 2 * N, s);
    if (!ws) return -5;
  }
  Epilogue ep{bias, (const __nv_bfloat16*)mask_src, out, out_f32, ldc, ld_mask, relu, aux_mode, S1, S2, ws, nullptr, 0, 1.f};
  rc = N <= 16 ? launch_tn_sel<16>(ta, B, M, N, K, ldb, ep, max_ctas, s)
     : N <= 32 ? launch_tn_sel<32>(ta, B, M, N, K, ldb, ep, max_ctas, s)
     : N <= 64 ? launch_tn_sel<64>(ta, B, M, N, K, ldb, ep, max_ctas, s)
               : launch_tn_sel<128>(ta, B, M, N, K, ldb, ep, max_ctas, s);
  if (rc || !S1) return rc;
  k_det_colsum<<<(N + 127) / 128, 128, 0, s>>>(ws, m_tiles, 2 * (int64_t)N, N, S1, S2, 1.f);
  DR_LAUNCH_CHECK();
  return 0;
}

// A/B switches for the GEMM variants (same effect as DEEPREC_GEMM_2CTA / DEEPREC_GEMM_BRES, settable at run time; return the previous value).
int dr_cuda_set_gemm_2cta(int on) { int prev = gemm_2cta_enabled(); gemm_2cta_enabled() = on ? 1 : 0; return prev; }
int dr_cuda_set_gemm_bres(int on) { int prev = gemm_bres_enabled(); gemm_bres_enabled() = on ? 1 : 0; return prev; }

// dW[N_out,K_in](ldw, fp32, accumulated into) += dY[batch,N_out](ldy)^T * X[batch,K_in](ldx)
int dr_cuda_gemm_dw(const void* dY, int64_t ldy, const void* X, int64_t ldx, int batch, int N_out, int K_in, float* dW, int64_t ldw,
                    int splits, cudaStream_t s) {
  if (batch <= 0 || N_out <= 0 || K_in <= 0) return 0;
  if ((ldy % 8) || (ldx % 8)) return -2;
  CUtensorMap ta, tb;
  int rc = make_tmap(&ta, dY, (uint64_t)N_out, (uint64_t)batch, (uint64_t)ldy * 2, 64, BLOCK_KB);
  if (rc) return rc;
  rc = make_tmap(&tb, X, (uint64_t)K_in, (uint64_t)batch, (uint64_t)ldx * 2, 64, BLOCK_KB);
  if (rc) return rc;
  const int m_tiles = (N_out + BLOCK_M - 1) / BLOCK_M;
  if (K_in <= 64) {
    if (splits <= 0) splits = max(1, num_sms() / m_tiles);
    return launch_nt<64>(ta, tb, N_out, K_in, batch, splits, dW, ldw, s);
  }
  const int n_tiles = (K_in + 127) / 128;
  if (splits <= 0) splits = max(1, num_sms() / (m_tiles * n_tiles));
  return launch_nt<128>(ta, tb, N_out, K_in, batch, splits, dW, ldw, s);
}

// FP8 (E4M3) GEMM for the serving MLP:  out[M,N] = (A_q[M,K] B_q[N,K]^T) * col_scale[n] + bias[n]  (ReLU)
//   A_q : activations quantised per tensor (static scale from calibration), B_q : weights quantised per output channel;
//   col_scale[n] = a_scale * w_scale[n] is folded on the host, so the epilogue is one FMA per element.  The output is bf16, or E4M3
//   re-quantised with the NEXT layer's activation scale (out = sat_e4m3(v * out_inv_scale)), so a chain of layers never leaves 8-bit
//   storage between GEMMs.  wgmma kind e4m3 (dense 8-bit rate = 2x bf16): one smem row = 128 B = 128 fp8 elements, 4 MMAs of K = 32
//   per stage.  A, B: K-major, lda/ldb multiples of 16 bytes; N % 16 == 0.
int dr_cuda_gemm_fp8_tn(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, const float* col_scale, const float* bias,
                        int relu, void* out, int64_t ldc, int out_fp8, float out_inv_scale, cudaStream_t s) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if ((lda % 16) || (ldb % 16) || (N % 16) || (ldc % 8) || (out_fp8 && (ldc % 16))) return -2;
  CUtensorMap ta;
  int rc = make_tmap(&ta, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, 128, BLOCK_M, CU_TENSOR_MAP_DATA_TYPE_UINT8);
  if (rc) return rc;
  Epilogue ep{bias, nullptr, out, nullptr, ldc, 0, relu, 0, nullptr, nullptr, nullptr, col_scale, out_fp8, out_inv_scale};
  if (N <= 16) return launch_tn<16, false, false, true>(ta, B, M, N, K, ldb, ep, num_sms(), s);
  if (N <= 32) return launch_tn<32, false, false, true>(ta, B, M, N, K, ldb, ep, num_sms(), s);
  if (N <= 64) return launch_tn<64, false, false, true>(ta, B, M, N, K, ldb, ep, num_sms(), s);
  return launch_tn<128, false, false, true>(ta, B, M, N, K, ldb, ep, num_sms(), s);
}

// out[M,N] (bf16, ldc) = blockscaled(A_q[M,Kp], sfa) * blockscaled(B_q[>= N,Kp], sfb)^T (+bias)(relu).  A_q / B_q: e4m3, K-major, row
// pitch Kp (multiple of 128); sfa / sfb: scale words in k_quantize_mxfp8's layout (gemm_mxfp8.cu); N % 8 == 0.
int dr_cuda_gemm_mxfp8_tn(const void* A, const void* sfa, const void* B, const void* sfb, int M, int N, int Kp, const float* bias, int relu, void* out,
                          int64_t ldc, int max_ctas, cudaStream_t s) {
  if (M <= 0 || N <= 0 || Kp <= 0) return 0;
  if ((Kp % 128) || (N % 8) || (ldc % 8)) return -2;
  if (max_ctas <= 0) max_ctas = num_sms();
  CUtensorMap ta;
  int rc = make_tmap(&ta, A, (uint64_t)Kp, (uint64_t)M, (uint64_t)Kp, 128, BLOCK_M, CU_TENSOR_MAP_DATA_TYPE_UINT8);
  if (rc) return rc;
  Epilogue ep{bias, nullptr, out, nullptr, ldc, 0, relu, 0, nullptr, nullptr, nullptr, nullptr, 0, 1.f, (const uint32_t*)sfa, (const uint32_t*)sfb};
  if (N <= 16) return launch_tn<16, false, false, true, true>(ta, B, M, N, Kp, Kp, ep, max_ctas, s);
  if (N <= 32) return launch_tn<32, false, false, true, true>(ta, B, M, N, Kp, Kp, ep, max_ctas, s);
  return launch_tn<64, false, false, true, true>(ta, B, M, N, Kp, Kp, ep, max_ctas, s);
}

}  // extern "C"
