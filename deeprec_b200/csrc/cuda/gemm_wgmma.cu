// Warpgroup-MMA / TMA GEMM kernels for the dense (MLP) path -- hand-written for sm_90a.
//
//   k_gemm_tn      D[M,N] = A[M,K] * B[N,K]^T (+bias)(ReLU)(* relu-mask)(column statistics)   bf16 in, fp32 register accumulate,
//                  bf16 out (optional fp32 copy); the same kernel with FP8 = true multiplies E4M3 operands and applies a per-column
//                  scale (serving MLP, dr_cuda_gemm_fp8_tn).
//                  Persistent and warp-specialised: warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = consumers that
//                  issue wgmma.mma_async straight from the 128B-swizzled K-major smem tiles and run the fused epilogue from their
//                  accumulator registers.  A 4-stage smem ring of mbarrier-guarded stages keeps the loads of the next tile in flight
//                  while the consumers finish the current one.
//                  bf16 streaming (the default): ping-pong consumers.  Each warpgroup owns whole 128-row tiles, alternate tiles of
//                  the schedule, so one warpgroup's epilogue overlaps the other's MMAs; the aux tile arrives by TMA into the
//                  warpgroup's output buffer and the bf16 tile leaves by TMA store.  FP8 / MX, BRES, CL2, the cross / residual /
//                  LayerNorm epilogues and unaligned aux operands: cooperative consumers, each warpgroup owns 64 rows of every tile
//                  and stores straight from registers.
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
#include <cstring>
#include <type_traits>

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

// 2-D tensor map: dims {inner, outer}, row pitch in bytes, box {box_inner, box_outer}, 128B swizzle unless given; out-of-bounds elements
// read as 0 and are not written by stores.
int make_tmap(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer, uint64_t pitch_bytes, uint32_t box_inner, uint32_t box_outer,
              CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_128B) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return -100;
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {pitch_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
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

// Epilogue kinds beyond the bias / ReLU / mask / statistics of kind 0.  The kind is a template parameter and only the new kinds take the
// wider parameter block, so the kind-0 instantiations compile exactly as before.  The aux operand (mask_src, ld_mask) is x_l for kEpiCross
// and the addend for kEpiResidual; both run with relu = 0 and aux_mode = 0.
enum { kEpiPlain = 0, kEpiCross = 1, kEpiResidual = 2, kEpiLayerNorm = 3 };
struct EpilogueX : Epilogue {
  const __nv_bfloat16* x0;        // kEpiCross: the x0 factor [M, ld_x0]
  __nv_bfloat16* u_out;           // kEpiCross: optional u = acc + bias [M, ld_u] (bf16), kept for the backward
  int64_t ld_x0, ld_u;
};
// kEpiLayerNorm: a row's N <= BLOCK_N columns sit in one tile, so its LayerNorm runs on the fp32 accumulators; relu applies after the norm.
struct EpilogueLN : Epilogue {
  const float* gamma;             // [N]
  const float* beta;              // [N]
  __nv_bfloat16* xhat;            // optional x^ = (h - mean) * rstd [M, ld_xhat] (bf16), kept for the backward
  float* rstd;                    // optional [M]
  int64_t ld_xhat;
  float eps;
};
template <int EPI>
using EpiT = std::conditional_t<EPI == kEpiPlain, Epilogue, std::conditional_t<EPI == kEpiLayerNorm, EpilogueLN, EpilogueX>>;

// UE8M0 scale byte -> 2^(b - 127)  (b = 0 is the denormal 2^-127)
__device__ __forceinline__ float ue8m0(uint32_t b) { return b ? __uint_as_float(b << 23) : 5.877471754111438e-39f; }
// scale word of row r, 128-wide k block kb (k_quantize_mxfp8 layout); byte j = 32-element sub-block j
__device__ __forceinline__ uint32_t mx_word(const uint32_t* sf, int r, int num_kb, int kb) {
  return __ldg(sf + ((int64_t)(r >> 7) * num_kb + kb) * 128 + (r & 31) * 4 + ((r & 127) >> 5));
}

// PP (ping-pong): each consumer warpgroup owns whole 128-row tiles and has its own output tile buffer (the aux tile lands there first)
// and its own statistics rows.  The output tile is stored by TMA in boxes of kBoxCols columns x 128 rows, kRowBytes per box row, with
// the tensor map's swizzle (128B / 64B / 32B for 64 / 32 / 16 columns): a warp's fragment accesses hit 32 different banks.
template <int BLOCK_N, bool BRES, bool PP = false>
struct SmemLayoutTN {
  static constexpr int kABytes = BLOCK_M * 128;
  static constexpr int kBBytes = BLOCK_N * 128;
  static constexpr int kSt = BRES ? 3 : kStages;
  static constexpr int kStageBytes = BRES ? kABytes : kABytes + kBBytes;
  static constexpr int kBResBytes = BRES ? kMaxKbRes * kBBytes : 0;
  static constexpr int kBoxCols = BLOCK_N < 64 ? BLOCK_N : 64;
  static constexpr int kRowBytes = kBoxCols * 2;
  static constexpr int kBoxBytes = BLOCK_M * kRowBytes;
  static constexpr int kOutBytes = PP ? BLOCK_M * BLOCK_N * 2 : 0;   // per consumer warpgroup
  static constexpr int kStatBytes = (PP ? 2 : 1) * 2 * 8 * BLOCK_N * 4;   // [warpgroup][S1 | S2][16-row group][column]
  static constexpr int kTotal = kBResBytes + kSt * kStageBytes + 2 * kOutBytes + kStatBytes + 256 /*barriers*/ + 1024 /*align slack*/;
};

// byte offset of (row, col) in a PP output tile buffer, in the layout the TMA swizzle gives it (16-byte chunk index ^ row bits)
template <int BLOCK_N>
__device__ __forceinline__ uint32_t out_tile_offset(int row, int col) {
  using L = SmemLayoutTN<BLOCK_N, false, true>;
  uint32_t off = (uint32_t)(row * L::kRowBytes + (col % L::kBoxCols) * 2);
  off ^= ((off >> 7) & (L::kRowBytes / 16 - 1)) << 4;
  return (uint32_t)(col / L::kBoxCols) * L::kBoxBytes + off;
}

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
// named barrier of one consumer warpgroup (PP: the two warpgroups never wait for each other)
__device__ __forceinline__ void wg_bar_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory"); }
// PP mainloop order: warpgroup wg waits on barrier 4 + wg until the other warpgroup has arrived there after its mainloop
__device__ __forceinline__ void order_wait(int wg) { asm volatile("bar.sync %0, 256;" ::"r"(4 + wg) : "memory"); }
__device__ __forceinline__ void order_signal(int wg) { asm volatile("bar.arrive %0, 256;" ::"r"(5 - wg) : "memory"); }
// this thread's bulk stores have finished reading shared memory (their global writes may still be in flight)
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
template <int R> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

__device__ __forceinline__ uint16_t pack_e4m3x2(float a, float b) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(b), "f"(a));
  return r;
}

template <int BLOCK_N, bool BRES, bool CL2, bool FP8, bool MX = false, bool PP = false, int EPI = kEpiPlain>
__global__ void __launch_bounds__(kGemmThreads, 1)
k_gemm_tn(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmOut,
          const __grid_constant__ CUtensorMap tmAux, int M, int N, int K, EpiT<EPI> ep) {
  static_assert(!PP || (!BRES && !CL2 && !FP8), "ping-pong consumers: bf16 streaming kernel only");
  static_assert(EPI == kEpiPlain || (!PP && !BRES && !CL2 && !FP8), "cross / residual / LayerNorm epilogues: bf16 cooperative streaming kernel only");
  using L = SmemLayoutTN<BLOCK_N, BRES, PP>;
  constexpr int kSt = L::kSt;
  constexpr int kAcc = BLOCK_N / 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem_al = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* bres_base = smem_al;                                  // [kMaxKbRes][BLOCK_N x 128 B] resident weight slab (BRES only)
  uint8_t* ring = smem_al + L::kBResBytes;
  uint8_t* out_tiles = ring + kSt * L::kStageBytes;              // PP: [warpgroup][kOutBytes]
  float* sS1 = reinterpret_cast<float*>(out_tiles + 2 * L::kOutBytes);
  float* sS2 = sS1 + 8 * BLOCK_N;
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sS1) + L::kStatBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kSt;
  uint64_t* bfull_bar = bars + 2 * kSt;
  uint64_t* aux_bar = bars + 2 * kSt + 1;                        // PP: [warpgroup] aux tile landed

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
    // a stage is released by every consumer warp that read it: the 8 of both warpgroups (x 2 CTAs for CL2), or the 4 of the one PP
    // warpgroup that owns its tile
    for (int i = 0; i < kSt; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], PP ? 4 : CL2 ? 16 : 8); }
    mbar_init(bfull_bar, 1);
    mbar_init(&aux_bar[0], 1);
    mbar_init(&aux_bar[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  if constexpr (CL2) cluster_sync_all();     // the peer's barriers are initialised before any multicast lands on them
  pdl_sync();      // everything above overlapped the previous kernel's tail; nothing before this touched global memory

  if (warp < 4) {
    // ================= TMA producer =================
    if constexpr (PP) setmaxnreg_dec<40>();    // registers go to the consumers, which hold a whole 128-row accumulator tile each
    if (warp == 0 && lane == 0) {
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
  } else if constexpr (PP) {
    // ================= ping-pong consumers: warpgroup wg owns the whole tiles wg, wg + 2, ... of this CTA's schedule =================
    // The producer fills the ring in schedule order, so while one warpgroup runs its epilogue the other's k-blocks are already landing
    // and its MMAs run.  Tile i of the schedule holds ring slots i * num_kb ... (i + 1) * num_kb - 1 (slot s: stage s % kSt, phase
    // (s / kSt) & 1).  The mainloops run in tile order (order_wait / order_signal): a parity wait on slot s is only sound once slot
    // s - kSt has completed, and every slot before tile i has when the mainloop of tile i - 1 is done.  The epilogue stages the bf16
    // tile in the warpgroup's smem buffer and stores it with TMA; with an aux operand the buffer first receives the aux tile (TMA,
    // aux_bar[wg]), and every thread overwrites exactly the aux elements it read.
    setmaxnreg_inc<232>();
    const int wg = (warp >> 2) - 1, wl = warp & 3, t = threadIdx.x & 127;
    uint8_t* obuf = out_tiles + wg * L::kOutBytes;
    float* wS1 = sS1 + wg * 2 * 8 * BLOCK_N;
    float* wS2 = wS1 + 8 * BLOCK_N;
    const bool has_aux = ep.mask_src != nullptr;
    const bool stats = ep.S1 != nullptr;
    uint32_t aux_phase = 0;
    for (int i = wg; unit0 + i * unit_step < num_units; i += 2) {
      const int u = unit0 + i * unit_step;
      const int m_blk = tile_m(u), n_blk = tile_n(u);
      if (has_aux && t == 0) {
        tma_store_wait_read();                          // the previous tile's store has left the buffer
        mbar_expect_tx(&aux_bar[wg], L::kOutBytes);
#pragma unroll
        for (int b = 0; b < BLOCK_N / L::kBoxCols; ++b)
          tma_load_2d(obuf + b * L::kBoxBytes, &tmAux, &aux_bar[wg], n_blk * BLOCK_N + b * L::kBoxCols, m_blk * BLOCK_M);
      }
      float acc[2][kAcc];                               // [64-row half][wgmma fragment]
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int r = 0; r < kAcc; ++r) acc[h][r] = 0.f;
      int prev = -1;
      if (i > 0) order_wait(wg);                        // the mainloop of tile i - 1 (the other warpgroup's) is done
      for (int kb = 0; kb < num_kb; ++kb) {
        const int slot = i * num_kb + kb, stage = slot % kSt;
        mbar_wait(&full_bar[stage], (uint32_t)(slot / kSt) & 1u);
        const uint32_t sa = smem_u32(ring + stage * L::kStageBytes);
        const uint64_t adesc0 = gmma_desc_sw128(sa, 16, 1024);
        const uint64_t adesc1 = gmma_desc_sw128(sa + 64 * 128, 16, 1024);
        const uint64_t bdesc = gmma_desc_sw128(sa + L::kABytes, 16, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma_bf16<BLOCK_N, 0, 0>(acc[0], adesc0 + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), 1);
          wgmma_bf16<BLOCK_N, 0, 0>(acc[1], adesc1 + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), 1);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
      }
      if (unit0 + (i + 1) * unit_step < num_units) order_signal(wg);   // only a tile that exists waits for this arrival
      wgmma_wait<0>();
      wgmma_fence_acc(acc[0]);
      wgmma_fence_acc(acc[1]);
      if (lane == 0) mbar_arrive(&empty_bar[prev]);

      if (has_aux) {
        mbar_wait(&aux_bar[wg], aux_phase);
        aux_phase ^= 1;
      } else {
        if (t == 0) tma_store_wait_read();
        wg_bar_sync(wg);
      }
      // ---- epilogue: the arithmetic and the statistics' summation order of the cooperative epilogue below, row group g = 4 half + wl.
      // It runs on 4 warps, one per SM sub-partition, so its time is latency, not issue: the aux mode, the statistics and whether the
      // tile lies wholly inside M x N are template arguments, so the element loop does not branch or reconverge on any of them.
      // The statistics use the shuffle tree of the cooperative epilogue (row lanes paired by xor 1, 2, 4 of lane / 4), but a pair of
      // lanes exchanges only the half of its column partials that the other lane keeps: 4 shuffles per 8 columns instead of 12, and
      // each add sees the same two operands, so the same bits.
      auto epilogue = [&](auto full_c, auto auxm_c, auto stats_c) {
        constexpr bool kFull = decltype(full_c)::value;
        constexpr int kAuxM = decltype(auxm_c)::value;  // 0: no aux element read   1: ReLU-backward mask   2: S2 partner
        constexpr bool kStats = decltype(stats_c)::value;
        const uint32_t obuf_s = smem_u32(obuf);
        const bool relu = ep.relu != 0;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int lrow0 = half * 64 + wl * 16 + (lane >> 2);
          const int row0 = m_blk * BLOCK_M + lrow0;
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j) {
            const int lcol = 8 * j + 2 * (lane & 3);
            const int col = n_blk * BLOCK_N + lcol;
            const bool col_ok = kFull || col < N;
            float b0 = 0.f, b1 = 0.f;
            if (col_ok && ep.bias) { b0 = __ldg(ep.bias + col); b1 = __ldg(ep.bias + col + 1); }
            float p1[2] = {0.f, 0.f}, p2[2] = {0.f, 0.f};
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = row0 + 8 * h;
              const bool ok = kFull || (col_ok && row < M);
              float v0 = acc[half][4 * j + 2 * h] + b0;
              float v1 = acc[half][4 * j + 2 * h + 1] + b1;
              v0 = relu ? fmaxf(v0, 0.f) : v0;
              v1 = relu ? fmaxf(v1, 0.f) : v1;
              const uint32_t sp = obuf_s + out_tile_offset<BLOCK_N>(lrow0 + 8 * h, lcol);
              float w0 = 0.f, w1 = 0.f;
              if (kAuxM != 0 && ok) {
                uint32_t raw;
                asm volatile("ld.shared.b32 %0, [%1];" : "=r"(raw) : "r"(sp));
                const float2 w = unpack_bf16x2(raw);
                w0 = w.x; w1 = w.y;
                if (kAuxM == 1) { v0 = w0 > 0.f ? v0 : 0.f; v1 = w1 > 0.f ? v1 : 0.f; }
              }
              // rows >= M and columns >= N are clipped by the store's tensor map
              asm volatile("st.shared.b32 [%0], %1;" ::"r"(sp), "r"(pack_bf16x2(v0, v1)));
              if (ok) {
                if (ep.out_f32) *reinterpret_cast<float2*>(ep.out_f32 + (int64_t)row * ep.ldc + col) = make_float2(v0, v1);
                if (kStats) {
                  p1[0] += v0; p1[1] += v1;
                  const float a0 = kAuxM == 2 ? w0 : v0, a1 = kAuxM == 2 ? w1 : v1;
                  p2[0] += v0 * a0; p2[1] += v1 * a1;
                }
              }
            }
            if (kStats) {
              // partial k = 2 s + c (s: S1 / S2, c: column 2 (lane & 3) + c).  Row bit 0 (lane xor 4): keep partials 2 b, 2 b + 1;
              // row bit 1 (xor 8): keep 2 b + c; row bit 2 (xor 16): both lanes keep it.  Lanes 0-15 then hold the group's sums.
              const bool b = (lane >> 2) & 1, c = (lane >> 3) & 1;
              const float s0 = b ? p1[0] : p2[0], s1 = b ? p1[1] : p2[1];
              float y0 = b ? p2[0] : p1[0], y1 = b ? p2[1] : p1[1];
              const float r0 = __shfl_xor_sync(0xffffffffu, s0, 4), r1 = __shfl_xor_sync(0xffffffffu, s1, 4);
              y0 += r0; y1 += r1;
              float z = c ? y1 : y0;
              z += __shfl_xor_sync(0xffffffffu, c ? y0 : y1, 8);
              z += __shfl_xor_sync(0xffffffffu, z, 16);
              if (lane < 16) (b ? wS2 : wS1)[(4 * half + wl) * BLOCK_N + lcol + (c ? 1 : 0)] = z;
            }
          }
        }
      };
      {
        using F = std::false_type;
        using T = std::true_type;
        using A0 = std::integral_constant<int, 0>;
        using A1 = std::integral_constant<int, 1>;
        using A2 = std::integral_constant<int, 2>;
        const bool full = (m_blk + 1) * BLOCK_M <= M && (n_blk + 1) * BLOCK_N <= N;
        const int auxm = !has_aux ? 0 : ep.aux_mode == 1 ? 1 : ep.aux_mode == 2 ? 2 : 0;
        auto by_aux = [&](auto full_c, auto stats_c) {
          if (auxm == 1) epilogue(full_c, A1{}, stats_c);
          else if (auxm == 2) epilogue(full_c, A2{}, stats_c);
          else epilogue(full_c, A0{}, stats_c);
        };
        if (full) { if (stats) by_aux(T{}, T{}); else by_aux(T{}, F{}); }
        else { if (stats) by_aux(F{}, T{}); else by_aux(F{}, F{}); }
      }
      fence_proxy_async();                              // the generic-proxy tile writes are visible to the TMA store
      wg_bar_sync(wg);
      if (t == 0) {
#pragma unroll
        for (int b = 0; b < BLOCK_N / L::kBoxCols; ++b)
          tma_store_2d(&tmOut, obuf + b * L::kBoxBytes, n_blk * BLOCK_N + b * L::kBoxCols, m_blk * BLOCK_M);
        tma_store_commit();
      }
      if (stats) {                                      // the tile's column sums, row groups added in row order -> workspace row m_blk
        for (int c = t; c < BLOCK_N; c += 128) {
          const int col = n_blk * BLOCK_N + c;
          if (col < N) {
            float a1 = 0.f, a2 = 0.f;
#pragma unroll
            for (int g = 0; g < 8; ++g) { a1 += wS1[g * BLOCK_N + c]; a2 += wS2[g * BLOCK_N + c]; }
            ep.stat_ws[(int64_t)m_blk * 2 * N + col] = a1;
            ep.stat_ws[(int64_t)m_blk * 2 * N + N + col] = a2;
          }
        }
        wg_bar_sync(wg);
      }
    }
    if (t == 0) tma_store_wait_all();                   // the output is in global memory before the CTA retires (PDL dependents read it)
  } else {
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
      if constexpr (EPI == kEpiLayerNorm) {
        // rows row0 and row0 + 8 of this thread: the 4 lanes of a quad hold all BLOCK_N columns of both.  h = acc + bias; the mean and the
        // two-pass variance over the N real columns are in-thread sums plus two shuffles inside the quad.
        const float inv_n = 1.f / (float)N;
        float sum[2] = {0.f, 0.f};
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int col = 8 * j + 2 * (lane & 3);
          if (col < N) {
            const float b0 = ep.bias ? __ldg(ep.bias + col) : 0.f, b1 = ep.bias ? __ldg(ep.bias + col + 1) : 0.f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              acc[4 * j + 2 * h] += b0; acc[4 * j + 2 * h + 1] += b1;
              sum[h] += acc[4 * j + 2 * h] + acc[4 * j + 2 * h + 1];
            }
          }
        }
        float mu[2], sq[2] = {0.f, 0.f}, rs[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 1);
          sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 2);
          mu[h] = sum[h] * inv_n;
        }
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          if (8 * j + 2 * (lane & 3) < N) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float d0 = acc[4 * j + 2 * h] - mu[h], d1 = acc[4 * j + 2 * h + 1] - mu[h];
              sq[h] = fmaf(d0, d0, fmaf(d1, d1, sq[h]));
            }
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          sq[h] += __shfl_xor_sync(0xffffffffu, sq[h], 1);
          sq[h] += __shfl_xor_sync(0xffffffffu, sq[h], 2);
          rs[h] = rsqrtf(sq[h] * inv_n + ep.eps);
          const int row = row0 + 8 * h;
          if (ep.rstd && (lane & 3) == 0 && row < M) ep.rstd[row] = rs[h];
        }
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int col = 8 * j + 2 * (lane & 3);
          if (col < N) {
            const float g0 = __ldg(ep.gamma + col), g1 = __ldg(ep.gamma + col + 1);
            const float e0 = __ldg(ep.beta + col), e1 = __ldg(ep.beta + col + 1);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = row0 + 8 * h;
              if (row < M) {
                const float x0 = (acc[4 * j + 2 * h] - mu[h]) * rs[h], x1 = (acc[4 * j + 2 * h + 1] - mu[h]) * rs[h];
                float y0 = fmaf(g0, x0, e0), y1 = fmaf(g1, x1, e1);
                if (ep.relu) { y0 = fmaxf(y0, 0.f); y1 = fmaxf(y1, 0.f); }
                *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(ep.out) + (int64_t)row * ep.ldc + col) = pack_bf16x2(y0, y1);
                if (ep.xhat) *reinterpret_cast<uint32_t*>(ep.xhat + (int64_t)row * ep.ld_xhat + col) = pack_bf16x2(x0, x1);
              }
            }
          }
        }
        continue;
      }
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
          if constexpr (EPI == kEpiCross) {               // u = acc + bias;  out = x0 * u + x_l
            if (ok) {
              if (ep.u_out) *reinterpret_cast<uint32_t*>(ep.u_out + (int64_t)row * ep.ld_u + col) = pack_bf16x2(v0, v1);
              const float2 x = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(ep.x0 + (int64_t)row * ep.ld_x0 + col));
              v0 = fmaf(x.x, v0, w0); v1 = fmaf(x.y, v1, w1);
            }
          } else if constexpr (EPI == kEpiResidual) {     // out = acc + aux
            v0 += w0; v1 += w1;
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

template <int BN, bool BRES, bool CL2, bool FP8, bool MX = false, bool PP = false, int EPI = kEpiPlain>
int launch_tn(const CUtensorMap& ta, const void* B, int M, int N, int K, int64_t ldb, const EpiT<EPI>& ep, int max_ctas, cudaStream_t s) {
  CUtensorMap tb, tout = {}, taux = {};
  const uint32_t box_rows = CL2 ? BN / 2 : BN;
  int rc = FP8 ? make_tmap(&tb, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb, 128, box_rows, CU_TENSOR_MAP_DATA_TYPE_UINT8)
               : make_tmap(&tb, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb * 2, BLOCK_K, box_rows);
  if (rc) return rc;
  using L = SmemLayoutTN<BN, BRES, PP>;
  static_assert(L::kTotal <= 227 * 1024, "shared-memory budget");
  if constexpr (PP) {       // output and aux tiles in the kernel's swizzled smem layout; dims {N, M}: stores never pass column N or row M
    const CUtensorMapSwizzle sw = L::kRowBytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : L::kRowBytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                                                                        : CU_TENSOR_MAP_SWIZZLE_32B;
    rc = make_tmap(&tout, ep.out, (uint64_t)N, (uint64_t)M, (uint64_t)ep.ldc * 2, L::kBoxCols, BLOCK_M, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, sw);
    if (rc) return rc;
    if (ep.mask_src) {
      rc = make_tmap(&taux, ep.mask_src, (uint64_t)N, (uint64_t)M, (uint64_t)ep.ld_mask * 2, L::kBoxCols, BLOCK_M, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, sw);
      if (rc) return rc;
    }
  }
  auto kern = k_gemm_tn<BN, BRES, CL2, FP8, MX, PP, EPI>;
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
    DR_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, ta, tb, tout, taux, M, N, K, ep));
  } else {
    DR_PDL_LAUNCH(kern, grid, kGemmThreads, L::kTotal, s, ta, tb, tout, taux, M, N, K, ep);
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
  // the ping-pong kernel reads the aux tile by TMA, which needs a 16-byte aligned base and pitch; the contract does not ask that of
  // mask_src / ld_mask, so any other aux operand runs the cooperative kernel (same results bit for bit)
  const bool aux_tma = !ep.mask_src || ((((uintptr_t)ep.mask_src) & 15) == 0 && ep.ld_mask % 8 == 0 && ep.ld_mask >= N);
  if (aux_tma) return launch_tn<BN, false, false, false, false, true>(ta, B, M, N, K, ldb, ep, max_ctas, s);
  return launch_tn<BN, false, false, false>(ta, B, M, N, K, ldb, ep, max_ctas, s);
}

// -------------------------------------------------------------------------------------------------
// Grouped GEMMs (expert MLPs: nn.fused_expert_mlps): G problems of one shape in one persistent launch.
//   k_gemm_tn_grouped        out_g = A_g B_g^T (+bias_g)(ReLU)(* relu-mask_g)(S1_g column sums) over the tiles (g, m, n), g-major; a tile
//                            runs the mainloop and the kind-0 epilogue of k_gemm_tn's cooperative consumers, so each group's output and
//                            statistics are bit-identical to a dr_cuda_gemm_tn_ex call on that group.  The kernel is separate from
//                            k_gemm_tn so that k_gemm_tn's instantiations stay exactly as they were.
//   k_gemm_nt_splitk_grouped k_gemm_nt_splitk with blockIdx.z = g * splits + split, then k_dw_reduce_grouped (blockIdx.y = g) adds each
//                            group's splits in order, as dr_cuda_gemm_dw does.
// The per-group tensor maps are __grid_constant__ kernel parameters: no host-to-device copy per call and no tensormap fence, and a captured
// CUDA graph holds them by value.  kMaxGroups is what fits the classic 4 KB parameter space: 12 x (2 x 128 B maps + 40 B of operands).
// -------------------------------------------------------------------------------------------------
constexpr int kMaxGroups = 12;

struct GroupTN {
  const float* bias;                  // [N] or null
  const __nv_bfloat16* mask;          // aux tile (aux_mode 1) or null
  __nv_bfloat16* out;
  int64_t ldc, ld_mask;
};
struct GroupedTN {
  CUtensorMap tmA[kMaxGroups];
  CUtensorMap tmB[kMaxGroups];
  GroupTN g[kMaxGroups];
  float* stat_ws;                     // [m_tiles][G N]: the S1 partials of group g in columns [g N, g N + N) (or null)
  int G, relu;
};
static_assert(sizeof(GroupedTN) + 3 * sizeof(int) <= 4096, "grouped GEMM parameters exceed the 4 KB kernel parameter space");

template <int BLOCK_N>
__global__ void __launch_bounds__(kGemmThreads, 1) k_gemm_tn_grouped(const __grid_constant__ GroupedTN p, int M, int N, int K) {
  using L = SmemLayoutTN<BLOCK_N, false>;
  constexpr int kSt = L::kSt;
  constexpr int kAcc = BLOCK_N / 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* ring = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* sS1 = reinterpret_cast<float*>(ring + kSt * L::kStageBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sS1) + L::kStatBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kSt;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_tiles = (M + BLOCK_M - 1) / BLOCK_M;
  const int n_tiles = (N + BLOCK_N - 1) / BLOCK_N;
  const int tiles = m_tiles * n_tiles;
  const int num_kb = (K + BLOCK_K - 1) / BLOCK_K;
  const int num_units = p.G * tiles;

  if (threadIdx.x == 0) {
    for (int g = 0; g < p.G; ++g) { tma_prefetch_desc(&p.tmA[g]); tma_prefetch_desc(&p.tmB[g]); }
    for (int i = 0; i < kSt; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_sync();

  if (warp < 4) {
    if (warp == 0 && lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int u = blockIdx.x; u < num_units; u += gridDim.x) {
        const int g = u / tiles, m_blk = (u % tiles) / n_tiles, n_blk = u % n_tiles;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = ring + stage * L::kStageBytes;
          mbar_expect_tx(&full_bar[stage], L::kStageBytes);
          tma_load_2d(sa, &p.tmA[g], &full_bar[stage], kb * BLOCK_K, m_blk * BLOCK_M);
          tma_load_2d(sa + L::kABytes, &p.tmB[g], &full_bar[stage], kb * BLOCK_K, n_blk * BLOCK_N);
          if (++stage == kSt) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    const int wg = (warp >> 2) - 1;
    const int wl = warp & 3;
    const int ct = threadIdx.x - 128;
    int stage = 0; uint32_t phase = 0;
    const bool stats = p.stat_ws != nullptr;
    for (int u = blockIdx.x; u < num_units; u += gridDim.x) {
      const int g = u / tiles, m_blk = (u % tiles) / n_tiles, n_blk = u % n_tiles;
      float acc[kAcc];
#pragma unroll
      for (int i = 0; i < kAcc; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(ring + stage * L::kStageBytes) + wg * 64 * 128;
        const uint32_t sb = smem_u32(ring + stage * L::kStageBytes) + L::kABytes;
        const uint64_t adesc = gmma_desc_sw128(sa, 16, 1024);
        const uint64_t bdesc = gmma_desc_sw128(sb, 16, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_bf16<BLOCK_N, 0, 0>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), 1);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == kSt) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if (lane == 0) mbar_arrive(&empty_bar[prev]);

      // ---- the kind-0 epilogue of k_gemm_tn: bias, ReLU, aux-mode-1 mask, S1 partials in the same order
      const GroupTN& q = p.g[g];
      const int row0 = m_blk * BLOCK_M + wg * 64 + wl * 16 + (lane >> 2);
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int col = n_blk * BLOCK_N + 8 * j + 2 * (lane & 3);
        const bool col_ok = col < N;
        float b0 = 0.f, b1 = 0.f;
        if (col_ok && q.bias) { b0 = __ldg(q.bias + col); b1 = __ldg(q.bias + col + 1); }
        float p1[2] = {0.f, 0.f};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = row0 + 8 * h;
          const bool ok = col_ok && row < M;
          float v0 = acc[4 * j + 2 * h] + b0;
          float v1 = acc[4 * j + 2 * h + 1] + b1;
          if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
          if (q.mask && ok) {
            const __nv_bfloat16* ms = q.mask + (int64_t)row * q.ld_mask + col;
            if (!(__bfloat162float(ms[0]) > 0.f)) v0 = 0.f;
            if (!(__bfloat162float(ms[1]) > 0.f)) v1 = 0.f;
          }
          if (ok) {
            *reinterpret_cast<uint32_t*>(q.out + (int64_t)row * q.ldc + col) = pack_bf16x2(v0, v1);
            if (stats) { p1[0] += v0; p1[1] += v1; }
          }
        }
        if (stats) {
#pragma unroll
          for (int c = 0; c < 2; ++c)
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) p1[c] += __shfl_xor_sync(0xffffffffu, p1[c], o);
          if (lane < 4) {
            float* r1 = sS1 + (warp - 4) * BLOCK_N + 8 * j + 2 * lane;
            r1[0] = p1[0]; r1[1] = p1[1];
          }
        }
      }
      if (stats) {
        consumer_bar_sync();
        for (int i = ct; i < BLOCK_N; i += 256) {
          const int col = n_blk * BLOCK_N + i;
          if (col < N) {
            float a1 = 0.f;
#pragma unroll
            for (int w = 0; w < 8; ++w) a1 += sS1[w * BLOCK_N + i];
            p.stat_ws[(int64_t)m_blk * p.G * N + (int64_t)g * N + col] = a1;
          }
        }
        consumer_bar_sync();
      }
    }
  }
}

struct GroupedNT {
  CUtensorMap tmA[kMaxGroups];
  CUtensorMap tmB[kMaxGroups];
};

template <int BLOCK_N>
__global__ void __launch_bounds__(kGemmThreads, 1)
k_gemm_nt_splitk_grouped(const __grid_constant__ GroupedNT p, int Mo, int No, int batch, int rows_per_split, int splits, float* __restrict__ part) {
  using L = SmemLayoutNT<BLOCK_N>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * L::kStageBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_blk = blockIdx.x, n_blk = blockIdx.y, g = blockIdx.z / splits, split = blockIdx.z % splits;
  const CUtensorMap* tmA = &p.tmA[g];
  const CUtensorMap* tmB = &p.tmB[g];
  const int b0 = split * rows_per_split;
  const int b1 = min(batch, b0 + rows_per_split);
  const int num_kb = (b1 - b0 + BLOCK_KB - 1) / BLOCK_KB;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(tmA); tma_prefetch_desc(tmB);
    for (int i = 0; i < kStages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_sync();
  if (num_kb <= 0) return;

  if (warp == 0) {
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sa = smem + stage * L::kStageBytes;
        uint8_t* sb = sa + L::kAChunks * kChunkBytes;
        mbar_expect_tx(&full_bar[stage], L::kStageBytes);
        const int brow = b0 + kb * BLOCK_KB;
#pragma unroll
        for (int c = 0; c < L::kAChunks; ++c) tma_load_2d(sa + c * kChunkBytes, tmA, &full_bar[stage], m_blk * BLOCK_M + c * 64, brow);
#pragma unroll
        for (int c = 0; c < L::kBChunks; ++c) tma_load_2d(sb + c * kChunkBytes, tmB, &full_bar[stage], n_blk * BLOCK_N + c * 64, brow);
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {
    const int wg = (warp >> 2) - 1, wl = warp & 3;
    float acc[BLOCK_N / 2];
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
    int stage = 0; uint32_t phase = 0, prev = 0;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * L::kStageBytes) + wg * kChunkBytes;
      const uint32_t sb = smem_u32(smem + stage * L::kStageBytes) + L::kAChunks * kChunkBytes;
      const uint64_t adesc = gmma_desc_sw128(sa, kChunkBytes, 1024);
      const uint64_t bdesc = gmma_desc_sw128(sb, kChunkBytes, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_KB / 16; ++k)
        wgmma_bf16<BLOCK_N, 1, 1>(acc, adesc + (uint64_t)(k * 128), bdesc + (uint64_t)(k * 128), 1);
      wgmma_commit();
      wgmma_wait<1>();
      if (kb > 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    float* gpart = part + (int64_t)g * splits * Mo * No;
    const int row0 = m_blk * BLOCK_M + wg * 64 + wl * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      const int col = n_blk * BLOCK_N + 8 * j + 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = row0 + 8 * h;
        if (row >= Mo) continue;
        float* dst = gpart + ((int64_t)split * Mo + row) * No + col;
        if (col < No) dst[0] = acc[4 * j + 2 * h];
        if (col + 1 < No) dst[1] = acc[4 * j + 2 * h + 1];
      }
    }
  }
}

struct GroupedDW { float* dW[kMaxGroups]; int64_t ldw[kMaxGroups]; };

// k_dw_reduce for group blockIdx.y: its splits added in order
__global__ void k_dw_reduce_grouped(const float* __restrict__ part, int splits, int Mo, int No, const __grid_constant__ GroupedDW d) {
  const int64_t n = (int64_t)Mo * No;
  const int g = blockIdx.y;
  const float* gp = part + (int64_t)g * splits * n;
  float* dW = d.dW[g];
  const int64_t ldw = d.ldw[g];
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float sum = 0.f;
    for (int k = 0; k < splits; ++k) sum += gp[k * n + i];
    dW[(i / No) * ldw + i % No] += sum;
  }
}

template <int BN>
int launch_tn_grouped(const GroupedTN& p, int M, int N, int K, int max_ctas, cudaStream_t s) {
  using L = SmemLayoutTN<BN, false>;
  static DrPerDeviceOnce attr_once; bool& attr_set = attr_once();
  if (!attr_set) {
    DR_CUDA_CHECK(cudaFuncSetAttribute(k_gemm_tn_grouped<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal));
    attr_set = true;
  }
  int grid = p.G * ((M + BLOCK_M - 1) / BLOCK_M) * ((N + BN - 1) / BN);
  if (grid > max_ctas) grid = max_ctas;
  DR_PDL_LAUNCH(k_gemm_tn_grouped<BN>, grid, kGemmThreads, L::kTotal, s, p, M, N, K);
  DR_LAUNCH_CHECK();
  return 0;
}

template <int BN>
int launch_nt_grouped(const GroupedNT& p, int G, int Mo, int No, int batch, int splits, const GroupedDW& d, cudaStream_t s) {
  using L = SmemLayoutNT<BN>;
  static DrPerDeviceOnce attr_once; bool& attr_set = attr_once();
  if (!attr_set) {
    DR_CUDA_CHECK(cudaFuncSetAttribute(k_gemm_nt_splitk_grouped<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal));
    attr_set = true;
  }
  int rows_per_split = ((batch + splits - 1) / splits + BLOCK_KB - 1) / BLOCK_KB * BLOCK_KB;     // as launch_nt
  splits = (batch + rows_per_split - 1) / rows_per_split;
  float* part = dr_workspace(kWsGemmDw, (size_t)G * splits * Mo * No, s);
  if (!part) return -5;
  dim3 grid((Mo + BLOCK_M - 1) / BLOCK_M, (No + BN - 1) / BN, G * splits);
  DR_PDL_LAUNCH((k_gemm_nt_splitk_grouped<BN>), grid, kGemmThreads, L::kTotal, s, p, Mo, No, batch, rows_per_split, splits, part);
  DR_LAUNCH_CHECK();
  const int64_t n = (int64_t)Mo * No;
  k_dw_reduce_grouped<<<dim3((unsigned)std::min<int64_t>((n + 255) / 256, num_sms() * 8), G), 256, 0, s>>>(part, splits, Mo, No, d);
  DR_LAUNCH_CHECK();
  return 0;
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
// Contract (the emulation stand-in in emu/emu_stubs.cu checks and computes the same):
//   -2  lda, ldb, ldc or N not a multiple of 8;  -3  A, B or out not 16-byte aligned;  -5  lda < K, ldb < K or ldc < N;
//   -4  S2 without S1, or aux_mode 2 without mask_src.
//   out and out_f32 share the row pitch ldc.  S1 / S2 are accumulated into (+=) and sum the fp32 epilogue values (after bias, ReLU and
//   mask, before the bf16 rounding of `out`) of rows < M only; S2 multiplies by the aux value in aux_mode 2, by the value itself otherwise.
//   Any N (a multiple of 8) may carry statistics, with or without out_f32.
int dr_cuda_gemm_tn_ex(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, const float* bias, int relu,
                       const void* mask_src, int64_t ld_mask, int aux_mode, void* out, int64_t ldc, float* out_f32, float* S1, float* S2,
                       int max_ctas, int force_v1, cudaStream_t s) {
  (void)force_v1;
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if ((lda % 8) || (ldb % 8) || (ldc % 8) || (N % 8)) return -2;
  if (((uintptr_t)A | (uintptr_t)B | (uintptr_t)out) & 15) return -3;
  if (lda < K || ldb < K || ldc < N) return -5;
  if ((S2 && !S1) || (aux_mode == 2 && !mask_src)) return -4;
  if (max_ctas <= 0) max_ctas = num_sms();
  CUtensorMap ta;
  int rc = make_tmap(&ta, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda * 2, BLOCK_K, BLOCK_M);
  if (rc) return rc;
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
  det_colsum(ws, m_tiles, 2 * (int64_t)N, {{0, N, S1}, {N, N, S2}}, s);
  DR_LAUNCH_CHECK();
  return 0;
}

// Low-rank cross layer epilogues (DLRM-DCNv2, models/dlrm_engine.py), on the cooperative kernel at every K:
//   kind 1 (cross):     out = x0 * (acc + bias) + xl        and, if u_out is given, u_out = acc + bias (bf16)
//   kind 2 (residual):  out = acc + xl
// with acc = A[M,K](lda) * B[N,K](ldb)^T in fp32 and the epilogue in fp32 from the bf16 operands, out rounded once to bf16.  bias may be
// null.  Contract of dr_cuda_gemm_tn_ex for A, B and out, and for the new operands:  -2  a pitch of xl, x0 or u_out not a multiple of 8;
// -3  xl, x0 or u_out not 16-byte aligned;  -5  ld_xl, ld_x0 or ld_u < N;  -4  an unknown kind, xl missing, or kind 1 without x0.
int dr_cuda_gemm_tn_cross(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, const float* bias, int kind,
                          const void* x0, int64_t ld_x0, const void* xl, int64_t ld_xl, void* out, int64_t ldc, void* u_out, int64_t ld_u,
                          int max_ctas, cudaStream_t s) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if ((kind != kEpiCross && kind != kEpiResidual) || !xl || (kind == kEpiCross && !x0)) return -4;
  if (kind != kEpiCross) { x0 = nullptr; u_out = nullptr; }
  if ((lda % 8) || (ldb % 8) || (ldc % 8) || (N % 8) || (ld_xl % 8) || (x0 && ld_x0 % 8) || (u_out && ld_u % 8)) return -2;
  if (((uintptr_t)A | (uintptr_t)B | (uintptr_t)out | (uintptr_t)xl | (uintptr_t)x0 | (uintptr_t)u_out) & 15) return -3;
  if (lda < K || ldb < K || ldc < N || ld_xl < N || (x0 && ld_x0 < N) || (u_out && ld_u < N)) return -5;
  if (max_ctas <= 0) max_ctas = num_sms();
  CUtensorMap ta;
  int rc = make_tmap(&ta, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda * 2, BLOCK_K, BLOCK_M);
  if (rc) return rc;
  EpilogueX ep;
  static_cast<Epilogue&>(ep) = Epilogue{bias, (const __nv_bfloat16*)xl, out, nullptr, ldc, ld_xl, 0, 0, nullptr, nullptr, nullptr, nullptr, 0, 1.f};
  ep.x0 = (const __nv_bfloat16*)x0; ep.u_out = (__nv_bfloat16*)u_out; ep.ld_x0 = ld_x0; ep.ld_u = ld_u;
#define TN_EPI(BN)                                                                                                             \
  (kind == kEpiCross ? launch_tn<BN, false, false, false, false, false, kEpiCross>(ta, B, M, N, K, ldb, ep, max_ctas, s)      \
                     : launch_tn<BN, false, false, false, false, false, kEpiResidual>(ta, B, M, N, K, ldb, ep, max_ctas, s))
  rc = N <= 16 ? TN_EPI(16) : N <= 32 ? TN_EPI(32) : N <= 64 ? TN_EPI(64) : TN_EPI(128);
#undef TN_EPI
  return rc;
}

// LayerNorm epilogue (MaskNet's MaskBlock, nn.FusedMaskBlock), on the cooperative kernel at every K:
//   h = acc + bias,  x^ = (h - mean_row(h)) * rstd,  rstd = 1 / sqrt(var_row(h) + eps),  out = relu?(gamma * x^ + beta)
// with acc = A[M,K](lda) * B[N,K](ldb)^T in fp32, the row mean and the two-pass variance sum((h - mean)^2) / N over the N columns from the
// fp32 accumulators, out rounded once to bf16.  bias may be null; x^ (bf16, pitch ld_xhat) and rstd (fp32 [M]) are optional.  out may be a
// column slice of a wider buffer (ldc > N).  Contract of dr_cuda_gemm_tn_ex for A, B and out, and:  -2  N > 128 (a row must fit one tile),
// N or a pitch of out / xhat not a multiple of 8;  -3  xhat not 16-byte aligned;  -5  ld_xhat < N;  -4  gamma or beta missing.
int dr_cuda_gemm_tn_ln(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, const float* bias, const float* gamma,
                       const float* beta, float eps, int relu, void* out, int64_t ldc, void* xhat, int64_t ld_xhat, float* rstd, int max_ctas,
                       cudaStream_t s) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if (!gamma || !beta) return -4;
  if ((lda % 8) || (ldb % 8) || (ldc % 8) || (N % 8) || N > 128 || (xhat && ld_xhat % 8)) return -2;
  if (((uintptr_t)A | (uintptr_t)B | (uintptr_t)out | (uintptr_t)xhat) & 15) return -3;
  if (lda < K || ldb < K || ldc < N || (xhat && ld_xhat < N)) return -5;
  if (max_ctas <= 0) max_ctas = num_sms();
  CUtensorMap ta;
  int rc = make_tmap(&ta, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda * 2, BLOCK_K, BLOCK_M);
  if (rc) return rc;
  EpilogueLN ep;
  static_cast<Epilogue&>(ep) = Epilogue{bias, nullptr, out, nullptr, ldc, 0, relu, 0, nullptr, nullptr, nullptr, nullptr, 0, 1.f};
  ep.gamma = gamma; ep.beta = beta; ep.xhat = (__nv_bfloat16*)xhat; ep.rstd = rstd; ep.ld_xhat = ld_xhat; ep.eps = eps;
  if (N <= 16) return launch_tn<16, false, false, false, false, false, kEpiLayerNorm>(ta, B, M, N, K, ldb, ep, max_ctas, s);
  if (N <= 32) return launch_tn<32, false, false, false, false, false, kEpiLayerNorm>(ta, B, M, N, K, ldb, ep, max_ctas, s);
  if (N <= 64) return launch_tn<64, false, false, false, false, false, kEpiLayerNorm>(ta, B, M, N, K, ldb, ep, max_ctas, s);
  return launch_tn<128, false, false, false, false, false, kEpiLayerNorm>(ta, B, M, N, K, ldb, ep, max_ctas, s);
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

// G GEMMs of one shape in one launch (k_gemm_tn_grouped): out[g][M,N] = A[g][M,K](lda[g]) * B[g][N,K](ldb[g])^T (+bias[g])(relu)(*mask[g]).
// The per-group arguments are host arrays of G entries; bias, mask_src (with ld_mask) and S1 may be null arrays, and bias[g] / mask_src[g]
// null entries.  A non-null mask_src[g] is the ReLU-backward mask of dr_cuda_gemm_tn_ex's aux_mode 1; S1[g] (all non-null when S1 is given)
// is accumulated into with the column sums of rows < M.  Each group's out and S1 are bit-identical to a dr_cuda_gemm_tn_ex call on it.
// Codes:  -6  G outside [1, kMaxGroups];  then per group in order the codes of dr_cuda_gemm_tn_ex:  -2  lda, ldb, ldc or N not a multiple
// of 8;  -3  A, B or out not 16-byte aligned;  -5  lda < K, ldb < K, ldc < N (or no workspace);  -4  S1 given with a null entry.
int dr_cuda_gemm_tn_grouped(int G, const void* const* A, const int64_t* lda, const void* const* B, const int64_t* ldb, int M, int N, int K,
                            const float* const* bias, int relu, const void* const* mask_src, const int64_t* ld_mask, void* const* out,
                            const int64_t* ldc, float* const* S1, int max_ctas, cudaStream_t s) {
  if (G < 1 || G > kMaxGroups) return -6;
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  for (int g = 0; g < G; ++g) {
    if ((lda[g] % 8) || (ldb[g] % 8) || (ldc[g] % 8) || (N % 8)) return -2;
    if (((uintptr_t)A[g] | (uintptr_t)B[g] | (uintptr_t)out[g]) & 15) return -3;
    if (lda[g] < K || ldb[g] < K || ldc[g] < N) return -5;
    if (S1 && !S1[g]) return -4;
  }
  if (max_ctas <= 0) max_ctas = num_sms();
  const int BN = N <= 16 ? 16 : N <= 32 ? 32 : N <= 64 ? 64 : 128;      // the tile width dr_cuda_gemm_tn_ex picks
  GroupedTN p;
  memset(&p, 0, sizeof(p));
  p.G = G; p.relu = relu;
  for (int g = 0; g < G; ++g) {
    int rc = make_tmap(&p.tmA[g], A[g], (uint64_t)K, (uint64_t)M, (uint64_t)lda[g] * 2, BLOCK_K, BLOCK_M);
    if (rc) return rc;
    rc = make_tmap(&p.tmB[g], B[g], (uint64_t)K, (uint64_t)N, (uint64_t)ldb[g] * 2, BLOCK_K, (uint32_t)BN);
    if (rc) return rc;
    p.g[g] = GroupTN{bias ? bias[g] : nullptr, mask_src ? (const __nv_bfloat16*)mask_src[g] : nullptr, (__nv_bfloat16*)out[g], ldc[g],
                     mask_src ? ld_mask[g] : 0};
  }
  const int m_tiles = (M + BLOCK_M - 1) / BLOCK_M;
  if (S1) {
    p.stat_ws = dr_workspace(kWsGemmStats, (size_t)m_tiles * G * N, s);
    if (!p.stat_ws) return -5;
  }
  int rc = BN == 16 ? launch_tn_grouped<16>(p, M, N, K, max_ctas, s)
         : BN == 32 ? launch_tn_grouped<32>(p, M, N, K, max_ctas, s)
         : BN == 64 ? launch_tn_grouped<64>(p, M, N, K, max_ctas, s)
                    : launch_tn_grouped<128>(p, M, N, K, max_ctas, s);
  if (rc || !S1) return rc;
  for (int g = 0; g < G; g += kDetColsumMaxRanges) {     // workspace row m_blk holds every group's tile sums: one range per group
    DetColsumRange r[kDetColsumMaxRanges] = {};
    for (int j = 0; j < kDetColsumMaxRanges && g + j < G; ++j) r[j] = DetColsumRange{(int64_t)(g + j) * N, N, S1[g + j]};
    det_colsum(p.stat_ws, m_tiles, (int64_t)G * N, r, s);
    DR_LAUNCH_CHECK();
  }
  return 0;
}

// G weight gradients of one shape (k_gemm_nt_splitk_grouped): dW[g][N_out,K_in](ldw[g], fp32, accumulated into) += dY[g]^T * X[g], with
// the split count and the in-order split sums of dr_cuda_gemm_dw, so each group's dW is bit-identical to a dr_cuda_gemm_dw call on it.
// Codes:  -6  G outside [1, kMaxGroups];  -2  ldy or ldx not a multiple of 8;  -5  no workspace.
int dr_cuda_gemm_dw_grouped(int G, const void* const* dY, const int64_t* ldy, const void* const* X, const int64_t* ldx, int batch, int N_out,
                            int K_in, float* const* dW, const int64_t* ldw, int splits, cudaStream_t s) {
  if (G < 1 || G > kMaxGroups) return -6;
  if (batch <= 0 || N_out <= 0 || K_in <= 0) return 0;
  for (int g = 0; g < G; ++g)
    if ((ldy[g] % 8) || (ldx[g] % 8)) return -2;
  GroupedNT p;
  memset(&p, 0, sizeof(p));
  GroupedDW d{};
  for (int g = 0; g < G; ++g) {
    int rc = make_tmap(&p.tmA[g], dY[g], (uint64_t)N_out, (uint64_t)batch, (uint64_t)ldy[g] * 2, 64, BLOCK_KB);
    if (rc) return rc;
    rc = make_tmap(&p.tmB[g], X[g], (uint64_t)K_in, (uint64_t)batch, (uint64_t)ldx[g] * 2, 64, BLOCK_KB);
    if (rc) return rc;
    d.dW[g] = dW[g]; d.ldw[g] = ldw[g];
  }
  const int m_tiles = (N_out + BLOCK_M - 1) / BLOCK_M;
  if (K_in <= 64) {
    if (splits <= 0) splits = max(1, num_sms() / m_tiles);
    return launch_nt_grouped<64>(p, G, N_out, K_in, batch, splits, d, s);
  }
  const int n_tiles = (K_in + 127) / 128;
  if (splits <= 0) splits = max(1, num_sms() / (m_tiles * n_tiles));
  return launch_nt_grouped<128>(p, G, N_out, K_in, batch, splits, d, s);
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
