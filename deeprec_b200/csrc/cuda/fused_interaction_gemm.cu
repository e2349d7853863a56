// k_dlrm_inter_gemm: embedding combine (+ROWS-flag wait) ⊕ DLRM dot interaction ⊕ top-MLP layer 0, ONE wgmma kernel (sm_90a).
//
// Reference dataflow replaced: SOK all2all(vectors) -> reorderKernel (all2all_output_dispatcher.cu:159-193) -> tf.matmul(X, X^T) +
// boolean_mask + concat (modelzoo/dlrm/train.py:121-133) -> cuBLAS Dense(512)+ReLU.  Unfused, this is three kernels (rank barrier,
// k_dot_fwd_tc writing Z, GEMM reading Z back); here the 128-sample Z tile is BUILT IN SHARED MEMORY in the 128B-swizzled K-major
// layout wgmma consumes, and multiplied by W0 without the GEMM ever reading it from HBM:
//
//   warpgroup 0      TMA producer (one thread): streams W0 [512 x 368] through a 7-stage ring of [128 n x 64 k] tiles (OOB K columns
//                    zero-filled)
//   warpgroups 1-2   per 128-sample tile, two phases:
//                    build -- warp = sample slot (16 samples per warp per tile): gather urow[inv[b][t]] rows straight out of the
//                    peer-written unique-row buffer (the kernel first waits for every owner's ROWS flag), compute the sample's
//                    32 x 32 x 16 Gram matrix with six warp-level mma.sync.m16n8k16 (lower-triangle tiles only) and scatter the strict
//                    lower triangle into the swizzled Z tile; one thread then TMA-stores the finished tile for the backward's dW0 GEMM;
//                    GEMM -- warpgroup g multiplies rows [64 g, 64 g + 64) of the Z tile by every 128-wide n block of W0 with
//                    wgmma.mma_async (fp32 register accumulators), then +bias -> ReLU -> bf16 stores of a0 [B, 512].
//                    The rows of the next tile's first samples are already in flight in registers while the GEMM phase runs.
#include <cuda.h>

#include "sp_sync.cuh"
#include "wgmma.cuh"

using namespace drc;

namespace {

__device__ __forceinline__ void consumer_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

constexpr int kD = 16;                  // embedding dim (= bottom MLP output)
constexpr int kTileM = 128;             // samples per tile
constexpr int kBN = 128;                // GEMM n-block
constexpr int kKB = 64;                 // GEMM k-block (one 128 B swizzle row)
constexpr int kStagesB = 7;             // 7 x 16 KB W0 tiles in flight: the per-SM L2->smem path needs ~100 KB outstanding to stay busy
constexpr int kThreads = 3 * 128;
constexpr int kMaxKb = 6;               // K <= 384

struct FusedSmem {
  static constexpr int kZBytes = kMaxKb * kTileM * 128;          // 98304
  static constexpr int kBStage = kBN * 128;                      // 16384
  static constexpr int kFBytes = 4 * 1024;                       // 8 builder warps x [32 rows][32 B] feature tile (x2 halves below)
  static constexpr int kOffB = kZBytes;
  static constexpr int kOffF = kOffB + kStagesB * kBStage;
  static constexpr int kOffBias = kOffF + 2 * kFBytes;
  static constexpr int kOffBar = kOffBias + 512 * 4;
  static constexpr int kTotal = kOffBar + 256 + 1024;
};

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
int make_tmap(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer, uint64_t pitch_bytes, uint32_t box_inner, uint32_t box_outer) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return -100;
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {pitch_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -101 - (int)r;
}

__global__ void __launch_bounds__(kThreads, 1)
k_dlrm_inter_gemm(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmZ, const __nv_bfloat16* __restrict__ x, int64_t ldx,
                  const __nv_bfloat16* __restrict__ urow, const int32_t* __restrict__ inv, int ldinv, int T, int64_t B, int Kz /* D + F(F-1)/2 */,
                  int N, const float* __restrict__ bias, __nv_bfloat16* __restrict__ out, int64_t ldo, int store_z, DrSpSync sync, int dbg) {
  using L = FusedSmem;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sZ = smem;
  uint8_t* sB = smem + L::kOffB;
  uint8_t* sF = smem + L::kOffF;                  // 8 KB: one 1 KB staging tile per builder warp
  float* s_bias = reinterpret_cast<float*>(smem + L::kOffBias);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::kOffBar);
  uint64_t* full_bar = bars;                       // [kStagesB]  W0 tile landed
  uint64_t* empty_bar = bars + kStagesB;           // [kStagesB]  W0 tile consumed

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int F = T + 1;
  const int64_t ntiles = (B + kTileM - 1) / kTileM;
  const int n_blks = (N + kBN - 1) / kBN;
  const int num_kb = (Kz + kKB - 1) / kKB;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmW); tma_prefetch_desc(&tmZ);
    for (int i = 0; i < kStagesB; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8); }
    fence_mbar_init();
  }
  // zero the Z tile once: the K padding columns [Kz, num_kb * 64) stay zero for the kernel's life, the feature tiles' padding rows too
  for (int i = threadIdx.x; i < (L::kZBytes + kStagesB * L::kBStage + 2 * L::kFBytes) / 16; i += blockDim.x) reinterpret_cast<int4*>(smem)[i] = make_int4(0, 0, 0, 0);
  __syncthreads();
  pdl_sync();
  if (sync.state) sp_wait_all(sync, SP_CH_ROWS);            // every owner has pushed this step's rows into my urow
  for (int i = threadIdx.x; i < 512; i += blockDim.x) s_bias[i] = (bias != nullptr && i < N) ? bias[i] : 0.f;
  fence_proxy_async();
  __syncthreads();

  if (warp == 0) {
    // ================= TMA producer: W0 tiles =================
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x)
        for (int nb = 0; nb < n_blks; ++nb)
          for (int kb = 0; kb < num_kb; ++kb) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            mbar_expect_tx(&full_bar[stage], L::kBStage);
            tma_load_2d(sB + stage * L::kBStage, &tmW, &full_bar[stage], kb * kKB, nb * kBN);
            if (++stage == kStagesB) { stage = 0; phase ^= 1; }
          }
    }
  } else if (warp >= 4) {
    // ================= builders + GEMM: gather + warp-level Gram (mma.sync) + lower-triangle scatter into the swizzled Z tile =================
    const int bw = warp - 4;                          // 0..7: this warp handles samples bw, bw + 8, ... of every tile
    const int wg = bw >> 2, wl = bw & 3, ct = threadIdx.x - 128;
    uint8_t* myF = sF + bw * 1024;                    // [32 feature rows][32 B] row-major staging tile of the current sample
    const int gI = lane >> 2, tI = lane & 3;          // mma.sync fragment coordinates
    // scatter plan of this lane's 12 accumulator pairs: byte offset inside a Z row of (fi, j) (k-block, 16 B chunk, element), before
    // the row-dependent XOR swizzle of bits 4-6
    uint32_t zoff[12], zoff1[12];
    {
      int e = 0;
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) {
          if (8 * ni > 16 * mi + 15) continue;
#pragma unroll
          for (int h = 0; h < 2; ++h, ++e) {
            const int fi = 16 * mi + gI + 8 * h, j = 8 * ni + 2 * tI;
            const uint32_t c = (uint32_t)(kD + fi * (fi - 1) / 2 + j), c1e = c + 1;
            const uint32_t o0 = ((c >> 6) * (uint32_t)(kTileM * 128)) | (((c >> 3) & 7u) << 4) | ((c & 7u) << 1);
            const uint32_t o1 = ((c1e >> 6) * (uint32_t)(kTileM * 128)) | (((c1e >> 3) & 7u) << 4) | ((c1e & 7u) << 1);
            const bool v0 = fi < F && j < fi, v1 = fi < F && j + 1 < fi;
            zoff[e] = o0 | (v0 ? 0x80000000u : 0u) | (v1 ? 0x40000000u : 0u) | ((v1 && (c & 1u) == 0) ? 0x20000000u : 0u);
            zoff1[e] = o1;
          }
        }
    }
    int stage = 0; uint32_t phase = 0;
    // Gather pipeline: a warp keeps a CHUNK of 4 samples in flight (rows of chunk k+1 and indices of chunk k+2 are loading while
    // chunk k is processed) -- one sample in flight per warp left the kernel bound by the L2 / NVLink-written-row latency.
    constexpr int SPW = kTileM / 8;                   // samples per warp per tile
    constexpr int CH = 4;                             // samples per chunk
    constexpr int CPT = SPW / CH;                     // chunks per tile
    int4 nr[CH][2];                                   // rows of the NEXT chunk to process
    int32_t gsn[CH];                                  // indices of the chunk after that
    auto sample_of = [&](int64_t tile, int i) -> int64_t { return tile * kTileM + bw + 8 * i; };
    // slot u of the two register arrays always holds sample u of some chunk: rows of the chunk being / about to be processed, and the
    // index of the same slot one chunk later; a slot is refilled the moment its sample has been staged
    auto fetch_idx1 = [&](int64_t tile, int k, int u) {
      const int64_t bb = tile < ntiles ? sample_of(tile, k * CH + u) : -1;
      gsn[u] = (bb >= 0 && bb < B && lane >= 1 && lane < F) ? inv[bb * ldinv + lane - 1] : -1;
    };
    auto fetch_rows1 = [&](int64_t tile, int k, int u) {
      const int64_t bb = tile < ntiles ? sample_of(tile, k * CH + u) : -1;
      nr[u][0] = nr[u][1] = make_int4(0, 0, 0, 0);
      if (!(dbg & 2) && bb >= 0 && bb < B && lane < F) {
        if (lane == 0) { nr[u][0] = ld_nc_v4(x + bb * ldx); nr[u][1] = ld_nc_v4(x + bb * ldx + 8); }
        else if (gsn[u] >= 0) { const __nv_bfloat16* src = urow + (int64_t)gsn[u] * kD; nr[u][0] = ld_v4_volatile(src); nr[u][1] = ld_v4_volatile(src + 8); }
      }
    };
    auto advance = [&](int64_t& tile, int& k) { if (++k >= CPT) { k = 0; tile += gridDim.x; } };
    {
      int64_t t1 = blockIdx.x; int k1 = 0;
#pragma unroll
      for (int u = 0; u < CH; ++u) fetch_idx1(t1, k1, u);
#pragma unroll
      for (int u = 0; u < CH; ++u) fetch_rows1(t1, k1, u);
      advance(t1, k1);
#pragma unroll
      for (int u = 0; u < CH; ++u) fetch_idx1(t1, k1, u);
    }
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      // the previous tile's GEMM (both warpgroups) and Z stores must have finished reading the Z tile before the first write of this one
      if (tile != (int64_t)blockIdx.x) consumer_bar_sync();
      for (int k = 0; k < CPT; ++k) {
        int64_t t1 = tile; int k1 = k; advance(t1, k1);        // next chunk (rows to fetch now)
        int64_t t2 = t1; int k2 = k1; advance(t2, k2);         // the chunk after it (indices to fetch now)
#pragma unroll
        for (int u = 0; u < CH; ++u) {
        const int i = k * CH + u;
        const int64_t b = sample_of(tile, i);
        const bool live = b < B;
        // ---- stage my feature row (padding lanes / dead samples write zeros); lane 0 keeps the dense vector for Z[:, 0:16]
        *reinterpret_cast<int4*>(myF + lane * 32) = nr[u][0];
        *reinterpret_cast<int4*>(myF + lane * 32 + 16) = nr[u][1];
        const int4 x0 = nr[u][0], x1 = nr[u][1];
        fetch_rows1(t1, k1, u);                          // refill the slot: rows one chunk ahead, index two chunks ahead
        fetch_idx1(t2, k2, u);
        __syncwarp();
        // ---- G = F F^T on the warp's tensor-core path: A fragments of the two 16-row tiles, B fragments of the four 8-column tiles
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
        const int zr = bw + 8 * i;                      // row of this sample in the tile
        uint8_t* zrow = sZ + zr * 128;
        const uint32_t rx = (uint32_t)(zr & 7) << 4;
        if (lane == 0) {                                // Z[:, 0:16] = x (16 B chunks 0 and 1 of k-block 0)
          *reinterpret_cast<int4*>(zrow + ((0u << 4) ^ rx)) = live ? x0 : make_int4(0, 0, 0, 0);
          *reinterpret_cast<int4*>(zrow + ((1u << 4) ^ rx)) = live ? x1 : make_int4(0, 0, 0, 0);
        }
        if (!(dbg & 1)) {
          int e = 0;
#pragma unroll
          for (int mi = 0; mi < 2; ++mi) {
#pragma unroll
            for (int ni = 0; ni < 4; ++ni) {
              if (8 * ni > 16 * mi + 15) continue;        // tile entirely above the diagonal (compile-time)
              float cacc[4] = {0.f, 0.f, 0.f, 0.f};
              asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                           : "+f"(cacc[0]), "+f"(cacc[1]), "+f"(cacc[2]), "+f"(cacc[3])
                           : "r"(af[mi][0]), "r"(af[mi][1]), "r"(af[mi][2]), "r"(af[mi][3]), "r"(bf[ni][0]), "r"(bf[ni][1]));
              // lane holds G[i][j], G[i][j+1] for i in {16 mi + gI, +8}, j = 8 ni + 2 tI: where they go is a per-lane constant
#pragma unroll
              for (int h = 0; h < 2; ++h, ++e) {
                const uint32_t po = zoff[e];                // bit 31: first element valid, bit 30: second valid, bit 29: one 4-byte store
                if (po & 0x80000000u) {
                  const uint32_t off0 = (po & 0x1FFFFu) ^ rx;
                  const float v0 = live ? cacc[2 * h] : 0.f, v1 = live ? cacc[2 * h + 1] : 0.f;
                  if (po & 0x20000000u) {
                    *reinterpret_cast<uint32_t*>(zrow + off0) = pack_bf16x2(v0, v1);
                  } else {
                    *reinterpret_cast<__nv_bfloat16*>(zrow + off0) = __float2bfloat16(v0);
                    if (po & 0x40000000u) *reinterpret_cast<__nv_bfloat16*>(zrow + (zoff1[e] ^ rx)) = __float2bfloat16(v1);
                  }
                }
              }
            }
          }
        }
        __syncwarp();                                   // the staging tile is rewritten by the next sample
        }
      }
      // ---- the Z tile is complete: hand it to the async proxy (TMA store, wgmma)
      fence_proxy_async();
      consumer_bar_sync();
      if (ct == 0 && store_z && !(dbg & 4)) {
        for (int kb = 0; kb < num_kb; ++kb) tma_store_2d(&tmZ, sZ + kb * (kTileM * 128), kb * kKB, (int)(tile * kTileM));
        tma_store_commit();
      }
      // ---- GEMM: rows [64 wg, 64 wg + 64) of the tile x every n block of W0
      const int64_t row0 = tile * kTileM + wg * 64 + wl * 16 + (lane >> 2);
      for (int nb = 0; nb < n_blks; ++nb) {
        float acc[kBN / 2];
#pragma unroll
        for (int i = 0; i < kBN / 2; ++i) acc[i] = 0.f;
        int prev = -1;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          const uint64_t adesc = gmma_desc_sw128(smem_u32(sZ + kb * (kTileM * 128) + wg * 64 * 128), 16, 1024);
          const uint64_t bdesc = gmma_desc_sw128(smem_u32(sB + stage * L::kBStage), 16, 1024);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < kKB / 16; ++k) wgmma_bf16<kBN, 0, 0>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), 1);
          wgmma_commit();
          wgmma_wait<1>();
          if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
          prev = stage;
          if (++stage == kStagesB) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_acc(acc);
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
        if (!(dbg & 8)) {
#pragma unroll
          for (int j = 0; j < kBN / 8; ++j) {
            const int col = nb * kBN + 8 * j + 2 * (lane & 3);
            if (col >= N) continue;                       // N is a multiple of 8
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int64_t row = row0 + 8 * h;
              if (row < B) {
                const float v0 = fmaxf(acc[4 * j + 2 * h] + s_bias[col], 0.f), v1 = fmaxf(acc[4 * j + 2 * h + 1] + s_bias[col + 1], 0.f);
                *reinterpret_cast<uint32_t*>(out + row * ldo + col) = pack_bf16x2(v0, v1);
              }
            }
          }
        }
      }
      if (ct == 0 && store_z && !(dbg & 4)) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");     // the stores have read the tile
    }
    if (ct == 0) tma_store_wait_all();
  }
}

}  // namespace

static int fused_dbg() { static int v = [] { const char* e = getenv("DEEPREC_FUSED_DBG"); return e ? atoi(e) : 0; }(); return v; }

extern "C" {

// out[B, N] = relu( Z W0^T + bias ),  Z[b] = [ x[b] | strict lower triangle of the Gram matrix of (x[b], urow[inv[b][0..T)]) | 0-pad ]
// W0: bf16 [N, ldw] K-major (ldw >= Kz, multiple of 8).  Z (optional, bf16 [B, ldz], ldz >= ceil(Kz/64)*64... columns beyond ldz are
// clipped by the tensor map) is written for the backward.  Requirements: D == 16, T + 1 <= 32, N <= 512, N % 8 == 0, Kz <= 384.
int dr_cuda_dlrm_inter_gemm(const void* x, int64_t ldx, const void* urow, const int32_t* inv, int ldinv, int T, int D, int64_t B, const void* W0,
                            int64_t ldw, int N, const float* bias, void* out, int64_t ldo, void* Z, int64_t ldz, const DrSpSync* sync,
                            cudaStream_t s) {
  const int F = T + 1;
  const int Kz = D + F * (F - 1) / 2;
  if (D != kD || F > 32 || N > 512 || (N % 8) || Kz > kMaxKb * kKB || (ldw % 8) || (ldo % 8) || (Z && (ldz % 8))) return -2;
  CUtensorMap tw, tz;
  int rc = make_tmap(&tw, W0, (uint64_t)Kz, (uint64_t)N, (uint64_t)ldw * 2, kKB, kBN);
  if (rc) return rc;
  // Z store map: inner extent = ldz so that the zero K-padding columns that exist in memory are written (as zeros) too
  rc = make_tmap(&tz, Z ? Z : out, (uint64_t)(Z ? ldz : ldo), (uint64_t)B, (uint64_t)(Z ? ldz : ldo) * 2, kKB, kTileM);
  if (rc) return rc;
  static DrPerDeviceOnce attr_once; bool& attr = attr_once();
  if (!attr) { DR_CUDA_CHECK(cudaFuncSetAttribute(k_dlrm_inter_gemm, cudaFuncAttributeMaxDynamicSharedMemorySize, FusedSmem::kTotal)); attr = true; }
  const int64_t ntiles = (B + kTileM - 1) / kTileM;
  const int grid = (int)(ntiles < num_sms() ? ntiles : num_sms());
  DrSpSync sy{}; if (sync) sy = *sync;
  DR_PDL_LAUNCH((k_dlrm_inter_gemm), grid, kThreads, FusedSmem::kTotal, s, tw, tz, (const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)urow, inv, ldinv, T, B, Kz,
                N, bias, (__nv_bfloat16*)out, ldo, Z ? 1 : 0, sy, fused_dbg());
  DR_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
