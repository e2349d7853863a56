// "Unique-first" model-parallel embedding pipeline over NVLink peer memory (sm_90a).
//
// The reference dedups ids before every EmbeddingVariable lookup / apply (python/training/optimizer.py:91,
// kernels/unique_ali_op_gpu.cu.cc: cub radix sort + adjacent-diff + scan) and SOK moves ids, vectors and gradients with three
// NCCL all-to-alls bracketed by pack/unpack kernels and a host sync (all2all_input_dispatcher.cu:227-285,
// all2all_output_dispatcher.cu:159-246).  Here the same dataflow is five kernels with no NCCL call and no host round trip:
//
//   k_sp_dedup   (requester)  sort-free dedup of the local [C][B] id columns in an L2-resident scratch hash: every distinct
//                             (table, key) gets a slot `gs`; inv[b][c] = gs; the winner appends (key, gs) to the bucket list of
//                             the owning rank (hash(key) % W), counts occurrences, and zeroes the key's gradient row.
//                             Last block raises DEDUP flags on every peer.
//   k_sp_lookup  (owner)      waits per source on its DEDUP flag, reads the source's bucket list + occurrence counts over NVLink,
//                             probes / inserts / admits in the device EmbeddingVariable, claims the per-step unique index, and
//                             stores the bf16 row straight into the SOURCE's urow[gs] (P2P stores).  Last block raises ROWS.
//   (interaction kernels gather urow[inv[b][c]] -- L2-resident, 32 B rows)
//   k_sp_segsum  (requester)  pre-reduces the per-sample gradient rows per distinct key into ugrad[gs] with in-warp match.any
//                             combining, so only UNIQUE rows ever cross NVLink.  Last block raises GRAD.  ugrad holds 64-bit fixed
//                             point (units of 2^-40): integer addition is associative, so a key's sum does not depend on the order
//                             in which warps add to it, and a training step computes the same gradients on every run.
//   k_sp_grad    (owner)      waits per source on its GRAD flag, pulls ugrad rows over NVLink and reduces the <= W contributions
//                             per key into gsum[unique]; the row-wise optimizer (k_apply) follows on the same stream.
//   k_sp_reset   (requester)  clears the touched scratch slots through the bucket lists (no 50 MB memset per step).
//
// With the bench's id distribution only ~15 % of the ids of a batch are distinct: NVLink traffic, owner-side probes and
// owner-side atomics all shrink by that factor, and what is left on the requester is perfectly balanced across ranks.
#include "sp_sync.cuh"

namespace {
constexpr float kUgradScale = 1099511627776.f;        // 2^40: |row sum| < 8e6, resolution 9e-13 (finer than a bf16 gradient of 1e-9)
__device__ __forceinline__ unsigned long long ugrad_fix(float v) { return (unsigned long long)(long long)rintf(v * kUgradScale); }
__device__ __forceinline__ float ugrad_float(unsigned long long q) { return (float)(long long)q * (1.f / kUgradScale); }
}  // namespace
#include "table.cuh"

using namespace drc;

extern "C" {
struct DrSpSlot {
  int64_t key;       // kEmptyKey = free
  int32_t count;     // occurrences in this batch
  int32_t pad;
};
// Geometry shared by all kernels of the pipeline.
struct DrSpGeom {
  const int32_t* col_table;   // [C] table index (0..T) of every id column
  const int64_t* hoff;        // [T + 1] scratch-slot offset of table t (capacity hoff[t+1]-hoff[t] is a power of two)
  const int64_t* boff;        // [T + 1] bucket-entry offset of table t: bucket (t, o) = [(boff[t] * W + o * bcap_t), + bcap_t)
  int32_t C, T, W, rank;
  int64_t B;
  int32_t dim, ldinv;
  int64_t pad_key;            // ids equal to this (or the reserved empty/tombstone keys) are padding: inv = -1
};
}

namespace {

__device__ __forceinline__ int sp_owner(int64_t key, int W) { return dr_sp_owner(key, W); }      // csrc/common/ev_types.h

// -----------------------------------------------------------------------------------------------------------------
// k_sp_dedup: a block owns 32 samples; warp w walks columns w, w+8, ...; lane = sample.
// -----------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_sp_dedup(const int64_t* __restrict__ ids /* [C][B] */, DrSpGeom g, DrSpSlot* __restrict__ scr,
                                                  int32_t* __restrict__ inv /* [B][ldinv] */, int32_t* __restrict__ invT /* [C][B] or null */,
                                                  int64_t* __restrict__ bkt_key,
                                                  int32_t* __restrict__ bkt_gs, int32_t* __restrict__ bcnt /* [T][W] */,
                                                  unsigned long long* __restrict__ ugrad, DrSpSync sync) {
  pdl_sync();
  extern __shared__ int32_t s_inv[];                         // [32][ldinv + 1]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int lds = g.ldinv + 1;
  const int64_t ntiles = (g.B + 31) / 32;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t b = tile * 32 + lane;
    const bool in_b = b < g.B;
    for (int c = warp; c < g.ldinv; c += 8) {
      int32_t gs = -1;
      bool winner = false;
      int owner = 0, t = 0;
      int64_t key = 0;
      bool live = false;
      if (c < g.C) {
        t = g.col_table[c];
        if (in_b) {
          key = ids[(int64_t)c * g.B + b];
          live = key != g.pad_key && key != kEmptyKey && key != kTombKey;
        }
      }
      const unsigned lm = __ballot_sync(0xffffffffu, live);
      if (live) {
        const unsigned same = __match_any_sync(lm, (unsigned long long)key);     // in-warp duplicates elect one prober
        const int leader = __ffs(same) - 1;
        if (lane == leader) {
          const int64_t base = g.hoff[t];
          const uint32_t mask = (uint32_t)(g.hoff[t + 1] - base) - 1u;
          uint32_t h = (uint32_t)(dr_mix64((uint64_t)key + 0x9e3779b97f4a7c15ULL) >> 20) & mask;
          DrSpSlot* sl;
          for (;;) {
            sl = scr + base + h;
            const int64_t k = ld_volatile_i64(&sl->key);
            if (k == key) break;
            if (k == kEmptyKey) {
              const unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(&sl->key), (unsigned long long)kEmptyKey, (unsigned long long)key);
              if ((int64_t)old == kEmptyKey) { winner = true; break; }
              if ((int64_t)old == key) break;
            }
            h = (h + 1) & mask;
          }
          gs = (int32_t)(base + h);
          atomicAdd(&sl->count, __popc(same));
          owner = sp_owner(key, g.W);
        }
        gs = __shfl_sync(same, gs, leader);
      }
      // winners append (key, gs) to the owner's bucket: one counter atomic per (warp, owner)
      const unsigned wm = __ballot_sync(0xffffffffu, winner);
      if (winner) {
        const unsigned grp = __match_any_sync(wm, owner);
        const int lead = __ffs(grp) - 1;
        int base_i = 0;
        if (lane == lead) base_i = atomicAdd(&bcnt[t * g.W + owner], __popc(grp));
        base_i = __shfl_sync(grp, base_i, lead);
        const int64_t bcap = g.boff[t + 1] - g.boff[t];
        const int64_t slot = g.boff[t] * g.W + (int64_t)owner * bcap + base_i + __popc(grp & ((1u << lane) - 1u));
        bkt_key[slot] = key;
        bkt_gs[slot] = gs;
        if (ugrad) {
          int4* z = reinterpret_cast<int4*>(ugrad + (int64_t)gs * g.dim);
          for (int q = 0; q < g.dim / 2; ++q) z[q] = make_int4(0, 0, 0, 0);
        }
      }
      s_inv[lane * lds + c] = gs;
      if (invT && c < g.C && in_b) invT[(int64_t)c * g.B + b] = gs;
    }
    __syncthreads();
    // coalesced write-out of the tile's 32 x ldinv index block
    const int n4 = g.ldinv >> 2;
    for (int e = threadIdx.x; e < 32 * n4; e += blockDim.x) {
      const int r = e / n4, c4 = (e % n4) * 4;
      const int64_t bb = tile * 32 + r;
      if (bb < g.B) {
        const int32_t* s = s_inv + r * lds + c4;
        *reinterpret_cast<int4*>(inv + bb * g.ldinv + c4) = make_int4(s[0], s[1], s[2], s[3]);
      }
    }
    __syncthreads();
  }
  sp_signal_last_block(sync, SP_CH_DEDUP);
}

// ---- compact work enumeration -------------------------------------------------------------------------------------------
// The bucket of (table, peer) is sized for the worst case (every id of the batch distinct and owned by one rank) but holds ~1/W of
// the distinct keys: enumerating capacity-sized chunk slots made the owner kernels O(T * W * B / chunk) -- at 8 ranks 90 % of a
// kernel's time was spent skipping empty slots.  Instead every block scans the T counts of the current peer into a chunk prefix
// (warp 0, shuffle scan) and walks only the chunks that exist; the table of a chunk is found by binary search in shared memory.
constexpr int kSpMaxTables = 256;
__device__ __forceinline__ int sp_prefix_chunks(const int32_t* s_cnt, int32_t* s_pre, int T, int unit) {
  __syncthreads();
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    const int per = (T + 31) / 32;
    const int lo = min(T, lane * per), hi = min(T, lo + per);
    int sum = 0;
    for (int t = lo; t < hi; ++t) sum += (s_cnt[t] + unit - 1) / unit;
    int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
    int run = incl - sum;
    for (int t = lo; t < hi; ++t) { s_pre[t] = run; run += (s_cnt[t] + unit - 1) / unit; }
    if (lane == 31) s_pre[T] = incl;
  }
  __syncthreads();
  return s_pre[T];
}
__device__ __forceinline__ int sp_chunk_table(const int32_t* s_pre, int T, int k) {      // the t with s_pre[t] <= k < s_pre[t + 1]
  int lo = 0, hi = T;
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (s_pre[mid] <= k) lo = mid; else hi = mid; }
  return lo;
}

// per-thread training bookkeeping of one (unique-per-source) key: freq += occurrences, dirty mark, per-step dedup claim
__device__ __forceinline__ void sp_touch(const DrDeviceTable& TB, bool touch, int64_t pos, int32_t occ, int table_index, int64_t* ulist,
                                         int32_t* nunique, int64_t ulist_cap) {
  bool claim = false;
  if (touch) {
    atomicAdd(&TB.slots[pos].freq, occ);
    int4 hi;                                                                             // {row_of, tag, dirty, pad}
    DR_LD_V4_VOLATILE(hi, &TB.slots[pos].row_of);
    if (hi.z == 0) DR_ST_RACY(TB.slots[pos].dirty, 1u);
    claim = ulist != nullptr && hi.y == -1 && atomicCAS(&TB.slots[pos].tag, -1, -2) == -1;
  }
  // one counter atomic per warp for the claims
  const unsigned cm = __ballot_sync(0xffffffffu, claim);
  if (cm == 0) return;
  const int lead = __ffs(cm) - 1;
  int base = 0;
  if ((threadIdx.x & 31) == lead) base = atomicAdd(nunique, __popc(cm));
  base = __shfl_sync(0xffffffffu, base, lead);
  if (claim) {
    const int u = base + __popc(cm & ((1u << (threadIdx.x & 31)) - 1u));
    if (u < ulist_cap) { ulist[u] = ((int64_t)table_index << 40) | pos; DR_ST_RACY(TB.slots[pos].tag, u); }
    else { DR_ST_RACY(TB.slots[pos].tag, -1); DR_ST_RACY(TB.counters[CTR_OVERFLOW], 2); }
  }
}

struct SpPeerLists { DrPeers bkt_key, bkt_gs, bcnt, scr, urow; };

// -----------------------------------------------------------------------------------------------------------------
// k_sp_lookup (owner): chunks are SOURCE-major (own rank first), so a block waits for a source's flag at most once and
// starts on the sources that are ready while a late rank is still deduplicating.
// -----------------------------------------------------------------------------------------------------------------
template <int LPR>
__global__ void __launch_bounds__(256) k_sp_lookup(const DrDeviceTable* __restrict__ tables, const int32_t* __restrict__ table_map, DrSpGeom g,
                                                   SpPeerLists P, int train, int32_t* __restrict__ own_pos, int32_t* __restrict__ own_gs,
                                                   int32_t* __restrict__ own_cnt, int64_t* __restrict__ ulist, int32_t* __restrict__ nunique,
                                                   int64_t ulist_cap, DrSpSync sync) {
  pdl_sync();
  __shared__ int32_t s_pos[256];
  __shared__ int64_t s_key[256];
  __shared__ int32_t s_gs[256];
  __shared__ int32_t s_cnt[kSpMaxTables];
  __shared__ int32_t s_pre[kSpMaxTables + 1];
  const int T = g.T, W = g.W, rank = g.rank;
  for (int si = 0; si < W; ++si) {
    const int s = (rank + si) % W;                            // own bucket first, then the peers in ring order
    __syncthreads();
    if (threadIdx.x == 0) sp_wait_one(sync, SP_CH_DEDUP, s);
    __syncthreads();
    for (int i = threadIdx.x; i < T; i += blockDim.x) {
      const int32_t c = (int32_t)ld_relaxed_sys(reinterpret_cast<const uint32_t*>(P.bcnt.ptr[s]) + i * W + rank);
      s_cnt[i] = c;
      if (blockIdx.x == 0) own_cnt[i * W + s] = c;
    }
    const int nchunks = sp_prefix_chunks(s_cnt, s_pre, T, 256);
    // rotate the starting block per peer so that the few chunks of every peer land on different blocks
    for (int k = (int)((blockIdx.x + gridDim.x - (unsigned)(si * 67) % gridDim.x) % gridDim.x); k < nchunks; k += gridDim.x) {
      const int t = sp_chunk_table(s_pre, T, k);
      const int64_t e0 = (int64_t)(k - s_pre[t]) * 256;
      const int64_t cnt = s_cnt[t];
      const DrDeviceTable& TB = tables[table_map[t]];
      const int64_t bcap = g.boff[t + 1] - g.boff[t];
      const int64_t src_off = g.boff[t] * W + (int64_t)rank * bcap;        // my bucket in the source's lists
      const int64_t own_off = g.boff[t] * W + (int64_t)s * bcap;           // this (table, source) segment of my own arrays
      {
        const int64_t e = e0 + threadIdx.x;
        const bool live = e < cnt;
        int64_t key = 0, pos = -2;
        int32_t gs = -1, occ = 1;
        bool touch = false;
        if (live) {
          key = reinterpret_cast<const int64_t*>(P.bkt_key.ptr[s])[src_off + e];
          gs = reinterpret_cast<const int32_t*>(P.bkt_gs.ptr[s])[src_off + e];
          if (!train || TB.is_inference) {
            pos = table_find(TB, key);
          } else {
            // the occurrence count is a second (dependent) NVLink round trip: issue it before the probe, consume it after
            occ = reinterpret_cast<const DrSpSlot*>(P.scr.ptr[s])[gs].count;
            bool inserted = false, skip = false;
            if (TB.filter_type == DR_FILTER_BLOOM) {
              pos = table_find(TB, key);
              if (pos < 0) {
                if (bloom_add_min(TB, key, (uint32_t)occ) < (uint32_t)TB.filter_freq) skip = true;
                else pos = table_find_or_insert(TB, key, &inserted);
              }
            } else {
              pos = table_find_or_insert(TB, key, &inserted);
            }
            if (!skip && pos < 0) TB.counters[CTR_OVERFLOW] = 1;
            if (inserted) atomicAdd(&TB.counters[CTR_NKEYS], 1);
            touch = !skip && pos >= 0;
          }
          own_pos[own_off + e] = (int32_t)pos;
          own_gs[own_off + e] = gs;
        }
        s_pos[threadIdx.x] = live ? (int32_t)pos : -2;
        s_key[threadIdx.x] = key;
        s_gs[threadIdx.x] = gs;
        if (train) sp_touch(TB, touch, pos, occ, table_map[t], ulist, nunique, ulist_cap);
      }
      __syncthreads();
      // LPR lanes per row: fp32 row -> bf16 into the SOURCE's unique-row buffer over NVLink
      constexpr int ROWS_PER_IT = 256 / LPR;
      const int lane = threadIdx.x % LPR;
      __nv_bfloat16* dst_base = reinterpret_cast<__nv_bfloat16*>(P.urow.ptr[s]);
#pragma unroll
      for (int it = 0; it < LPR; ++it) {
        const int li = it * ROWS_PER_IT + threadIdx.x / LPR;
        if (s_pos[li] != -2) {
          const float* src = table_read_ptr(TB, s_key[li], s_pos[li]);
          const float4 v = src ? *reinterpret_cast<const float4*>(src + 4 * lane)
                               : make_float4(TB.no_permission, TB.no_permission, TB.no_permission, TB.no_permission);
          __nv_bfloat16* dst = dst_base + (int64_t)s_gs[li] * (4 * LPR) + 4 * lane;
          *reinterpret_cast<uint2*>(dst) = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
        }
      }
      __syncthreads();
    }
  }
  sp_signal_last_block(sync, SP_CH_ROWS);
}

// -----------------------------------------------------------------------------------------------------------------
// k_sp_segsum (requester): ugrad[gs] += per-sample gradient rows, pre-reduced per distinct key BEFORE anything crosses NVLink
// (the reference sums duplicates with unique + unsorted_segment_sum on the OWNER after shipping every row:
// all2all_output_dispatcher.cu:233-246, kit_cc/framework/compat/kernels/unsorted_segment_sum.cu).
// One warp = 32 consecutive samples of one id column (coalesced 32 B bf16 rows of the feature-major demb buffer).  Lanes holding
// the same key are found with match.any; every group's leader sums its members' rows out of a 1 KB shared-memory tile and issues
// ONE vectorised L2 reduction per 16 B chunk -- no shared-memory atomics (fp32 ATOMS are CAS loops), no sort.
// -----------------------------------------------------------------------------------------------------------------
template <int LPR /* dim / 4 */>
__global__ void __launch_bounds__(256) k_sp_segsum(const __nv_bfloat16* __restrict__ demb /* [C][B][dim] */, const int32_t* __restrict__ invT /* [C][B] */,
                                                   DrSpGeom g, unsigned long long* __restrict__ ugrad, DrSpSync sync) {
  pdl_sync();
  constexpr int dim = 4 * LPR;
  constexpr int V = dim / 8;                                   // int4 (8 bf16) chunks per row
  __shared__ __align__(16) int4 s_row[8][32][V];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t tiles = (g.B + 31) / 32;
  const int64_t units = tiles * g.C;
  for (int64_t u = (int64_t)blockIdx.x * 8 + warp; u < units; u += (int64_t)gridDim.x * 8) {
    const int c = (int)(u / tiles);
    const int64_t b = (u % tiles) * 32 + lane;
    int32_t gs = -1;
    if (b < g.B) gs = invT[(int64_t)c * g.B + b];
    const bool live = gs >= 0;
    const unsigned lm = __ballot_sync(0xffffffffu, live);
    if (live) {
      const int4* src = reinterpret_cast<const int4*>(demb + ((int64_t)c * g.B + b) * dim);
#pragma unroll
      for (int v = 0; v < V; ++v) s_row[warp][lane][v] = ld_nc_v4(src + v);
    }
    __syncwarp();
    if (live) {
      const unsigned same = __match_any_sync(lm, gs);
      if (lane == __ffs(same) - 1) {                            // leader of this key inside the tile
        float acc[dim];
#pragma unroll
        for (int d = 0; d < dim; ++d) acc[d] = 0.f;
        for (unsigned m = same; m; m &= m - 1) {
          const int src_lane = __ffs(m) - 1;
#pragma unroll
          for (int v = 0; v < V; ++v) {
            const int4 raw = s_row[warp][src_lane][v];
            const uint32_t w[4] = {(uint32_t)raw.x, (uint32_t)raw.y, (uint32_t)raw.z, (uint32_t)raw.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) { const float2 f = unpack_bf16x2(w[e]); acc[8 * v + 2 * e] += f.x; acc[8 * v + 2 * e + 1] += f.y; }
          }
        }
        unsigned long long* dst = ugrad + (int64_t)gs * dim;
#pragma unroll
        for (int d = 0; d < dim; ++d) atomicAdd(dst + d, ugrad_fix(acc[d]));
      }
    }
    __syncwarp();
  }
  sp_signal_last_block(sync, SP_CH_GRAD);
}

// -----------------------------------------------------------------------------------------------------------------
// k_sp_gather (requester): out[b][c][:] = urow[inv[b][c]]  (padding -> zeros) -- the sample-major [B, C, dim] activation generic dense
// networks consume (models/rec_engine.py).  Waits in-kernel for every owner's ROWS flag, like the fused interaction kernels do.
// -----------------------------------------------------------------------------------------------------------------
template <int LPR>
__global__ void __launch_bounds__(256) k_sp_gather(const __nv_bfloat16* __restrict__ urow, const int32_t* __restrict__ inv, int ldinv, int C, int64_t B,
                                                   __nv_bfloat16* __restrict__ out, DrSpSync sync) {
  pdl_sync();
  sp_wait_all(sync, SP_CH_ROWS);
  constexpr int dim = 4 * LPR;
  const int lane = threadIdx.x % LPR;
  const int64_t n = B * C;
  for (int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / LPR; i < n; i += (int64_t)gridDim.x * blockDim.x / LPR) {
    const int64_t b = i / C; const int c = (int)(i % C);
    const int32_t gs = inv[b * ldinv + c];
    uint2 v = make_uint2(0u, 0u);
    if (gs >= 0) DR_LD_V2_VOLATILE_U32(v, urow + (int64_t)gs * dim + 4 * lane);
    *reinterpret_cast<uint2*>(out + i * dim + 4 * lane) = v;
  }
}

// -----------------------------------------------------------------------------------------------------------------
// k_sp_grad (owner): gsum[tag(pos)] += ugrad_of_source[gs]      (fp32 rows, pre-reduced per key on the source)
// -----------------------------------------------------------------------------------------------------------------
template <int LPR>
__global__ void __launch_bounds__(256) k_sp_grad(const DrDeviceTable* __restrict__ tables, const int32_t* __restrict__ table_map, DrSpGeom g,
                                                 DrPeers ugrad, const int32_t* __restrict__ own_pos, const int32_t* __restrict__ own_gs,
                                                 const int32_t* __restrict__ own_cnt, float* __restrict__ gsum, DrSpSync sync) {
  pdl_sync();
  constexpr int IPC = 256 / LPR;
  constexpr int dim = 4 * LPR;
  __shared__ int32_t s_cnt[kSpMaxTables];
  __shared__ int32_t s_pre[kSpMaxTables + 1];
  const int T = g.T, W = g.W, rank = g.rank;
  const int lane = threadIdx.x % LPR;
  for (int si = 0; si < W; ++si) {
    const int s = (rank + si) % W;
    __syncthreads();
    if (threadIdx.x == 0) sp_wait_one(sync, SP_CH_GRAD, s);
    __syncthreads();
    for (int i = threadIdx.x; i < T; i += blockDim.x) s_cnt[i] = own_cnt[i * W + s];
    const int nchunks = sp_prefix_chunks(s_cnt, s_pre, T, IPC);
    for (int k = (int)((blockIdx.x + gridDim.x - (unsigned)(si * 67) % gridDim.x) % gridDim.x); k < nchunks; k += gridDim.x) {
      const int t = sp_chunk_table(s_pre, T, k);
      const int64_t e = (int64_t)(k - s_pre[t]) * IPC + threadIdx.x / LPR;
      if (e >= s_cnt[t]) continue;
      const int64_t bcap = g.boff[t + 1] - g.boff[t];
      const int64_t own_off = g.boff[t] * W + (int64_t)s * bcap + e;
      const int32_t p = own_pos[own_off];
      if (p < 0) continue;
      // the peer row does not depend on the tag: both loads are in flight together
      const unsigned long long* q = reinterpret_cast<const unsigned long long*>(ugrad.ptr[s]) + (int64_t)own_gs[own_off] * dim + 4 * lane;
      const float4 v = make_float4(ugrad_float(q[0]), ugrad_float(q[1]), ugrad_float(q[2]), ugrad_float(q[3]));
      const int32_t u = tables[table_map[t]].slots[p].tag;
      if (u < 0) continue;
      if (W == 1) *reinterpret_cast<float4*>(gsum + (int64_t)u * dim + 4 * lane) = v;     // one contribution per key: plain store (gsum is zero)
      else red_add_v4_f32(gsum + (int64_t)u * dim + 4 * lane, v.x, v.y, v.z, v.w);
    }
  }
}

// -----------------------------------------------------------------------------------------------------------------
// k_sp_reset (requester): free the scratch slots this batch touched; the last block zeroes the bucket counters.
// -----------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_sp_reset(DrSpGeom g, DrSpSlot* __restrict__ scr, const int32_t* __restrict__ bkt_gs,
                                                  int32_t* __restrict__ bcnt, int32_t* __restrict__ state) {
  pdl_sync();
  __shared__ int32_t s_cnt[kSpMaxTables];
  __shared__ int32_t s_pre[kSpMaxTables + 1];
  const int T = g.T, W = g.W;
  for (int o = 0; o < W; ++o) {
    __syncthreads();
    for (int i = threadIdx.x; i < T; i += blockDim.x) s_cnt[i] = bcnt[i * W + o];
    const int nchunks = sp_prefix_chunks(s_cnt, s_pre, T, 256);
    for (int k = (int)((blockIdx.x + gridDim.x - (unsigned)(o * 67) % gridDim.x) % gridDim.x); k < nchunks; k += gridDim.x) {
      const int t = sp_chunk_table(s_pre, T, k);
      const int64_t e = (int64_t)(k - s_pre[t]) * 256 + threadIdx.x;
      if (e >= s_cnt[t]) continue;
      const int64_t bcap = g.boff[t + 1] - g.boff[t];
      const int32_t gs = bkt_gs[g.boff[t] * W + (int64_t)o * bcap + e];
      DrSpSlot z; z.key = kEmptyKey; z.count = 0; z.pad = 0;
      *reinterpret_cast<int4*>(&scr[gs]) = *reinterpret_cast<int4*>(&z);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const int prev = atomicAdd(&state[8 + SP_CH_AUX], 1);
    if (prev == (int)gridDim.x - 1) {
      state[8 + SP_CH_AUX] = 0;
      __threadfence();
      for (int i = 0; i < T * W; ++i) bcnt[i] = 0;
    }
  }
}

__global__ void k_sp_signal(DrSpSync sync, int ch) {
  pdl_sync();
  sp_signal_last_block(sync, ch);
}
__global__ void k_sp_step_end(int32_t* state) {
  pdl_sync();
  state[0] += 1;
}
__global__ void k_sp_init_scratch(DrSpSlot* scr, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    scr[i].key = kEmptyKey; scr[i].count = 0; scr[i].pad = 0;
  }
}

// number of distinct (table, key) pairs of the current batch and ids per batch (diagnostics for bench.py: unique_ratio)
__global__ void k_sp_stats(DrSpGeom g, const int32_t* __restrict__ bcnt, int64_t* __restrict__ out) {
  int64_t n = 0;
  for (int i = 0; i < g.T * g.W; ++i) n += bcnt[i];
  out[0] = n;
}

inline int sp_grid(int64_t blocks) {
  const int64_t cap = (int64_t)num_sms() * sparse_blocks_per_sm();
  if (blocks < 1) blocks = 1;
  return (int)(blocks > cap ? cap : blocks);
}

}  // namespace

extern "C" {

int dr_sp_init_scratch(void* scr, int64_t n, cudaStream_t s) {
  k_sp_init_scratch<<<num_sms() * 4, 256, 0, s>>>((DrSpSlot*)scr, n);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_sp_dedup(const int64_t* ids, const DrSpGeom* g, void* scr, int32_t* inv, int32_t* invT, int64_t* bkt_key, int32_t* bkt_gs, int32_t* bcnt,
                void* ugrad, const DrSpSync* sync, cudaStream_t s) {
  if (g->ldinv % 4 || g->ldinv < g->C || g->dim % 4) return -2;
  const size_t smem = (size_t)32 * (g->ldinv + 1) * 4;
  if (smem > 48 * 1024) return -3;
  DR_PDL_LAUNCH((k_sp_dedup), sp_grid((g->B + 31) / 32), 256, smem, s, ids, *g, (DrSpSlot*)scr, inv, invT, bkt_key, bkt_gs, bcnt, (unsigned long long*)ugrad, *sync);
  DR_LAUNCH_CHECK();
  return 0;
}

// demb: bf16 [C][B][dim] per-sample gradient rows (feature-major); accumulates into ugrad and raises the GRAD flags
int dr_sp_segsum(const void* demb, const int32_t* invT, const DrSpGeom* g, void* ugrad, const DrSpSync* sync, cudaStream_t s) {
  const int64_t units = ((g->B + 31) / 32) * g->C;
  const int grid = sp_grid((units + 7) / 8);
#define SPS(L) DR_PDL_LAUNCH((k_sp_segsum<L>), grid, 256, 0, s, (const __nv_bfloat16*)demb, invT, *g, (unsigned long long*)ugrad, *sync)
  switch (g->dim / 4) {
    case 2: SPS(2); break; case 4: SPS(4); break; case 8: SPS(8); break; case 16: SPS(16); break;
    default: return -3;
  }
#undef SPS
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_sp_lookup(const DrDeviceTable* tables_dev, const int32_t* table_map, const DrSpGeom* g, int64_t max_bcap, const DrPeers* bkt_key,
                 const DrPeers* bkt_gs, const DrPeers* bcnt, const DrPeers* scr, const DrPeers* urow, int train, int32_t* own_pos, int32_t* own_gs,
                 int32_t* own_cnt, int64_t* ulist, int32_t* nunique, int64_t ulist_cap, const DrSpSync* sync, cudaStream_t s) {
  if (g->T > kSpMaxTables || g->W > 16) return -2;
  SpPeerLists P{*bkt_key, *bkt_gs, *bcnt, *scr, *urow};
  const int64_t chunks = (int64_t)g->T * g->W * ((max_bcap + 255) / 256);
  const int grid = sp_grid(chunks);
#define SPL(L) DR_PDL_LAUNCH((k_sp_lookup<L>), grid, 256, 0, s, tables_dev, table_map, *g, P, train, own_pos, own_gs, own_cnt, ulist, nunique, ulist_cap, *sync)
  switch (g->dim / 4) {
    case 2: SPL(2); break; case 4: SPL(4); break; case 8: SPL(8); break; case 16: SPL(16); break; case 32: SPL(32); break;
    default: return -3;
  }
#undef SPL
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_sp_grad(const DrDeviceTable* tables_dev, const int32_t* table_map, const DrSpGeom* g, int64_t max_bcap, const DrPeers* ugrad,
               const int32_t* own_pos, const int32_t* own_gs, const int32_t* own_cnt, float* gsum, const DrSpSync* sync, cudaStream_t s) {
  const int lpr = g->dim / 4;
  if (lpr < 2 || lpr > 32 || (lpr & (lpr - 1))) return -3;
  const int ipc = 256 / lpr;
  const int64_t chunks = (int64_t)g->T * g->W * ((max_bcap + ipc - 1) / ipc);
  const int grid = sp_grid(chunks);
#define SPG(L) DR_PDL_LAUNCH((k_sp_grad<L>), grid, 256, 0, s, tables_dev, table_map, *g, *ugrad, own_pos, own_gs, own_cnt, gsum, *sync)
  switch (lpr) {
    case 2: SPG(2); break; case 4: SPG(4); break; case 8: SPG(8); break; case 16: SPG(16); break; case 32: SPG(32); break;
    default: return -3;
  }
#undef SPG
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_sp_gather(const void* urow, const int32_t* inv, const DrSpGeom* g, void* out, const DrSpSync* sync, cudaStream_t s) {
  const int lpr = g->dim / 4;
  const int64_t n = g->B * g->C;
  const int grid = sp_grid((n * lpr + 255) / 256);
#define SPGA(L) DR_PDL_LAUNCH((k_sp_gather<L>), grid, 256, 0, s, (const __nv_bfloat16*)urow, inv, g->ldinv, g->C, g->B, (__nv_bfloat16*)out, *sync)
  switch (lpr) {
    case 2: SPGA(2); break; case 4: SPGA(4); break; case 8: SPGA(8); break; case 16: SPGA(16); break; case 32: SPGA(32); break;
    default: return -3;
  }
#undef SPGA
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_sp_reset(const DrSpGeom* g, int64_t max_bcap, void* scr, const int32_t* bkt_gs, int32_t* bcnt, int32_t* state, cudaStream_t s) {
  const int64_t chunks = (int64_t)g->T * g->W * ((max_bcap + 255) / 256);
  DR_PDL_LAUNCH((k_sp_reset), sp_grid(chunks), 256, 0, s, *g, (DrSpSlot*)scr, bkt_gs, bcnt, state);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_sp_signal(const DrSpSync* sync, int ch, cudaStream_t s) {
  DR_PDL_LAUNCH((k_sp_signal), 1, 32, 0, s, *sync, ch);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_sp_step_end(int32_t* state, cudaStream_t s) {
  DR_PDL_LAUNCH((k_sp_step_end), 1, 1, 0, s, state);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_sp_stats(const DrSpGeom* g, const int32_t* bcnt, int64_t* out, cudaStream_t s) {
  k_sp_stats<<<1, 1, 0, s>>>(*g, bcnt, out);
  DR_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
