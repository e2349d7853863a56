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
//   k_sp_linear_fwd / k_sp_linear_bwd (requester)  a linear (wide) embedding group: the per-sample sum of element 0 of the unique rows,
//                             and its fp32 gradient scattered into element 0 of ugrad -- in place of gather / segsum.
//   k_sp_pool / k_sp_pool_segsum (requester)  multi-hot bags: runs of consecutive id columns pooled (sum / mean / sqrtn) into one [B, F, dim]
//                             activation slot each, and the pooled gradient scaled back onto every column of its bag -- in place of gather /
//                             segsum.
//
// With the bench's id distribution only ~15 % of the ids of a batch are distinct: NVLink traffic, owner-side probes and
// owner-side atomics all shrink by that factor, and what is left on the requester is perfectly balanced across ranks.
#include "sp_sync.cuh"

namespace {
// 2^40: resolution 9e-13 (finer than a bf16 gradient of 1e-9).  A key's gradient sum must stay below 2^22 (4.2e6) in magnitude; the
// engines scale the loss by 1 / (global batch) (DLRMEngine._head), so a per-sample gradient is O(1 / batch) and a key's sum O(1).
// A 32-row partial beyond +-2^22 is clamped to it (a defined saturation instead of an out-of-range float -> integer conversion, which
// is undefined on the host); NaN converts to 0 as the device cvt does.  The 64-bit sum of the partials itself wraps beyond 2^23.
constexpr float kUgradScale = 1099511627776.f;
constexpr float kUgradMax = 4611686018427387904.f;           // 2^22 * 2^40 = 2^62
__device__ __forceinline__ unsigned long long ugrad_fix(float v) {
  float x = v * kUgradScale;
  if (!(fabsf(x) <= kUgradMax)) x = x != x ? 0.f : copysignf(kUgradMax, x);
  return (unsigned long long)(long long)rintf(x);
}
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
// Multi-hot bags: bag f pools the id columns [off[f], off[f+1]) into activation slot f; together the F bags cover the C columns in order.
struct DrSpBags {
  const int32_t* off;         // [F + 1]
  const int32_t* comb;        // [F] 0 = sum, 1 = mean, 2 = sqrtn
  const int32_t* col_bag;     // [C] bag of id column c
  int32_t F;
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
// One warp = 32 consecutive samples of one id column (coalesced bf16 rows of the feature-major demb buffer, staged in shared memory).
// Lanes holding the same key are found with match.any.  The tile's key groups are then summed with the lanes on consecutive elements of
// a row: a lane adds one element of its group's members in ascending lane order (an fp32 sum from 0, so the bits do not depend on how
// lanes are assigned), converts it to fixed point and reduces it into ugrad.  One reduction instruction covers whole rows (two 128 B rows
// at dim 16) instead of 32 scattered 8-byte ones; no shared-memory atomics (fp32 ATOMS are CAS loops), no sort.
// Rows wider than 64 (dim 128) are staged and summed in 64-wide passes: a whole tile would need 64 KB of shared memory.
// -----------------------------------------------------------------------------------------------------------------
template <int LPR /* dim / 4 */>
__global__ void __launch_bounds__(256) k_sp_segsum(const __nv_bfloat16* __restrict__ demb /* [C][B][dim] */, const int32_t* __restrict__ invT /* [C][B] */,
                                                   DrSpGeom g, unsigned long long* __restrict__ ugrad, DrSpSync sync) {
  pdl_sync();
  constexpr int dim = 4 * LPR;
  constexpr int PD = dim < 64 ? dim : 64;                      // row elements per pass
  constexpr int V = PD / 8;                                    // int4 (8 bf16) chunks per row and pass
  constexpr int EL = PD < 32 ? PD : 32;                        // lanes per row
  constexpr int EPL = PD / EL;                                 // elements per lane
  constexpr int RPI = 32 / EL;                                 // rows per reduction instruction
  static_assert(dim % PD == 0, "dim: a multiple of the pass width");
  __shared__ __align__(16) int4 s_row[8][32][V];
  __shared__ int32_t s_lead[8][32];                            // lane of the j-th key group's leader (groups in ascending leader lane)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int sub = lane / EL, e0 = lane % EL;
  const int64_t tiles = (g.B + 31) / 32;
  const int64_t units = tiles * g.C;
  for (int64_t u = (int64_t)blockIdx.x * 8 + warp; u < units; u += (int64_t)gridDim.x * 8) {
    const int c = (int)(u / tiles);
    const int64_t b = (u % tiles) * 32 + lane;
    int32_t gs = -1;
    if (b < g.B) gs = invT[(int64_t)c * g.B + b];
    const bool live = gs >= 0;
    const unsigned lm = __ballot_sync(0xffffffffu, live);
    unsigned same = 0;
    if (live) same = __match_any_sync(lm, gs);
    const bool leader = live && lane == __ffs(same) - 1;
    const unsigned lead = __ballot_sync(0xffffffffu, leader);
    if (leader) s_lead[warp][__popc(lead & ((1u << lane) - 1u))] = lane;
    const int ngroups = __popc(lead);
    for (int p = 0; p < dim / PD; ++p) {
      if (live) {
        const int4* src = reinterpret_cast<const int4*>(demb + ((int64_t)c * g.B + b) * dim + p * PD);
#pragma unroll
        for (int v = 0; v < V; ++v) s_row[warp][lane][v] = ld_nc_v4(src + v);
      }
      __syncwarp();
      for (int j0 = 0; j0 < ngroups; j0 += RPI) {
        const int j = j0 + sub;
        const int ll = s_lead[warp][j < ngroups ? j : j0];
        const unsigned members = __shfl_sync(0xffffffffu, same, ll);
        const int32_t key = __shfl_sync(0xffffffffu, gs, ll);
        if (j < ngroups) {
          float acc[EPL];
#pragma unroll
          for (int k = 0; k < EPL; ++k) acc[k] = 0.f;
          for (unsigned m = members; m; m &= m - 1) {
            const uint16_t* r = reinterpret_cast<const uint16_t*>(s_row[warp][__ffs(m) - 1]);
#pragma unroll
            for (int k = 0; k < EPL; ++k) acc[k] += __uint_as_float((uint32_t)r[e0 + EL * k] << 16);      // bf16 -> fp32 is exact
          }
          unsigned long long* dst = ugrad + (int64_t)key * dim + p * PD + e0;
#pragma unroll
          for (int k = 0; k < EPL; ++k) atomicAdd(dst + EL * k, ugrad_fix(acc[k]));
        }
      }
      __syncwarp();
    }
  }
  sp_signal_last_block(sync, SP_CH_GRAD);
}

// -----------------------------------------------------------------------------------------------------------------
// k_sp_gather (requester): out[b * ldo + c * dim + :] = urow[inv[b][c]]  (padding -> zeros) -- the sample-major [B, C, dim] activation generic
// dense networks consume (models/rec_engine.py, ldo = C * dim), or the embedding columns of a wider row (DLRM-DCNv2's x0).  Waits in-kernel
// for every owner's ROWS flag, like the fused interaction kernels do.
// -----------------------------------------------------------------------------------------------------------------
template <int LPR>
__global__ void __launch_bounds__(256) k_sp_gather(const __nv_bfloat16* __restrict__ urow, const int32_t* __restrict__ inv, int ldinv, int C, int64_t B,
                                                   __nv_bfloat16* __restrict__ out, int64_t ldo, DrSpSync sync) {
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
    *reinterpret_cast<uint2*>(out + b * ldo + (int64_t)c * dim + 4 * lane) = v;
  }
}

// -----------------------------------------------------------------------------------------------------------------
// k_sp_pool (requester): out[b][f][:] = w * (sum over the live columns c of bag f of urow[inv[b][c]]), added in column order in fp32 and rounded
// once to bf16.  n = the live ids of the bag: padding (inv < 0) neither adds nor counts, a key a CounterFilter has not admitted counts with its
// no_permission row.  w = 1, 1/n or 1/sqrt(n) for sum / mean / sqrtn (correctly rounded), 0 for an empty bag; it is stored to w_out[f][b]
// for the backward, which cannot cheaply recount n per column.  One LPR-lane group per (b, f), so the result does not depend on the grid.
// Waits in-kernel for every owner's ROWS flag, like k_sp_gather.
// -----------------------------------------------------------------------------------------------------------------
template <int LPR>
__global__ void __launch_bounds__(256) k_sp_pool(const __nv_bfloat16* __restrict__ urow, const int32_t* __restrict__ inv, int ldinv, int64_t B,
                                                 DrSpBags bags, __nv_bfloat16* __restrict__ out, float* __restrict__ w_out, DrSpSync sync) {
  pdl_sync();
  sp_wait_all(sync, SP_CH_ROWS);
  constexpr int dim = 4 * LPR;
  const int lane = threadIdx.x % LPR;
  const int F = bags.F;
  const int64_t n = B * F;
  for (int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / LPR; i < n; i += (int64_t)gridDim.x * blockDim.x / LPR) {
    const int64_t b = i / F; const int f = (int)(i % F);
    const int32_t* ib = inv + b * ldinv;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    int live = 0;
    for (int c = bags.off[f], ce = bags.off[f + 1]; c < ce; ++c) {
      const int32_t gs = ib[c];
      if (gs < 0) continue;
      uint2 v;
      DR_LD_V2_VOLATILE_U32(v, urow + (int64_t)gs * dim + 4 * lane);       // peer-written row: bypass L1, as k_sp_gather does
      const float2 x = unpack_bf16x2(v.x), y = unpack_bf16x2(v.y);
      a0 += x.x; a1 += x.y; a2 += y.x; a3 += y.y;
      ++live;
    }
    const int comb = bags.comb[f];
    const float w = live == 0 ? 0.f : comb == 0 ? 1.f : comb == 1 ? __frcp_rn((float)live) : __frcp_rn(__fsqrt_rn((float)live));
    *reinterpret_cast<uint2*>(out + i * dim + 4 * lane) = make_uint2(pack_bf16x2(a0 * w, a1 * w), pack_bf16x2(a2 * w, a3 * w));
    if (lane == 0) w_out[(int64_t)f * B + b] = w;
  }
}

// -----------------------------------------------------------------------------------------------------------------
// k_sp_pool_segsum (requester): k_sp_segsum for pooled bags.  Column c of sample b contributes its bag's gradient row dpool[bag(c)][b] times
// w[bag(c)][b] (each element rounded once to fp32, no fused multiply-add), so with sum bags (w = 1) a key's sum equals k_sp_segsum's on the bag
// gradient repeated per column, bit for bit.  Same unit of work (one warp = 32 consecutive samples of one column), match.any leader sums,
// 64-bit fixed-point atomics; the last block raises GRAD.
// -----------------------------------------------------------------------------------------------------------------
template <int LPR /* dim / 4 */>
__global__ void __launch_bounds__(256) k_sp_pool_segsum(const __nv_bfloat16* __restrict__ dpool /* [F][B][dim] */, const float* __restrict__ wbag /* [F][B] */,
                                                        const int32_t* __restrict__ invT /* [C][B] */, DrSpGeom g, DrSpBags bags,
                                                        unsigned long long* __restrict__ ugrad, DrSpSync sync) {
  pdl_sync();
  constexpr int dim = 4 * LPR;
  constexpr int V = dim / 8;                                   // int4 (8 bf16) chunks per row
  __shared__ __align__(16) int4 s_row[8][32][V];
  __shared__ float s_w[8][32];
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
      const int64_t r = (int64_t)bags.col_bag[c] * g.B + b;
      const int4* src = reinterpret_cast<const int4*>(dpool + r * dim);
#pragma unroll
      for (int v = 0; v < V; ++v) s_row[warp][lane][v] = ld_nc_v4(src + v);
      s_w[warp][lane] = wbag[r];
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
          const float w = s_w[warp][src_lane];
#pragma unroll
          for (int v = 0; v < V; ++v) {
            const int4 raw = s_row[warp][src_lane][v];
            const uint32_t q[4] = {(uint32_t)raw.x, (uint32_t)raw.y, (uint32_t)raw.z, (uint32_t)raw.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float2 f = unpack_bf16x2(q[e]);
              acc[8 * v + 2 * e] += __fmul_rn(f.x, w);
              acc[8 * v + 2 * e + 1] += __fmul_rn(f.y, w);
            }
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
// k_sp_linear_fwd (requester): out[b] = sum_c float(urow[inv[b][c]][0])  -- the linear (wide) logit of a sample, read in place from the
// unique rows instead of gathering a [B, C, dim] activation.  One thread per sample adds its columns in order in fp32, so the result is
// the sequential float sum whatever the launch geometry.  Padding (inv < 0) adds nothing.  Waits in-kernel for every owner's ROWS flag.
// -----------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_sp_linear_fwd(const __nv_bfloat16* __restrict__ urow, const int32_t* __restrict__ inv, int ldinv, int C,
                                                       int64_t B, int dim, float* __restrict__ out, DrSpSync sync) {
  pdl_sync();
  sp_wait_all(sync, SP_CH_ROWS);
  for (int64_t b = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
    const int32_t* ib = inv + b * ldinv;
    float acc = 0.f;
    for (int c = 0; c < C; ++c) {
      const int32_t gs = ib[c];
      if (gs < 0) continue;
      uint2 v;
      DR_LD_V2_VOLATILE_U32(v, urow + (int64_t)gs * dim);       // peer-written row: bypass L1, as k_sp_gather does
      acc += unpack_bf16x2(v.x).x;
    }
    out[b] = acc;
  }
}

// -----------------------------------------------------------------------------------------------------------------
// k_sp_linear_bwd (requester): ugrad[gs][0] += fix(dlogit[b]) for every (c, b) with gs = invT[c][b] >= 0.  The per-sample gradient is
// fp32 and each term is converted to 64-bit fixed point before anything is combined, so a key's sum is exactly the integer sum of its
// terms whatever the grid or warp layout.  One warp = 32 consecutive samples of one column; lanes holding the same key are combined
// with match.any so a hot key costs one atomic per warp.  Elements 1..dim-1 keep the zero k_sp_dedup wrote.  Last block raises GRAD.
// -----------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_sp_linear_bwd(const float* __restrict__ dlogit, const int32_t* __restrict__ invT, DrSpGeom g,
                                                       unsigned long long* __restrict__ ugrad, DrSpSync sync) {
  pdl_sync();
  __shared__ uint64_t s_q[8][32];                             // (one-token type: the emulation build gives it per-block storage)
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
    if (live) s_q[warp][lane] = ugrad_fix(dlogit[b]);
    __syncwarp();
    if (live) {
      const unsigned same = __match_any_sync(lm, gs);
      if (lane == __ffs(same) - 1) {                            // leader of this key inside the tile: integer sum of its members' terms
        unsigned long long sum = 0;
        for (unsigned m = same; m; m &= m - 1) sum += s_q[warp][__ffs(m) - 1];
        atomicAdd(ugrad + (int64_t)gs * g.dim, sum);
      }
    }
    __syncwarp();
  }
  sp_signal_last_block(sync, SP_CH_GRAD);
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
  const int64_t cap = (int64_t)sparse_sm_count() * sparse_blocks_per_sm();
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
    case 2: SPS(2); break; case 4: SPS(4); break; case 8: SPS(8); break; case 16: SPS(16); break; case 32: SPS(32); break;
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
    case 1: SPL(1); break; case 2: SPL(2); break; case 4: SPL(4); break; case 8: SPL(8); break; case 16: SPL(16); break; case 32: SPL(32); break;
    default: return -3;
  }
#undef SPL
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_sp_grad(const DrDeviceTable* tables_dev, const int32_t* table_map, const DrSpGeom* g, int64_t max_bcap, const DrPeers* ugrad,
               const int32_t* own_pos, const int32_t* own_gs, const int32_t* own_cnt, float* gsum, const DrSpSync* sync, cudaStream_t s) {
  const int lpr = g->dim / 4;
  if (lpr < 1 || lpr > 32 || (lpr & (lpr - 1))) return -3;
  const int ipc = 256 / lpr;
  const int64_t chunks = (int64_t)g->T * g->W * ((max_bcap + ipc - 1) / ipc);
  const int grid = sp_grid(chunks);
#define SPG(L) DR_PDL_LAUNCH((k_sp_grad<L>), grid, 256, 0, s, tables_dev, table_map, *g, *ugrad, own_pos, own_gs, own_cnt, gsum, *sync)
  switch (lpr) {
    case 1: SPG(1); break; case 2: SPG(2); break; case 4: SPG(4); break; case 8: SPG(8); break; case 16: SPG(16); break; case 32: SPG(32); break;
    default: return -3;
  }
#undef SPG
  DR_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"

namespace {
int sp_gather(const void* urow, const int32_t* inv, const DrSpGeom* g, void* out, int64_t ldo, const DrSpSync* sync, cudaStream_t s) {
  const int lpr = g->dim / 4;
  const int64_t n = g->B * g->C;
  const int grid = sp_grid((n * lpr + 255) / 256);
#define SPGA(L) DR_PDL_LAUNCH((k_sp_gather<L>), grid, 256, 0, s, (const __nv_bfloat16*)urow, inv, g->ldinv, g->C, g->B, (__nv_bfloat16*)out, ldo, *sync)
  switch (lpr) {
    case 2: SPGA(2); break; case 4: SPGA(4); break; case 8: SPGA(8); break; case 16: SPGA(16); break; case 32: SPGA(32); break;
    default: return -3;
  }
#undef SPGA
  DR_LAUNCH_CHECK();
  return 0;
}
}  // namespace

extern "C" {

int dr_sp_gather(const void* urow, const int32_t* inv, const DrSpGeom* g, void* out, const DrSpSync* sync, cudaStream_t s) {
  return sp_gather(urow, inv, g, out, (int64_t)g->C * g->dim, sync, s);
}

// dr_sp_gather into rows of pitch ldo (elements): out[b * ldo + c * dim + :] = urow[inv[b][c]].  -2: ldo not a multiple of 4 or < C * dim,
// or out not 8-byte aligned.
int dr_sp_gather_pitched(const void* urow, const int32_t* inv, const DrSpGeom* g, void* out, int64_t ldo, const DrSpSync* sync, cudaStream_t s) {
  if ((ldo % 4) || ldo < (int64_t)g->C * g->dim || ((uintptr_t)out & 7)) return -2;
  return sp_gather(urow, inv, g, out, ldo, sync, s);
}

// out: bf16 [B][F][dim] pooled bags, w_out: fp32 [F][B] the factor each bag was scaled by; waits for every owner's ROWS flag
int dr_sp_pool(const void* urow, const int32_t* inv, const DrSpGeom* g, const DrSpBags* bags, void* out, float* w_out, const DrSpSync* sync,
               cudaStream_t s) {
  if (bags->F <= 0 || bags->F > g->C || g->ldinv < g->C) return -2;
  const int lpr = g->dim / 4;
  const int64_t n = g->B * bags->F;
  const int grid = sp_grid((n * lpr + 255) / 256);
#define SPP(L) DR_PDL_LAUNCH((k_sp_pool<L>), grid, 256, 0, s, (const __nv_bfloat16*)urow, inv, g->ldinv, g->B, *bags, (__nv_bfloat16*)out, w_out, *sync)
  switch (g->dim % 4 ? 0 : lpr) {
    case 2: SPP(2); break; case 4: SPP(4); break; case 8: SPP(8); break; case 16: SPP(16); break; case 32: SPP(32); break;
    default: return -3;
  }
#undef SPP
  DR_LAUNCH_CHECK();
  return 0;
}

// dpool: bf16 [F][B][dim] gradient of the pooled bags, w: fp32 [F][B] as dr_sp_pool stored it; accumulates into ugrad and raises the GRAD flags
int dr_sp_pool_segsum(const void* dpool, const float* w, const int32_t* invT, const DrSpGeom* g, const DrSpBags* bags, void* ugrad,
                      const DrSpSync* sync, cudaStream_t s) {
  if (bags->F <= 0 || bags->F > g->C) return -2;
  const int64_t units = ((g->B + 31) / 32) * g->C;
  const int grid = sp_grid((units + 7) / 8);
#define SPPS(L) DR_PDL_LAUNCH((k_sp_pool_segsum<L>), grid, 256, 0, s, (const __nv_bfloat16*)dpool, w, invT, *g, *bags, (unsigned long long*)ugrad, *sync)
  switch (g->dim % 4 ? 0 : g->dim / 4) {
    case 2: SPPS(2); break; case 4: SPPS(4); break; case 8: SPPS(8); break; case 16: SPPS(16); break;
    default: return -3;
  }
#undef SPPS
  DR_LAUNCH_CHECK();
  return 0;
}

// out_f32[b] = sum_c float(urow[inv[b][c]][0]): the linear logit of every local sample (fp32 [B]); waits for every owner's ROWS flag
int dr_sp_linear_fwd(const void* urow, const int32_t* inv, const DrSpGeom* g, float* out_f32, const DrSpSync* sync, cudaStream_t s) {
  if (g->dim % 4 || g->dim <= 0 || g->ldinv < g->C) return -2;
  DR_PDL_LAUNCH((k_sp_linear_fwd), sp_grid((g->B + 255) / 256), 256, 0, s, (const __nv_bfloat16*)urow, inv, g->ldinv, g->C, g->B, g->dim, out_f32, *sync);
  DR_LAUNCH_CHECK();
  return 0;
}

// dlogit_f32: fp32 [B] gradient of the linear logits; adds it to element 0 of ugrad[invT[c][b]] for every live id and raises the GRAD flags
int dr_sp_linear_bwd(const float* dlogit_f32, const int32_t* invT, const DrSpGeom* g, void* ugrad, const DrSpSync* sync, cudaStream_t s) {
  if (g->dim % 4 || g->dim <= 0) return -2;
  const int64_t units = ((g->B + 31) / 32) * g->C;
  DR_PDL_LAUNCH((k_sp_linear_bwd), sp_grid((units + 7) / 8), 256, 0, s, dlogit_f32, invT, *g, (unsigned long long*)ugrad, *sync);
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
