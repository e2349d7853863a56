// All-gather -> lookup / partial combine -> reduce-scatter embedding over NVLink peer memory.
//
// The reference's OTHER model-parallel dataflow (SOK v1 `DistributedEmbedding`, SURVEY 2.15 C5 / C6): every rank all-gathers the sparse ids of
// the whole global batch (3 x ncclAllGather: values, row indices, counts -- all_gather_dispatcher.cu:128-140), looks up and partially combines
// the keys ITS shard owns for every sample of every rank, then reduce-scatters the [W * B, D] partial sums (ncclReduceScatter + an all-reduce of
// the row offsets, reduce_scatter_dispatcher.cu:42-84); the backward all-gathers the top gradients.  Here the three collectives disappear into
// the kernels:
//   k_ag_lookup  (owner)      reads every peer's (key, row) list IN PLACE over NVLink (no gathered copy exists), probes / inserts the keys it owns
//                             (admission, frequency, dedup claim: table_touch_aggregated) and accumulates their rows into partial[src][row];
//   k_ag_reduce  (requester)  out[b] = sum over owners of their partial[me][b], pulled straight from the owners' memory: the reduce-scatter;
//   k_ag_grad    (owner)      pulls the top-gradient row of every (source, sample) it contributed to and adds it to the claimed key's gradient
//                             sum; the row optimizer (k_apply) follows.
// Synchronisation: the release / acquire flags of sp_sync.cuh (IDS raised after a rank staged its ids, ROWS after an owner's lookup, GRAD after a
// requester staged its gradients, AUX = "I have consumed every owner's partial" so that owners may zero it for the next step).
// The unique-first pipeline (sparse_pipeline.cu) moves strictly less data and is what the engines use; this is the SOK-compatible variant for
// multi-hot columns whose per-sample combine is worth doing at the owner (the partial sums that cross NVLink are one row per (owner, sample),
// however many ids the sample has).
#include "sp_sync.cuh"
#include "table.cuh"

using namespace drc;

extern "C" {
struct DrAgGeom {
  int32_t W, rank, dim, table_index;   // table_index: position of the table in the StepContext's struct array (ulist encoding)
  int64_t B;                           // samples per rank
  int64_t nnz_cap;                     // capacity of every rank's (key, row) lists
};
// symmetric buffers (one allocation per rank, peer-mapped): keys int64 [nnz_cap], rows int32 [nnz_cap], meta int32 [4] ([0] = nnz),
// partial fp32 [W][B][D] (owner side: contributions to source s's samples), grad fp32 [B][D] (requester side: top gradients)
struct DrAgPeers { DrPeers keys, rows, meta, partial, grad; };
}

namespace {

enum { AG_CH_IDS = 0, AG_CH_ROWS = 1, AG_CH_GRAD = 2, AG_CH_DONE = 4 };

__device__ __forceinline__ int ag_owner(int64_t key, int W) {
  return W == 1 ? 0 : (int)((dr_mix64((uint64_t)key ^ 0x7f4a7c159e3779b9ULL) >> 33) % (uint64_t)W);
}

// wait until `src` has finished phase `ch` of the PREVIOUS step (flags are monotonic: value >= state[0])
__device__ __forceinline__ void ag_wait_prev(const DrSpSync& s, int ch, int src) {
  const uint32_t ep = (uint32_t)ld_volatile_i32(&s.state[0]);
  const uint32_t* f = reinterpret_cast<const uint32_t*>(s.flags.ptr[s.rank]) + ch * 16 + src;
  while ((int32_t)(ld_acquire_sys(f) - ep) < 0) __nanosleep(40);
}

// zero my partial sums once every requester has consumed the previous step's
__global__ void __launch_bounds__(256) k_ag_zero(float* __restrict__ partial, int64_t n, DrSpSync sync) {
  if ((int)threadIdx.x < sync.W) ag_wait_prev(sync, AG_CH_DONE, threadIdx.x);
  __syncthreads();
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) partial[i] = 0.f;
}

// owner: one warp per 32 entries of a source's list
__global__ void __launch_bounds__(256) k_ag_lookup(const DrDeviceTable* __restrict__ tables, DrAgGeom g, DrAgPeers P, int train, int32_t* __restrict__ own_pos /* [W][nnz_cap] */,
                                                   int32_t* __restrict__ own_row /* [W][nnz_cap] */, int32_t* __restrict__ own_cnt /* [W] */, int64_t* __restrict__ ulist,
                                                   int32_t* __restrict__ nunique, int64_t ulist_cap, DrSpSync sync) {
  const DrDeviceTable& TB = tables[g.table_index];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const int W = g.W, D = g.dim;
  float* partial = reinterpret_cast<float*>(P.partial.ptr[g.rank]);
  for (int si = 0; si < W; ++si) {
    const int s = (g.rank + si) % W;                          // own list first, then the peers in ring order
    __syncthreads();
    if (threadIdx.x == 0) sp_wait_one(sync, AG_CH_IDS, s);
    __syncthreads();
    int64_t n = (int64_t)ld_relaxed_sys(reinterpret_cast<const uint32_t*>(P.meta.ptr[s]));
    if (n > g.nnz_cap) n = g.nnz_cap;
    if (blockIdx.x == 0 && threadIdx.x == 0) own_cnt[s] = (int32_t)n;
    const int64_t* keys = reinterpret_cast<const int64_t*>(P.keys.ptr[s]);
    const int32_t* rows = reinterpret_cast<const int32_t*>(P.rows.ptr[s]);
    for (int64_t base = ((int64_t)blockIdx.x * wpb + warp) * 32; base < n; base += (int64_t)gridDim.x * wpb * 32) {
      const int64_t e = base + lane;
      int64_t key = 0, pos = -1;
      int32_t row = -1;
      bool mine = false, touch = false;
      if (e < n) {
        key = keys[e]; row = rows[e];
        mine = key != kEmptyKey && key != kTombKey && row >= 0 && row < g.B && ag_owner(key, W) == g.rank;
        if (mine) {
          if (!train || TB.is_inference) {
            pos = table_find(TB, key);
          } else {
            bool inserted = false, skip = false;
            if (TB.filter_type == DR_FILTER_BLOOM) {
              pos = table_find(TB, key);
              if (pos < 0) {
                if (bloom_add_min(TB, key, 1u) < (uint32_t)TB.filter_freq) skip = true;
                else pos = table_find_or_insert(TB, key, &inserted);
              }
            } else {
              pos = table_find_or_insert(TB, key, &inserted);
            }
            if (!skip && pos < 0) TB.counters[CTR_OVERFLOW] = 1;
            if (inserted) atomicAdd(&TB.counters[CTR_NKEYS], 1);
            touch = !skip && pos >= 0;
          }
        }
        own_pos[(int64_t)s * g.nnz_cap + e] = mine ? (int32_t)pos : -2;        // -2: not mine, -1: mine but absent (default / no-permission row)
        own_row[(int64_t)s * g.nnz_cap + e] = row;
      }
      if (train) table_touch_aggregated(TB, touch, pos, g.table_index, ulist, nunique, ulist_cap);      // all 32 lanes
      // accumulate the rows of this warp's entries into partial[s][row]: the lanes walk the embedding dimension
      for (int j = 0; j < 32; ++j) {
        const int m = __shfl_sync(0xffffffffu, (int)mine, j);
        if (!m) continue;
        const int64_t kj = __shfl_sync(0xffffffffu, key, j), pj = __shfl_sync(0xffffffffu, pos, j);
        const int rj = __shfl_sync(0xffffffffu, row, j);
        const float* src = table_read_ptr(TB, kj, pj);
        float* dst = partial + ((int64_t)s * g.B + rj) * D;
        for (int d = lane; d < D; d += 32) atomicAdd(dst + d, src ? src[d] : TB.no_permission);
      }
    }
  }
  sp_signal_last_block(sync, AG_CH_ROWS);
}

// requester: the reduce-scatter as a pull -- out[b] = scale[b] * sum_r partial_r[me][b]
__global__ void __launch_bounds__(256) k_ag_reduce(DrAgGeom g, DrAgPeers P, const float* __restrict__ scale /* [B] or null */, float* __restrict__ out /* [B][D] */,
                                                   DrSpSync sync) {
  sp_wait_all(sync, AG_CH_ROWS);
  const int64_t n = g.B * (int64_t)g.dim;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int r = 0; r < g.W; ++r) acc += reinterpret_cast<const float*>(P.partial.ptr[r])[(int64_t)g.rank * n + i];
    out[i] = scale ? acc * scale[i / g.dim] : acc;
  }
  sp_signal_last_block(sync, AG_CH_DONE);
}

// owner: the gradient of every entry I contributed is the top gradient of its (source, sample): pull it, add it to the key's claimed sum
__global__ void __launch_bounds__(256) k_ag_grad(const DrDeviceTable* __restrict__ tables, DrAgGeom g, DrAgPeers P, const int32_t* __restrict__ own_pos,
                                                 const int32_t* __restrict__ own_row, const int32_t* __restrict__ own_cnt, float* __restrict__ gsum, int64_t ulist_cap,
                                                 DrSpSync sync) {
  sp_wait_all(sync, AG_CH_GRAD);
  const DrDeviceTable& TB = tables[g.table_index];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const int D = g.dim;
  for (int s = 0; s < g.W; ++s) {
    const int64_t n = own_cnt[s];
    const float* gr = reinterpret_cast<const float*>(P.grad.ptr[s]);
    for (int64_t e = (int64_t)blockIdx.x * wpb + warp; e < n; e += (int64_t)gridDim.x * wpb) {      // one warp per entry: lanes walk the dimension
      const int32_t pos = own_pos[(int64_t)s * g.nnz_cap + e];
      if (pos < 0) continue;
      const int32_t u = TB.slots[pos].tag;
      if (u < 0 || u >= ulist_cap) continue;                                                          // not admitted / claim list overflowed
      const float* src = gr + (int64_t)own_row[(int64_t)s * g.nnz_cap + e] * D;
      for (int d = lane; d < D; d += 32) atomicAdd(gsum + (int64_t)u * D + d, src[d]);
    }
  }
}

inline int ag_grid(int64_t work_items) {
  int64_t b = (work_items + 255) / 256;
  const int64_t cap = (int64_t)num_sms() * sparse_blocks_per_sm();
  return (int)(b < 1 ? 1 : b > cap ? cap : b);
}

}  // namespace

extern "C" {

int dr_ag_sizeof_geom() { return (int)sizeof(DrAgGeom); }

int dr_ag_lookup(const DrDeviceTable* tables_dev, const DrAgGeom* g, const DrAgPeers* P, int train, int32_t* own_pos, int32_t* own_row, int32_t* own_cnt, int64_t* ulist,
                 int32_t* nunique, int64_t ulist_cap, const DrSpSync* sync, cudaStream_t s) {
  if (g->W > 16 || g->dim <= 0 || g->B <= 0 || g->nnz_cap <= 0) return -2;
  float* partial = reinterpret_cast<float*>(P->partial.ptr[g->rank]);
  const int64_t n = (int64_t)g->W * g->B * g->dim;
  k_ag_zero<<<ag_grid(n), 256, 0, s>>>(partial, n, *sync);
  k_ag_lookup<<<ag_grid(g->nnz_cap), 256, 0, s>>>(tables_dev, *g, *P, train, own_pos, own_row, own_cnt, ulist, nunique, ulist_cap, *sync);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_ag_reduce(const DrAgGeom* g, const DrAgPeers* P, const float* scale, float* out, const DrSpSync* sync, cudaStream_t s) {
  k_ag_reduce<<<ag_grid(g->B * g->dim), 256, 0, s>>>(*g, *P, scale, out, *sync);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_ag_grad(const DrDeviceTable* tables_dev, const DrAgGeom* g, const DrAgPeers* P, const int32_t* own_pos, const int32_t* own_row, const int32_t* own_cnt, float* gsum,
               int64_t ulist_cap, const DrSpSync* sync, cudaStream_t s) {
  k_ag_grad<<<ag_grid(g->nnz_cap * 32), 256, 0, s>>>(tables_dev, *g, *P, own_pos, own_row, own_cnt, gsum, ulist_cap, *sync);
  DR_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
