// Device-side multi-tier EmbeddingVariable storage: an HBM cache tier (DrDeviceTable, bounded row slab) over a host DRAM tier
// (HostEV, csrc/host/host_engine.cc), driven by kernels and ONE native background thread -- no Python on the per-step path.
//
// Reference: MultiTierStorage / HbmDramStorage / BatchCache / EvictionManager (framework/embedding/multi_tier_storage.h:45-330,
// hbm_dram_storage.h:229-306, cache.h:133,272, eviction_manager.h:39-131, multi_tier_storage.cu.cc:43-121).  There the index of BOTH
// tiers is a CPU hash map, every GPU lookup first copies its ids D2H and blocks on the host probe (kv_variable_lookup_ops.cc:404-412),
// and a polling eviction thread demotes <= 10 000 ids per pass.  Here:
//
//   prefetch (one batch ahead, side stream)   k_tier_miss_list probes the HBM tier's own hash table; hits are PINNED for the coming
//       step (slot.pad = epoch -- the reference's add_to_prefetch_list); only the miss keys leave the GPU, written straight into mapped
//       pinned memory.  The background thread dedups them, reads the rows the DRAM tier holds (HostEV::ExportKeys) into a pinned staging
//       block and flags the batch ready.
//   commit (step boundary, main stream)        one cudaMemcpyAsync H2D per column of the staging block + the import kernel + a pin
//       kernel: every row the next step reads is resident before its graph launches.  Nothing is copied when nothing missed.
//   evict (step boundary, when the slab passes its high watermark)   k_tier_hist builds a log2 histogram of the eviction score over
//       the resident, un-pinned rows (LFU: frequency, LRU: age in steps); k_tier_threshold picks the score cut that frees the requested
//       number of rows; k_tier_evict compacts the victims (key, full-stride row, freq, version) into a device block, returns their rows
//       to the free list and tombstones their keys; D2H on the same stream; the background thread commits them to the DRAM tier
//       (HostEV::Import) when the copy's event fires -- strictly BEFORE it serves the next prefetch, so a key can never be looked for
//       in the host tier while it is still in flight.
//
// World > 1 (row-wise model parallelism: rank r holds the keys with dr_sp_owner(key, W) == r of every table, and with them BOTH tiers of those
// keys).  A key must be promoted by its OWNER, whichever ranks' batches it appears in, so the prefetch is a fused id all-gather + probe over
// peer memory -- no gathered copy of the ids, no NCCL call: k_tier_publish copies the rank's next-batch ids into its symmetric buffer (double
// buffered by epoch parity) and its last block raises the rank's epoch flag on every peer (st.release.sys); k_tier_wait (ONE block, so the spin can
// never starve the training step's kernels of SMs) polls the W flags; k_tier_miss_list_mp walks every rank's id buffer in place over NVLink and
// keeps the keys this rank owns.  Everything after the miss list (staging, import, pin, eviction) is rank-local.  Reuse of a parity buffer two
// prefetches later is safe because a step of the sparse pipeline cannot complete on any rank before every rank has launched it, which a rank
// does only after commit() saw its own probe kernel of the previous epoch finish.
#include <atomic>
#include <condition_variable>
#include <deque>
#include <mutex>
#include <thread>
#include <vector>
#include <algorithm>

#include "table.cuh"
#include "sp_sync.cuh"

using namespace drc;

namespace {

// ---- kernels -----------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_tier_miss_list(DrDeviceTable TB, const int64_t* __restrict__ keys, int64_t n, int64_t pad_key, uint32_t epoch,
                                                        int64_t* __restrict__ miss_keys /* mapped pinned */, int32_t* __restrict__ counters /* [0] misses [1] hits (device) */,
                                                        int64_t miss_cap) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t key = keys[i];
    if (key == pad_key || key == kEmptyKey || key == kTombKey) continue;
    const int64_t pos = table_find(TB, key);
    if (pos >= 0 && TB.slots[pos].row_of >= 0) {
      DR_ST_RACY(TB.slots[pos].pad, epoch);           // pinned until the step that consumes this batch has run (duplicates store the same value)
      atomicAdd(&counters[1], 1);
    } else {
      const int m = atomicAdd(&counters[0], 1);
      if (m < miss_cap) miss_keys[m] = key;
    }
  }
}

// ---- world > 1: publish my ids / wait for every rank's / probe the keys I own out of all of them ------------------------------------------------
__global__ void __launch_bounds__(256) k_tier_publish(const int64_t* __restrict__ keys, int64_t n, int64_t* __restrict__ mine /* my symmetric slot of this parity */,
                                                      DrPeers flags, int32_t* __restrict__ done /* device counter */, uint32_t epoch, int W, int rank) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) mine[i] = keys[i];
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();                                      // this block's ids before the count
    const int prev = atomicAdd(done, 1);
    if (prev == (int)gridDim.x - 1) {
      *done = 0;
      __threadfence_system();                                    // every block's ids before the flag
      for (int r = 0; r < W; ++r) st_release_sys(reinterpret_cast<uint32_t*>(flags.ptr[r]) + rank, epoch);
    }
  }
}

__global__ void k_tier_wait(DrPeers flags, uint32_t epoch, int W, int rank) {
  if ((int)threadIdx.x < W) {
    const uint32_t* f = reinterpret_cast<const uint32_t*>(flags.ptr[rank]) + threadIdx.x;
    while ((int32_t)(ld_acquire_sys(f) - epoch) < 0) __nanosleep(200);
  }
}

__global__ void __launch_bounds__(256) k_tier_miss_list_mp(DrDeviceTable TB, DrPeers ids /* int64 [2][n] per rank */, int64_t n, int parity, int64_t pad_key,
                                                           uint32_t epoch, int W, int rank, int64_t* __restrict__ miss_keys, int32_t* __restrict__ counters,
                                                           int64_t miss_cap) {
  const int64_t total = n * W;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int s = (int)(i / n);
    const int64_t key = reinterpret_cast<const int64_t*>(ids.ptr[(rank + s) % W])[(int64_t)parity * n + (i - (int64_t)s * n)];     // own list first, peers in ring order
    if (key == pad_key || key == kEmptyKey || key == kTombKey || dr_sp_owner(key, W) != rank) continue;
    const int64_t pos = table_find(TB, key);
    if (pos >= 0 && TB.slots[pos].row_of >= 0) {
      DR_ST_RACY(TB.slots[pos].pad, epoch);
      atomicAdd(&counters[1], 1);
    } else {
      const int m = atomicAdd(&counters[0], 1);
      if (m < miss_cap) miss_keys[m] = key;
    }
  }
}

__global__ void __launch_bounds__(256) k_tier_pin(DrDeviceTable TB, const int64_t* __restrict__ keys, int64_t n, uint32_t epoch) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t pos = table_find(TB, keys[i]);
    if (pos >= 0) TB.slots[pos].pad = epoch;
  }
}

// eviction score bucket: LFU -> floor(log2(freq + 1)), LRU -> 63 - floor(log2(age + 1)) (older = smaller = evicted first)
__device__ __forceinline__ int tier_bucket(const DrSlot& s, int strategy, int64_t step) {
  if (strategy == 0) return 63 - __clzll((unsigned long long)max(s.freq, 0) + 1ull);
  const long long age = max((long long)step - (long long)s.version, 0ll);
  return 63 - (63 - __clzll((unsigned long long)age + 1ull));
}
__device__ __forceinline__ bool tier_evictable(const DrSlot& s, uint32_t epoch_min) {
  return s.key != kEmptyKey && s.key != kTombKey && s.row_of >= 0 && s.tag == -1 && s.pad < epoch_min;
}

__global__ void __launch_bounds__(256) k_tier_hist(DrDeviceTable TB, int strategy, int64_t step, uint32_t epoch_min, int32_t* __restrict__ hist /* [64] */) {
  __shared__ int32_t sh[64];
  if (threadIdx.x < 64) sh[threadIdx.x] = 0;
  __syncthreads();
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < TB.capacity; p += (int64_t)gridDim.x * blockDim.x) {
    const DrSlot s = TB.slots[p];
    if (tier_evictable(s, epoch_min)) atomicAdd(&sh[tier_bucket(s, strategy, step)], 1);
  }
  __syncthreads();
  if (threadIdx.x < 64 && sh[threadIdx.x]) atomicAdd(&hist[threadIdx.x], sh[threadIdx.x]);
}

// ctl[0] = bucket cut (evict buckets <= cut), ctl[1] = rows allowed from the cut bucket itself, ctl[2] = victim counter, ctl[3] = cut-bucket counter
__global__ void k_tier_threshold(const int32_t* __restrict__ hist, int32_t need, int32_t* __restrict__ ctl) {
  int acc = 0, cut = -1, partial = 0;
  for (int b = 0; b < 64; ++b) {
    if (acc + hist[b] >= need) { cut = b; partial = need - acc; break; }
    acc += hist[b];
  }
  if (cut < 0) { cut = 63; partial = 0x7fffffff; }            // fewer evictable rows than requested: take them all
  ctl[0] = cut; ctl[1] = partial; ctl[2] = 0; ctl[3] = 0;
}

__global__ void __launch_bounds__(256) k_tier_evict(DrDeviceTable TB, int strategy, int64_t step, uint32_t epoch_min, int32_t* __restrict__ ctl, int32_t cap,
                                                    int64_t* __restrict__ ev_keys, float* __restrict__ ev_rows, int64_t* __restrict__ ev_freq,
                                                    int64_t* __restrict__ ev_ver) {
  const int cut = ctl[0], partial = ctl[1];
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < TB.capacity; p += (int64_t)gridDim.x * blockDim.x) {
    const DrSlot s = TB.slots[p];
    if (!tier_evictable(s, epoch_min)) continue;
    const int b = tier_bucket(s, strategy, step);
    if (b > cut) continue;
    if (b == cut && atomicAdd(&ctl[3], 1) >= partial) continue;
    const int v = atomicAdd(&ctl[2], 1);
    if (v >= cap) continue;
    ev_keys[v] = s.key; ev_freq[v] = s.freq; ev_ver[v] = s.version;
    const float* row = TB.rows + (int64_t)s.row_of * TB.stride;
    float* dst = ev_rows + (int64_t)v * TB.stride;
    for (int d = 0; d < TB.stride; d += 4) *reinterpret_cast<float4*>(dst + d) = *reinterpret_cast<const float4*>(row + d);
    // give the row back and drop the key (a later lookup misses -> the row comes back from the DRAM tier)
    const int32_t top = atomicAdd(&TB.counters[CTR_FREE_TOP], 1);
    TB.free_list[top] = s.row_of;
    atomicSub(&TB.counters[CTR_NADMITTED], 1); atomicSub(&TB.counters[CTR_NKEYS], 1);
    DrSlot z; z.key = kTombKey; z.freq = 0; z.version = -1; z.row_of = -1; z.tag = -1; z.dirty = 0; z.pad = 0;
    TB.slots[p] = z;
  }
}

// ---- native manager --------------------------------------------------------------------------------------------------------
typedef void (*fn_export_t)(void*, const int64_t*, int64_t, float*, int64_t*, int64_t*, uint8_t*);
typedef int64_t (*fn_import_t)(void*, const int64_t*, const float*, int64_t, const int64_t*, const int64_t*, int64_t, int, int, int);

struct TierManager {
  void* host_ev; fn_export_t fexport; fn_import_t fimport;
  int stride; int64_t miss_cap, evict_cap;
  // prefetch path
  int64_t* h_miss = nullptr; int64_t* d_miss_alias = nullptr;     // mapped pinned (host / device views)
  int32_t* d_counters = nullptr; int32_t* h_counters = nullptr;    // device counters + pinned copy
  int64_t *h_imp_keys = nullptr, *h_imp_freq = nullptr, *h_imp_ver = nullptr; float* h_imp_rows = nullptr;
  int64_t *d_imp_keys = nullptr, *d_imp_freq = nullptr, *d_imp_ver = nullptr; float* d_imp_rows = nullptr; int32_t* d_kept = nullptr;
  cudaEvent_t ev_miss = nullptr, ev_imp_copied = nullptr; bool imp_copy_pending = false;
  // eviction path
  int32_t *d_hist = nullptr, *d_ctl = nullptr, *h_ctl = nullptr;
  int64_t *d_ev_keys = nullptr, *d_ev_freq = nullptr, *d_ev_ver = nullptr; float* d_ev_rows = nullptr;
  int64_t *h_ev_keys = nullptr, *h_ev_freq = nullptr, *h_ev_ver = nullptr; float* h_ev_rows = nullptr;
  cudaEvent_t ev_evict = nullptr;
  // thread + queue
  std::thread th; std::mutex mu; std::condition_variable cv;
  std::deque<int> q;                                  // 0 = prefetch batch, 1 = eviction commit, 2 = quit
  bool prefetch_inflight = false, prefetch_ready = false, evict_inflight = false;
  int64_t n_import = 0;
  std::vector<int64_t> uniq; std::vector<uint8_t> found;
  int device = 0;
  // statistics
  std::atomic<int64_t> hits{0}, misses{0}, promoted{0}, demoted{0}, h2d_bytes{0}, d2h_bytes{0}, evict_passes{0};

  void Loop() {
    cudaSetDevice(device);
    for (;;) {
      int job;
      { std::unique_lock<std::mutex> l(mu); cv.wait(l, [&] { return !q.empty(); }); job = q.front(); q.pop_front(); }
      if (job == 2) return;
      if (job == 1) {            // ---- eviction commit: rows have landed in pinned memory when the event fires
        cudaEventSynchronize(ev_evict);
        const int64_t n = std::min<int64_t>(h_ctl[2], evict_cap);
        if (n > 0) {
          fimport(host_ev, h_ev_keys, h_ev_rows, stride, h_ev_freq, h_ev_ver, n, 0, 1, /*keep versions, mark dirty (incremental checkpoints)*/ 2);
          demoted += n; d2h_bytes += n * ((int64_t)stride * 4 + 24);
        }
        { std::lock_guard<std::mutex> l(mu); evict_inflight = false; }
        cv.notify_all();
        continue;
      }
      // ---- prefetch: miss keys are in mapped pinned memory once the probe kernel's event fires
      cudaEventSynchronize(ev_miss);
      const int64_t nm = std::min<int64_t>(h_counters[0], miss_cap);
      const bool overflow = h_counters[0] > miss_cap;               // a dropped miss would be re-created from the default row: refuse (commit returns -20)
      hits += h_counters[1]; misses += h_counters[0];
      uniq.assign(h_miss, h_miss + nm);
      std::sort(uniq.begin(), uniq.end());
      uniq.erase(std::unique(uniq.begin(), uniq.end()), uniq.end());
      int64_t ni = 0;
      if (!uniq.empty()) {
        if (imp_copy_pending) { cudaEventSynchronize(ev_imp_copied); imp_copy_pending = false; }     // the staging block is still being read by the last H2D
        const int64_t nu = (int64_t)uniq.size();
        found.resize((size_t)nu);
        // export straight into the staging block, then compact the rows the DRAM tier really holds to the front
        fexport(host_ev, uniq.data(), nu, h_imp_rows, h_imp_freq, h_imp_ver, found.data());
        for (int64_t i = 0; i < nu; ++i) {
          if (!found[(size_t)i]) continue;
          if (ni != i) {
            memcpy(h_imp_rows + ni * stride, h_imp_rows + i * stride, (size_t)stride * 4);
            h_imp_freq[ni] = h_imp_freq[i]; h_imp_ver[ni] = h_imp_ver[i];
          }
          h_imp_keys[ni] = uniq[(size_t)i];
          ++ni;
        }
      }
      { std::lock_guard<std::mutex> l(mu); n_import = overflow ? -20 : ni; prefetch_ready = true; prefetch_inflight = false; }
      cv.notify_all();
    }
  }
};

template <typename T> int alloc_pinned(T** p, size_t n) { return (int)cudaHostAlloc((void**)p, n * sizeof(T), cudaHostAllocMapped); }
template <typename T> int alloc_dev(T** p, size_t n) { return (int)cudaMalloc((void**)p, n * sizeof(T)); }
inline int grid_of(int64_t n) { int64_t b = (n + 255) / 256; if (b < 1) b = 1; const int64_t cap = (int64_t)num_sms() * sparse_blocks_per_sm(); return (int)(b > cap ? cap : b); }

}  // namespace

extern "C" {

void* dr_tier_create(void* host_ev, void* fn_export, void* fn_import, int stride, int64_t miss_cap, int64_t evict_cap, int device) {
  auto* m = new TierManager();
  m->host_ev = host_ev; m->fexport = (fn_export_t)fn_export; m->fimport = (fn_import_t)fn_import;
  m->stride = stride; m->miss_cap = miss_cap; m->evict_cap = evict_cap; m->device = device;
  int rc = 0;
  rc |= alloc_pinned(&m->h_miss, (size_t)miss_cap);
  rc |= (int)cudaHostGetDevicePointer((void**)&m->d_miss_alias, m->h_miss, 0);
  rc |= alloc_dev(&m->d_counters, 4); rc |= alloc_pinned(&m->h_counters, 4);
  rc |= alloc_pinned(&m->h_imp_keys, (size_t)miss_cap); rc |= alloc_pinned(&m->h_imp_freq, (size_t)miss_cap); rc |= alloc_pinned(&m->h_imp_ver, (size_t)miss_cap);
  rc |= alloc_pinned(&m->h_imp_rows, (size_t)miss_cap * stride);
  rc |= alloc_dev(&m->d_imp_keys, (size_t)miss_cap); rc |= alloc_dev(&m->d_imp_freq, (size_t)miss_cap); rc |= alloc_dev(&m->d_imp_ver, (size_t)miss_cap);
  rc |= alloc_dev(&m->d_imp_rows, (size_t)miss_cap * stride); rc |= alloc_dev(&m->d_kept, 4);
  rc |= alloc_dev(&m->d_hist, 64); rc |= alloc_dev(&m->d_ctl, 4); rc |= alloc_pinned(&m->h_ctl, 4);
  rc |= alloc_dev(&m->d_ev_keys, (size_t)evict_cap); rc |= alloc_dev(&m->d_ev_freq, (size_t)evict_cap); rc |= alloc_dev(&m->d_ev_ver, (size_t)evict_cap);
  rc |= alloc_dev(&m->d_ev_rows, (size_t)evict_cap * stride);
  rc |= alloc_pinned(&m->h_ev_keys, (size_t)evict_cap); rc |= alloc_pinned(&m->h_ev_freq, (size_t)evict_cap); rc |= alloc_pinned(&m->h_ev_ver, (size_t)evict_cap);
  rc |= alloc_pinned(&m->h_ev_rows, (size_t)evict_cap * stride);
  rc |= (int)cudaEventCreateWithFlags(&m->ev_miss, cudaEventDisableTiming);
  rc |= (int)cudaEventCreateWithFlags(&m->ev_imp_copied, cudaEventDisableTiming);
  rc |= (int)cudaEventCreateWithFlags(&m->ev_evict, cudaEventDisableTiming);
  if (rc) { fprintf(stderr, "[deeprec_cuda] dr_tier_create: allocation failed (%d)\n", rc); delete m; return nullptr; }
  m->h_ctl[2] = 0;
  m->th = std::thread([m] { m->Loop(); });
  return m;
}

void dr_tier_destroy(void* h) {
  auto* m = static_cast<TierManager*>(h);
  { std::lock_guard<std::mutex> l(m->mu); m->q.push_back(2); }
  m->cv.notify_all();
  if (m->th.joinable()) m->th.join();
  cudaFreeHost(m->h_miss); cudaFree(m->d_counters); cudaFreeHost(m->h_counters);
  cudaFreeHost(m->h_imp_keys); cudaFreeHost(m->h_imp_freq); cudaFreeHost(m->h_imp_ver); cudaFreeHost(m->h_imp_rows);
  cudaFree(m->d_imp_keys); cudaFree(m->d_imp_freq); cudaFree(m->d_imp_ver); cudaFree(m->d_imp_rows); cudaFree(m->d_kept);
  cudaFree(m->d_hist); cudaFree(m->d_ctl); cudaFreeHost(m->h_ctl);
  cudaFree(m->d_ev_keys); cudaFree(m->d_ev_freq); cudaFree(m->d_ev_ver); cudaFree(m->d_ev_rows);
  cudaFreeHost(m->h_ev_keys); cudaFreeHost(m->h_ev_freq); cudaFreeHost(m->h_ev_ver); cudaFreeHost(m->h_ev_rows);
  cudaEventDestroy(m->ev_miss); cudaEventDestroy(m->ev_imp_copied); cudaEventDestroy(m->ev_evict);
  delete m;
}

// Probe `keys` (device, n entries, duplicates / padding allowed) against the HBM tier on `side`: hits are pinned for `epoch`, misses go to
// the background thread.  One batch may be in flight at a time (commit it before the next prefetch).
int dr_tier_prefetch(void* h, const DrDeviceTable* tb, const int64_t* keys, int64_t n, int64_t pad_key, uint32_t epoch, cudaStream_t side) {
  auto* m = static_cast<TierManager*>(h);
  {
    std::unique_lock<std::mutex> l(m->mu);
    if (m->prefetch_inflight || m->prefetch_ready) return -10;      // protocol: prefetch -> commit -> prefetch ...
    m->prefetch_inflight = true;
  }
  DR_CUDA_CHECK(cudaMemsetAsync(m->d_counters, 0, 16, side));
  if (n > 0) k_tier_miss_list<<<grid_of(n), 256, 0, side>>>(*tb, keys, n, pad_key, epoch, m->d_miss_alias, m->d_counters, m->miss_cap);
  DR_LAUNCH_CHECK();
  DR_CUDA_CHECK(cudaMemcpyAsync(m->h_counters, m->d_counters, 16, cudaMemcpyDeviceToHost, side));
  DR_CUDA_CHECK(cudaEventRecord(m->ev_miss, side));
  { std::lock_guard<std::mutex> l(m->mu); m->q.push_back(0); }
  m->cv.notify_all();
  return 0;
}

// World > 1: `keys` are THIS rank's next-batch ids (n entries, the same n on every rank); `ids` is a symmetric int64 [2][n] buffer and `flags` a
// symmetric zero-initialised uint32 [16] buffer (parallel.p2p.P2PComm.symmetric).  Every rank calls this once per epoch.
int dr_tier_prefetch_mp(void* h, const DrDeviceTable* tb, const int64_t* keys, int64_t n, int64_t pad_key, uint32_t epoch, const DrPeers* ids,
                        const DrPeers* flags, int W, int rank, cudaStream_t side) {
  auto* m = static_cast<TierManager*>(h);
  if (W < 1 || W > 16 || rank < 0 || rank >= W || n < 0) return -11;
  {
    std::unique_lock<std::mutex> l(m->mu);
    if (m->prefetch_inflight || m->prefetch_ready) return -10;
    m->prefetch_inflight = true;
  }
  const int parity = (int)(epoch & 1u);
  DR_CUDA_CHECK(cudaMemsetAsync(m->d_counters, 0, 16, side));
  k_tier_publish<<<grid_of(n), 256, 0, side>>>(keys, n, reinterpret_cast<int64_t*>(ids->ptr[rank]) + (int64_t)parity * n, *flags, m->d_counters + 2, epoch, W, rank);
  k_tier_wait<<<1, 32, 0, side>>>(*flags, epoch, W, rank);
  if (n > 0) k_tier_miss_list_mp<<<grid_of(n * W), 256, 0, side>>>(*tb, *ids, n, parity, pad_key, epoch, W, rank, m->d_miss_alias, m->d_counters, m->miss_cap);
  DR_LAUNCH_CHECK();
  DR_CUDA_CHECK(cudaMemcpyAsync(m->h_counters, m->d_counters, 16, cudaMemcpyDeviceToHost, side));
  DR_CUDA_CHECK(cudaEventRecord(m->ev_miss, side));
  { std::lock_guard<std::mutex> l(m->mu); m->q.push_back(0); }
  m->cv.notify_all();
  return 0;
}

// Step boundary: make the prefetched batch resident (waits for the background thread's staging, then enqueues H2D + import + pin on
// `main`).  Returns the number of rows promoted, or < 0 on error.
int64_t dr_tier_commit(void* h, const DrDeviceTable* tb, uint32_t epoch, cudaStream_t main) {
  auto* m = static_cast<TierManager*>(h);
  int64_t n;
  {
    std::unique_lock<std::mutex> l(m->mu);
    if (!m->prefetch_inflight && !m->prefetch_ready) return 0;
    m->cv.wait(l, [&] { return m->prefetch_ready; });
    n = m->n_import; m->prefetch_ready = false;
  }
  if (n < 0) { fprintf(stderr, "[deeprec_cuda] dr_tier_commit: the miss list of the prefetched batch overflowed (max_batch_keys = %lld): raise it\n", (long long)m->miss_cap); return n; }
  if (n > 0) {
    if (cudaMemcpyAsync(m->d_imp_keys, m->h_imp_keys, (size_t)n * 8, cudaMemcpyHostToDevice, main) != cudaSuccess) return -1;
    cudaMemcpyAsync(m->d_imp_freq, m->h_imp_freq, (size_t)n * 8, cudaMemcpyHostToDevice, main);
    cudaMemcpyAsync(m->d_imp_ver, m->h_imp_ver, (size_t)n * 8, cudaMemcpyHostToDevice, main);
    cudaMemcpyAsync(m->d_imp_rows, m->h_imp_rows, (size_t)n * m->stride * 4, cudaMemcpyHostToDevice, main);
    cudaEventRecord(m->ev_imp_copied, main); m->imp_copy_pending = true;
    extern int dr_cuda_table_import(const DrDeviceTable*, const int64_t*, const float*, int, const int64_t*, const int64_t*, int64_t, int, int, int, int32_t*, cudaStream_t);
    if (dr_cuda_table_import(tb, m->d_imp_keys, m->d_imp_rows, m->stride, m->d_imp_freq, m->d_imp_ver, n, 0, 1, 0, m->d_kept, main) != 0) return -2;
    k_tier_pin<<<grid_of(n), 256, 0, main>>>(*tb, m->d_imp_keys, n, epoch);
    m->promoted += n; m->h2d_bytes += n * ((int64_t)m->stride * 4 + 24);
  }
  return n;
}

// Step boundary: free `need` rows of the HBM tier (rows pinned for epoch >= epoch_min are kept).  strategy 0 = LFU, 1 = LRU.
int dr_tier_evict(void* h, const DrDeviceTable* tb, int32_t need, uint32_t epoch_min, int64_t step, int strategy, cudaStream_t main) {
  auto* m = static_cast<TierManager*>(h);
  if (need <= 0) return 0;
  if (need > m->evict_cap) need = (int32_t)m->evict_cap;
  {
    std::unique_lock<std::mutex> l(m->mu);
    m->cv.wait(l, [&] { return !m->evict_inflight; });              // the previous batch of victims has been committed to the DRAM tier
    m->evict_inflight = true;
  }
  DR_CUDA_CHECK(cudaMemsetAsync(m->d_hist, 0, 64 * 4, main));
  const int g = grid_of(tb->capacity);
  k_tier_hist<<<g, 256, 0, main>>>(*tb, strategy, step, epoch_min, m->d_hist);
  k_tier_threshold<<<1, 1, 0, main>>>(m->d_hist, need, m->d_ctl);
  k_tier_evict<<<g, 256, 0, main>>>(*tb, strategy, step, epoch_min, m->d_ctl, (int32_t)m->evict_cap, m->d_ev_keys, m->d_ev_rows, m->d_ev_freq, m->d_ev_ver);
  DR_LAUNCH_CHECK();
  DR_CUDA_CHECK(cudaMemcpyAsync(m->h_ctl, m->d_ctl, 16, cudaMemcpyDeviceToHost, main));
  // the victim count is only known on the device: copy the requested upper bound (need <= evict_cap rows)
  DR_CUDA_CHECK(cudaMemcpyAsync(m->h_ev_keys, m->d_ev_keys, (size_t)need * 8, cudaMemcpyDeviceToHost, main));
  DR_CUDA_CHECK(cudaMemcpyAsync(m->h_ev_freq, m->d_ev_freq, (size_t)need * 8, cudaMemcpyDeviceToHost, main));
  DR_CUDA_CHECK(cudaMemcpyAsync(m->h_ev_ver, m->d_ev_ver, (size_t)need * 8, cudaMemcpyDeviceToHost, main));
  DR_CUDA_CHECK(cudaMemcpyAsync(m->h_ev_rows, m->d_ev_rows, (size_t)need * m->stride * 4, cudaMemcpyDeviceToHost, main));
  DR_CUDA_CHECK(cudaEventRecord(m->ev_evict, main));
  m->evict_passes++;
  { std::lock_guard<std::mutex> l(m->mu); m->q.push_back(1); }
  m->cv.notify_all();
  return 0;
}

// Block until every queued job (prefetch staging, eviction commit) has been processed by the background thread.
void dr_tier_drain(void* h) {
  auto* m = static_cast<TierManager*>(h);
  std::unique_lock<std::mutex> l(m->mu);
  m->cv.wait(l, [&] { return m->q.empty() && !m->evict_inflight && !m->prefetch_inflight; });
}

void dr_tier_stats(void* h, int64_t* out /* [8] */) {
  auto* m = static_cast<TierManager*>(h);
  out[0] = m->hits; out[1] = m->misses; out[2] = m->promoted; out[3] = m->demoted; out[4] = m->h2d_bytes; out[5] = m->d2h_bytes; out[6] = m->evict_passes; out[7] = 0;
}

}  // extern "C"
