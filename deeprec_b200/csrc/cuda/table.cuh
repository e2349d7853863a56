// Device-resident EmbeddingVariable: open-addressing key table + SoA metadata + slab row store.
//
// Replaces (behaviourally) the reference's GPUHashTable / GPUHashMapKV built on cuco::dynamic_map
// (framework/embedding/gpu_hash_table.{h,cu.cc}, gpu_hash_map_kv.h) and its bank allocator.
// Differences by design:
//   * no host synchronisation on insert/growth (reference: cudaDeviceSynchronize per submap,
//     gpu_hash_table.cu.cc:485): capacity is pre-sized, growth is a device-side rehash at a step
//     boundary triggered from a lazily-read counter;
//   * admission (counter / counting-Bloom), frequency, version and the dedup "claim" are fused
//     into the find-or-insert kernel; rows are allocated lazily at apply time (only admitted keys
//     own a row), mirroring counter_filter_policy.h:106-139.
#pragma once
#include "common.cuh"

extern "C" {
// One hash-table slot = ONE 32-byte DRAM sector: the probe that finds the key has also fetched every piece of metadata the
// lookup / claim / apply kernels need (an SoA layout costs 4-5 random sectors per key).
struct __align__(32) DrSlot {
  int64_t key;             // kEmptyKey / kTombKey / key
  int32_t freq;
  int32_t version;         // global step of last update, -1 = never
  int32_t row_of;          // row index, -1 = not admitted yet
  int32_t tag;             // per-step unique index (dedup claim), -1 = unclaimed
  uint32_t dirty;          // touched since last (incremental) checkpoint
  uint32_t pad;
};
// Mirrored by ctypes (deeprec_b200/_cuda_sigs.py::DeviceTableStruct) -- keep in sync.
struct DrDeviceTable {
  DrSlot* slots;           // [capacity]
  float* rows;             // [row_capacity, stride]
  int32_t* free_list;      // [row_capacity]
  int32_t* counters;       // [8]: 0 next_row, 1 free_top, 2 n_keys, 3 n_admitted, 4 overflow, 5 n_unique, 6 n_miss, 7 spare
  const float* default_matrix;  // [default_value_dim, dim]
  uint32_t* bloom;         // [bloom_m] counting-Bloom counters (or null)
  int64_t capacity;        // power of two
  int64_t row_capacity;
  int64_t default_value_dim;
  int64_t bloom_m;
  int32_t dim;
  int32_t stride;
  int32_t num_slots;
  int32_t has_scalars;
  int32_t filter_type;
  int32_t filter_freq;
  int32_t bloom_k;
  int32_t is_inference;
  float no_permission;
  float slot_init[4];
  int32_t steps_to_live;
  float l2_weight_threshold;
};
}

namespace drc {

enum { CTR_NEXT_ROW = 0, CTR_FREE_TOP = 1, CTR_NKEYS = 2, CTR_NADMITTED = 3, CTR_OVERFLOW = 4, CTR_NUNIQUE = 5, CTR_NMISS = 6 };

__device__ __forceinline__ int64_t table_find(const DrDeviceTable& T, int64_t key) {
  const uint64_t mask = (uint64_t)T.capacity - 1;
  uint64_t pos = dr_mix64((uint64_t)key) & mask;
  for (int64_t probes = 0; probes < T.capacity; ++probes, pos = (pos + 1) & mask) {
    int64_t k = T.slots[pos].key;
    if (k == key) return (int64_t)pos;
    if (k == kEmptyKey) return -1;
  }
  return -1;
}

// find or CAS-insert; returns position or -1 if the table is full.  *inserted set for the winner.
__device__ __forceinline__ int64_t table_find_or_insert(const DrDeviceTable& T, int64_t key, bool* inserted) {
  const uint64_t mask = (uint64_t)T.capacity - 1;
  uint64_t pos = dr_mix64((uint64_t)key) & mask;
  *inserted = false;
  for (int64_t probes = 0; probes < T.capacity; ++probes) {
    int64_t k = ld_volatile_i64(&T.slots[pos].key);
    if (k == key) return (int64_t)pos;
    if (k == kEmptyKey) {
      unsigned long long old = atomicCAS((unsigned long long*)&T.slots[pos].key, (unsigned long long)kEmptyKey, (unsigned long long)key);
      if ((int64_t)old == kEmptyKey) { *inserted = true; return (int64_t)pos; }
      if ((int64_t)old == key) return (int64_t)pos;
      // another key took the slot: fall through to the next position
    }
    pos = (pos + 1) & mask;
  }
  return -1;
}

__device__ __forceinline__ uint32_t bloom_add_min(const DrDeviceTable& T, int64_t key, uint32_t count) {
  uint32_t mn = 0xFFFFFFFFu;
  for (int i = 0; i < T.bloom_k; ++i) {
    uint64_t idx = dr_hash_seed((uint64_t)key, (uint64_t)i) % (uint64_t)T.bloom_m;
    uint32_t v = atomicAdd(&T.bloom[idx], count) + count;
    mn = min(mn, v);
  }
  return mn;
}
__device__ __forceinline__ uint32_t bloom_min(const DrDeviceTable& T, int64_t key) {
  uint32_t mn = 0xFFFFFFFFu;
  for (int i = 0; i < T.bloom_k; ++i) {
    uint64_t idx = dr_hash_seed((uint64_t)key, (uint64_t)i) % (uint64_t)T.bloom_m;
    mn = min(mn, T.bloom[idx]);
  }
  return mn;
}

// Row allocation (called by one lane per unique key in the apply kernel).
__device__ __forceinline__ int32_t table_alloc_row(const DrDeviceTable& T) {
  int32_t top = atomicSub(&T.counters[CTR_FREE_TOP], 1);
  if (top > 0) return T.free_list[top - 1];
  atomicAdd(&T.counters[CTR_FREE_TOP], 1);
  int32_t r = atomicAdd(&T.counters[CTR_NEXT_ROW], 1);
  if ((int64_t)r >= T.row_capacity) { T.counters[CTR_OVERFLOW] = 1; return -1; }
  return r;
}

// What a forward read returns for position `pos` (or absent key): pointer to a row of `dim` floats,
// or nullptr meaning "fill with no_permission".
__device__ __forceinline__ const float* table_read_ptr(const DrDeviceTable& T, int64_t key, int64_t pos) {
  int32_t r = pos >= 0 ? T.slots[pos].row_of : -1;
  if (r >= 0) return T.rows + (int64_t)r * T.stride;
  if (T.filter_type != DR_FILTER_NONE && T.filter_freq > 0) return nullptr;
  return T.default_matrix + dr_default_row(key, T.default_value_dim) * T.dim;
}


// ---- training-side bookkeeping of one probe result, aggregated over the warp -------------------------------------
// All 32 lanes call this (valid = lane has a live key at `pos` of table TB; every valid lane of a warp addresses the
// SAME table).  Lanes holding the same position elect a leader that performs ONE freq += count, the dirty mark and the
// per-step dedup claim: hot keys of tiny tables would otherwise serialise tens of thousands of same-address atomics.
__device__ __forceinline__ void table_touch_aggregated(const DrDeviceTable& TB, bool valid, int64_t pos, int table_index, int64_t* ulist,
                                                       int32_t* nunique, int64_t ulist_cap) {
  const unsigned lane = threadIdx.x & 31;
  // lanes of a warp may straddle two tables when a segment boundary is not 32-aligned: the table is part of the match key
  const int64_t mkey = valid ? (((int64_t)table_index << 40) | pos) : -(int64_t)(lane + 1);            // invalid lanes match nobody
  const unsigned same = __match_any_sync(0xffffffffu, mkey);
  if (!valid) return;
  if ((unsigned)(__ffs(same) - 1) != lane) return;                    // not the leader of this position
  atomicAdd(&TB.slots[pos].freq, __popc(same));
  // read-before-write: a hot key's slot is hammered by every warp of the batch; once it is dirty / claimed, later warps
  // must not add a store and a CAS to the same-sector serialisation queue (the probe already pulled the sector in)
  int4 hi;                                                                             // {row_of, tag, dirty, pad}
  DR_LD_V4_VOLATILE(hi, &TB.slots[pos].row_of);
  if (hi.z == 0) DR_ST_RACY(TB.slots[pos].dirty, 1u);
  if (ulist != nullptr && hi.y == -1 && atomicCAS(&TB.slots[pos].tag, -1, -2) == -1) {
    const int u = atomicAdd(nunique, 1);
    if (u < ulist_cap) { ulist[u] = ((int64_t)table_index << 40) | pos; DR_ST_RACY(TB.slots[pos].tag, u); }
    else { DR_ST_RACY(TB.slots[pos].tag, -1); DR_ST_RACY(TB.counters[CTR_OVERFLOW], 2); }
  }
}

// ---- block-aggregated variant ---------------------------------------------------------------------------------------
// Same bookkeeping, aggregated over the whole 256-thread block through a small shared-memory hash: warp leaders (one per
// distinct position in the warp) deposit (table, pos) -> count; after a barrier each shared entry performs ONE global
// freq += count / dirty / claim.  A hot key (power-law ids, tiny tables) costs one global atomic per block iteration instead
// of one per warp -- same-address L2 atomics serialise at ~14 ns each, which is what bounds the probe kernels on skewed data.
// Every thread of the block must call it (it synchronises); invalid lanes pass valid = false.
constexpr int kTouchSlots = 512;
struct TouchSmem { unsigned long long key[kTouchSlots]; int32_t count[kTouchSlots]; };

__device__ __forceinline__ void table_touch_block(const DrDeviceTable* __restrict__ tables, bool valid, int64_t pos, int table_index, int64_t* ulist,
                                                  int32_t* nunique, int64_t ulist_cap, TouchSmem& sm) {
  constexpr unsigned long long kNone = ~0ull;
  for (int e = threadIdx.x; e < kTouchSlots; e += blockDim.x) { sm.key[e] = kNone; sm.count[e] = 0; }
  __syncthreads();
  const unsigned lane = threadIdx.x & 31;
  const int64_t mkey = valid ? (((int64_t)table_index << 40) | pos) : -(int64_t)(lane + 1);
  const unsigned same = __match_any_sync(0xffffffffu, mkey);
  if (valid && (unsigned)(__ffs(same) - 1) == lane) {
    uint32_t h = (uint32_t)(dr_mix64((uint64_t)mkey) >> 40) & (kTouchSlots - 1);
    for (int probe = 0; probe < kTouchSlots; ++probe, h = (h + 1) & (kTouchSlots - 1)) {
      const unsigned long long old = atomicCAS(&sm.key[h], kNone, (unsigned long long)mkey);
      if (old == kNone || old == (unsigned long long)mkey) { atomicAdd(&sm.count[h], __popc(same)); break; }
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < kTouchSlots; e += blockDim.x) {
    const unsigned long long k = sm.key[e];
    if (k == kNone) continue;
    const int t = (int)(k >> 40);
    const int64_t p = (int64_t)(k & ((1ull << 40) - 1));
    const DrDeviceTable& TB = tables[t];
    atomicAdd(&TB.slots[p].freq, sm.count[e]);
    int4 hi;                                                                            // {row_of, tag, dirty, pad}
    DR_LD_V4_VOLATILE(hi, &TB.slots[p].row_of);
    if (hi.z == 0) DR_ST_RACY(TB.slots[p].dirty, 1u);
    if (ulist != nullptr && hi.y == -1 && atomicCAS(&TB.slots[p].tag, -1, -2) == -1) {
      const int u = atomicAdd(nunique, 1);
      if (u < ulist_cap) { ulist[u] = (int64_t)k; DR_ST_RACY(TB.slots[p].tag, u); }
      else { DR_ST_RACY(TB.slots[p].tag, -1); DR_ST_RACY(TB.counters[CTR_OVERFLOW], 2); }
    }
  }
  __syncthreads();
}

// ---- per-block combining cache for gradient accumulation ----------------------------------------------------------------
// Direct-mapped on the unique index u: s_tag[C] (init -1), s_acc[C * dim] (init 0).  A group of LPR lanes adds its float4
// chunks either into the cached row (shared-memory atomics) or, on a slot conflict, straight into gsum with red.global.
// flush_combining_cache() pushes every cached row with ONE vectorised global reduction per chunk.
template <int LPR>
__device__ __forceinline__ void combine_add(int32_t* s_tag, float* s_acc, int C, int dim, int32_t u, int lane, unsigned gmask, int gleader,
                                            const float4* chunks, int nchunks_per_lane, float* __restrict__ gsum) {
  int hit = 0;
  const int slot = u & (C - 1);
  if (C > 0) {      // C == 0: caller decided this table is too large for combining to pay off -> straight to L2 reductions
    if (lane == 0) { const int32_t old = atomicCAS(&s_tag[slot], -1, u); hit = (old == -1 || old == u); }
    hit = __shfl_sync(gmask, hit, gleader);
  }
  const int nvec = dim >> 2;
#pragma unroll 4
  for (int k = 0; k < nchunks_per_lane; ++k) {
    const int c = lane + k * LPR;
    if (c >= nvec) break;
    const float4 g = chunks[k];
    if (hit) {
      float* d = s_acc + (int64_t)slot * dim + 4 * c;
      atomicAdd(d, g.x); atomicAdd(d + 1, g.y); atomicAdd(d + 2, g.z); atomicAdd(d + 3, g.w);
    } else {
      red_add_v4_f32(gsum + (int64_t)u * dim + 4 * c, g.x, g.y, g.z, g.w);
    }
  }
}
__device__ __forceinline__ void flush_combining_cache(const int32_t* s_tag, const float* s_acc, int C, int dim, float* __restrict__ gsum) {
  const int nvec = dim >> 2;
  for (int e = threadIdx.x; e < C * nvec; e += blockDim.x) {
    const int slot = e / nvec, c = e % nvec;
    const int32_t u = s_tag[slot];
    if (u >= 0) {
      const float* s = s_acc + (int64_t)slot * dim + 4 * c;
      red_add_v4_f32(gsum + (int64_t)u * dim + 4 * c, s[0], s[1], s[2], s[3]);
    }
  }
}
inline int combining_cache_slots(int dim) { int c = 512; while (c > 16 && (int64_t)c * dim * 4 > 32768) c >>= 1; return c; }

}  // namespace drc
