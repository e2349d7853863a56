// sm_90a kernels for the device EmbeddingVariable: fused find-or-insert (+admission, frequency,
// version, dedup claim), row gather, metadata queries, rehash, eviction scan, snapshot, import.
//
// Reference kernels replaced: K1-K5 of SURVEY §2.14 (gpu_hash_table.cu.cc:187-658).

#include "table.cuh"

using namespace drc;

namespace {

__device__ __forceinline__ int seg_of(const int64_t* offsets, int T, int64_t i, int64_t uniform) {
  if (offsets == nullptr) return (int)(i / uniform);
  int lo = 0, hi = T;                  // largest t with offsets[t] <= i
  while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (offsets[mid] <= i) lo = mid; else hi = mid; }
  return lo;
}

// -----------------------------------------------------------------------------------------------
// K_lookup: one thread per key.  train=1: insert-if-absent (subject to Bloom admission), freq += 1,
// version = step, dirty = 1 and claim a per-step unique index for the backward dedup.
// train=0: read-only probe (inference / eval; INFERENCE_MODE never creates).
// out_pos[i] = table position or -1.
// -----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_lookup(const DrDeviceTable* __restrict__ tables, const int32_t* __restrict__ table_map, int T,
                                                const int64_t* __restrict__ keys, const int64_t* __restrict__ offsets,
                                                int64_t uniform, int64_t n, int train, const int64_t* __restrict__ step_ptr,
                                                int32_t* __restrict__ out_pos, int64_t* __restrict__ ulist,
                                                int32_t* __restrict__ group_nunique, int64_t ulist_cap) {
  pdl_sync();
  (void)step_ptr;
  __shared__ TouchSmem s_touch;
  // whole blocks iterate together (n rounded up to the block size): the training bookkeeping is aggregated over the block
  const int64_t nb = train ? (n + blockDim.x - 1) / blockDim.x * blockDim.x : n;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nb; i += (int64_t)gridDim.x * blockDim.x) {
    const bool live = i < n;
    const int64_t ii = live ? i : n - 1;
    const int tl = seg_of(offsets, T, ii, uniform);
    const int t = table_map ? table_map[tl] : tl;      // index into the context-wide table array
    const DrDeviceTable& TB = tables[t];
    const int64_t key = keys[ii];
    int64_t pos = -1;
    bool touch = false;
    if (live) {
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
      out_pos[i] = (int32_t)pos;
    }
    if (train) table_touch_block(tables, touch, pos, t, ulist, group_nunique, ulist_cap, s_touch);
  }
}

// -----------------------------------------------------------------------------------------------
// K_gather: LPR lanes per row (float4 per lane).  out element (b, t) at out + b*stride_b + t*stride_t.
// -----------------------------------------------------------------------------------------------
template <int LPR, bool BF16>
__global__ void __launch_bounds__(256) k_gather(const DrDeviceTable* __restrict__ tables, const int32_t* __restrict__ table_map, int T,
                                                const int64_t* __restrict__ keys, const int32_t* __restrict__ pos,
                                                const int64_t* __restrict__ offsets, int64_t uniform, int64_t n,
                                                void* __restrict__ out, int64_t stride_b, int64_t stride_t, int flat_out) {
  pdl_sync();
  const int lane = threadIdx.x % LPR;
  const int64_t gid = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / LPR;
  const int64_t gstride = (int64_t)gridDim.x * blockDim.x / LPR;
  for (int64_t i = gid; i < n; i += gstride) {
    const int t = seg_of(offsets, T, i, uniform);
    const DrDeviceTable& TB = tables[table_map ? table_map[t] : t];
    const float* src = table_read_ptr(TB, keys[i], pos[i]);
    int64_t o;
    if (flat_out) o = i * TB.dim;
    else { int64_t b = offsets ? i - offsets[t] : i % uniform; o = b * stride_b + (int64_t)t * stride_t; }
    const int nvec = TB.dim >> 2;
    for (int c = lane; c < nvec; c += LPR) {
      float4 v = src ? *reinterpret_cast<const float4*>(src + 4 * c)
                     : make_float4(TB.no_permission, TB.no_permission, TB.no_permission, TB.no_permission);
      if (BF16) {
        uint2 p = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
        *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(out) + o + 4 * c) = p;
      } else {
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + o + 4 * c) = v;
      }
    }
  }
}

__global__ void k_get_meta(DrDeviceTable TB, const int64_t* __restrict__ keys, int64_t n, int64_t* __restrict__ freq,
                           int64_t* __restrict__ version, int32_t* __restrict__ row) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t pos = table_find(TB, keys[i]);
    if (freq) freq[i] = pos >= 0 ? TB.slots[pos].freq : (TB.bloom ? (int64_t)bloom_min(TB, keys[i]) : 0);
    if (version) version[i] = pos >= 0 ? TB.slots[pos].version : -1;
    if (row) row[i] = pos >= 0 ? TB.slots[pos].row_of : -1;
  }
}

// gather one slot (0 = embedding) of the rows of `keys` (inspection / tests)
__global__ void k_gather_slot(DrDeviceTable TB, const int64_t* __restrict__ keys, int64_t n, int slot, float* __restrict__ out) {
  int64_t total = n * TB.dim;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    int64_t i = e / TB.dim; int d = (int)(e % TB.dim);
    int64_t pos = table_find(TB, keys[i]);
    int32_t r = pos >= 0 ? TB.slots[pos].row_of : -1;
    out[e] = r >= 0 ? TB.rows[(int64_t)r * TB.stride + slot * TB.dim + d] : (slot == 0 ? 0.f : TB.slot_init[slot - 1]);
  }
}

// -----------------------------------------------------------------------------------------------
// Rehash old -> new (growth, or tombstone purge after eviction).  Metadata moves with the key.
// -----------------------------------------------------------------------------------------------
__global__ void k_rehash(DrDeviceTable OLD, DrDeviceTable NEW) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < OLD.capacity; p += (int64_t)gridDim.x * blockDim.x) {
    int64_t key = OLD.slots[p].key;
    if (key == kEmptyKey || key == kTombKey) continue;
    bool ins;
    int64_t q = table_find_or_insert(NEW, key, &ins);
    if (q < 0) { NEW.counters[CTR_OVERFLOW] = 1; continue; }
    NEW.slots[q].freq = OLD.slots[p].freq; NEW.slots[q].version = OLD.slots[p].version; NEW.slots[q].row_of = OLD.slots[p].row_of;
    NEW.slots[q].dirty = OLD.slots[p].dirty; NEW.slots[q].tag = -1;
  }
}

// -----------------------------------------------------------------------------------------------
// Eviction scan (runs inside save, single_tier_storage.h:235-261): GlobalStep and/or L2 policy.
// Evicted keys become tombstones, their rows go back to the free list.
// -----------------------------------------------------------------------------------------------
__global__ void k_shrink(DrDeviceTable TB, int step, int32_t* __restrict__ n_evicted) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < TB.capacity; p += (int64_t)gridDim.x * blockDim.x) {
    int64_t key = TB.slots[p].key;
    if (key == kEmptyKey || key == kTombKey) continue;
    bool evict = false;
    int32_t r = TB.slots[p].row_of;
    if (TB.steps_to_live > 0) {
      int32_t v = TB.slots[p].version;
      if (v == -1) TB.slots[p].version = step;
      else if (step - v > TB.steps_to_live) evict = true;
    }
    if (!evict && TB.l2_weight_threshold >= 0.f && r >= 0) {
      const float* row = TB.rows + (int64_t)r * TB.stride; float s = 0.f;
      for (int d = 0; d < TB.dim; ++d) s += row[d] * row[d];
      if (0.5f * s < TB.l2_weight_threshold) evict = true;
    }
    if (evict) {
      TB.slots[p].key = kTombKey;
      if (r >= 0) {
        int32_t top = atomicAdd(&TB.counters[CTR_FREE_TOP], 1);
        TB.free_list[top] = r;
        atomicSub(&TB.counters[CTR_NADMITTED], 1);
      }
      TB.slots[p].row_of = -1; TB.slots[p].freq = 0; TB.slots[p].version = -1; TB.slots[p].dirty = 0; TB.slots[p].tag = -1;
      atomicSub(&TB.counters[CTR_NKEYS], 1);
      atomicAdd(n_evicted, 1);
    }
  }
}

// Copy-on-write import (serving delta update under live requests, model_instance.cc:429-446): the new row is written to a FRESH slab
// row and published with one atomic exchange of slot.row_of -- a concurrent reader (k_lookup + k_gather of a session's stream) sees
// the old row or the new row, never a torn one.  The replaced rows are returned through `retired` and recycled by the caller once
// every session has passed a quiescent point.
__global__ void k_import_cow(DrDeviceTable TB, const int64_t* __restrict__ keys, const float* __restrict__ rows, int ncols, int64_t n,
                             int32_t* __restrict__ retired, int32_t* __restrict__ n_retired, int32_t* __restrict__ n_kept) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t key = keys[i];
    bool ins;
    const int64_t p = table_find_or_insert(TB, key, &ins);
    if (p < 0) { TB.counters[CTR_OVERFLOW] = 1; continue; }
    if (ins) atomicAdd(&TB.counters[CTR_NKEYS], 1);
    const int32_t r_new = table_alloc_row(TB);
    if (r_new < 0) continue;
    const int32_t r_old = TB.slots[p].row_of;
    float* row = TB.rows + (int64_t)r_new * TB.stride;
    if (r_old >= 0) { const float* o = TB.rows + (int64_t)r_old * TB.stride; for (int d = 0; d < TB.stride; ++d) row[d] = o[d]; }
    else {
      const float* def = TB.default_matrix + dr_default_row(key, TB.default_value_dim) * TB.dim;
      for (int d = 0; d < TB.dim; ++d) row[d] = def[d];
      for (int d = TB.dim; d < TB.stride; ++d) row[d] = 0.f;
    }
    const float* src = rows + (int64_t)i * ncols;
    const int m = ncols < TB.stride ? ncols : TB.stride;
    for (int d = 0; d < m; ++d) row[d] = src[d];
    __threadfence();                                            // the row is complete before it becomes reachable
    const int32_t prev = atomicExch(&TB.slots[p].row_of, r_new);
    if (prev >= 0) retired[atomicAdd(n_retired, 1)] = prev; else atomicAdd(&TB.counters[CTR_NADMITTED], 1);
    atomicAdd(n_kept, 1);
  }
}
__global__ void k_free_rows(DrDeviceTable TB, const int32_t* __restrict__ rows, const int32_t* __restrict__ n_ptr) {
  const int n = *n_ptr;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int32_t top = atomicAdd(&TB.counters[CTR_FREE_TOP], 1);
    TB.free_list[top] = rows[i];
  }
}

__global__ void k_remove(DrDeviceTable TB, const int64_t* __restrict__ keys, int64_t n, int32_t* __restrict__ n_removed) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t p = table_find(TB, keys[i]);
    if (p < 0) continue;
    unsigned long long old = atomicCAS((unsigned long long*)&TB.slots[p].key, (unsigned long long)keys[i], (unsigned long long)kTombKey);
    if ((int64_t)old != keys[i]) continue;
    int32_t r = TB.slots[p].row_of;
    if (r >= 0) { int32_t top = atomicAdd(&TB.counters[CTR_FREE_TOP], 1); TB.free_list[top] = r; atomicSub(&TB.counters[CTR_NADMITTED], 1); }
    TB.slots[p].row_of = -1; TB.slots[p].freq = 0; TB.slots[p].version = -1; TB.slots[p].dirty = 0; TB.slots[p].tag = -1;
    atomicSub(&TB.counters[CTR_NKEYS], 1);
    atomicAdd(n_removed, 1);
  }
}

// -----------------------------------------------------------------------------------------------
// Snapshot (K5 analogue): compacts admitted keys (with full rows) and filtered keys.
// counts[0] admitted, counts[1] filtered.  Pass null outputs to only count.
// -----------------------------------------------------------------------------------------------
__global__ void k_snapshot(DrDeviceTable TB, int dirty_only, int part_id, int part_num, int32_t* __restrict__ counts,
                           int64_t* __restrict__ keys, float* __restrict__ rows, int64_t* __restrict__ freqs,
                           int64_t* __restrict__ versions, int64_t* __restrict__ fkeys, int64_t* __restrict__ ffreqs,
                           int64_t* __restrict__ fversions) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < TB.capacity; p += (int64_t)gridDim.x * blockDim.x) {
    int64_t key = TB.slots[p].key;
    if (key == kEmptyKey || key == kTombKey) continue;
    if (part_num > 1 && dr_ckpt_bucket(key) % part_num != part_id) continue;
    if (dirty_only && !TB.slots[p].dirty) continue;
    int32_t r = TB.slots[p].row_of;
    if (r >= 0) {
      int32_t o = atomicAdd(&counts[0], 1);
      if (keys) {
        keys[o] = key; freqs[o] = TB.slots[p].freq; versions[o] = TB.slots[p].version;
        const float* src = TB.rows + (int64_t)r * TB.stride; float* dst = rows + (int64_t)o * TB.stride;
        for (int d = 0; d < TB.stride; ++d) dst[d] = src[d];
      }
    } else {
      int32_t o = atomicAdd(&counts[1], 1);
      if (fkeys) { fkeys[o] = key; ffreqs[o] = TB.slots[p].freq; fversions[o] = TB.slots[p].version; }
    }
  }
}

// Snapshot of the admitted keys whose version (the global step of their last update, written by k_apply) is >= min_version: the rows a
// serving delta needs, selected without reading or clearing the dirty bits that incremental checkpoints consume.  counts[0] = rows.
__global__ void k_snapshot_since(DrDeviceTable TB, int64_t min_version, int32_t* __restrict__ counts, int64_t* __restrict__ keys, float* __restrict__ rows,
                                 int64_t* __restrict__ freqs, int64_t* __restrict__ versions) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < TB.capacity; p += (int64_t)gridDim.x * blockDim.x) {
    const int64_t key = TB.slots[p].key;
    if (key == kEmptyKey || key == kTombKey) continue;
    const int32_t r = TB.slots[p].row_of, v = TB.slots[p].version;
    if (r < 0 || (int64_t)v < min_version) continue;
    const int32_t o = atomicAdd(&counts[0], 1);
    if (keys) {
      keys[o] = key; freqs[o] = TB.slots[p].freq; versions[o] = v;
      const float* src = TB.rows + (int64_t)r * TB.stride; float* dst = rows + (int64_t)o * TB.stride;
      for (int d = 0; d < TB.stride; ++d) dst[d] = src[d];
    }
  }
}

// rows (full stride) + metadata of specific keys (multi-tier demotion / promotion); found[i] = key owns a row
__global__ void k_export_keys(DrDeviceTable TB, const int64_t* __restrict__ keys, int64_t n, float* __restrict__ rows, int64_t* __restrict__ freqs,
                              int64_t* __restrict__ versions, uint8_t* __restrict__ found) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t p = table_find(TB, keys[i]);
    int32_t r = p >= 0 ? TB.slots[p].row_of : -1;
    found[i] = r >= 0;
    freqs[i] = p >= 0 ? TB.slots[p].freq : 0;
    versions[i] = p >= 0 ? TB.slots[p].version : -1;
    if (r >= 0) { const float* src = TB.rows + (int64_t)r * TB.stride; float* dst = rows + i * TB.stride; for (int d = 0; d < TB.stride; ++d) dst[d] = src[d]; }
  }
}

__global__ void k_clear_dirty(DrDeviceTable TB) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < TB.capacity; p += (int64_t)gridDim.x * blockDim.x) TB.slots[p].dirty = 0;
}

// Import rows (restore / elastic import / incremental replay).  rows == null imports filtered keys.
__global__ void k_import(DrDeviceTable TB, const int64_t* __restrict__ keys, const float* __restrict__ rows, int ncols,
                         const int64_t* __restrict__ freqs, const int64_t* __restrict__ versions, int64_t n,
                         int part_id, int part_num, int reset_version, int32_t* __restrict__ n_kept) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t key = keys[i];
    if (part_num > 1 && dr_ckpt_bucket(key) % part_num != part_id) continue;
    bool ins;
    int64_t p = table_find_or_insert(TB, key, &ins);
    if (p < 0) { TB.counters[CTR_OVERFLOW] = 1; continue; }
    if (ins) atomicAdd(&TB.counters[CTR_NKEYS], 1);
    TB.slots[p].freq = freqs ? (int32_t)min(freqs[i], (int64_t)INT32_MAX) : 0;
    TB.slots[p].version = reset_version ? -1 : (versions ? (int32_t)versions[i] : -1);
    if (rows) {
      int32_t r = TB.slots[p].row_of;
      if (r < 0) {
        r = table_alloc_row(TB);
        if (r < 0) continue;
        TB.slots[p].row_of = r; atomicAdd(&TB.counters[CTR_NADMITTED], 1);
        float* row = TB.rows + (int64_t)r * TB.stride;
        const float* def = TB.default_matrix + dr_default_row(key, TB.default_value_dim) * TB.dim;
        for (int d = 0; d < TB.dim; ++d) row[d] = def[d];
        for (int s = 0; s < TB.num_slots; ++s) for (int d = 0; d < TB.dim; ++d) row[(1 + s) * TB.dim + d] = TB.slot_init[s];
        for (int d = TB.dim * (1 + TB.num_slots); d < TB.stride; ++d) row[d] = 0.f;
      }
      float* row = TB.rows + (int64_t)r * TB.stride;
      const float* src = rows + (int64_t)i * ncols;
      int m = ncols < TB.stride ? ncols : TB.stride;
      for (int d = 0; d < m; ++d) row[d] = src[d];
    }
    atomicAdd(n_kept, 1);
  }
}

// empty slot = {kEmptyKey, freq 0, version -1, row_of -1, tag -1, dirty 0}: two 16 B stores per slot
__global__ void k_init_slots(DrSlot* slots, int64_t n) {
  const int4 lo = make_int4((int)(uint32_t)((uint64_t)kEmptyKey & 0xffffffffu), (int)(uint32_t)((uint64_t)kEmptyKey >> 32), 0, -1);
  const int4 hi = make_int4(-1, -1, 0, 0);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int4* p = reinterpret_cast<int4*>(slots + i);
    p[0] = lo; p[1] = hi;
  }
}

__global__ void k_fill_i64(int64_t* p, int64_t v, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}

inline int grid_for(int64_t n, int block, int max_blocks = 0) {
  if (max_blocks <= 0) max_blocks = num_sms() * sparse_blocks_per_sm();
  int64_t b = (n + block - 1) / block;
  if (b < 1) b = 1;
  if (b > max_blocks) b = max_blocks;
  return (int)b;
}

}  // namespace

extern "C" {

int dr_cuda_table_init_slots(void* slots, int64_t n, cudaStream_t s) {
  k_init_slots<<<grid_for(n, 256, num_sms() * 8), 256, 0, s>>>((DrSlot*)slots, n);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_fill_i64(int64_t* p, int64_t v, int64_t n, cudaStream_t s) {
  k_fill_i64<<<grid_for(n, 256), 256, 0, s>>>(p, v, n);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_table_lookup(const DrDeviceTable* tables_dev, const int32_t* table_map, int T, const int64_t* keys, const int64_t* offsets, int64_t uniform,
                         int64_t n, int train, const int64_t* step_ptr, int32_t* out_pos, int64_t* ulist, int32_t* group_nunique,
                         int64_t ulist_cap, cudaStream_t s) {
  if (n == 0) return 0;
  DR_PDL_LAUNCH((k_lookup), grid_for(n, 256), 256, 0, s, tables_dev, table_map, T, keys, offsets, uniform, n, train, step_ptr, out_pos, ulist, group_nunique, ulist_cap);
  DR_LAUNCH_CHECK();
  return 0;
}

// out_bf16: 0 fp32, 1 bf16.  dim4 = dim/4 selects lanes-per-row.
int dr_cuda_table_gather(const DrDeviceTable* tables_dev, const int32_t* table_map, int T, int dim, const int64_t* keys, const int32_t* pos,
                         const int64_t* offsets, int64_t uniform, int64_t n, void* out, int out_bf16, int64_t stride_b,
                         int64_t stride_t, int flat_out, cudaStream_t s) {
  if (n == 0) return 0;
  int nvec = dim / 4;
  int lpr = 1; while (lpr < nvec && lpr < 32) lpr <<= 1;
  int grid = grid_for(n * lpr, 256);
#define LAUNCH(L)                                                                                                      \
  if (out_bf16) DR_PDL_LAUNCH((k_gather<L, true>), grid, 256, 0, s, tables_dev, table_map, T, keys, pos, offsets, uniform, n, out, stride_b, stride_t, flat_out); \
  else DR_PDL_LAUNCH((k_gather<L, false>), grid, 256, 0, s, tables_dev, table_map, T, keys, pos, offsets, uniform, n, out, stride_b, stride_t, flat_out);
  switch (lpr) {
    case 1: LAUNCH(1) break; case 2: LAUNCH(2) break; case 4: LAUNCH(4) break; case 8: LAUNCH(8) break;
    case 16: LAUNCH(16) break; default: LAUNCH(32) break;
  }
#undef LAUNCH
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_table_get_meta(const DrDeviceTable* t_host, const int64_t* keys, int64_t n, int64_t* freq, int64_t* version, int32_t* row, cudaStream_t s) {
  if (n == 0) return 0;
  k_get_meta<<<grid_for(n, 256), 256, 0, s>>>(*t_host, keys, n, freq, version, row);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_table_gather_slot(const DrDeviceTable* t_host, const int64_t* keys, int64_t n, int slot, float* out, cudaStream_t s) {
  if (n == 0) return 0;
  k_gather_slot<<<grid_for(n * t_host->dim, 256), 256, 0, s>>>(*t_host, keys, n, slot, out);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_table_rehash(const DrDeviceTable* old_host, const DrDeviceTable* new_host, cudaStream_t s) {
  k_rehash<<<grid_for(old_host->capacity, 256), 256, 0, s>>>(*old_host, *new_host);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_table_shrink(const DrDeviceTable* t_host, int step, int32_t* n_evicted, cudaStream_t s) {
  k_shrink<<<grid_for(t_host->capacity, 256), 256, 0, s>>>(*t_host, step, n_evicted);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_table_remove(const DrDeviceTable* t_host, const int64_t* keys, int64_t n, int32_t* n_removed, cudaStream_t s) {
  if (n == 0) return 0;
  k_remove<<<grid_for(n, 256), 256, 0, s>>>(*t_host, keys, n, n_removed);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_table_snapshot(const DrDeviceTable* t_host, int dirty_only, int part_id, int part_num, int32_t* counts,
                           int64_t* keys, float* rows, int64_t* freqs, int64_t* versions, int64_t* fkeys, int64_t* ffreqs,
                           int64_t* fversions, cudaStream_t s) {
  k_snapshot<<<grid_for(t_host->capacity, 256), 256, 0, s>>>(*t_host, dirty_only, part_id, part_num, counts, keys, rows, freqs,
                                                            versions, fkeys, ffreqs, fversions);
  DR_LAUNCH_CHECK();
  return 0;
}

// Pass null outputs to only count (counts[0]), then allocate and call again with counts zeroed -- as dr_cuda_table_snapshot.
int dr_cuda_table_snapshot_since(const DrDeviceTable* t_host, int64_t min_version, int32_t* counts, int64_t* keys, float* rows, int64_t* freqs,
                                 int64_t* versions, cudaStream_t s) {
  k_snapshot_since<<<grid_for(t_host->capacity, 256), 256, 0, s>>>(*t_host, min_version, counts, keys, rows, freqs, versions);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_table_export_keys(const DrDeviceTable* t_host, const int64_t* keys, int64_t n, float* rows, int64_t* freqs, int64_t* versions,
                               uint8_t* found, cudaStream_t s) {
  if (n == 0) return 0;
  k_export_keys<<<grid_for(n, 256), 256, 0, s>>>(*t_host, keys, n, rows, freqs, versions, found);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_table_clear_dirty(const DrDeviceTable* t_host, cudaStream_t s) {
  k_clear_dirty<<<grid_for(t_host->capacity, 256), 256, 0, s>>>(*t_host);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_table_import(const DrDeviceTable* t_host, const int64_t* keys, const float* rows, int ncols, const int64_t* freqs,
                         const int64_t* versions, int64_t n, int part_id, int part_num, int reset_version, int32_t* n_kept,
                         cudaStream_t s) {
  if (n == 0) return 0;
  k_import<<<grid_for(n, 256), 256, 0, s>>>(*t_host, keys, rows, ncols, freqs, versions, n, part_id, part_num, reset_version, n_kept);
  DR_LAUNCH_CHECK();
  return 0;
}

// retired: int32 [>= n] device buffer, n_retired / n_kept: device counters (zeroed by the caller)
int dr_cuda_table_import_cow(const DrDeviceTable* t_host, const int64_t* keys, const float* rows, int ncols, int64_t n, int32_t* retired,
                             int32_t* n_retired, int32_t* n_kept, cudaStream_t s) {
  if (n == 0) return 0;
  k_import_cow<<<grid_for(n, 256), 256, 0, s>>>(*t_host, keys, rows, ncols, n, retired, n_retired, n_kept);
  DR_LAUNCH_CHECK();
  return 0;
}
int dr_cuda_table_free_rows(const DrDeviceTable* t_host, const int32_t* rows, const int32_t* n_dev, int64_t max_n, cudaStream_t s) {
  if (max_n == 0) return 0;
  k_free_rows<<<grid_for(max_n, 256), 256, 0, s>>>(*t_host, rows, n_dev);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_sizeof_table() { return (int)sizeof(DrDeviceTable); }

}  // extern "C"
