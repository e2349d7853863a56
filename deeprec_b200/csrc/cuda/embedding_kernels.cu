// Fused multi-table gather + combine (GroupEmbedding / fused_embedding_lookup_sparse on device).
//
// Replaces K11-K15 of SURVEY §2.14 (kernels/group_embedding/*_base_ops.cu.h, kernels/fused_embedding/*):
// ONE launch covers every table of a group; a sub-warp of LPR lanes owns one bag (table t, sample b),
// walks its ids, reads rows straight out of the slab through the probe result and applies
// sum / mean / sqrtn with optional per-id weights.  The forward also emits the per-id backward scale
// (weight / denominator) and sample index so the backward is the same k_accumulate used by the
// one-hot path (no separate "per-nnz grad" tensor is materialised, unlike the reference's
// ComputeEVGradFn -> unsorted_segment_sum chain).
#include "table.cuh"

using namespace drc;

namespace {

template <int LPR, bool BF16>
__global__ void __launch_bounds__(256) k_combine_fwd(const DrDeviceTable* __restrict__ tables, const int32_t* __restrict__ table_map, int T, int64_t B, int dim,
                                                     const int64_t* __restrict__ keys, const int32_t* __restrict__ pos,
                                                     const int64_t* __restrict__ bag_offsets,   // [T*B + 1]
                                                     const float* __restrict__ weights,         // [nnz] or null
                                                     const int32_t* __restrict__ combiners,     // [T] 0 sum 1 mean 2 sqrtn
                                                     void* __restrict__ out, int64_t stride_b, int64_t stride_t,
                                                     float* __restrict__ nnz_scale, int32_t* __restrict__ nnz_row) {
  const int lane = threadIdx.x % LPR;
  const int64_t gid = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / LPR;
  const int64_t gstride = (int64_t)gridDim.x * blockDim.x / LPR;
  const int nvec = dim >> 2;
  const int64_t nbags = (int64_t)T * B;
  for (int64_t bag = gid; bag < nbags; bag += gstride) {
    const int t = (int)(bag / B);
    const int64_t b = bag % B;
    const DrDeviceTable& TB = tables[table_map ? table_map[t] : t];
    const int64_t j0 = bag_offsets[bag], j1 = bag_offsets[bag + 1];
    const int comb = combiners[t];
    float den = 0.f;
    for (int64_t j = j0; j < j1; ++j) {
      float w = weights ? weights[j] : 1.0f;
      den += comb == 2 ? w * w : w;
    }
    float inv = 1.0f;
    if (comb == 1) inv = den > 0.f ? 1.0f / den : 0.f;
    else if (comb == 2) inv = den > 0.f ? rsqrtf(den) : 0.f;
    // up to 4 float4 chunks per lane (dim <= 512 with LPR = 32)
    float4 acc[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int64_t j = j0; j < j1; ++j) {
      const float w = weights ? weights[j] : 1.0f;
      const float* src = table_read_ptr(TB, keys[j], pos[j]);
      if (lane == 0) { nnz_scale[j] = w * inv; nnz_row[j] = (int32_t)b; }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        int c = lane + k * LPR;
        if (c < nvec) {
          float4 v = src ? *reinterpret_cast<const float4*>(src + 4 * c)
                         : make_float4(TB.no_permission, TB.no_permission, TB.no_permission, TB.no_permission);
          acc[k].x += w * v.x; acc[k].y += w * v.y; acc[k].z += w * v.z; acc[k].w += w * v.w;
        }
      }
    }
    const int64_t o = b * stride_b + (int64_t)t * stride_t;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      int c = lane + k * LPR;
      if (c < nvec) {
        float4 v = make_float4(acc[k].x * inv, acc[k].y * inv, acc[k].z * inv, acc[k].w * inv);
        if (BF16) {
          *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(out) + o + 4 * c) = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
        } else {
          *reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + o + 4 * c) = v;
        }
      }
    }
  }
}

// Unique-with-counts for plain tensors (Variable-backed tables, host-tier miss lists): open-addressing
// scratch table keyed by value.  out_inverse[i] = unique index; counts[u]; n_unique in counter[0].
__global__ void __launch_bounds__(256) k_unique_insert(const int64_t* __restrict__ vals, int64_t n, int64_t* __restrict__ tkeys,
                                                       int32_t* __restrict__ tvals, int64_t cap, int32_t* __restrict__ counter,
                                                       int64_t* __restrict__ out_unique, int32_t* __restrict__ first_pos) {
  const uint64_t mask = (uint64_t)cap - 1;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t key = vals[i];
    uint64_t p = dr_mix64((uint64_t)key) & mask;
    for (;;) {
      int64_t k = ld_volatile_i64(&tkeys[p]);
      if (k == key) break;
      if (k == kEmptyKey) {
        unsigned long long old = atomicCAS((unsigned long long*)&tkeys[p], (unsigned long long)kEmptyKey, (unsigned long long)key);
        if ((int64_t)old == kEmptyKey) {
          int u = atomicAdd(counter, 1);
          out_unique[u] = key; tvals[p] = u;
          break;
        }
        if ((int64_t)old == key) break;
      }
      p = (p + 1) & mask;
    }
    first_pos[i] = (int32_t)p;
  }
}
__global__ void __launch_bounds__(256) k_unique_resolve(int64_t n, const int32_t* __restrict__ first_pos, const int32_t* __restrict__ tvals,
                                                        int32_t* __restrict__ inverse, int32_t* __restrict__ counts) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int u = tvals[first_pos[i]];
    inverse[i] = u;
    atomicAdd(&counts[u], 1);
  }
}

// segment-sum of rows by inverse index: out[inverse[i]] += rows[i]
template <int LPR>
__global__ void __launch_bounds__(256) k_segment_sum(const float* __restrict__ rows, const int32_t* __restrict__ inverse, int64_t n,
                                                     int dim, float* __restrict__ out) {
  const int lane = threadIdx.x % LPR;
  const int64_t gid = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / LPR;
  const int64_t gstride = (int64_t)gridDim.x * blockDim.x / LPR;
  const int nvec = dim >> 2;
  for (int64_t i = gid; i < n; i += gstride) {
    float* dst = out + (int64_t)inverse[i] * dim;
    for (int c = lane; c < nvec; c += LPR) {
      float4 v = *reinterpret_cast<const float4*>(rows + i * dim + 4 * c);
      red_add_v4_f32(dst + 4 * c, v.x, v.y, v.z, v.w);
    }
  }
}

inline int grid_for(int64_t n, int block, int max_blocks = 0) {
  if (max_blocks <= 0) max_blocks = num_sms() * sparse_blocks_per_sm();
  int64_t b = (n + block - 1) / block;
  if (b < 1) b = 1;
  if (b > max_blocks) b = max_blocks;
  return (int)b;
}
inline int lanes_for(int dim) { int nvec = dim / 4, l = 1; while (l < nvec && l < 32) l <<= 1; return l; }

}  // namespace

extern "C" {

int dr_cuda_combine_fwd(const DrDeviceTable* tables_dev, const int32_t* table_map, int T, int64_t B, int dim, const int64_t* keys, const int32_t* pos,
                        const int64_t* bag_offsets, const float* weights, const int32_t* combiners, void* out, int out_bf16,
                        int64_t stride_b, int64_t stride_t, float* nnz_scale, int32_t* nnz_row, cudaStream_t s) {
  if (T * B == 0) return 0;
  if (dim > 512 || dim % 4) return -1;
  int lpr = lanes_for(dim);
  int grid = grid_for((int64_t)T * B * lpr, 256);
#define LAUNCH(L)                                                                                                          \
  if (out_bf16) k_combine_fwd<L, true><<<grid, 256, 0, s>>>(tables_dev, table_map, T, B, dim, keys, pos, bag_offsets, weights, combiners, out, stride_b, stride_t, nnz_scale, nnz_row); \
  else k_combine_fwd<L, false><<<grid, 256, 0, s>>>(tables_dev, table_map, T, B, dim, keys, pos, bag_offsets, weights, combiners, out, stride_b, stride_t, nnz_scale, nnz_row);
  switch (lpr) {
    case 1: LAUNCH(1) break; case 2: LAUNCH(2) break; case 4: LAUNCH(4) break; case 8: LAUNCH(8) break;
    case 16: LAUNCH(16) break; default: LAUNCH(32) break;
  }
#undef LAUNCH
  DR_LAUNCH_CHECK();
  return 0;
}

// scratch: tkeys[cap] (pre-filled with kEmptyKey), tvals[cap], first_pos[n], counter[1]=0, counts[n]=0
int dr_cuda_unique(const int64_t* vals, int64_t n, int64_t* tkeys, int32_t* tvals, int64_t cap, int32_t* counter,
                   int64_t* out_unique, int32_t* first_pos, int32_t* inverse, int32_t* counts, cudaStream_t s) {
  if (n == 0) return 0;
  k_unique_insert<<<grid_for(n, 256), 256, 0, s>>>(vals, n, tkeys, tvals, cap, counter, out_unique, first_pos);
  DR_LAUNCH_CHECK();
  k_unique_resolve<<<grid_for(n, 256), 256, 0, s>>>(n, first_pos, tvals, inverse, counts);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_segment_sum(const float* rows, const int32_t* inverse, int64_t n, int dim, float* out, cudaStream_t s) {
  if (n == 0) return 0;
  if (dim % 4) return -1;
  int lpr = lanes_for(dim);
  int grid = grid_for(n * lpr, 256);
  switch (lpr) {
    case 1: k_segment_sum<1><<<grid, 256, 0, s>>>(rows, inverse, n, dim, out); break;
    case 2: k_segment_sum<2><<<grid, 256, 0, s>>>(rows, inverse, n, dim, out); break;
    case 4: k_segment_sum<4><<<grid, 256, 0, s>>>(rows, inverse, n, dim, out); break;
    case 8: k_segment_sum<8><<<grid, 256, 0, s>>>(rows, inverse, n, dim, out); break;
    case 16: k_segment_sum<16><<<grid, 256, 0, s>>>(rows, inverse, n, dim, out); break;
    default: k_segment_sum<32><<<grid, 256, 0, s>>>(rows, inverse, n, dim, out); break;
  }
  DR_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
