// Sparse utility kernels of the input / embedding front-end, sm_90a.  One C entry per op, every data-dependent size stays on the device
// (the python wrapper reads the count once, where the reference blocks on a D2H copy of the cub select result).
//
// Reference kernels replaced (SURVEY §2.14 K14 / K16):
//   fused-embedding pre ops    kernels/fused_embedding/fused_embedding_pre_ops_gpus.cu.cc:23-123  (InitFlagsToOneInt4, DetectInvalid,
//                              FusedMultiFunctionalKernel: prune invalid ids / non-positive weights + fill empty rows; cub select + scan)
//   SparseFillEmptyRows (GPU)  kernels/sparse_fill_empty_rows_op_util.cu.cc
//   SparseSlice (GPU)          kernels/sparse_slice_op_gpu.cu.cc
//   SparseReshape              kernels/sparse_reshape_op.cc (index re-linearisation)
//   SparseSegment{Sum,Mean,SqrtN}(+Grad) GPU rewrites  kernels/segment_reduction_ops_gpu.cu.{h,cc}
//
// Design: prune + fill is ONE ordered compaction -- per-row kept counts (atomics), three exclusive scans (cub::DeviceScan: kept flags, kept per
// row, output rows per row), one emit kernel that writes kept entries and default entries directly at their final, row-ordered position (the
// reference concatenates the fills and re-sorts).  Segment reductions walk sorted segment ids with a warp per output row (no atomics forward;
// the gradient scatters with red.global.add.v4).
#ifndef DR_CUDA_EMU
#include <cub/device/device_scan.cuh>
#endif

#include "common.cuh"

using namespace drc;

namespace {

inline int grid_el(int64_t n, int block = 256) { const int64_t b = (n + block - 1) / block; return (int)(b < 1 ? 1 : b > num_sms() * 8 ? num_sms() * 8 : b); }
inline size_t align256(size_t n) { return (n + 255) / 256 * 256; }

// ---------------------------------------------------------------------------------------------- prune + fill-empty-rows
__global__ void __launch_bounds__(256) k_spu_flags(const int64_t* __restrict__ values, const int64_t* __restrict__ rows, const float* __restrict__ weights, int64_t nnz,
                                                   int64_t B, int prune, int32_t* __restrict__ keep, int32_t* __restrict__ cnt) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nnz; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = rows[i];
    int k = r >= 0 && r < B;
    if (prune) k = k && values[i] >= 0 && (!weights || weights[i] > 0.f);
    keep[i] = k;
    if (k) atomicAdd(cnt + r, 1);
  }
}

__global__ void __launch_bounds__(256) k_spu_rows(const int32_t* __restrict__ cnt, int64_t B, int fill, int32_t* __restrict__ row_out_in, int32_t* __restrict__ empty) {
  for (int64_t b = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
    const int e = cnt[b] == 0;
    row_out_in[b] = cnt[b] + (fill && e ? 1 : 0);
    if (empty) empty[b] = e;
  }
}

__global__ void __launch_bounds__(256) k_spu_emit(const int64_t* __restrict__ values, const int64_t* __restrict__ rows, const float* __restrict__ weights, int64_t nnz,
                                                  int64_t B, int fill, int64_t default_id, const int32_t* __restrict__ keep, const int32_t* __restrict__ scan_keep,
                                                  const int32_t* __restrict__ cnt, const int32_t* __restrict__ row_kept, const int32_t* __restrict__ row_out,
                                                  const int32_t* __restrict__ row_out_in, int64_t* __restrict__ out_values, int64_t* __restrict__ out_rows,
                                                  float* __restrict__ out_weights, int64_t* __restrict__ out_count) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, nth = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = tid; i < nnz; i += nth) {
    if (!keep[i]) continue;
    const int64_t r = rows[i];
    const int64_t pos = (int64_t)row_out[r] + (scan_keep[i] - row_kept[r]);      // rows are non-decreasing: rank inside the row = global rank - kept before the row
    out_values[pos] = values[i]; out_rows[pos] = r;
    if (out_weights) out_weights[pos] = weights ? weights[i] : 1.f;
  }
  if (fill)
    for (int64_t b = tid; b < B; b += nth) {
      if (cnt[b]) continue;
      const int64_t pos = row_out[b];
      out_values[pos] = default_id; out_rows[pos] = b;
      if (out_weights) out_weights[pos] = 1.f;
    }
  if (tid == 0) *out_count = B > 0 ? (int64_t)row_out[B - 1] + row_out_in[B - 1] : 0;
}

// ---------------------------------------------------------------------------------------------- COO slice / reshape
// keep entries inside the box [start, start + size) (per dimension), shift their indices by -start
__global__ void __launch_bounds__(256) k_spu_slice_flags(const int64_t* __restrict__ idx, int64_t nnz, int R, const int64_t* __restrict__ start,
                                                         const int64_t* __restrict__ size, int32_t* __restrict__ keep) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nnz; i += (int64_t)gridDim.x * blockDim.x) {
    int k = 1;
    for (int d = 0; d < R; ++d) { const int64_t v = idx[i * R + d]; k = k && v >= start[d] && v < start[d] + size[d]; }
    keep[i] = k;
  }
}
template <typename V>
__global__ void __launch_bounds__(256) k_spu_slice_emit(const int64_t* __restrict__ idx, const V* __restrict__ vals, int64_t nnz, int R, const int64_t* __restrict__ start,
                                                        const int32_t* __restrict__ keep, const int32_t* __restrict__ scan_keep, int64_t* __restrict__ out_idx,
                                                        V* __restrict__ out_vals, int64_t* __restrict__ out_count) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  for (int64_t i = tid; i < nnz; i += (int64_t)gridDim.x * blockDim.x) {
    if (!keep[i]) continue;
    const int64_t pos = scan_keep[i];
    for (int d = 0; d < R; ++d) out_idx[pos * R + d] = idx[i * R + d] - start[d];
    out_vals[pos] = vals[i];
  }
  if (tid == 0) *out_count = nnz > 0 ? (int64_t)scan_keep[nnz - 1] + keep[nnz - 1] : 0;
}

// indices [nnz, R0] under shape0 -> indices [nnz, R1] under shape1 (same number of elements): linearise, de-linearise
__global__ void __launch_bounds__(256) k_spu_reshape(const int64_t* __restrict__ idx, int64_t nnz, int R0, const int64_t* __restrict__ shape0, int R1,
                                                     const int64_t* __restrict__ shape1, int64_t* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nnz; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t lin = 0;
    for (int d = 0; d < R0; ++d) lin = lin * shape0[d] + idx[i * R0 + d];
    for (int d = R1 - 1; d >= 0; --d) { out[i * R1 + d] = lin % shape1[d]; lin /= shape1[d]; }
  }
}

// ---------------------------------------------------------------------------------------------- sparse segment reductions
// out[s] = scale(s) * sum_{i: seg[i] == s} data[indices[i]]   (seg sorted; mode 0 sum, 1 mean, 2 sqrtn).  One warp per output segment:
// binary search of the segment's [lo, hi) range, lanes stride the feature dimension.
__device__ __forceinline__ int64_t lower_bound_i64(const int64_t* a, int64_t n, int64_t v) {
  int64_t lo = 0, hi = n;
  while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (a[mid] < v) lo = mid + 1; else hi = mid; }
  return lo;
}
__global__ void __launch_bounds__(256) k_spu_segment_fwd(const float* __restrict__ data, int64_t N, int D, const int64_t* __restrict__ indices,
                                                         const int64_t* __restrict__ seg, int64_t nnz, int64_t S, int mode, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t s = warp; s < S; s += nwarps) {
    const int64_t lo = lower_bound_i64(seg, nnz, s), hi = lower_bound_i64(seg, nnz, s + 1);
    const float cntf = (float)(hi - lo);
    const float scale = (mode == 0 || hi == lo) ? 1.f : mode == 1 ? 1.f / cntf : rsqrtf(cntf);
    for (int c = lane; c < D; c += 32) {
      float acc = 0.f;
      for (int64_t i = lo; i < hi; ++i) { const int64_t r = indices[i]; if (r >= 0 && r < N) acc += data[r * D + c]; }
      out[s * D + c] = acc * scale;
    }
  }
}
// d_data[indices[i]] += scale(seg[i]) * g[seg[i]]
__global__ void __launch_bounds__(256) k_spu_segment_bwd(const float* __restrict__ g, int64_t S, int D, const int64_t* __restrict__ indices, const int64_t* __restrict__ seg,
                                                         int64_t nnz, int64_t N, int mode, float* __restrict__ d_data) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = warp; i < nnz; i += nwarps) {
    const int64_t s = seg[i], r = indices[i];
    if (s < 0 || s >= S || r < 0 || r >= N) continue;
    float scale = 1.f;
    if (mode) {
      const float cntf = (float)(lower_bound_i64(seg, nnz, s + 1) - lower_bound_i64(seg, nnz, s));
      scale = mode == 1 ? 1.f / cntf : rsqrtf(cntf);
    }
    for (int c = lane; c < D; c += 32) atomicAdd(d_data + r * D + c, g[s * D + c] * scale);
  }
}

struct PfWs { int32_t *keep, *scan_keep, *cnt, *row_kept, *row_out_in, *row_out; void* cub; size_t cub_bytes; };
inline size_t cub_scan_bytes(int64_t n) {
  size_t b = 0;
  cub::DeviceScan::ExclusiveSum((void*)nullptr, b, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(n > 0 ? n : 1));
  return b;
}
inline PfWs carve(void* ws, int64_t nnz, int64_t B) {
  uint8_t* p = static_cast<uint8_t*>(ws);
  PfWs w{};
  auto take = [&](size_t bytes) { void* q = p; p += align256(bytes); return q; };
  w.keep = (int32_t*)take((size_t)(nnz > 0 ? nnz : 1) * 4); w.scan_keep = (int32_t*)take((size_t)(nnz > 0 ? nnz : 1) * 4);
  w.cnt = (int32_t*)take((size_t)(B > 0 ? B : 1) * 4); w.row_kept = (int32_t*)take((size_t)(B > 0 ? B : 1) * 4);
  w.row_out_in = (int32_t*)take((size_t)(B > 0 ? B : 1) * 4); w.row_out = (int32_t*)take((size_t)(B > 0 ? B : 1) * 4);
  w.cub_bytes = cub_scan_bytes(nnz > B ? nnz : B); w.cub = take(w.cub_bytes);
  return w;
}

}  // namespace

extern "C" {

// bytes of device workspace dr_cuda_sparse_prune_fill / dr_cuda_sparse_slice need for (nnz, B)
int64_t dr_cuda_sparse_utils_workspace(int64_t nnz, int64_t B) {
  const size_t n1 = (size_t)(nnz > 0 ? nnz : 1), b1 = (size_t)(B > 0 ? B : 1);
  return (int64_t)(2 * align256(n1 * 4) + 4 * align256(b1 * 4) + align256(cub_scan_bytes(nnz > B ? nnz : B)) + 256);
}

// (values, rows (non-decreasing), weights?) [nnz] over B rows -> pruned (ids < 0, weights <= 0 dropped when `prune`) and, when `fill`, every
// empty row gets one (default_id, weight 1) entry; outputs are row-ordered, sized >= nnz + B; *out_count (device) = number of entries.
// empty_indicator [B] (optional): 1 where the row had no kept entry.
int dr_cuda_sparse_prune_fill(const int64_t* values, const int64_t* rows, const float* weights, int64_t nnz, int64_t B, int prune, int fill, int64_t default_id,
                              int64_t* out_values, int64_t* out_rows, float* out_weights, int32_t* empty_indicator, int64_t* out_count, void* workspace,
                              cudaStream_t s) {
  if (B <= 0) { DR_CUDA_CHECK(cudaMemsetAsync(out_count, 0, 8, s)); return 0; }
  if (nnz >= (int64_t)1 << 31 || B >= (int64_t)1 << 31) return -2;
  PfWs w = carve(workspace, nnz, B);
  DR_CUDA_CHECK(cudaMemsetAsync(w.cnt, 0, (size_t)B * 4, s));
  if (nnz > 0) {
    k_spu_flags<<<grid_el(nnz), 256, 0, s>>>(values, rows, weights, nnz, B, prune, w.keep, w.cnt);
    DR_LAUNCH_CHECK();
    size_t cb = w.cub_bytes;
    DR_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(w.cub, cb, w.keep, w.scan_keep, (int)nnz, s));
  }
  k_spu_rows<<<grid_el(B), 256, 0, s>>>(w.cnt, B, fill, w.row_out_in, empty_indicator);
  DR_LAUNCH_CHECK();
  size_t cb = w.cub_bytes;
  DR_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(w.cub, cb, w.cnt, w.row_kept, (int)B, s));
  cb = w.cub_bytes;
  DR_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(w.cub, cb, w.row_out_in, w.row_out, (int)B, s));
  k_spu_emit<<<grid_el(nnz > B ? nnz : B), 256, 0, s>>>(values, rows, weights, nnz, B, fill, default_id, w.keep, w.scan_keep, w.cnt, w.row_kept, w.row_out, w.row_out_in,
                                                      out_values, out_rows, out_weights, out_count);
  DR_LAUNCH_CHECK();
  return 0;
}

// COO slice: indices [nnz, R] int64, values [nnz] (elem_bytes 4 or 8), start / size [R] on the DEVICE.  Outputs sized nnz; *out_count on the device.
int dr_cuda_sparse_slice(const int64_t* indices, const void* values, int elem_bytes, int64_t nnz, int R, const int64_t* start_dev, const int64_t* size_dev,
                         int64_t* out_indices, void* out_values, int64_t* out_count, void* workspace, cudaStream_t s) {
  if (nnz <= 0) { DR_CUDA_CHECK(cudaMemsetAsync(out_count, 0, 8, s)); return 0; }
  if (nnz >= (int64_t)1 << 31 || R <= 0 || R > 8 || (elem_bytes != 4 && elem_bytes != 8)) return -2;
  PfWs w = carve(workspace, nnz, 1);
  k_spu_slice_flags<<<grid_el(nnz), 256, 0, s>>>(indices, nnz, R, start_dev, size_dev, w.keep);
  DR_LAUNCH_CHECK();
  size_t cb = w.cub_bytes;
  DR_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(w.cub, cb, w.keep, w.scan_keep, (int)nnz, s));
  if (elem_bytes == 4)
    k_spu_slice_emit<uint32_t><<<grid_el(nnz), 256, 0, s>>>(indices, (const uint32_t*)values, nnz, R, start_dev, w.keep, w.scan_keep, out_indices, (uint32_t*)out_values, out_count);
  else
    k_spu_slice_emit<uint64_t><<<grid_el(nnz), 256, 0, s>>>(indices, (const uint64_t*)values, nnz, R, start_dev, w.keep, w.scan_keep, out_indices, (uint64_t*)out_values, out_count);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_sparse_reshape(const int64_t* indices, int64_t nnz, int R0, const int64_t* shape0_dev, int R1, const int64_t* shape1_dev, int64_t* out_indices,
                           cudaStream_t s) {
  if (nnz <= 0) return 0;
  if (R0 <= 0 || R1 <= 0 || R0 > 8 || R1 > 8) return -2;
  k_spu_reshape<<<grid_el(nnz), 256, 0, s>>>(indices, nnz, R0, shape0_dev, R1, shape1_dev, out_indices);
  DR_LAUNCH_CHECK();
  return 0;
}

// mode: 0 sum, 1 mean, 2 sqrtn.  segment_ids sorted ascending (as tf.sparse.segment_* requires).  out [S, D] is fully written.
int dr_cuda_sparse_segment_fwd(const float* data, int64_t N, int D, const int64_t* indices, const int64_t* segment_ids, int64_t nnz, int64_t S, int mode, float* out,
                               cudaStream_t s) {
  if (S <= 0 || D <= 0) return 0;
  k_spu_segment_fwd<<<grid_el(S * 32), 256, 0, s>>>(data, N, D, indices, segment_ids, nnz, S, mode, out);
  DR_LAUNCH_CHECK();
  return 0;
}

// d_data [N, D] must be zeroed by the caller (or hold a running sum): the kernel accumulates.
int dr_cuda_sparse_segment_bwd(const float* g, int64_t S, int D, const int64_t* indices, const int64_t* segment_ids, int64_t nnz, int64_t N, int mode, float* d_data,
                               cudaStream_t s) {
  if (nnz <= 0 || D <= 0) return 0;
  k_spu_segment_bwd<<<grid_el(nnz * 32), 256, 0, s>>>(g, S, D, indices, segment_ids, nnz, N, mode, d_data);
  DR_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
