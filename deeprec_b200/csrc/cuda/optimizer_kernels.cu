// Sparse optimizer path on the device tables: sort-free dedup (claim -> accumulate -> apply) and the
// eight row-wise update rules; plus the fused multi-tensor dense optimizer.
//
// Replaces K7/K8/K9/K10 of SURVEY §2.14 (batch.cu.cc:80-212, training_ali_ops_gpu.cu.cc:48-591,
// unique_ali_op_gpu.cu.cc).  The reference dedups with cub radix sort + adjacent-diff + scan and a
// separate segment-sum; here the forward probe already claimed a unique index per touched key
// (k_lookup), the backward scatters gradients with vectorised L2 reductions (red.global.add.v4.f32)
// into a compact [n_unique, dim] buffer, and ONE apply kernel per step admits/allocates/initialises
// rows, runs the rule, clears the claim and re-zeroes the buffer.
#include "table.cuh"

using namespace drc;

namespace {

__device__ __forceinline__ int seg_of(const int64_t* offsets, int T, int64_t i, int64_t uniform) {
  if (offsets == nullptr) return (int)(i / uniform);
  int lo = 0, hi = T;
  while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (offsets[mid] <= i) lo = mid; else hi = mid; }
  return lo;
}

// -----------------------------------------------------------------------------------------------
// K_accumulate: gsum[tag[pos_i]] += scale_i * grad(b_i, t_i).   LPR lanes per item, float4 each.
// grad element (b, t) at grad + b*stride_b + t*stride_t  (flat_in: grad + i*dim).
// -----------------------------------------------------------------------------------------------
template <int LPR, bool BF16>
__global__ void __launch_bounds__(256) k_accumulate(const DrDeviceTable* __restrict__ tables, const int32_t* __restrict__ table_map, int T, int dim,
                                                    const int32_t* __restrict__ pos, const int64_t* __restrict__ offsets,
                                                    int64_t uniform, int64_t n, const void* __restrict__ grad,
                                                    int64_t stride_b, int64_t stride_t, int flat_in,
                                                    const int32_t* __restrict__ row_ids, const float* __restrict__ scale,
                                                    float* __restrict__ gsum, int C) {
  pdl_sync();
  // per-block combining cache (see table.cuh): hot keys are reduced in shared memory and flushed once per block
  extern __shared__ __align__(16) uint8_t smem_raw[];
  float* s_acc = reinterpret_cast<float*>(smem_raw);
  int32_t* s_tag = reinterpret_cast<int32_t*>(smem_raw + (size_t)C * dim * 4);
  for (int e = threadIdx.x; e < C * dim; e += blockDim.x) s_acc[e] = 0.f;
  for (int e = threadIdx.x; e < C; e += blockDim.x) s_tag[e] = -1;
  __syncthreads();
  const int lane = threadIdx.x % LPR;
  const int gleader = (threadIdx.x & 31) / LPR * LPR;
  const unsigned gmask = LPR == 32 ? 0xffffffffu : (((1u << LPR) - 1u) << gleader);
  const int64_t gid = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / LPR;
  const int64_t gstride = (int64_t)gridDim.x * blockDim.x / LPR;
  const int nvec = dim >> 2;
  for (int64_t i = gid; i < n; i += gstride) {
    const int32_t p = pos[i];
    if (p < 0) continue;
    const int t = seg_of(offsets, T, i, uniform);
    const DrDeviceTable& TBa = tables[table_map ? table_map[t] : t];
    const int32_t u = TBa.slots[p].tag;
    if (u < 0) continue;
    const int Ce = TBa.capacity <= (1 << 17) ? C : 0;      // combining only pays for small (hot-key) tables
    int64_t o;
    if (flat_in) o = i * dim;
    else {
      int64_t b = row_ids ? row_ids[i] : (offsets ? i - offsets[t] : i % uniform);
      o = b * stride_b + (int64_t)t * stride_t;
    }
    const float sc = scale ? scale[i] : 1.0f;
    float4 chunks[4];
    int k = 0;
    for (int c = lane; c < nvec && k < 4; c += LPR, ++k) {
      float4 g;
      if (BF16) {
        uint2 raw = *reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(grad) + o + 4 * c);
        float2 a = unpack_bf16x2(raw.x), b2 = unpack_bf16x2(raw.y);
        g = make_float4(a.x, a.y, b2.x, b2.y);
      } else {
        g = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(grad) + o + 4 * c);
      }
      chunks[k] = make_float4(g.x * sc, g.y * sc, g.z * sc, g.w * sc);
    }
    combine_add<LPR>(s_tag, s_acc, Ce, dim, u, lane, gmask, gleader, chunks, k, gsum);
  }
  __syncthreads();
  flush_combining_cache(s_tag, s_acc, C, dim, gsum);
}

// -----------------------------------------------------------------------------------------------
// K_apply: one LPR-lane group per unique key.
// -----------------------------------------------------------------------------------------------
template <int LPR>
__global__ void __launch_bounds__(256) k_apply(const DrDeviceTable* __restrict__ tables, const int64_t* __restrict__ ulist,
                                               const int32_t* __restrict__ n_unique_ptr, int64_t ulist_cap,
                                               float* __restrict__ gsum, int dim, const DrOptHyper* __restrict__ hp_dev) {
  pdl_sync();
  const DrOptHyper hp = *hp_dev;      // device-resident so a captured CUDA graph sees the live step / beta powers
  const int lane = threadIdx.x % LPR;
  const int64_t gid = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / LPR;
  const int64_t gstride = (int64_t)gridDim.x * blockDim.x / LPR;
  int64_t nu = *n_unique_ptr; if (nu > ulist_cap) nu = ulist_cap;
  const int nvec = dim >> 2;
  const float alpha = dr_adam_alpha(hp);
  const unsigned gmask = LPR == 32 ? 0xffffffffu : (((1u << LPR) - 1u) << ((threadIdx.x & 31) / LPR * LPR));
  for (int64_t u = gid; u < nu; u += gstride) {
    const int64_t packed = ulist[u];
    const int t = (int)(packed >> 40);
    const int64_t pos = packed & ((int64_t(1) << 40) - 1);
    const DrDeviceTable& TB = tables[t];
    float* g = gsum + u * dim;
    int32_t r = 0;
    if (lane == 0) {
      r = TB.slots[pos].row_of;
      if (r < 0) {
        bool admit = TB.filter_type == DR_FILTER_COUNTER ? TB.slots[pos].freq >= TB.filter_freq : true;
        if (admit) {
          r = table_alloc_row(TB);
          if (r >= 0) { TB.slots[pos].row_of = r; atomicAdd(&TB.counters[CTR_NADMITTED], 1); r = -(r + 2); }   // negative => fresh
        } else {
          r = -1;
        }
      }
      TB.slots[pos].tag = -1;   // release the per-step claim
      TB.slots[pos].version = (int32_t)hp.global_step;   // UpdateVersion(value_ptr, gs) for every touched key, admitted or not
    }
    r = __shfl_sync(gmask, r, (threadIdx.x & 31) / LPR * LPR);
    bool fresh = r <= -2;
    if (fresh) r = -(r + 2);
    if (r < 0) {   // not admitted (or out of rows): drop gradient, keep buffer clean
      for (int c = lane; c < nvec; c += LPR) *reinterpret_cast<float4*>(g + 4 * c) = make_float4(0.f, 0.f, 0.f, 0.f);
      continue;
    }
    float* row = TB.rows + (int64_t)r * TB.stride;
    if (fresh) {
      const int64_t key = TB.slots[pos].key;
      const float* def = TB.default_matrix + dr_default_row(key, TB.default_value_dim) * TB.dim;
      for (int c = lane; c < nvec; c += LPR) {
        *reinterpret_cast<float4*>(row + 4 * c) = *reinterpret_cast<const float4*>(def + 4 * c);
        for (int s = 0; s < TB.num_slots; ++s) {
          float v = TB.slot_init[s];
          *reinterpret_cast<float4*>(row + (1 + s) * dim + 4 * c) = make_float4(v, v, v, v);
        }
      }
      if (lane == 0) for (int d = dim * (1 + TB.num_slots); d < TB.stride; ++d) row[d] = 0.f;
      __syncwarp(gmask);
    }
    bool decay_now = false;
    if (hp.kind == DR_OPT_ADAGRAD_DECAY && TB.has_scalars) {
      float* sc = row + dim * (1 + TB.num_slots);
      float pw = sc[0];
      decay_now = hp.decay_step > 0 && (float)(hp.global_step / hp.decay_step) > pw;
      __syncwarp(gmask);
      if (decay_now && lane == 0) sc[0] = pw + 1.0f;
    }
    if (hp.kind == DR_OPT_FTRL) {
      // phase 1: linear update + row norm (group-lasso form, training_ali_ops.cc:559-585)
      float sq = 0.f;
      for (int c = lane; c < nvec; c += LPR) {
        float4 gv = *reinterpret_cast<float4*>(g + 4 * c);
        float4 w = *reinterpret_cast<float4*>(row + 4 * c);
        float4 a = *reinterpret_cast<float4*>(row + dim + 4 * c);
        float4 l = *reinterpret_cast<float4*>(row + 2 * dim + 4 * c);
        float na;
        dr_ftrl_linear(hp, gv.x, w.x, a.x, l.x, na); dr_ftrl_linear(hp, gv.y, w.y, a.y, l.y, na);
        dr_ftrl_linear(hp, gv.z, w.z, a.z, l.z, na); dr_ftrl_linear(hp, gv.w, w.w, a.w, l.w, na);
        *reinterpret_cast<float4*>(row + 2 * dim + 4 * c) = l;
        sq += l.x * l.x + l.y * l.y + l.z * l.z + l.w * l.w;
      }
      for (int o = LPR / 2; o > 0; o >>= 1) sq += __shfl_xor_sync(gmask, sq, o);
      const float norm = sqrtf(sq);
      for (int c = lane; c < nvec; c += LPR) {
        float4 gv = *reinterpret_cast<float4*>(g + 4 * c);
        float4 w = *reinterpret_cast<float4*>(row + 4 * c);
        float4 a = *reinterpret_cast<float4*>(row + dim + 4 * c);
        float4 l = *reinterpret_cast<float4*>(row + 2 * dim + 4 * c);
        float gx = gv.x + 2.f * hp.l2_shrinkage * w.x, gy = gv.y + 2.f * hp.l2_shrinkage * w.y;
        float gz = gv.z + 2.f * hp.l2_shrinkage * w.z, gw = gv.w + 2.f * hp.l2_shrinkage * w.w;
        w.x = dr_ftrl_weight(hp, l.x, a.x + gx * gx, norm); w.y = dr_ftrl_weight(hp, l.y, a.y + gy * gy, norm);
        w.z = dr_ftrl_weight(hp, l.z, a.z + gz * gz, norm); w.w = dr_ftrl_weight(hp, l.w, a.w + gw * gw, norm);
        a.x += gv.x * gv.x; a.y += gv.y * gv.y; a.z += gv.z * gv.z; a.w += gv.w * gv.w;
        *reinterpret_cast<float4*>(row + 4 * c) = w;
        *reinterpret_cast<float4*>(row + dim + 4 * c) = a;
        *reinterpret_cast<float4*>(g + 4 * c) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      continue;
    }
    const int ns = TB.num_slots;
    for (int c = lane; c < nvec; c += LPR) {
      float4 gv = *reinterpret_cast<float4*>(g + 4 * c);
      float4 w = *reinterpret_cast<float4*>(row + 4 * c);
      float4 s0 = ns > 0 ? *reinterpret_cast<float4*>(row + dim + 4 * c) : make_float4(0.f, 0.f, 0.f, 0.f);
      float4 s1 = ns > 1 ? *reinterpret_cast<float4*>(row + 2 * dim + 4 * c) : make_float4(0.f, 0.f, 0.f, 0.f);
      dr_apply_elem(hp.kind, hp, alpha, decay_now, gv.x, w.x, s0.x, s1.x);
      dr_apply_elem(hp.kind, hp, alpha, decay_now, gv.y, w.y, s0.y, s1.y);
      dr_apply_elem(hp.kind, hp, alpha, decay_now, gv.z, w.z, s0.z, s1.z);
      dr_apply_elem(hp.kind, hp, alpha, decay_now, gv.w, w.w, s0.w, s1.w);
      *reinterpret_cast<float4*>(row + 4 * c) = w;
      if (ns > 0) *reinterpret_cast<float4*>(row + dim + 4 * c) = s0;
      if (ns > 1) *reinterpret_cast<float4*>(row + 2 * dim + 4 * c) = s1;
      *reinterpret_cast<float4*>(g + 4 * c) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}

// reset of the per-step unique counter happens in a 1-thread tail so the whole step is graph-capturable
__global__ void k_reset_counter(int32_t* c) {
  pdl_sync();
  *c = 0;
}

// end-of-step bookkeeping on the device: the dense AdagradDecay power follows the decay this step's dense apply made,
// global_step += 1, Adam-family beta powers advance
__global__ void k_advance_hyper(DrOptHyper* hp) {
  pdl_sync();
  if (dr_dense_decay_now(*hp)) hp->dense_decay_power += 1;
  hp->global_step += 1;
  if (hp->kind == DR_OPT_ADAM || hp->kind == DR_OPT_ADAMW || hp->kind == DR_OPT_ADAM_ASYNC || hp->kind == DR_OPT_ADAM_ASYNC_RMSPROP) {
    hp->beta1_power *= hp->beta1;
    hp->beta2_power *= hp->beta2;
  }
}

// -----------------------------------------------------------------------------------------------
// Dense multi-tensor optimizer on flat fp32 buffers (K9 analogue: ApplyAdamAsync etc.), optionally
// emitting bf16 shadow weights (W and W^T are produced by the GEMM-layout kernel in dense_kernels.cu).
// -----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_dense_apply(float* __restrict__ w, const float* __restrict__ grad,
                                                     float* __restrict__ s0, float* __restrict__ s1, int64_t n,
                                                     const DrOptHyper* __restrict__ hp_dev, float grad_scale,
                                                     __nv_bfloat16* __restrict__ w_bf16) {
  pdl_sync();
  const DrOptHyper hp = *hp_dev;
  const float alpha = dr_adam_alpha(hp);
  const bool decay_now = dr_dense_decay_now(hp);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float g = grad[i] * grad_scale;
    float wv = w[i];
    float a = s0 ? s0[i] : 0.f, b = s1 ? s1[i] : 0.f;
    dr_apply_elem(hp.kind, hp, alpha, decay_now, g, wv, a, b);
    w[i] = wv;
    if (s0) s0[i] = a;
    if (s1) s1[i] = b;
    if (w_bf16) w_bf16[i] = __float2bfloat16(wv);
  }
}

inline int grid_for(int64_t n, int block, int max_blocks = 0) {
  if (max_blocks <= 0) max_blocks = sparse_sm_count() * sparse_blocks_per_sm();
  int64_t b = (n + block - 1) / block;
  if (b < 1) b = 1;
  if (b > max_blocks) b = max_blocks;
  return (int)b;
}
inline int lanes_for(int dim) { int nvec = dim / 4, l = 1; while (l < nvec && l < 32) l <<= 1; return l; }

}  // namespace

extern "C" {

int dr_cuda_sparse_accumulate(const DrDeviceTable* tables_dev, const int32_t* table_map, int T, int dim, const int32_t* pos, const int64_t* offsets,
                              int64_t uniform, int64_t n, const void* grad, int grad_bf16, int64_t stride_b, int64_t stride_t,
                              int flat_in, const int32_t* row_ids, const float* scale, float* gsum, cudaStream_t s) {
  if (n == 0) return 0;
  if (dim > 512) return -1;
  int lpr = lanes_for(dim);
  int grid = grid_for(n * lpr, 256);
  const int C = combining_cache_slots(dim);
  const size_t smem = (size_t)C * dim * 4 + (size_t)C * 4;
#define LAUNCH(L)                                                                                                  \
  if (grad_bf16) DR_PDL_LAUNCH((k_accumulate<L, true>), grid, 256, smem, s, tables_dev, table_map, T, dim, pos, offsets, uniform, n, grad, stride_b, stride_t, flat_in, row_ids, scale, gsum, C); \
  else DR_PDL_LAUNCH((k_accumulate<L, false>), grid, 256, smem, s, tables_dev, table_map, T, dim, pos, offsets, uniform, n, grad, stride_b, stride_t, flat_in, row_ids, scale, gsum, C);
  switch (lpr) {
    case 1: LAUNCH(1) break; case 2: LAUNCH(2) break; case 4: LAUNCH(4) break; case 8: LAUNCH(8) break;
    case 16: LAUNCH(16) break; default: LAUNCH(32) break;
  }
#undef LAUNCH
  DR_LAUNCH_CHECK();
  return 0;
}

// max_unique bounds the grid; the kernel reads the true count from device memory (no host sync).
int dr_cuda_sparse_apply(const DrDeviceTable* tables_dev, const int64_t* ulist, int32_t* n_unique_dev, int64_t ulist_cap,
                         float* gsum, int dim, const DrOptHyper* hp_dev, int64_t max_unique, int reset_counter, cudaStream_t s) {
  int lpr = lanes_for(dim);
  int grid = grid_for(max_unique * lpr, 256, sparse_sm_count() * (sparse_blocks_per_sm() < 8 ? sparse_blocks_per_sm() : 8));
  switch (lpr) {
    case 1: DR_PDL_LAUNCH((k_apply<1>), grid, 256, 0, s, tables_dev, ulist, n_unique_dev, ulist_cap, gsum, dim, hp_dev); break;
    case 2: DR_PDL_LAUNCH((k_apply<2>), grid, 256, 0, s, tables_dev, ulist, n_unique_dev, ulist_cap, gsum, dim, hp_dev); break;
    case 4: DR_PDL_LAUNCH((k_apply<4>), grid, 256, 0, s, tables_dev, ulist, n_unique_dev, ulist_cap, gsum, dim, hp_dev); break;
    case 8: DR_PDL_LAUNCH((k_apply<8>), grid, 256, 0, s, tables_dev, ulist, n_unique_dev, ulist_cap, gsum, dim, hp_dev); break;
    case 16: DR_PDL_LAUNCH((k_apply<16>), grid, 256, 0, s, tables_dev, ulist, n_unique_dev, ulist_cap, gsum, dim, hp_dev); break;
    default: DR_PDL_LAUNCH((k_apply<32>), grid, 256, 0, s, tables_dev, ulist, n_unique_dev, ulist_cap, gsum, dim, hp_dev); break;
  }
  DR_LAUNCH_CHECK();
  if (reset_counter) { DR_PDL_LAUNCH((k_reset_counter), 1, 1, 0, s, n_unique_dev); DR_LAUNCH_CHECK(); }
  return 0;
}

int dr_cuda_advance_hyper(DrOptHyper* hp_dev, cudaStream_t s) {
  DR_PDL_LAUNCH((k_advance_hyper), 1, 1, 0, s, hp_dev);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_cuda_dense_apply(float* w, const float* grad, float* s0, float* s1, int64_t n, const DrOptHyper* hp_dev, float grad_scale,
                        void* w_bf16, cudaStream_t s) {
  if (n == 0) return 0;
  DR_PDL_LAUNCH((k_dense_apply), grid_for(n, 256), 256, 0, s, w, grad, s0, s1, n, hp_dev, grad_scale, (__nv_bfloat16*)w_bf16);
  DR_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
