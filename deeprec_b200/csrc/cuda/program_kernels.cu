// Op-program serving on the GPU: the non-GEMM ops of an exported inference graph (serving/export.py::export_saved_model_program) over
// bf16 [B, ld] activation buffers.  The LINEAR ops run on the wgmma GEMM (gemm_wgmma.cu, bias + ReLU in its epilogue); everything
// here is bandwidth-trivial glue between them (a DeepFM forward at batch 2048 moves < 4 MB through these kernels).
//
// Reference: the processor runs ANY SavedModel graph per session on the session's device (serving/processor/serving/model_session.cc:377-386,
// tensorflow/core/common_runtime/direct_session.cc:563-620); the CPU interpreter of the same program is csrc/host/cpu_serving.cc::RunProgram.
//
// Buffer convention: bf16, row-major, ld = width rounded up to 8 (TMA / 16-byte rule of the GEMM); pad columns are zero and stay zero
// (every kernel writes columns [0, width) only; LINEAR writes its zero-padded output channels, which are exact zeros).
#include "common.cuh"

using namespace drc;

namespace {

__device__ __forceinline__ float ldb(const __nv_bfloat16* p) { return __bfloat162float(*p); }
__device__ __forceinline__ void stb(__nv_bfloat16* p, float v) { *p = __float2bfloat16(v); }

// dst[b, off + k] = src[b, start + k], k < w   (CONCAT piece / SLICE)
__global__ void __launch_bounds__(256) k_prog_copy_cols(const __nv_bfloat16* __restrict__ src, int64_t lds, int start, int w, __nv_bfloat16* __restrict__ dst,
                                                        int64_t ldd, int off, int64_t B) {
  const int64_t n = B * (int64_t)w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / w; const int k = (int)(i - b * w);
    dst[b * ldd + off + k] = src[b * lds + start + k];
  }
}

// y = x * scale[k] + shift[k]   (BatchNorm with moving statistics that could not be folded into a Linear)
__global__ void __launch_bounds__(256) k_prog_affine(const __nv_bfloat16* __restrict__ x, int64_t ldx, int w, const float* __restrict__ sc,
                                                     const float* __restrict__ sh, __nv_bfloat16* __restrict__ y, int64_t ldy, int64_t B) {
  const int64_t n = B * (int64_t)w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / w; const int k = (int)(i - b * w);
    stb(y + b * ldy + k, ldb(x + b * ldx + k) * sc[k] + sh[k]);
  }
}

// FM second-order term per embedding dimension: 0.5 ((sum_t v_t)^2 - sum_t v_t^2); emb [B, T * D]
__global__ void __launch_bounds__(256) k_prog_fm(const __nv_bfloat16* __restrict__ e, int64_t lde, int T, int D, __nv_bfloat16* __restrict__ y, int64_t ldy, int64_t B) {
  const int64_t n = B * (int64_t)D;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / D; const int k = (int)(i - b * D);
    const __nv_bfloat16* row = e + b * lde + k;
    float sum = 0.f, sq = 0.f;
    for (int t = 0; t < T; ++t) { const float v = ldb(row + (int64_t)t * D); sum += v; sq += v * v; }
    stb(y + b * ldy + k, 0.5f * (sum * sum - sq));
  }
}

// kind 0: a + b, 1: a * b, 2: a * b + c
__global__ void __launch_bounds__(256) k_prog_binary(int kind, const __nv_bfloat16* __restrict__ a, int64_t lda, const __nv_bfloat16* __restrict__ b, int64_t ldb_,
                                                     const __nv_bfloat16* __restrict__ c, int64_t ldc, int w, __nv_bfloat16* __restrict__ y, int64_t ldy, int64_t B) {
  const int64_t n = B * (int64_t)w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / w; const int k = (int)(i - r * w);
    const float av = ldb(a + r * lda + k), bv = ldb(b + r * ldb_ + k);
    float v = kind == 0 ? av + bv : av * bv;
    if (kind == 2) v += ldb(c + r * ldc + k);
    stb(y + r * ldy + k, v);
  }
}

// DCN cross layer, one warp per row: y = x0 * (xl . w) + bias + xl
__global__ void __launch_bounds__(256) k_prog_cross(const __nv_bfloat16* __restrict__ x0, int64_t ld0, const __nv_bfloat16* __restrict__ xl, int64_t ldl, int w,
                                                    const float* __restrict__ wv, const float* __restrict__ bv, __nv_bfloat16* __restrict__ y, int64_t ldy, int64_t B) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < B; r += nwarps) {
    float dot = 0.f;
    for (int k = lane; k < w; k += 32) dot += ldb(xl + r * ldl + k) * wv[k];
#pragma unroll
    for (int o = 16; o; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    for (int k = lane; k < w; k += 32) stb(y + r * ldy + k, ldb(x0 + r * ld0 + k) * dot + bv[k] + ldb(xl + r * ldl + k));
  }
}

// LayerNorm (biased variance) + optional ReLU, one warp per row
__global__ void __launch_bounds__(256) k_prog_layernorm(const __nv_bfloat16* __restrict__ x, int64_t ldx, int w, const float* __restrict__ g,
                                                        const float* __restrict__ bt, float eps, int relu, __nv_bfloat16* __restrict__ y, int64_t ldy, int64_t B) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < B; r += nwarps) {
    float sum = 0.f;
    for (int k = lane; k < w; k += 32) sum += ldb(x + r * ldx + k);
#pragma unroll
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / (float)w;
    float var = 0.f;
    for (int k = lane; k < w; k += 32) { const float d = ldb(x + r * ldx + k) - mean; var += d * d; }
#pragma unroll
    for (int o = 16; o; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
    const float rs = rsqrtf(var / (float)w + eps);
    for (int k = lane; k < w; k += 32) {
      float v = (ldb(x + r * ldx + k) - mean) * rs * g[k] + bt[k];
      if (relu && v < 0.f) v = 0.f;
      stb(y + r * ldy + k, v);
    }
  }
}

// prob[b] = sigmoid(x[b, 0])
__global__ void __launch_bounds__(256) k_prog_sigmoid0(const __nv_bfloat16* __restrict__ x, int64_t ldx, int64_t B, float* __restrict__ prob) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < B; i += (int64_t)gridDim.x * blockDim.x)
    prob[i] = 1.f / (1.f + __expf(-ldb(x + i * ldx)));
}

// ---- sequence models (DIN) -------------------------------------------------------------------------------------------------------------
// mask[b, l] = ids[(start + l) * stride + b] >= 0, b < rows   (ids: [C][stride] lookup columns of the request; rows < stride when a
// sample-aware program evaluates the mask of a user-side history once per request)
__global__ void __launch_bounds__(256) k_prog_valid_mask(const int64_t* __restrict__ ids, int64_t stride, int64_t rows, int start, int L, __nv_bfloat16* __restrict__ y,
                                                         int64_t ldy) {
  const int64_t n = rows * (int64_t)L;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / L; const int l = (int)(i - b * L);
    stb(y + b * ldy + l, ids[(int64_t)(start + l) * stride + b] >= 0 ? 1.f : 0.f);
  }
}
// position-wise concat: y[b, l, :] = [a[b, l, :wa] | c[b, l, :wb]]
__global__ void __launch_bounds__(256) k_prog_seq_zip(const __nv_bfloat16* __restrict__ a, int64_t lda, int wa, const __nv_bfloat16* __restrict__ c, int64_t ldc, int wb,
                                                      int L, __nv_bfloat16* __restrict__ y, int64_t ldy, int64_t B) {
  const int w = wa + wb; const int64_t n = B * (int64_t)L * w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / ((int64_t)L * w); const int r = (int)(i - b * (int64_t)L * w); const int l = r / w, k = r - l * w;
    y[b * ldy + r] = k < wa ? a[b * lda + l * wa + k] : c[b * ldc + l * wb + (k - wa)];
  }
}
// y[b, l, :] = x[b, l, :] * mask[b, l]
__global__ void __launch_bounds__(256) k_prog_seq_mask(const __nv_bfloat16* __restrict__ x, int64_t ldx, const __nv_bfloat16* __restrict__ m, int64_t ldm, int L, int w,
                                                       __nv_bfloat16* __restrict__ y, int64_t ldy, int64_t B) {
  const int64_t n = B * (int64_t)L * w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / ((int64_t)L * w); const int r = (int)(i - b * (int64_t)L * w);
    stb(y + b * ldy + r, ldb(x + b * ldx + r) * ldb(m + b * ldm + r / w));
  }
}
// y[b, :] = sum_l x[b, l, :]
__global__ void __launch_bounds__(256) k_prog_seq_sum(const __nv_bfloat16* __restrict__ x, int64_t ldx, int L, int w, __nv_bfloat16* __restrict__ y, int64_t ldy, int64_t B) {
  const int64_t n = B * (int64_t)w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / w; const int k = (int)(i - b * w);
    float acc = 0.f;
    for (int l = 0; l < L; ++l) acc += ldb(x + b * ldx + (int64_t)l * w + k);
    stb(y + b * ldy + k, acc);
  }
}
__global__ void __launch_bounds__(256) k_prog_prelu(const __nv_bfloat16* __restrict__ x, int64_t ldx, int w, const float* __restrict__ alpha, __nv_bfloat16* __restrict__ y,
                                                    int64_t ldy, int64_t B) {
  const int64_t n = B * (int64_t)w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / w; const int k = (int)(i - b * w);
    const float v = ldb(x + b * ldx + k);
    stb(y + b * ldy + k, v > 0.f ? v : alpha[k] * v);
  }
}
// staging for the fp32 attention kernel (attention_kernels.cu): bf16 [B, ld] <-> dense fp32 [B, w]; mask -> uint8
__global__ void __launch_bounds__(256) k_prog_to_f32(const __nv_bfloat16* __restrict__ x, int64_t ldx, int w, float* __restrict__ y, int64_t B) {
  const int64_t n = B * (int64_t)w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) { const int64_t b = i / w; y[i] = ldb(x + b * ldx + (i - b * w)); }
}
__global__ void __launch_bounds__(256) k_prog_from_f32(const float* __restrict__ x, int w, __nv_bfloat16* __restrict__ y, int64_t ldy, int64_t B) {
  const int64_t n = B * (int64_t)w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) { const int64_t b = i / w; stb(y + b * ldy + (i - b * w), x[i]); }
}
__global__ void __launch_bounds__(256) k_prog_to_u8(const __nv_bfloat16* __restrict__ x, int64_t ldx, int w, uint8_t* __restrict__ y, int64_t B) {
  const int64_t n = B * (int64_t)w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) { const int64_t b = i / w; y[i] = ldb(x + b * ldx + (i - b * w)) > 0.f ? 1 : 0; }
}

// host-resident tables (device placement optimisation): rows looked up on the CPU arrive sample-major fp32 [B, T * D]; the DLRM path wants them
// feature-major bf16 [T][B][D]
__global__ void __launch_bounds__(256) k_prog_emb_feature_major(const float* __restrict__ x, int T, int D, int64_t B, __nv_bfloat16* __restrict__ y) {
  const int64_t n = B * (int64_t)T * D;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / ((int64_t)T * D); const int r = (int)(i - b * (int64_t)T * D); const int t = r / D, d = r - t * D;
    stb(y + ((int64_t)t * B + b) * D + d, x[i]);
  }
}

// row-wise softmax (mixture-of-experts gates), one warp per row
__global__ void __launch_bounds__(256) k_prog_softmax(const __nv_bfloat16* __restrict__ x, int64_t ldx, int w, __nv_bfloat16* __restrict__ y, int64_t ldy, int64_t B) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < B; r += nwarps) {
    float mx = -3.4e38f;
    for (int k = lane; k < w; k += 32) mx = fmaxf(mx, ldb(x + r * ldx + k));
#pragma unroll
    for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float den = 0.f;
    for (int k = lane; k < w; k += 32) den += __expf(ldb(x + r * ldx + k) - mx);
#pragma unroll
    for (int o = 16; o; o >>= 1) den += __shfl_xor_sync(0xffffffffu, den, o);
    const float inv = 1.f / den;
    for (int k = lane; k < w; k += 32) stb(y + r * ldy + k, __expf(ldb(x + r * ldx + k) - mx) * inv);
  }
}
// y[b, 0] = cos(a[b, :], c[b, :]) with each norm clamped at 1e-8, one warp per row
__global__ void __launch_bounds__(256) k_prog_cosine(const __nv_bfloat16* __restrict__ a, int64_t lda, const __nv_bfloat16* __restrict__ c, int64_t ldc, int w,
                                                     __nv_bfloat16* __restrict__ y, int64_t ldy, int64_t B) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < B; r += nwarps) {
    float xy = 0.f, xx = 0.f, yy = 0.f;
    for (int k = lane; k < w; k += 32) { const float p = ldb(a + r * lda + k), q = ldb(c + r * ldc + k); xy += p * q; xx += p * p; yy += q * q; }
#pragma unroll
    for (int o = 16; o; o >>= 1) { xy += __shfl_xor_sync(0xffffffffu, xy, o); xx += __shfl_xor_sync(0xffffffffu, xx, o); yy += __shfl_xor_sync(0xffffffffu, yy, o); }
    if (lane == 0) stb(y + r * ldy, xy / (fmaxf(sqrtf(xx), 1e-8f) * fmaxf(sqrtf(yy), 1e-8f)));
  }
}
// prob[b * no + o] = sigmoid(x[b, o]), o < no   (multi-task programs: no probabilities per row)
__global__ void __launch_bounds__(256) k_prog_sigmoid_cols(const __nv_bfloat16* __restrict__ x, int64_t ldx, int no, int64_t B, float* __restrict__ prob) {
  const int64_t n = B * (int64_t)no;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / no;
    prob[i] = 1.f / (1.f + __expf(-ldb(x + b * ldx + (i - b * no))));
  }
}

// ---- recurrent / transformer sequence models (DIEN, BST) -------------------------------------------------------------------------------------
// GRU recurrence over the pre-computed input projection gi [B * L, 3H] (the wgmma GEMM x W_ih^T + b_ih): one block per sample, W_hh^T in
// shared memory ([k][j]: consecutive threads read consecutive gate columns), two barriers per time step.  PyTorch gate order r, z, n:
//   r = s(gi_r + W_hr h + b_hr), z = s(gi_z + W_hz h + b_hz), n = tanh(gi_n + r (W_hn h + b_hn)), h' = (1 - z) n + z h
__global__ void __launch_bounds__(256) k_prog_gru(const __nv_bfloat16* __restrict__ gi, int64_t ldg, const float* __restrict__ whh /* [3H][H] */,
                                                  const float* __restrict__ bhh, int L, int H, __nv_bfloat16* __restrict__ y, int64_t ldy, int64_t B) {
  extern __shared__ float sm_gru[];
  float* sW = sm_gru;                       // [H][3H]
  float* sh = sW + 3 * H * H;               // [H] hidden state
  float* sg = sh + H;                       // [3H] W_hh h + b_hh
  const int H3 = 3 * H;
  for (int i = threadIdx.x; i < H3 * H; i += blockDim.x) { const int j = i / H, k = i - j * H; sW[k * H3 + j] = whh[i]; }
  __syncthreads();
  for (int64_t b = blockIdx.x; b < B; b += gridDim.x) {
    for (int j = threadIdx.x; j < H; j += blockDim.x) sh[j] = 0.f;
    __syncthreads();
    for (int t = 0; t < L; ++t) {
      for (int j = threadIdx.x; j < H3; j += blockDim.x) {
        float a = bhh[j];
        for (int k = 0; k < H; ++k) a = fmaf(sW[k * H3 + j], sh[k], a);
        sg[j] = a;
      }
      __syncthreads();
      const __nv_bfloat16* g = gi + (b * L + t) * ldg;
      for (int j = threadIdx.x; j < H; j += blockDim.x) {
        const float r = 1.f / (1.f + __expf(-(ldb(g + j) + sg[j])));
        const float z = 1.f / (1.f + __expf(-(ldb(g + H + j) + sg[H + j])));
        const float n = tanhf(ldb(g + 2 * H + j) + r * sg[2 * H + j]);
        const float h = (1.f - z) * n + z * sh[j];
        sh[j] = h;
        stb(y + b * ldy + (int64_t)t * H + j, h);
      }
      __syncthreads();
    }
  }
}
// y[b, :] = x[b, last(b), :], last = max(sum_l mask[b, l], 1) - 1   (one warp per row)
__global__ void __launch_bounds__(256) k_prog_seq_last(const __nv_bfloat16* __restrict__ x, int64_t ldx, const __nv_bfloat16* __restrict__ m, int64_t ldm, int L, int w,
                                                       __nv_bfloat16* __restrict__ y, int64_t ldy, int64_t B) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < B; r += nwarps) {
    int cnt = 0;
    for (int l = lane; l < L; l += 32) cnt += ldb(m + r * ldm + l) > 0.f ? 1 : 0;
#pragma unroll
    for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    const int last = (cnt > 1 ? cnt : 1) - 1;
    for (int k = lane; k < w; k += 32) y[r * ldy + k] = x[r * ldx + (int64_t)last * w + k];
  }
}
// y[b, :] = mean over the valid positions of x[b, l, :]
__global__ void __launch_bounds__(256) k_prog_seq_mean(const __nv_bfloat16* __restrict__ x, int64_t ldx, const __nv_bfloat16* __restrict__ m, int64_t ldm, int L, int w,
                                                       __nv_bfloat16* __restrict__ y, int64_t ldy, int64_t B) {
  const int64_t n = B * (int64_t)w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / w; const int k = (int)(i - b * w);
    float acc = 0.f; int cnt = 0;
    for (int l = 0; l < L; ++l) if (ldb(m + b * ldm + l) > 0.f) { acc += ldb(x + b * ldx + (int64_t)l * w + k); ++cnt; }
    stb(y + b * ldy + k, acc / (float)(cnt > 1 ? cnt : 1));
  }
}
// multi-head self-attention core: qkv [B, S * 3E] (per position [q | k | v]), valid [B, S] -> [B, S * E].  One block per sample, the sample's qkv
// staged in shared memory as fp32; one thread per (head, query position) runs an online softmax over the valid keys (dh <= 64).
constexpr int kMhaMaxDh = 64;
__global__ void __launch_bounds__(256) k_prog_mha(const __nv_bfloat16* __restrict__ qkv, int64_t ldq, const __nv_bfloat16* __restrict__ valid, int64_t ldv, int S, int E,
                                                  int heads, __nv_bfloat16* __restrict__ y, int64_t ldy, int64_t B) {
  extern __shared__ float sm_mha[];
  float* sx = sm_mha;                       // [S][3E]
  float* sv = sx + (size_t)S * 3 * E;       // [S] validity
  const int dh = E / heads; const float scale = rsqrtf((float)dh);
  for (int64_t b = blockIdx.x; b < B; b += gridDim.x) {
    for (int i = threadIdx.x; i < S * 3 * E; i += blockDim.x) sx[i] = ldb(qkv + b * ldq + i);
    for (int i = threadIdx.x; i < S; i += blockDim.x) sv[i] = ldb(valid + b * ldv + i);
    __syncthreads();
    for (int it = threadIdx.x; it < heads * S; it += blockDim.x) {
      const int hd = it / S, s1 = it - hd * S;
      const float* q = sx + (size_t)s1 * 3 * E + hd * dh;
      float acc[kMhaMaxDh];
      for (int c = 0; c < dh; ++c) acc[c] = 0.f;
      float mx = -3.4e38f, den = 0.f;
      for (int s2 = 0; s2 < S; ++s2) {
        if (!(sv[s2] > 0.f)) continue;
        const float* kk = sx + (size_t)s2 * 3 * E + E + hd * dh;
        float dot = 0.f;
        for (int c = 0; c < dh; ++c) dot = fmaf(q[c], kk[c], dot);
        dot *= scale;
        const float nm = fmaxf(mx, dot), corr = __expf(mx - nm), pe = __expf(dot - nm);
        const float* vv = kk + E;
        for (int c = 0; c < dh; ++c) acc[c] = acc[c] * corr + pe * vv[c];
        den = den * corr + pe; mx = nm;
      }
      const float inv = den > 0.f ? 1.f / den : 0.f;
      for (int c = 0; c < dh; ++c) stb(y + b * ldy + (int64_t)s1 * E + hd * dh + c, acc[c] * inv);
    }
    __syncthreads();
  }
}

inline int grid_el(int64_t n) { const int64_t b = (n + 255) / 256; return (int)(b < 1 ? 1 : b > num_sms() * 8 ? num_sms() * 8 : b); }
inline int grid_rows(int64_t rows) { return grid_el(rows * 32); }

}  // namespace

extern "C" {

int dr_prog_copy_cols(const void* src, int64_t lds, int start, int w, void* dst, int64_t ldd, int off, int64_t B, cudaStream_t s) {
  if (B <= 0 || w <= 0) return 0;
  k_prog_copy_cols<<<grid_el(B * w), 256, 0, s>>>((const __nv_bfloat16*)src, lds, start, w, (__nv_bfloat16*)dst, ldd, off, B);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_prog_affine(const void* x, int64_t ldx, int w, const float* scale, const float* shift, void* y, int64_t ldy, int64_t B, cudaStream_t s) {
  if (B <= 0 || w <= 0) return 0;
  k_prog_affine<<<grid_el(B * w), 256, 0, s>>>((const __nv_bfloat16*)x, ldx, w, scale, shift, (__nv_bfloat16*)y, ldy, B);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_prog_fm(const void* emb, int64_t lde, int T, int D, void* y, int64_t ldy, int64_t B, cudaStream_t s) {
  if (B <= 0 || T <= 0 || D <= 0) return 0;
  k_prog_fm<<<grid_el(B * D), 256, 0, s>>>((const __nv_bfloat16*)emb, lde, T, D, (__nv_bfloat16*)y, ldy, B);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_prog_binary(int kind, const void* a, int64_t lda, const void* b, int64_t ldb, const void* c, int64_t ldc, int w, void* y, int64_t ldy, int64_t B,
                   cudaStream_t s) {
  if (B <= 0 || w <= 0) return 0;
  if (kind < 0 || kind > 2 || (kind == 2 && !c)) return -2;
  k_prog_binary<<<grid_el(B * w), 256, 0, s>>>(kind, (const __nv_bfloat16*)a, lda, (const __nv_bfloat16*)b, ldb, (const __nv_bfloat16*)c, ldc, w, (__nv_bfloat16*)y,
                                               ldy, B);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_prog_cross(const void* x0, int64_t ld0, const void* xl, int64_t ldl, int w, const float* wv, const float* bv, void* y, int64_t ldy, int64_t B, cudaStream_t s) {
  if (B <= 0 || w <= 0) return 0;
  k_prog_cross<<<grid_rows(B), 256, 0, s>>>((const __nv_bfloat16*)x0, ld0, (const __nv_bfloat16*)xl, ldl, w, wv, bv, (__nv_bfloat16*)y, ldy, B);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_prog_layernorm(const void* x, int64_t ldx, int w, const float* gamma, const float* beta, float eps, int relu, void* y, int64_t ldy, int64_t B, cudaStream_t s) {
  if (B <= 0 || w <= 0) return 0;
  k_prog_layernorm<<<grid_rows(B), 256, 0, s>>>((const __nv_bfloat16*)x, ldx, w, gamma, beta, eps, relu, (__nv_bfloat16*)y, ldy, B);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_prog_valid_mask(const int64_t* ids, int64_t stride, int64_t rows, int start, int L, void* y, int64_t ldy, cudaStream_t s) {
  if (rows <= 0 || L <= 0) return 0;
  if (rows > stride) return -2;
  k_prog_valid_mask<<<grid_el(rows * L), 256, 0, s>>>(ids, stride, rows, start, L, (__nv_bfloat16*)y, ldy);
  DR_LAUNCH_CHECK();
  return 0;
}
int dr_prog_seq_zip(const void* a, int64_t lda, int wa, const void* c, int64_t ldc, int wb, int L, void* y, int64_t ldy, int64_t B, cudaStream_t s) {
  if (B <= 0 || L <= 0) return 0;
  k_prog_seq_zip<<<grid_el(B * L * (wa + wb)), 256, 0, s>>>((const __nv_bfloat16*)a, lda, wa, (const __nv_bfloat16*)c, ldc, wb, L, (__nv_bfloat16*)y, ldy, B);
  DR_LAUNCH_CHECK();
  return 0;
}
int dr_prog_seq_mask(const void* x, int64_t ldx, const void* m, int64_t ldm, int L, int w, void* y, int64_t ldy, int64_t B, cudaStream_t s) {
  if (B <= 0 || L <= 0 || w <= 0) return 0;
  k_prog_seq_mask<<<grid_el(B * L * w), 256, 0, s>>>((const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)m, ldm, L, w, (__nv_bfloat16*)y, ldy, B);
  DR_LAUNCH_CHECK();
  return 0;
}
int dr_prog_seq_sum(const void* x, int64_t ldx, int L, int w, void* y, int64_t ldy, int64_t B, cudaStream_t s) {
  if (B <= 0 || L <= 0 || w <= 0) return 0;
  k_prog_seq_sum<<<grid_el(B * w), 256, 0, s>>>((const __nv_bfloat16*)x, ldx, L, w, (__nv_bfloat16*)y, ldy, B);
  DR_LAUNCH_CHECK();
  return 0;
}
int dr_prog_prelu(const void* x, int64_t ldx, int w, const float* alpha, void* y, int64_t ldy, int64_t B, cudaStream_t s) {
  if (B <= 0 || w <= 0) return 0;
  k_prog_prelu<<<grid_el(B * w), 256, 0, s>>>((const __nv_bfloat16*)x, ldx, w, alpha, (__nv_bfloat16*)y, ldy, B);
  DR_LAUNCH_CHECK();
  return 0;
}
int dr_prog_to_f32(const void* x, int64_t ldx, int w, float* y, int64_t B, cudaStream_t s) {
  if (B <= 0 || w <= 0) return 0;
  k_prog_to_f32<<<grid_el(B * w), 256, 0, s>>>((const __nv_bfloat16*)x, ldx, w, y, B);
  DR_LAUNCH_CHECK();
  return 0;
}
int dr_prog_from_f32(const float* x, int w, void* y, int64_t ldy, int64_t B, cudaStream_t s) {
  if (B <= 0 || w <= 0) return 0;
  k_prog_from_f32<<<grid_el(B * w), 256, 0, s>>>(x, w, (__nv_bfloat16*)y, ldy, B);
  DR_LAUNCH_CHECK();
  return 0;
}
int dr_prog_to_u8(const void* x, int64_t ldx, int w, uint8_t* y, int64_t B, cudaStream_t s) {
  if (B <= 0 || w <= 0) return 0;
  k_prog_to_u8<<<grid_el(B * w), 256, 0, s>>>((const __nv_bfloat16*)x, ldx, w, y, B);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_prog_gru(const void* gi, int64_t ldg, const float* whh, const float* bhh, int L, int H, void* y, int64_t ldy, int64_t B, cudaStream_t s) {
  if (B <= 0 || L <= 0 || H <= 0) return 0;
  const size_t bytes = ((size_t)3 * H * H + 4 * (size_t)H) * sizeof(float);
  if (bytes > 200 * 1024) return -1;                                // W_hh must fit in shared memory (H <= 126)
  static DrPerDeviceOnce attr_once; bool& attr = attr_once();
  if (!attr) { DR_CUDA_CHECK(cudaFuncSetAttribute(k_prog_gru, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); attr = true; }
  k_prog_gru<<<(int)(B < num_sms() * 4 ? B : num_sms() * 4), 256, bytes, s>>>((const __nv_bfloat16*)gi, ldg, whh, bhh, L, H, (__nv_bfloat16*)y, ldy, B);
  DR_LAUNCH_CHECK();
  return 0;
}
int dr_prog_seq_last(const void* x, int64_t ldx, const void* m, int64_t ldm, int L, int w, void* y, int64_t ldy, int64_t B, cudaStream_t s) {
  if (B <= 0 || L <= 0 || w <= 0) return 0;
  k_prog_seq_last<<<grid_rows(B), 256, 0, s>>>((const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)m, ldm, L, w, (__nv_bfloat16*)y, ldy, B);
  DR_LAUNCH_CHECK();
  return 0;
}
int dr_prog_seq_mean(const void* x, int64_t ldx, const void* m, int64_t ldm, int L, int w, void* y, int64_t ldy, int64_t B, cudaStream_t s) {
  if (B <= 0 || L <= 0 || w <= 0) return 0;
  k_prog_seq_mean<<<grid_el(B * w), 256, 0, s>>>((const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)m, ldm, L, w, (__nv_bfloat16*)y, ldy, B);
  DR_LAUNCH_CHECK();
  return 0;
}
int dr_prog_mha(const void* qkv, int64_t ldq, const void* valid, int64_t ldv, int S, int E, int heads, void* y, int64_t ldy, int64_t B, cudaStream_t s) {
  if (B <= 0 || S <= 0 || E <= 0) return 0;
  if (heads <= 0 || E % heads || E / heads > kMhaMaxDh) return -2;
  const size_t bytes = ((size_t)S * 3 * E + (size_t)S) * sizeof(float);
  if (bytes > 200 * 1024) return -1;
  static DrPerDeviceOnce attr_once; bool& attr = attr_once();
  if (!attr) { DR_CUDA_CHECK(cudaFuncSetAttribute(k_prog_mha, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); attr = true; }
  k_prog_mha<<<(int)(B < num_sms() * 4 ? B : num_sms() * 4), 256, bytes, s>>>((const __nv_bfloat16*)qkv, ldq, (const __nv_bfloat16*)valid, ldv, S, E, heads, (__nv_bfloat16*)y, ldy, B);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_prog_emb_feature_major(const float* x, int T, int D, int64_t B, void* y, cudaStream_t s) {
  if (B <= 0 || T <= 0 || D <= 0) return 0;
  k_prog_emb_feature_major<<<grid_el(B * T * D), 256, 0, s>>>(x, T, D, B, (__nv_bfloat16*)y);
  DR_LAUNCH_CHECK();
  return 0;
}
int dr_prog_softmax(const void* x, int64_t ldx, int w, void* y, int64_t ldy, int64_t B, cudaStream_t s) {
  if (B <= 0 || w <= 0) return 0;
  k_prog_softmax<<<grid_rows(B), 256, 0, s>>>((const __nv_bfloat16*)x, ldx, w, (__nv_bfloat16*)y, ldy, B);
  DR_LAUNCH_CHECK();
  return 0;
}
int dr_prog_cosine(const void* a, int64_t lda, const void* c, int64_t ldc, int w, void* y, int64_t ldy, int64_t B, cudaStream_t s) {
  if (B <= 0 || w <= 0) return 0;
  k_prog_cosine<<<grid_rows(B), 256, 0, s>>>((const __nv_bfloat16*)a, lda, (const __nv_bfloat16*)c, ldc, w, (__nv_bfloat16*)y, ldy, B);
  DR_LAUNCH_CHECK();
  return 0;
}
int dr_prog_sigmoid_cols(const void* x, int64_t ldx, int no, int64_t B, float* prob, cudaStream_t s) {
  if (B <= 0 || no <= 0) return 0;
  k_prog_sigmoid_cols<<<grid_el(B * no), 256, 0, s>>>((const __nv_bfloat16*)x, ldx, no, B, prob);
  DR_LAUNCH_CHECK();
  return 0;
}

int dr_prog_sigmoid0(const void* x, int64_t ldx, int64_t B, float* prob, cudaStream_t s) {
  if (B <= 0) return 0;
  k_prog_sigmoid0<<<grid_el(B), 256, 0, s>>>((const __nv_bfloat16*)x, ldx, B, prob);
  DR_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
