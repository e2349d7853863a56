// Native serving runtime: Processor C ABI + SessionGroup + model updater (full / delta hot-swap) for the DLRM family.
//
// Parity map (behaviour) to the reference's serving/processor (17.6 kLoC, SURVEY §2.10, §3.6, Appendix A.11-12):
//   C ABI  initialize / process / batch_process / get_serving_model_info, return 200 / 500     serving/processor.cc:9-100
//   ModelConfig JSON (session_num, select_session_policy MOD|RR, gpu id, update threads/interval, warm-up) serving/model_config.cc
//   SessionGroup: N sessions = N CUDA streams with private activation / pinned IO buffers over ONE shared, read-only set
//     of tables + weights (direct_session_group.{h,cc}; "sessions share variables, own streams/threads")
//   ModelUpdater::WorkLoop: poll the version file; new FULL version -> build a fresh model, warm it up, atomically swap,
//     old one reaped when its last request finishes (shared_ptr refcount); new DELTA -> patch rows of the live tables +
//     swap the (small) dense parameter block, no warm-up (model_instance.cc:406-446); invalid versions are skipped.
//   Tracer: per-request stage timings, dumped every N requests (serving/tracer.h).
// The reference embeds the TF runtime and runs a SavedModel graph; here inference is the sm_90a kernel sequence of the
// flagship engine (BatchNorm folded at load time, read-only probes), so a request is ~16 kernel launches on the
// session's stream.
#include <dlfcn.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cmath>
#include <cstdlib>
#include <memory>
#include <mutex>
#include <sstream>
#include <string>
#include <thread>
#include <vector>

#include "../common/bundle.h"
#include "../common/model_config.h"
#include "../common/predict_pb.h"
#include "../common/saved_model.h"
#include "table.cuh"

// kernel launchers from the other translation units of this library
extern "C" {
int dr_cuda_fill_i64(int64_t* p, int64_t v, int64_t n, cudaStream_t s);
int dr_cuda_table_init_slots(void* slots, int64_t n, cudaStream_t s);
int dr_cuda_gemm_fp8_tn(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, const float* col_scale, const float* bias,
                        int relu, void* out, int64_t ldc, int out_fp8, float out_inv_scale, cudaStream_t s);
int dr_cuda_quantize_e4m3(const void* x, int is_bf16, int64_t M, int C, int64_t ldx, void* y, int Cp, float inv_scale, cudaStream_t s);
int dr_cuda_quantize_weights_e4m3(const float* w, int N, int K, int64_t ldw, void* q, int Kp, float* scale, cudaStream_t s);
int dr_cuda_absmax_bf16(const void* x, int64_t n, float* out, cudaStream_t s);
int dr_cuda_table_lookup(const DrDeviceTable* tables_dev, const int32_t* table_map, int T, const int64_t* keys, const int64_t* offsets, int64_t uniform,
                         int64_t n, int train, const int64_t* step_ptr, int32_t* out_pos, int64_t* ulist, int32_t* group_nunique, int64_t ulist_cap, cudaStream_t s);
int dr_cuda_table_gather(const DrDeviceTable* tables_dev, const int32_t* table_map, int T, int dim, const int64_t* keys, const int32_t* pos,
                         const int64_t* offsets, int64_t uniform, int64_t n, void* out, int out_bf16, int64_t stride_b, int64_t stride_t, int flat_out, cudaStream_t s);
int dr_cuda_table_import_cow(const DrDeviceTable* t_host, const int64_t* keys, const float* rows, int ncols, int64_t n, int32_t* retired,
                             int32_t* n_retired, int32_t* n_kept, cudaStream_t s);
int dr_cuda_table_free_rows(const DrDeviceTable* t_host, const int32_t* rows, const int32_t* n_dev, int64_t max_n, cudaStream_t s);
int dr_cuda_table_import(const DrDeviceTable* t_host, const int64_t* keys, const float* rows, int ncols, const int64_t* freqs, const int64_t* versions,
                         int64_t n, int part_id, int part_num, int reset_version, int32_t* n_kept, cudaStream_t s);
int dr_cuda_gemm_tn_ex(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, const float* bias, int relu, const void* mask_src,
                       int64_t ld_mask, int aux_mode, void* out, int64_t ldc, float* out_f32, float* S1, float* S2, int max_ctas, int force_v1, cudaStream_t s);
int dr_cuda_cast_pad(const float* x, int64_t B, int C, void* y, int Cp, cudaStream_t s);
int dr_cuda_bn_apply(const void* a, int64_t B, int N, int64_t lda, const float* scale, const float* shift, void* y, int64_t ldy, cudaStream_t s);
int dr_cuda_dot_interaction_fwd(const void* x, int64_t ldx, const void* emb, int64_t emb_stride_t, int64_t emb_stride_b, int T, int D, int64_t B, void* Z,
                                int64_t ldz, cudaStream_t s);
int dr_prog_copy_cols(const void* src, int64_t lds, int start, int w, void* dst, int64_t ldd, int off, int64_t B, cudaStream_t s);
int dr_prog_affine(const void* x, int64_t ldx, int w, const float* scale, const float* shift, void* y, int64_t ldy, int64_t B, cudaStream_t s);
int dr_prog_fm(const void* emb, int64_t lde, int T, int D, void* y, int64_t ldy, int64_t B, cudaStream_t s);
int dr_prog_binary(int kind, const void* a, int64_t lda, const void* b, int64_t ldb, const void* c, int64_t ldc, int w, void* y, int64_t ldy, int64_t B, cudaStream_t s);
int dr_prog_cross(const void* x0, int64_t ld0, const void* xl, int64_t ldl, int w, const float* wv, const float* bv, void* y, int64_t ldy, int64_t B, cudaStream_t s);
int dr_prog_layernorm(const void* x, int64_t ldx, int w, const float* gamma, const float* beta, float eps, int relu, void* y, int64_t ldy, int64_t B, cudaStream_t s);
int dr_prog_sigmoid0(const void* x, int64_t ldx, int64_t B, float* prob, cudaStream_t s);
int dr_prog_valid_mask(const int64_t* ids, int64_t stride, int64_t rows, int start, int L, void* y, int64_t ldy, cudaStream_t s);
int dr_prog_seq_zip(const void* a, int64_t lda, int wa, const void* c, int64_t ldc, int wb, int L, void* y, int64_t ldy, int64_t B, cudaStream_t s);
int dr_prog_seq_mask(const void* x, int64_t ldx, const void* m, int64_t ldm, int L, int w, void* y, int64_t ldy, int64_t B, cudaStream_t s);
int dr_prog_seq_sum(const void* x, int64_t ldx, int L, int w, void* y, int64_t ldy, int64_t B, cudaStream_t s);
int dr_prog_prelu(const void* x, int64_t ldx, int w, const float* alpha, void* y, int64_t ldy, int64_t B, cudaStream_t s);
int dr_prog_to_f32(const void* x, int64_t ldx, int w, float* y, int64_t B, cudaStream_t s);
int dr_prog_from_f32(const float* x, int w, void* y, int64_t ldy, int64_t B, cudaStream_t s);
int dr_prog_to_u8(const void* x, int64_t ldx, int w, uint8_t* y, int64_t B, cudaStream_t s);
int dr_prog_softmax(const void* x, int64_t ldx, int w, void* y, int64_t ldy, int64_t B, cudaStream_t s);
int dr_prog_cosine(const void* a, int64_t lda, const void* c, int64_t ldc, int w, void* y, int64_t ldy, int64_t B, cudaStream_t s);
int dr_prog_sigmoid_cols(const void* x, int64_t ldx, int no, int64_t B, float* prob, cudaStream_t s);
int dr_prog_emb_feature_major(const float* x, int T, int D, int64_t B, void* y, cudaStream_t s);
int dr_prog_gru(const void* gi, int64_t ldg, const float* whh, const float* bhh, int L, int H, void* y, int64_t ldy, int64_t B, cudaStream_t s);
int dr_prog_seq_last(const void* x, int64_t ldx, const void* m, int64_t ldm, int L, int w, void* y, int64_t ldy, int64_t B, cudaStream_t s);
int dr_prog_seq_mean(const void* x, int64_t ldx, const void* m, int64_t ldm, int L, int w, void* y, int64_t ldy, int64_t B, cudaStream_t s);
int dr_prog_seq_sqrtn(const void* x, int64_t ldx, const void* m, int64_t ldm, int L, int w, void* y, int64_t ldy, int64_t B, cudaStream_t s);
int dr_cuda_gemm_tn_cross(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, const float* bias, int kind,
                          const void* x0, int64_t ld_x0, const void* xl, int64_t ld_xl, void* out, int64_t ldc, void* u_out, int64_t ld_u,
                          int max_ctas, cudaStream_t s);
int dr_prog_mha(const void* qkv, int64_t ldq, const void* valid, int64_t ldv, int S, int E, int heads, void* y, int64_t ldy, int64_t B, cudaStream_t s);
int dr_cuda_din_attention_fwd_w(const float* q, const float* k, const uint8_t* mask, int64_t B, int L, int D, const float* W1, const float* b1, int H1,
                                const float* W2, const float* b2, int H2, const float* w3, float b3, float* out, float* weights_out, cudaStream_t s);
int dr_cuda_din_attention_fwd(const float* q, const float* k, const uint8_t* mask, int64_t B, int L, int D, const float* W1, const float* b1, int H1,
                              const float* W2, const float* b2, int H2, const float* w3, float b3, float* out, cudaStream_t s);
int dr_cuda_head(const void* h, int64_t ldh, int64_t B, int K, const float* w, const float* bias, const float* labels, float inv_batch, float* prob,
                 float* loss_sum, void* dh, float* dw, float* db, int relu_mask, int train, float* dbias_h, cudaStream_t s);
}

namespace serve {
using namespace drsm;

// ---- device placement optimisation (ModelConfig "enable_device_placement_optimization", the reference's gpu_device_placement_pass.cc: the embedding
// layer stays on the CPU for GPU inference) -- the tables live in the HOST engine (libdeeprec_host.so next to this library, bound at run time so
// that the GPU library keeps no link-time dependency on it): tables larger than HBM, or one copy shared by the replicas of every GPU of a box.
// A request looks its rows up on the caller's thread, ships them as one H2D copy and runs the dense part on the GPU as usual.
struct HostApi {
  void* (*create)(const DrEvConfig*) = nullptr; void (*destroy)(void*) = nullptr; void (*set_default)(void*, const float*) = nullptr;
  int64_t (*import)(void*, const int64_t*, const float*, int64_t, const int64_t*, const int64_t*, int64_t, int, int, int) = nullptr;
  int64_t (*import_cow)(void*, const int64_t*, const float*, int64_t, int64_t) = nullptr;
  void (*group_lookup)(void**, int, const int64_t*, int64_t, float*) = nullptr;
  bool ok = false;
  static HostApi& Get() {
    static HostApi api = [] {
      HostApi a;
      Dl_info info{};
      std::string dir = ".";
      if (dladdr((void*)&HostApi::Get, &info) && info.dli_fname) { dir = info.dli_fname; const size_t p = dir.find_last_of('/'); dir = p == std::string::npos ? "." : dir.substr(0, p); }
      void* h = dlopen((dir + "/libdeeprec_host.so").c_str(), RTLD_NOW | RTLD_LOCAL);
      if (!h) { fprintf(stderr, "[deeprec_serving] device placement optimisation needs %s/libdeeprec_host.so: %s\n", dir.c_str(), dlerror()); return a; }
      a.create = (decltype(a.create))dlsym(h, "dr_host_ev_create"); a.destroy = (decltype(a.destroy))dlsym(h, "dr_host_ev_destroy");
      a.set_default = (decltype(a.set_default))dlsym(h, "dr_host_ev_set_default"); a.import = (decltype(a.import))dlsym(h, "dr_host_ev_import");
      a.import_cow = (decltype(a.import_cow))dlsym(h, "dr_host_ev_import_cow"); a.group_lookup = (decltype(a.group_lookup))dlsym(h, "dr_host_group_lookup");
      a.ok = a.create && a.destroy && a.set_default && a.import && a.import_cow && a.group_lookup;
      return a;
    }();
    return api;
  }
};

#define SV_CUDA(expr) do { cudaError_t _e = (expr); if (_e != cudaSuccess) { fprintf(stderr, "[deeprec_serving] %s: %s\n", #expr, cudaGetErrorString(_e)); return false; } } while (0)

static uint16_t f2bf(float f) { uint32_t u; memcpy(&u, &f, 4); uint32_t r = 0x7FFF + ((u >> 16) & 1); return (uint16_t)((u + r) >> 16); }

struct DevBuf {      // owning, move-only device allocation
  void* p = nullptr; size_t n = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), n(o.n) { o.p = nullptr; o.n = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept { if (this != &o) { if (p) cudaFree(p); p = o.p; n = o.n; o.p = nullptr; o.n = 0; } return *this; }
  bool alloc(size_t bytes) { if (p) { cudaFree(p); p = nullptr; } n = bytes; return cudaMalloc(&p, bytes ? bytes : 16) == cudaSuccess; }
  ~DevBuf() { if (p) cudaFree(p); }
  template <typename T> T* as() const { return static_cast<T*>(p); }
};
template <typename T> static bool Upload(DevBuf& b, const std::vector<T>& h) {
  if (!b.alloc(h.size() * sizeof(T))) return false;
  return cudaMemcpy(b.p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice) == cudaSuccess;
}

struct LayerW {
  int N, K, Kp; DevBuf w_bf16, bias;
  int Np = 0;              // program LINEAR: output channels padded to a tile the GEMM tests cover (16 | 32 | multiple of 8 above)
  // fp8 serving path: E4M3 weights [N, Kp16] quantised per output channel; col_scale[n] = w_scale[n] * in_scale
  int Kp16 = 0; DevBuf w_fp8, w_scale, col_scale;
};
static inline int pad16(int n) { return (n + 15) / 16 * 16; }

// static activation scales (amax / 448 with head-room) measured by Calibrate(); index: 0 = x0, 1.. = bottom activations
struct ActScales { std::vector<float> bot_in, top_in; bool valid = false; };

// dense parameter block (small; swapped as a whole on full AND delta updates)
struct DenseParams {
  std::vector<LayerW> bot, top;
  DevBuf last_scale, last_shift, head_w, head_b;
  bool fp8 = false;        // fp8 tensors + scales below are populated
  ActScales act;
  // program models: per-op weights (LINEAR: bf16 [pad8(N), pad8(K)] + bias[pad8(N)]; affine / layernorm / cross: two fp32 vectors), buffer widths
  struct PW { LayerW L; DevBuf v0, v1; std::vector<DevBuf> att; int H1 = 0, H2 = 0; float b3 = 0.f; };    // gru: L = input projection [3H, I], v0 = W_hh, v1 = b_hh, H1 = H    // att: W1 b1 W2 b2 w3 of a din_attention op
  std::vector<PW> pdata; std::vector<int> width;
};

struct TableDev {
  DrDeviceTable t{}; DevBuf slots, rows, free_list, counters, def;
  int64_t n_rows = 0;
  std::vector<int64_t> sample_keys;     // a few stored keys: calibration / warm-up batches look up rows that exist
};

struct DeviceModel {
  Arch arch; int64_t version = -1; std::string path;
  std::shared_ptr<DenseParams> dense;
  std::vector<std::unique_ptr<TableDev>> tables;
  DevBuf structs;      // DrDeviceTable[T] on the device
  DevBuf col_table;    // int32 [C]: table of every lookup column (program models; identity otherwise)
  // device placement optimisation: the tables live in the host engine instead (HostEV handles, owned), col_handles[c] = table of lookup column c
  bool host_resident = false; std::vector<void*> host_tables, col_handles;
  ~DeviceModel() { if (host_resident) for (void* h : host_tables) if (h) HostApi::Get().destroy(h); }
};

// fp8 path: E4M3 copy of a layer's fp32 weights W' [N, Kp], one scale per output channel
static bool QuantizeLayer(LayerW& L, const std::vector<float>& w_folded /*[N, Kp]*/) {
  L.Kp16 = pad16(L.Kp);
  DevBuf tmp;
  if (!Upload(tmp, w_folded) || !L.w_fp8.alloc((size_t)L.N * L.Kp16) || !L.w_scale.alloc((size_t)L.N * 4) || !L.col_scale.alloc((size_t)L.N * 4)) return false;
  if (dr_cuda_quantize_weights_e4m3(tmp.as<float>(), L.N, L.Kp, L.Kp, L.w_fp8.p, L.Kp16, L.w_scale.as<float>(), 0) != 0) return false;
  return cudaDeviceSynchronize() == cudaSuccess;
}

// col_scale[n] = w_scale[n] * in_scale for every layer, from the calibrated activation scales
static bool ApplyActScales(DenseParams& dp) {
  auto one = [](LayerW& L, float in_scale) {
    std::vector<float> ws((size_t)L.N);
    if (cudaMemcpy(ws.data(), L.w_scale.p, ws.size() * 4, cudaMemcpyDeviceToHost) != cudaSuccess) return false;
    for (auto& v : ws) v *= in_scale;
    return cudaMemcpy(L.col_scale.p, ws.data(), ws.size() * 4, cudaMemcpyHostToDevice) == cudaSuccess;
  };
  for (size_t l = 0; l < dp.bot.size(); ++l) if (!one(dp.bot[l], dp.act.bot_in[l])) return false;
  for (size_t l = 0; l < dp.top.size(); ++l) if (!one(dp.top[l], dp.act.top_in[l])) return false;
  dp.fp8 = true;
  return true;
}

// Row pitch of a program buffer (bf16 elements).  Buffers 0 / 1 are the cast dense inputs and the gathered embeddings; every other buffer
// is padded like a GEMM output: 16 | 32 for narrow layers (full N tiles of the direct-store kernel), a multiple of 8 above (TMA 16-byte rule).
static int prog_npad(int w) { return w <= 16 ? 16 : w <= 32 ? 32 : pad8(w); }
static int prog_ld(const Arch& a, const std::vector<int>& width, int id) { return id == 0 ? pad8(a.num_dense) : id == 1 ? a.C * a.D : prog_npad(width[(size_t)id]); }

// Device layout of a program model's weights: LINEAR as bf16 [Np, Kp] with zero pad rows / columns, GRU's input projection as bf16 [3H, I],
// the other vectors fp32.  The checks here are the kernels' own: a sequence buffer is a [B * len, w] matrix only when its rows are not
// padded, the GEMM's 8-element rule, the recurrence kernel's H <= 126 and the attention kernel's head width <= 64.
static bool BuildProgram(dr::BundleReader& r, const Arch& a, std::shared_ptr<DenseParams>* out) {
  ProgramData p;
  if (!ReadProgram(r, a, &p)) return false;
  auto dp = std::make_shared<DenseParams>();
  dp->pdata.resize(a.ops.size());
  for (size_t i = 0; i < a.ops.size(); ++i) {
    const POp& op = a.ops[i]; const OpTensors& t = p.ops[i]; auto& d = dp->pdata[i];
    const int w0 = p.width[(size_t)op.in[0]];
    const bool unpadded = prog_ld(a, p.width, op.in[0]) == w0;
    d.H1 = t.H1; d.H2 = t.H2;
    if ((!t.v0.empty() && !Upload(d.v0, t.v0)) || (!t.v1.empty() && !Upload(d.v1, t.v1))) return false;
    switch (op.kind) {
      case P_LINEAR: {                                               // len > 1: [B, len * K] == [B * len, K], no output padding either
        const int S = op.len > 0 ? op.len : 1, N = t.N, K = t.K;
        if (S > 1 && (!unpadded || K % 8 || prog_npad(N) != N || prog_npad(S * N) != S * N)) return false;
        const int Np = prog_npad(N), Kp = S > 1 ? K : prog_ld(a, p.width, op.in[0]);
        std::vector<uint16_t> wb((size_t)Np * Kp, 0); std::vector<float> bias((size_t)Np, 0.f);     // zero rows / columns: pad outputs are exact zeros
        for (int n = 0; n < N; ++n) { bias[(size_t)n] = t.b[(size_t)n]; for (int k = 0; k < K; ++k) wb[(size_t)n * Kp + k] = f2bf(t.W[(size_t)n * K + k]); }
        d.L.N = N; d.L.K = K; d.L.Kp = Kp; d.L.Np = Np;
        if (!Upload(d.L.w_bf16, wb) || !Upload(d.L.bias, bias)) return false;
        break;
      }
      case P_LAYERNORM: if (op.len > 1 && !unpadded) return false; break;
      case P_GRU: {                                                  // input projection on the GEMM ([B * L, I] x W_ih^T + b_ih -> [B * L, 3H]), recurrence kernel
        if (!unpadded || t.K % 8 || t.N % 8 || t.H1 > 126) return false;
        std::vector<uint16_t> wb(t.W.size());
        for (size_t k = 0; k < wb.size(); ++k) wb[k] = f2bf(t.W[k]);
        d.L.N = t.N; d.L.K = t.K; d.L.Kp = t.K; d.L.Np = t.N;
        if (!Upload(d.L.w_bf16, wb) || !Upload(d.L.bias, t.b)) return false;
        break;
      }
      case P_MHA: if (w0 / (3 * op.len) / op.heads > 64) return false; break;
      case P_CROSS_LINEAR: {                                         // dr_cuda_gemm_tn_cross over the padded widths: A = t [B, Kp], kernel [Np, Kp], x0 / x_l / out [B, Np]
        const int N = t.N, K = t.K, Np = prog_npad(N), Kp = prog_ld(a, p.width, op.in[2]);
        const int64_t ld_x0 = prog_ld(a, p.width, op.in[0]), ld_xl = prog_ld(a, p.width, op.in[1]);
        if (Kp % 8 || Np % 8 || ld_x0 % 8 || ld_xl % 8 || ld_x0 < Np || ld_xl < Np || Kp < K) {
          fprintf(stderr, "[deeprec_serving] cross_linear op %s: the cross GEMM needs pitches that are multiples of 8 and at least the padded width "
                          "(N %d padded to %d, rank %d, pitches x0 %lld, x_l %lld, t %d)\n", op.name.c_str(), N, Np, K, (long long)ld_x0, (long long)ld_xl, Kp);
          return false;
        }
        std::vector<uint16_t> wb((size_t)Np * Kp, 0); std::vector<float> bias((size_t)Np, 0.f);     // zero pad rows / bias: pad outputs stay x_l's zeros
        for (int n = 0; n < N; ++n) { bias[(size_t)n] = t.b[(size_t)n]; for (int k = 0; k < K; ++k) wb[(size_t)n * Kp + k] = f2bf(t.W[(size_t)n * K + k]); }
        d.L.N = N; d.L.K = K; d.L.Kp = Kp; d.L.Np = Np;
        if (!Upload(d.L.w_bf16, wb) || !Upload(d.L.bias, bias)) return false;
        break;
      }
      case P_DIN_ATT:
        d.b3 = t.att[5][0]; d.att.resize(5);
        for (int k = 0; k < 5; ++k) if (!Upload(d.att[(size_t)k], t.att[(size_t)k])) return false;
        break;
      default: break;
    }
  }
  dp->width = std::move(p.width);
  *out = dp;
  return true;
}

// DLRM: bf16 weights (and their E4M3 copy for the fp8 path) of the BatchNorm-folded layers
static bool BuildDense(dr::BundleReader& r, const Arch& a, std::shared_ptr<DenseParams>* out, bool want_fp8 = false) {
  if (a.program) return BuildProgram(r, a, out);
  DlrmDense t;
  if (!ReadDlrmDense(r, a, &t)) return false;
  auto dp = std::make_shared<DenseParams>();
  auto layer = [&](const DenseLayer& s, LayerW& L) {
    L.N = s.N; L.K = s.K; L.Kp = s.Kp;
    std::vector<uint16_t> wb(s.W.size());
    for (size_t i = 0; i < wb.size(); ++i) wb[i] = f2bf(s.W[i]);
    return Upload(L.w_bf16, wb) && Upload(L.bias, s.b) && (!want_fp8 || QuantizeLayer(L, s.W));
  };
  dp->bot.resize(t.bot.size()); dp->top.resize(t.top.size());
  for (size_t l = 0; l < t.bot.size(); ++l) if (!layer(t.bot[l], dp->bot[l])) return false;
  for (size_t l = 0; l < t.top.size(); ++l) if (!layer(t.top[l], dp->top[l])) return false;
  if (!Upload(dp->last_scale, t.last_scale) || !Upload(dp->last_shift, t.last_shift) || !Upload(dp->head_w, t.head_w) || !Upload(dp->head_b, t.head_b)) return false;
  *out = dp;
  return true;
}

static int64_t NextPow2(int64_t n) { int64_t p = 1; while (p < n) p <<= 1; return p; }

static bool BuildTable(const TableData& in, int D, TableDev* td, int64_t extra_rows) {
  const int64_t n = (int64_t)in.keys.size();
  const int64_t rows = n + extra_rows, cap = NextPow2(std::max<int64_t>(1024, 2 * rows));
  auto& T = td->t;
  if (!td->slots.alloc((size_t)cap * sizeof(DrSlot)) ||
      !td->rows.alloc((size_t)rows * D * 4) || !td->free_list.alloc(rows * 4 + 16) || !td->counters.alloc(32) || !Upload(td->def, in.def)) return false;
  dr_cuda_table_init_slots(td->slots.p, cap, 0);
  cudaMemset(td->counters.p, 0, 32);
  T.slots = td->slots.as<DrSlot>();
  T.rows = td->rows.as<float>(); T.free_list = td->free_list.as<int32_t>();
  T.counters = td->counters.as<int32_t>(); T.default_matrix = td->def.as<float>(); T.bloom = nullptr;
  T.capacity = cap; T.row_capacity = rows; T.default_value_dim = (int64_t)in.def.size() / D; T.bloom_m = 0;
  T.dim = D; T.stride = D; T.num_slots = 0; T.has_scalars = 0; T.filter_type = 0; T.filter_freq = 0; T.bloom_k = 0; T.is_inference = 1;
  T.no_permission = 0.f; T.steps_to_live = 0; T.l2_weight_threshold = -1.f;
  td->n_rows = n;
  if (n) {
    DevBuf dk, dv, df, dver, kept;
    if (!Upload(dk, in.keys) || !Upload(dv, in.values) || !kept.alloc(4)) return false;
    cudaMemset(kept.p, 0, 4);
    if (!in.freqs.empty()) Upload(df, in.freqs);
    if (!in.versions.empty()) Upload(dver, in.versions);
    if (dr_cuda_table_import(&T, dk.as<int64_t>(), dv.as<float>(), D, in.freqs.empty() ? nullptr : df.as<int64_t>(), in.versions.empty() ? nullptr : dver.as<int64_t>(),
                             n, 0, 1, 0, kept.as<int32_t>(), 0) != 0) return false;
    SV_CUDA(cudaDeviceSynchronize());
  }
  return true;
}

// host-resident twin of BuildTable (device placement optimisation): the rows go into a HostEV of the host engine
static void* BuildHostTable(const TableData& in, int D) {
  HostApi& api = HostApi::Get();
  if (!api.ok) return nullptr;
  DrEvConfig c{};
  c.dim = D; c.num_slots = 0; c.has_scalars = 0; c.init_capacity = std::max<int64_t>(1024, (int64_t)in.keys.size() * 2);
  c.default_value_dim = (int64_t)in.def.size() / D; c.num_partitions = 16; c.record_freq = 1; c.record_version = 1; c.l2_weight_threshold = -1.f;
  void* h = api.create(&c);
  if (!h) return nullptr;
  api.set_default(h, in.def.data());
  if (!in.keys.empty())
    api.import(h, in.keys.data(), in.values.data(), D, in.freqs.empty() ? nullptr : in.freqs.data(), in.versions.empty() ? nullptr : in.versions.data(),
               (int64_t)in.keys.size(), 0, 1, 0);
  return h;
}

static std::shared_ptr<DeviceModel> LoadModel(const std::string& dir, int64_t extra_rows, bool want_fp8 = false, bool host_tables = false) {
  auto m = std::make_shared<DeviceModel>();
  const Arch& a = m->arch;
  std::string prefix;
  // a program's embedding buffer doubles as a GEMM operand: its row pitch C * D must obey the 16-byte rule; rows are gathered as float4 groups
  if (!ParseArch(dir, &m->arch, &m->version, &prefix) || (a.program && (a.D % 4 || (a.C * a.D) % 8))) {
    fprintf(stderr, "[deeprec_serving] bad saved_model.json in %s\n", dir.c_str()); return nullptr;
  }
  dr::BundleReader r(prefix);
  if (!r.ok()) { fprintf(stderr, "[deeprec_serving] cannot open bundle %s\n", prefix.c_str()); return nullptr; }
  if (!BuildDense(r, a, &m->dense, want_fp8 && !a.program)) { fprintf(stderr, "[deeprec_serving] dense parameters incomplete in %s\n", prefix.c_str()); return nullptr; }
  m->host_resident = host_tables;                                    // device placement optimisation: embedding layer on the CPU
  std::vector<DrDeviceTable> structs;
  for (int t = 0; t < a.T; ++t) {
    m->tables.emplace_back(new TableDev());
    TableDev& dev = *m->tables.back();
    TableData td;
    if (!ReadTable(r, t, a.D, &td)) { fprintf(stderr, "[deeprec_serving] table %d incomplete\n", t); return nullptr; }
    dev.sample_keys.assign(td.keys.begin(), td.keys.begin() + std::min<size_t>(td.keys.size(), 512));
    if (host_tables) {
      void* h = BuildHostTable(td, a.D);
      if (!h) { fprintf(stderr, "[deeprec_serving] host table %d not created (libdeeprec_host.so missing?)\n", t); return nullptr; }
      m->host_tables.push_back(h);
    } else {
      if (!BuildTable(td, a.D, &dev, extra_rows)) { fprintf(stderr, "[deeprec_serving] table %d not created\n", t); return nullptr; }
      structs.push_back(dev.t);
    }
  }
  if (host_tables) {
    for (int c = 0; c < a.C; ++c) m->col_handles.push_back(m->host_tables[(size_t)a.col_table[(size_t)c]]);
  } else {
    std::vector<int32_t> ct(a.col_table.begin(), a.col_table.end());
    if (!Upload(m->structs, structs) || !Upload(m->col_table, ct)) return nullptr;
  }
  m->path = dir;
  return m;
}

// ---------------------------------------------------------------------------------------------------------------
struct Session {
  cudaStream_t stream = nullptr; int max_batch = 0; std::mutex mu;
  DevBuf dense_in, ids, x0, emb, pos, Z, prob, loss, labels, y_last;
  std::vector<DevBuf> a_bot, a_top;
  DevBuf x0_q, Z_q, amax; std::vector<DevBuf> q_bot, q_top;        // fp8 path: E4M3 activations between the GEMMs
  float* h_dense = nullptr; int64_t* h_ids = nullptr; float* h_prob = nullptr;    // pinned
  float* h_emb = nullptr; DevBuf emb_f32;                            // host-resident tables: looked-up rows [B, C, D] fp32 (pinned) and their device copy
  // rows of this chunk from the host engine -> one H2D copy -> bf16 in the layout the dense part expects (program: [B, C * D]; DLRM: [T][B][D])
  bool HostLookup(const DeviceModel& m, int B) {
    const Arch& a = m.arch; cudaStream_t s = stream;
    const size_t n = (size_t)B * a.C * a.D;
    if (!h_emb) { SV_CUDA(cudaMallocHost(&h_emb, (size_t)max_batch * a.C * a.D * 4)); if (!emb_f32.alloc((size_t)max_batch * a.C * a.D * 4)) return false; }
    HostApi::Get().group_lookup(const_cast<void**>(m.col_handles.data()), a.C, h_ids, B, h_emb);
    SV_CUDA(cudaMemcpyAsync(emb_f32.p, h_emb, n * 4, cudaMemcpyHostToDevice, s));
    const int rc = a.program ? dr_prog_from_f32(emb_f32.as<float>(), a.C * a.D, emb.p, (int64_t)a.C * a.D, B, s)
                             : dr_prog_emb_feature_major(emb_f32.as<float>(), a.C, a.D, B, emb.p, s);
    return rc == 0;
  }
  bool Init(const Arch& a, int maxB) {
    max_batch = maxB;
    SV_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    bool ok = dense_in.alloc((size_t)maxB * a.num_dense * 4) && ids.alloc((size_t)a.C * maxB * 8) && x0.alloc((size_t)maxB * pad8(a.num_dense) * 2) &&
              emb.alloc((size_t)a.C * maxB * a.D * 2) && pos.alloc((size_t)a.C * maxB * 4) && Z.alloc((size_t)maxB * a.Zp * 2) && prob.alloc((size_t)maxB * a.n_out * 4) &&
              loss.alloc(16) && labels.alloc((size_t)maxB * 4) && y_last.alloc((size_t)maxB * a.D * 2);
    a_bot.resize(a.bot.size()); a_top.resize(a.top.size());
    for (size_t l = 0; l < a.bot.size(); ++l) ok = ok && a_bot[l].alloc((size_t)maxB * a.bot[l] * 2);
    for (size_t l = 0; l < a.top.size(); ++l) ok = ok && a_top[l].alloc((size_t)maxB * a.top[l] * 2);
    q_bot.resize(a.bot.size()); q_top.resize(a.top.size());
    ok = ok && x0_q.alloc((size_t)maxB * pad16(a.num_dense)) && Z_q.alloc((size_t)maxB * pad16(a.Zp)) && amax.alloc(64);
    for (size_t l = 0; l < a.bot.size(); ++l) ok = ok && q_bot[l].alloc((size_t)maxB * pad16(a.bot[l]));
    for (size_t l = 0; l < a.top.size(); ++l) ok = ok && q_top[l].alloc((size_t)maxB * pad16(a.top[l]));
    if (!ok) return false;
    cudaMemset(labels.p, 0, (size_t)maxB * 4);
    SV_CUDA(cudaMallocHost(&h_dense, (size_t)maxB * a.num_dense * 4));
    SV_CUDA(cudaMallocHost(&h_ids, (size_t)a.C * maxB * 8));
    SV_CUDA(cudaMallocHost(&h_prob, (size_t)maxB * a.n_out * 4));
    return true;
  }
  ~Session() { if (h_dense) cudaFreeHost(h_dense); if (h_ids) cudaFreeHost(h_ids); if (h_prob) cudaFreeHost(h_prob); if (h_emb) cudaFreeHost(h_emb); if (stream) cudaStreamDestroy(stream); }

  // ---- op-program models: buffers 0 / 1 alias x0 / emb, the others are (max_batch x prog_ld(width)) bf16, zeroed once (pad columns stay zero) ----
  std::vector<DevBuf> pbuf; std::vector<int> pbuf_width;
  DevBuf att_q, att_k, att_o, att_m, att_w;                          // fp32 / uint8 staging of the din_attention kernel (att_w: its softmax weights)
  DevBuf gru_gi;                                                     // bf16 [max_batch * L, 3H]: input projection of a gru op
  bool RunProgram(const DeviceModel& m, const DenseParams& dp, const int Bfull) {
    const Arch& a = m.arch; cudaStream_t s = stream;
    if (pbuf_width != dp.width) {                                     // first program run, or a full update changed the layer widths
      SV_CUDA(cudaStreamSynchronize(s));
      pbuf.clear(); pbuf.resize(dp.width.size());
      for (size_t i = 2; i < dp.width.size(); ++i) {
        const size_t bytes = (size_t)max_batch * prog_ld(a, dp.width, (int)i) * 2;
        if (!pbuf[i].alloc(bytes)) return false;
        SV_CUDA(cudaMemsetAsync(pbuf[i].p, 0, bytes, s));
      }
      size_t wq = 0, wk = 0, wl = 0, wg = 0;
      for (size_t oi = 0; oi < a.ops.size(); ++oi) {
        const POp& op = a.ops[oi];
        if (op.kind == P_DIN_ATT) { wq = std::max(wq, (size_t)dp.width[(size_t)op.in[0]]); wk = std::max(wk, (size_t)dp.width[(size_t)op.in[1]]); wl = std::max(wl, (size_t)dp.width[(size_t)op.in[2]]); }
        if (op.kind == P_GRU) wg = std::max(wg, (size_t)op.len * 3 * (size_t)dp.pdata[oi].H1);
      }
      if (wq && (!att_q.alloc((size_t)max_batch * wq * 4) || !att_k.alloc((size_t)max_batch * wk * 4) || !att_o.alloc((size_t)max_batch * wq * 4) || !att_m.alloc((size_t)max_batch * wl) ||
                 !att_w.alloc((size_t)max_batch * wl * 4))) return false;
      if (wg && !gru_gi.alloc((size_t)max_batch * wg * 2)) return false;
      pbuf_width = dp.width;
    }
    auto buf = [&](int id) -> void* { return id == 0 ? x0.p : id == 1 ? emb.p : pbuf[(size_t)id].p; };
    auto ld = [&](int id) -> int64_t { return prog_ld(a, dp.width, id); };
    int rc = 0;
    const int64_t n = (int64_t)a.C * Bfull;
    const int32_t* ct = m.col_table.as<int32_t>();                   // lookup column -> table
    if (m.host_resident) { if (!HostLookup(m, Bfull)) return false; }
    else {
      rc |= dr_cuda_table_lookup(m.structs.as<DrDeviceTable>(), ct, a.C, ids.as<int64_t>(), nullptr, Bfull, n, 0, nullptr, pos.as<int32_t>(), nullptr, nullptr, 0, s);
      // sample-major embeddings [B, C * D]: element (b, c) at b * (C * D) + c * D
      rc |= dr_cuda_table_gather(m.structs.as<DrDeviceTable>(), ct, a.C, a.D, ids.as<int64_t>(), pos.as<int32_t>(), nullptr, Bfull, n, emb.p, 1, (int64_t)a.C * a.D, a.D, 0, s);
    }
    rc |= dr_cuda_cast_pad(dense_in.as<float>(), Bfull, a.num_dense, x0.p, pad8(a.num_dense), s);
    for (size_t oi = 0; oi < a.ops.size() && rc == 0; ++oi) {
      const POp& op = a.ops[oi]; const auto& pd = dp.pdata[oi];
      const int B = op.rows1 ? 1 : Bfull;                            // sample-aware compression: user-side ops once per request (row 0 of their inputs)
      void* out = buf(op.out); const int W = dp.width[(size_t)op.out]; const int64_t ldo = ld(op.out);
      const void* a0 = buf(op.in[0]); const int w0 = dp.width[(size_t)op.in[0]]; const int64_t ld0 = ld(op.in[0]);
      switch (op.kind) {
        case P_LINEAR:                                               // wgmma GEMM, bias (+ ReLU) in the epilogue; N padded to 8 with zero rows
          if (op.len > 1)                                            // sequence form: [B, S * K] is a [B * S, K] matrix (un-padded buffers, checked at load)
            rc |= dr_cuda_gemm_tn_ex(a0, pd.L.K, pd.L.w_bf16.p, pd.L.Kp, B * op.len, pd.L.Np, pd.L.Kp, pd.L.bias.as<float>(), op.relu ? 1 : 0, nullptr, 0, 0, out, pd.L.N,
                                     nullptr, nullptr, nullptr, 0, 0, s);
          else
            rc |= dr_cuda_gemm_tn_ex(a0, ld0, pd.L.w_bf16.p, pd.L.Kp, B, pd.L.Np, pd.L.Kp, pd.L.bias.as<float>(), op.relu ? 1 : 0, nullptr, 0, 0, out, ldo,
                                     nullptr, nullptr, nullptr, 0, 0, s);
          break;
        case P_GRU: {
          const int L = op.len, I = w0 / L, H = pd.H1;
          rc |= dr_cuda_gemm_tn_ex(a0, I, pd.L.w_bf16.p, I, B * L, 3 * H, I, pd.L.bias.as<float>(), 0, nullptr, 0, 0, gru_gi.p, 3 * H, nullptr, nullptr, nullptr, 0, 0, s);
          rc |= dr_prog_gru(gru_gi.p, 3 * H, pd.v0.as<float>(), pd.v1.as<float>(), L, H, out, ldo, B, s);
          break;
        }
        case P_SEQ_LAST: rc |= dr_prog_seq_last(a0, ld0, buf(op.in[1]), ld(op.in[1]), op.len, W, out, ldo, B, s); break;
        case P_SEQ_MEAN:
          if (op.mode == 1) rc |= dr_prog_seq_sqrtn(a0, ld0, buf(op.in[1]), ld(op.in[1]), op.len, W, out, ldo, B, s);
          else rc |= dr_prog_seq_mean(a0, ld0, buf(op.in[1]), ld(op.in[1]), op.len, W, out, ldo, B, s);
          break;
        case P_CROSS_LINEAR:                                         // x0 * (t W^T + b) + x_l in the GEMM epilogue (the DCNv2 training forward)
          rc |= dr_cuda_gemm_tn_cross(buf(op.in[2]), ld(op.in[2]), pd.L.w_bf16.p, pd.L.Kp, B, pd.L.Np, pd.L.Kp, pd.L.bias.as<float>(), 1, a0, ld0,
                                      buf(op.in[1]), ld(op.in[1]), out, ldo, nullptr, 0, 0, s);
          break;
        case P_MHA: rc |= dr_prog_mha(a0, ld0, buf(op.in[1]), ld(op.in[1]), op.len, W / op.len, op.heads, out, ldo, B, s); break;
        case P_CONCAT: {
          int off = 0;
          for (int src : op.in) { const int w = dp.width[(size_t)src]; rc |= dr_prog_copy_cols(buf(src), ld(src), 0, w, out, ldo, off, B, s); off += w; }
          break;
        }
        case P_AFFINE: rc |= dr_prog_affine(a0, ld0, W, pd.v0.as<float>(), pd.v1.as<float>(), out, ldo, B, s); break;
        case P_FM: rc |= dr_prog_fm(a0, ld0, a.C, a.D, out, ldo, B, s); break;
        case P_CROSS: rc |= dr_prog_cross(a0, ld0, buf(op.in[1]), ld(op.in[1]), W, pd.v0.as<float>(), pd.v1.as<float>(), out, ldo, B, s); break;
        case P_ADD: rc |= dr_prog_binary(0, a0, ld0, buf(op.in[1]), ld(op.in[1]), nullptr, 0, W, out, ldo, B, s); break;
        case P_MUL: rc |= dr_prog_binary(1, a0, ld0, buf(op.in[1]), ld(op.in[1]), nullptr, 0, W, out, ldo, B, s); break;
        case P_MUL_ADD: rc |= dr_prog_binary(2, a0, ld0, buf(op.in[1]), ld(op.in[1]), buf(op.in[2]), ld(op.in[2]), W, out, ldo, B, s); break;
        case P_SLICE: rc |= dr_prog_copy_cols(a0, ld0, op.start, W, out, ldo, 0, B, s); break;
        case P_LAYERNORM:
          if (op.len > 1) rc |= dr_prog_layernorm(a0, W / op.len, W / op.len, pd.v0.as<float>(), pd.v1.as<float>(), op.eps, op.relu ? 1 : 0, out, W / op.len, (int64_t)B * op.len, s);
          else rc |= dr_prog_layernorm(a0, ld0, W, pd.v0.as<float>(), pd.v1.as<float>(), op.eps, op.relu ? 1 : 0, out, ldo, B, s);
          break;
        case P_VALID_MASK: rc |= dr_prog_valid_mask(ids.as<int64_t>(), Bfull, B, op.start, W, out, ldo, s); break;
        case P_TILE: rc |= dr_prog_copy_cols(a0, /*row pitch 0: broadcast row 0*/ 0, 0, W, out, ldo, 0, B, s); break;
        case P_SEQ_ZIP: { const int L = op.len, wb = dp.width[(size_t)op.in[1]]; rc |= dr_prog_seq_zip(a0, ld0, w0 / L, buf(op.in[1]), ld(op.in[1]), wb / L, L, out, ldo, B, s); break; }
        case P_SEQ_MASK: rc |= dr_prog_seq_mask(a0, ld0, buf(op.in[1]), ld(op.in[1]), op.len, W / op.len, out, ldo, B, s); break;
        case P_SEQ_SUM: rc |= dr_prog_seq_sum(a0, ld0, op.len, W, out, ldo, B, s); break;
        case P_PRELU: rc |= dr_prog_prelu(a0, ld0, W, pd.v0.as<float>(), out, ldo, B, s); break;
        case P_SOFTMAX: rc |= dr_prog_softmax(a0, ld0, W, out, ldo, B, s); break;
        case P_COSINE: rc |= dr_prog_cosine(a0, ld0, buf(op.in[1]), ld(op.in[1]), w0, out, ldo, B, s); break;
        case P_DIN_ATT: {                                            // fp32 staging -> the fused attention kernel (attention_kernels.cu) -> bf16
          const int L = dp.width[(size_t)op.in[2]], Wq = w0;         // mode 1 (DIEN): the output is the softmax weights [B, L], not the weighted sum [B, Wq]
          rc |= dr_prog_to_f32(a0, ld0, Wq, att_q.as<float>(), B, s);
          rc |= dr_prog_to_f32(buf(op.in[1]), ld(op.in[1]), L * Wq, att_k.as<float>(), B, s);
          rc |= dr_prog_to_u8(buf(op.in[2]), ld(op.in[2]), L, att_m.as<uint8_t>(), B, s);
          rc |= dr_cuda_din_attention_fwd_w(att_q.as<float>(), att_k.as<float>(), att_m.as<uint8_t>(), B, L, Wq, pd.att[0].as<float>(), pd.att[1].as<float>(), pd.H1,
                                            pd.att[2].as<float>(), pd.att[3].as<float>(), pd.H2, pd.att[4].as<float>(), pd.b3, att_o.as<float>(),
                                            op.mode == 1 ? att_w.as<float>() : nullptr, s);
          if (op.mode == 1) rc |= dr_prog_from_f32(att_w.as<float>(), L, out, ldo, B, s);
          else rc |= dr_prog_from_f32(att_o.as<float>(), Wq, out, ldo, B, s);
          break;
        }
        default: rc = -1;
      }
      (void)w0;
    }
    rc |= dr_prog_sigmoid_cols(buf(a.out_buf), ld(a.out_buf), a.n_out, Bfull, prob.as<float>(), s);
    return rc == 0;
  }

  // inputs already in h_dense / h_ids ([T][B] feature-major); result in h_prob
  bool Run(const DeviceModel& m, const DenseParams& dp, int B, bool force_bf16 = false) {
    const Arch& a = m.arch; cudaStream_t s = stream;
    SV_CUDA(cudaMemcpyAsync(dense_in.p, h_dense, (size_t)B * a.num_dense * 4, cudaMemcpyHostToDevice, s));
    SV_CUDA(cudaMemcpyAsync(ids.p, h_ids, (size_t)a.C * B * 8, cudaMemcpyHostToDevice, s));
    if (a.program) {
      if (!RunProgram(m, dp, B)) return false;
      SV_CUDA(cudaMemcpyAsync(h_prob, prob.p, (size_t)B * a.n_out * 4, cudaMemcpyDeviceToHost, s));
      SV_CUDA(cudaStreamSynchronize(s));
      return true;
    }
    int rc = 0;
    const int64_t n = (int64_t)a.T * B;
    if (m.host_resident) { if (!HostLookup(m, B)) return false; }
    else {
      rc |= dr_cuda_table_lookup(m.structs.as<DrDeviceTable>(), nullptr, a.T, ids.as<int64_t>(), nullptr, B, n, 0, nullptr, pos.as<int32_t>(), nullptr, nullptr, 0, s);
      rc |= dr_cuda_table_gather(m.structs.as<DrDeviceTable>(), nullptr, a.T, a.D, ids.as<int64_t>(), pos.as<int32_t>(), nullptr, B, n, emb.p, 1, 0, 0, 1, s);
    }
    const void* x; int64_t ldx;
    if (dp.fp8 && !force_bf16) {
      // ---- E4M3 path: every hidden activation stays 8-bit; each GEMM epilogue re-quantises with the next layer's static scale
      const int c0 = pad16(a.num_dense);
      rc |= dr_cuda_quantize_e4m3(dense_in.p, 0, B, a.num_dense, a.num_dense, x0_q.p, c0, 1.0f / dp.act.bot_in[0], s);
      x = x0_q.p; ldx = c0;
      const size_t nb = dp.bot.size();
      for (size_t l = 0; l < nb; ++l) {
        const LayerW& L = dp.bot[l];
        const bool last = l + 1 == nb;        // the last bottom layer feeds BatchNorm + the bf16 interaction kernel
        rc |= dr_cuda_gemm_fp8_tn(x, ldx, L.w_fp8.p, L.Kp16, B, L.N, L.Kp16, L.col_scale.as<float>(), L.bias.as<float>(), 1,
                                  last ? a_bot[l].p : q_bot[l].p, last ? L.N : pad16(L.N), last ? 0 : 1, last ? 1.f : 1.0f / dp.act.bot_in[l + 1], s);
        x = last ? a_bot[l].p : q_bot[l].p; ldx = last ? L.N : pad16(L.N);
      }
      rc |= dr_cuda_bn_apply(x, B, a.D, a.D, dp.last_scale.as<float>(), dp.last_shift.as<float>(), y_last.p, a.D, s);
      rc |= dr_cuda_dot_interaction_fwd(y_last.p, a.D, emb.p, (int64_t)B * a.D, a.D, a.T, a.D, B, Z.p, a.Zp, s);
      rc |= dr_cuda_quantize_e4m3(Z.p, 1, B, a.Zp, a.Zp, Z_q.p, pad16(a.Zp), 1.0f / dp.act.top_in[0], s);
      x = Z_q.p; ldx = pad16(a.Zp);
      const size_t nt = dp.top.size();
      for (size_t l = 0; l < nt; ++l) {
        const LayerW& L = dp.top[l];
        const bool last = l + 1 == nt;        // the head kernel consumes bf16
        rc |= dr_cuda_gemm_fp8_tn(x, ldx, L.w_fp8.p, L.Kp16, B, L.N, L.Kp16, L.col_scale.as<float>(), L.bias.as<float>(), 1,
                                  last ? a_top[l].p : q_top[l].p, last ? L.N : pad16(L.N), last ? 0 : 1, last ? 1.f : 1.0f / dp.act.top_in[l + 1], s);
        x = last ? a_top[l].p : q_top[l].p; ldx = last ? L.N : pad16(L.N);
      }
    } else {
    rc |= dr_cuda_cast_pad(dense_in.as<float>(), B, a.num_dense, x0.p, pad8(a.num_dense), s);
    x = x0.p; ldx = pad8(a.num_dense);
    for (size_t l = 0; l < dp.bot.size(); ++l) {
      const LayerW& L = dp.bot[l];
      rc |= dr_cuda_gemm_tn_ex(x, ldx, L.w_bf16.p, L.Kp, B, L.N, L.Kp, L.bias.as<float>(), 1, nullptr, 0, 0, a_bot[l].p, L.N, nullptr, nullptr, nullptr, 0, 0, s);
      x = a_bot[l].p; ldx = L.N;
    }
    rc |= dr_cuda_bn_apply(x, B, a.D, a.D, dp.last_scale.as<float>(), dp.last_shift.as<float>(), y_last.p, a.D, s);
    rc |= dr_cuda_dot_interaction_fwd(y_last.p, a.D, emb.p, (int64_t)B * a.D, a.D, a.T, a.D, B, Z.p, a.Zp, s);
    x = Z.p; ldx = a.Zp;
    for (size_t l = 0; l < dp.top.size(); ++l) {
      const LayerW& L = dp.top[l];
      rc |= dr_cuda_gemm_tn_ex(x, ldx, L.w_bf16.p, L.Kp, B, L.N, L.Kp, L.bias.as<float>(), 1, nullptr, 0, 0, a_top[l].p, L.N, nullptr, nullptr, nullptr, 0, 0, s);
      x = a_top[l].p; ldx = L.N;
    }
    }
    rc |= dr_cuda_head(x, ldx, B, (int)ldx, dp.head_w.as<float>(), dp.head_b.as<float>(), labels.as<float>(), 1.0f / B, prob.as<float>(), loss.as<float>(),
                       nullptr, nullptr, nullptr, 0, 0, nullptr, s);
    if (rc) return false;
    SV_CUDA(cudaMemcpyAsync(h_prob, prob.p, (size_t)B * 4, cudaMemcpyDeviceToHost, s));
    SV_CUDA(cudaStreamSynchronize(s));
    return true;
  }
};

// Static activation scales for the fp8 path: run the bf16 forward on a calibration batch and take amax of every tensor that is
// stored in E4M3 (network input, hidden activations, interaction output); scale = 2 * amax / 448 (2x head-room: E4M3 keeps 3
// mantissa bits down to 2^-6 of full scale, so head-room is cheap, saturation is not).
static bool Calibrate(Session& ss, const DeviceModel& m, DenseParams& dp, int B) {
  const Arch& a = m.arch;
  if (!ss.Run(m, dp, B, /*force_bf16=*/true)) return false;
  auto amax_of = [&](const DevBuf& buf, int64_t n, float* out) {
    if (dr_cuda_absmax_bf16(buf.p, n, ss.amax.as<float>(), ss.stream) != 0) return false;
    if (cudaMemcpyAsync(out, ss.amax.p, 4, cudaMemcpyDeviceToHost, ss.stream) != cudaSuccess) return false;
    return cudaStreamSynchronize(ss.stream) == cudaSuccess;
  };
  auto to_scale = [](float amax) { return std::max(amax, 1e-6f) * 2.0f / 448.0f; };
  dp.act.bot_in.assign(dp.bot.size(), 1.f); dp.act.top_in.assign(dp.top.size(), 1.f);
  float v = 0.f;
  if (!amax_of(ss.x0, (int64_t)B * pad8(a.num_dense), &v)) return false;
  dp.act.bot_in[0] = to_scale(v);
  for (size_t l = 0; l + 1 < dp.bot.size(); ++l) { if (!amax_of(ss.a_bot[l], (int64_t)B * dp.bot[l].N, &v)) return false; dp.act.bot_in[l + 1] = to_scale(v); }
  if (!amax_of(ss.Z, (int64_t)B * a.Zp, &v)) return false;
  dp.act.top_in[0] = to_scale(v);
  for (size_t l = 0; l + 1 < dp.top.size(); ++l) { if (!amax_of(ss.a_top[l], (int64_t)B * dp.top[l].N, &v)) return false; dp.act.top_in[l + 1] = to_scale(v); }
  dp.act.valid = true;
  return ApplyActScales(dp);
}

struct Config {
  bool fp8 = false, host_tables = false;                 // host_tables: "enable_device_placement_optimization" -- embedding lookups on the CPU
  int session_num = 2, select_policy = 0 /*0 RR, 1 MOD*/, gpu_id = 0, max_batch = 4096, update_interval_ms = 1000, extra_rows = 1 << 16;
  int timeline_start_step = -1, timeline_interval_step = 0, timeline_trace_count = 0;
  std::string savedmodel_dir, checkpoint_dir, warmup_file_name, timeline_path;
};

struct ServingModel {
  Config cfg;
  drcfg::Compat compat;                    // reference ModelConfig keys without a 1:1 field (csrc/common/model_config.h)
  std::shared_ptr<DeviceModel> model;      // swapped atomically on full update (std::atomic_load / atomic_store)
  std::vector<std::unique_ptr<Session>> sessions;
  std::atomic<uint64_t> rr{0}, requests{0}, failures{0}, full_updates{0}, delta_updates{0};
  std::atomic<int64_t> delta_version{-1};
  int64_t rejected_version = -1;           // updater thread only: last version refused because it changes the architecture
  struct Retired { int t; std::shared_ptr<DevBuf> rows; int64_t n; };
  std::vector<Retired> retired;            // updater thread only: slab rows replaced by the last delta (copy-on-write), freed at the next one
  std::thread updater; std::atomic<bool> stop{false};
  std::mutex tmu; std::vector<std::string> trace;
  ~ServingModel() { stop = true; if (updater.joinable()) updater.join(); }
};

static int Predict(ServingModel* sm, const void* in, int in_size, void** out, int* out_size, int hint) {
  auto m = std::atomic_load(&sm->model);
  if (!m || in_size < (int)sizeof(drpb::WireReq)) return 500;
  drpb::WireReq h; memcpy(&h, in, sizeof(h));
  const Arch& a = m->arch;
  const size_t need = sizeof(h) + (size_t)h.batch * h.num_dense * 4 + (size_t)h.num_sparse * h.batch * 8;
  if (h.magic != drpb::kWireReqMagic || (int)h.num_dense != a.num_dense || (int)h.num_sparse != a.R || h.batch == 0 || (size_t)in_size < need) return 500;
  uint64_t pick = sm->cfg.select_policy == 1 ? (hint >= 0 ? (uint64_t)hint : std::hash<std::thread::id>()(std::this_thread::get_id())) : sm->rr.fetch_add(1);
  const size_t ns = sm->sessions.size();
  Session* sp = sm->sessions[pick % ns].get();
  std::vector<float> probs((size_t)h.batch * a.n_out);
  auto t0 = std::chrono::steady_clock::now();
  {
    // MOD: the caller / hint owns its session.  RR: start at the round-robin slot and take the first IDLE session (a serial caller still
    // rotates through the sessions; concurrent callers no longer queue behind a busy session while another one is free)
    std::unique_lock<std::mutex> l(sp->mu, std::defer_lock);
    if (sm->cfg.select_policy == 1) l.lock();
    else {
      bool got = false;
      for (size_t i = 0; i < ns && !got; ++i) {
        Session* c = sm->sessions[(pick + i) % ns].get();
        std::unique_lock<std::mutex> t(c->mu, std::try_to_lock);
        if (t.owns_lock()) { l = std::move(t); sp = c; got = true; }
      }
      if (!got) l.lock();
    }
    Session& s = *sp;
    cudaSetDevice(sm->cfg.gpu_id);
    auto dense = std::atomic_load(&m->dense);
    const uint8_t* p = static_cast<const uint8_t*>(in) + sizeof(h);
    for (uint32_t off = 0; off < h.batch; off += s.max_batch) {          // requests larger than a session's buffers are chunked
      const int B = (int)std::min<uint32_t>(s.max_batch, h.batch - off);
      memcpy(s.h_dense, p + (size_t)off * a.num_dense * 4, (size_t)B * a.num_dense * 4);
      const int64_t* ids = reinterpret_cast<const int64_t*>(p + (size_t)h.batch * a.num_dense * 4);
      for (int c = 0; c < a.C; ++c) memcpy(s.h_ids + (size_t)c * B, ids + (size_t)a.id_map[(size_t)c] * h.batch + off, (size_t)B * 8);
      if (!s.Run(*m, *dense, B)) { sm->failures++; return 500; }
      memcpy(probs.data() + (size_t)off * a.n_out, s.h_prob, (size_t)B * a.n_out * 4);
    }
  }
  const uint64_t rq = ++sm->requests;
  if (sm->cfg.timeline_interval_step > 0 && (int64_t)rq >= sm->cfg.timeline_start_step && (rq % sm->cfg.timeline_interval_step) == 0 &&
      (int)sm->trace.size() < sm->cfg.timeline_trace_count) {
    double us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
    std::lock_guard<std::mutex> l(sm->tmu);
    char line[160]; snprintf(line, sizeof(line), "{\"request\": %llu, \"batch\": %u, \"latency_us\": %.1f, \"model_version\": %lld}", (unsigned long long)rq, h.batch, us, (long long)m->version);
    sm->trace.emplace_back(line);
    if (!sm->cfg.timeline_path.empty()) { FILE* f = fopen(sm->cfg.timeline_path.c_str(), "a"); if (f) { fprintf(f, "%s\n", line); fclose(f); } }
  }
  drpb::WireResp rh{drpb::kWireRespMagic, h.batch, 200, (uint32_t)(a.n_out > 1 ? a.n_out : 0), m->version};        // reserved = probabilities per row (0: one)
  *out_size = (int)(sizeof(rh) + probs.size() * 4);
  *out = malloc(*out_size);
  memcpy(*out, &rh, sizeof(rh)); memcpy(static_cast<uint8_t*>(*out) + sizeof(rh), probs.data(), probs.size() * 4);
  return 200;
}

// delta update: rows of the touched keys are patched into the LIVE tables; the dense block is rebuilt and swapped
static bool ApplyDelta(ServingModel* sm, const std::string& prefix, int64_t version) {
  auto m = std::atomic_load(&sm->model);
  if (!m) return false;
  dr::BundleReader r(prefix);
  if (!r.ok()) return false;
  cudaSetDevice(sm->cfg.gpu_id);
  // rows replaced by the PREVIOUS delta: no request that could still read them is in flight once every session has been idle once
  if (!sm->retired.empty()) {
    for (auto& sp : sm->sessions) { std::lock_guard<std::mutex> l(sp->mu); cudaStreamSynchronize(sp->stream); }
    for (auto& rt : sm->retired)
      if (rt.t < (int)m->tables.size()) dr_cuda_table_free_rows(&m->tables[rt.t]->t, rt.rows->as<int32_t>(), rt.rows->as<int32_t>() + rt.n, rt.n, 0);
    cudaDeviceSynchronize();
    sm->retired.clear();
  }
  for (int t = 0; t < m->arch.T; ++t) {
    std::vector<int64_t> keys; std::vector<float> vals;
    if (!ReadDeltaRows(r, t, m->arch.D, &keys, &vals)) return false;
    if (keys.empty()) continue;
    if (m->host_resident) {                                          // host engine: copy-on-write import, readers never see a torn row
      HostApi::Get().import_cow(m->host_tables[(size_t)t], keys.data(), vals.data(), m->arch.D, (int64_t)keys.size());
      continue;
    }
    // copy-on-write: live sessions keep reading complete rows (old or new) while the delta lands; the replaced rows are recycled at
    // the NEXT delta, after every session has passed a quiescent point (Quiesce below) -- CPU runtime: dr_host_ev_import_cow
    DevBuf dk, dv, cnt;
    auto retired = std::make_shared<DevBuf>();
    if (!Upload(dk, keys) || !Upload(dv, vals) || !cnt.alloc(16) || !retired->alloc(keys.size() * 4 + 16)) return false;
    cudaMemset(cnt.p, 0, 16);
    int32_t* n_retired = retired->as<int32_t>() + keys.size();            // counter lives behind the list
    cudaMemset(n_retired, 0, 4);
    if (dr_cuda_table_import_cow(&m->tables[t]->t, dk.as<int64_t>(), dv.as<float>(), m->arch.D, (int64_t)keys.size(), retired->as<int32_t>(), n_retired,
                                 cnt.as<int32_t>(), 0) != 0) return false;
    cudaDeviceSynchronize();
    sm->retired.push_back({t, retired, (int64_t)keys.size()});
  }
  std::shared_ptr<DenseParams> dp;
  if (HasDenseBlock(r, m->arch) && BuildDense(r, m->arch, &dp, sm->cfg.fp8)) {
    if (sm->cfg.fp8 && !m->arch.program) {       // delta updates keep the calibrated activation scales of the serving model (no warm-up on deltas)
      auto old = std::atomic_load(&m->dense);
      dp->act = old->act;
      if (!dp->act.valid || !ApplyActScales(*dp)) return false;
    }
    std::atomic_store(&m->dense, dp);
  }
  sm->delta_version = version;
  sm->delta_updates++;
  return true;
}

// Warm-up / calibration batch: the request stored in warmup_file_name (wire format of process()) when present, else a
// deterministic synthetic batch -- dense features spread over the log-transformed Criteo range, ids cycling over stored keys.
static int FillWarmupBatch(ServingModel* sm, const DeviceModel& m, Session& s) {
  const Arch& a = m.arch;
  int B = std::min(256, s.max_batch);
  std::string raw;
  if (!sm->cfg.warmup_file_name.empty() && drjson::ReadFile(sm->cfg.warmup_file_name, &raw) && raw.size() >= sizeof(drpb::WireReq)) {
    drpb::WireReq h; memcpy(&h, raw.data(), sizeof(h));
    const size_t need = sizeof(h) + (size_t)h.batch * h.num_dense * 4 + (size_t)h.num_sparse * h.batch * 8;
    if (h.magic == drpb::kWireReqMagic && (int)h.num_dense == a.num_dense && (int)h.num_sparse == a.R && h.batch > 0 && raw.size() >= need) {
      B = std::min<int>(h.batch, s.max_batch);
      const float* d = reinterpret_cast<const float*>(raw.data() + sizeof(h));
      const int64_t* ids = reinterpret_cast<const int64_t*>(raw.data() + sizeof(h) + (size_t)h.batch * h.num_dense * 4);
      memcpy(s.h_dense, d, (size_t)B * a.num_dense * 4);
      for (int c = 0; c < a.C; ++c) memcpy(s.h_ids + (size_t)c * B, ids + (size_t)a.id_map[(size_t)c] * h.batch, (size_t)B * 8);
      return B;
    }
  }
  for (int b = 0; b < B; ++b)
    for (int j = 0; j < a.num_dense; ++j) s.h_dense[(size_t)b * a.num_dense + j] = (float)((b * 31 + j * 17) % 97) / 97.0f * 8.0f;
  for (int c = 0; c < a.C; ++c) {
    const auto& sk = m.tables[(size_t)a.col_table[(size_t)c]]->sample_keys;
    for (int b = 0; b < B; ++b) s.h_ids[(size_t)c * B + b] = sk.empty() ? 0 : sk[(size_t)(b * 7 + c) % sk.size()];
  }
  return B;
}

static bool WarmUp(ServingModel* sm, const std::shared_ptr<DeviceModel>& m, const ActScales* reuse = nullptr) {
  bool first = true;
  for (auto& s : sm->sessions) {
    std::lock_guard<std::mutex> l(s->mu);
    const int B = FillWarmupBatch(sm, *m, *s);
    auto dense = std::atomic_load(&m->dense);
    if (sm->cfg.fp8 && !m->arch.program && first && !dense->fp8) {
      if (reuse && reuse->valid && reuse->bot_in.size() == dense->bot.size() && reuse->top_in.size() == dense->top.size()) {
        dense->act = *reuse;
        if (!ApplyActScales(*dense)) return false;
      } else if (!Calibrate(*s, *m, *dense, B)) {
        fprintf(stderr, "[deeprec_serving] fp8 calibration failed\n");
        return false;
      }
    }
    first = false;
    if (!s->Run(*m, *dense, B)) return false;
  }
  return true;
}

static void UpdaterLoop(ServingModel* sm) {
  int bad = 0;
  auto load_full = [&](int64_t v, const std::string& dir) {
    auto cur = std::atomic_load(&sm->model);
    cudaSetDevice(sm->cfg.gpu_id);
    auto nm = LoadModel(dir, sm->cfg.extra_rows, sm->cfg.fp8, sm->cfg.host_tables);
    if (!nm) { if (++bad > 3) fprintf(stderr, "[deeprec_serving] skipping invalid model version %lld\n", (long long)v); return; }
    bad = 0;
    // The sessions' device / pinned buffers were sized from the architecture they were initialised with (Session::Init): a version with
    // more tables, a larger D, more dense columns or wider layers would overflow them.  Such a version is rejected (logged once) -- the
    // reference would build a fresh SessionGroup (serving/processor/serving/model_instance.cc:406-427); restart the processor for it.
    const Arch& o = cur->arch; const Arch& n = nm->arch;
    if (n.num_dense != o.num_dense || n.T != o.T || n.D != o.D || n.bot != o.bot || n.top != o.top || n.Zp != o.Zp || n.program != o.program || n.R != o.R || n.C != o.C || n.n_out != o.n_out) {
      if (sm->rejected_version != v) {
        fprintf(stderr, "[deeprec_serving] model version %lld changes the architecture (tables %d->%d, D %d->%d, dense %d->%d): rejected, sessions keep serving version %lld\n",
                (long long)v, o.T, n.T, o.D, n.D, o.num_dense, n.num_dense, (long long)cur->version);
        sm->rejected_version = v;
      }
      return;
    }
    if (!WarmUp(sm, nm)) return;
    std::atomic_store(&sm->model, nm);          // requests in flight keep the old model alive through their shared_ptr
    sm->retired.clear();
    sm->delta_version = -1;
    sm->full_updates++;
  };
  RunUpdater(sm->cfg.checkpoint_dir.empty() ? sm->cfg.savedmodel_dir : sm->cfg.checkpoint_dir, sm->cfg.update_interval_ms, sm->stop, sm->model, sm->delta_version,
             load_full, [&](int64_t v, const std::string& prefix) { ApplyDelta(sm, prefix, v); });
}

// protobuf PredictRequest (reference predict.proto wire format) -> compact request -> Predict -> PredictResponse
static int PredictProto(ServingModel* sm, const void* in, int in_size, void** out, int* out_size, int hint) {
  auto m = std::atomic_load(&sm->model);
  if (!m) return 500;
  drpb::Request rq;
  std::string wire, err, pb;
  if (!drpb::ParseRequest(in, (size_t)in_size, &rq) || !drpb::RequestToWire(rq, m->arch.num_dense, m->arch.R, &wire, &err)) { sm->failures++; return 500; }
  void* w_out = nullptr; int w_size = 0;
  const int rc = Predict(sm, wire.data(), (int)wire.size(), &w_out, &w_size, hint);
  if (rc != 200) { free(w_out); return rc; }
  const bool ok = drpb::WireToResponse(w_out, (size_t)w_size, rq.output_filter, &pb);
  free(w_out);
  if (!ok) return 500;
  *out_size = (int)pb.size();
  *out = malloc(pb.size() ? pb.size() : 1);
  memcpy(*out, pb.data(), pb.size());
  return 200;
}

static int PredictAny(ServingModel* sm, const void* in, int in_size, void** out, int* out_size, int hint) {
  return drpb::IsWireRequest(in, (size_t)std::max(in_size, 0)) ? Predict(sm, in, in_size, out, out_size, hint) : PredictProto(sm, in, in_size, out, out_size, hint);
}

}  // namespace serve

extern "C" {

// model_entry: saved-model directory (may be empty if the JSON config names it).  Returns an opaque model handle.
void* initialize(const char* model_entry, const char* model_config, int* state) {
  using namespace serve;
  auto* sm = new ServingModel();
  drjson::JVal j;
  if (model_config && *model_config && !drjson::ParseJson(model_config, &j)) { *state = -1; delete sm; return nullptr; }
  Config& c = sm->cfg;
  sm->compat = drcfg::ParseCompat(j, "deeprec_cuda_serving");                 // every reference ModelConfig key classified (csrc/common/model_config.h)
  if (!sm->compat.error.empty()) { *state = -1; delete sm; return nullptr; }
  c.session_num = (int)j.n("session_num", 2); c.gpu_id = (int)j.n("gpu_id", sm->compat.first_gpu >= 0 ? sm->compat.first_gpu : 0); c.max_batch = (int)j.n("max_batch", 4096);
  c.select_policy = j.s("select_session_policy", "RR") == "MOD" ? 1 : 0;
  c.update_interval_ms = (int)j.n("model_update_interval_ms", 1000); c.extra_rows = (int)j.n("delta_extra_rows", 1 << 16);
  c.savedmodel_dir = j.s("savedmodel_dir", model_entry ? model_entry : ""); c.checkpoint_dir = j.s("checkpoint_dir", "");
  c.warmup_file_name = j.s("warmup_file_name", ""); c.timeline_path = j.s("timeline_path", "");
  c.timeline_start_step = (int)j.n("timeline_start_step", -1); c.timeline_interval_step = (int)j.n("timeline_interval_step", 0);
  c.timeline_trace_count = (int)j.n("timeline_trace_count", 0);
  if (cudaSetDevice(c.gpu_id) != cudaSuccess) { *state = -1; delete sm; return nullptr; }
  c.fp8 = j.s("mlp_dtype", "bf16") == "fp8";
  c.host_tables = j.n("enable_device_placement_optimization", 0) != 0 || j.s("embedding_placement", "device") == "host";
  auto m = LoadModel(c.savedmodel_dir, c.extra_rows, c.fp8, c.host_tables);
  if (!m) { *state = -1; delete sm; return nullptr; }
  for (int i = 0; i < std::max(1, c.session_num); ++i) {
    sm->sessions.emplace_back(new Session());
    if (!sm->sessions.back()->Init(m->arch, c.max_batch)) { *state = -1; delete sm; return nullptr; }
  }
  if (!WarmUp(sm, m)) { *state = -1; delete sm; return nullptr; }
  std::atomic_store(&sm->model, m);
  if (c.update_interval_ms > 0) sm->updater = std::thread(UpdaterLoop, sm);
  *state = 0;
  return sm;
}

int process(void* model_buf, const void* input_data, int input_size, void** output_data, int* output_size) {
  if (!model_buf) return 500;
  return serve::PredictAny(static_cast<serve::ServingModel*>(model_buf), input_data, input_size, output_data, output_size, -1);
}

int batch_process(void* model_buf, const void* input_data[], int* input_size, void* output_data[], int* output_size) {
  // input_size[0] = number of requests, followed by their sizes (reference: one call, several PredictRequests)
  if (!model_buf || !input_size) return 500;
  int n = input_size[0], rc = 200;
  for (int i = 0; i < n; ++i) {
    int r = serve::PredictAny(static_cast<serve::ServingModel*>(model_buf), input_data[i], input_size[i + 1], &output_data[i], &output_size[i], i);
    if (r != 200) rc = r;
  }
  return rc;
}

int get_serving_model_info(void* model_buf, void** output_data, int* output_size) {
  if (!model_buf) return 500;
  auto* sm = static_cast<serve::ServingModel*>(model_buf);
  auto m = std::atomic_load(&sm->model);
  std::ostringstream os;
  os << "{\"model_version\": " << (m ? m->version : -1) << ", \"delta_version\": " << sm->delta_version.load() << ", \"model_path\": \"" << (m ? m->path : "")
     << "\", \"sessions\": " << sm->sessions.size() << ", \"requests\": " << sm->requests.load() << ", \"failures\": " << sm->failures.load()
     << ", \"mlp_dtype\": \"" << (sm->cfg.fp8 ? "fp8" : "bf16") << "\", \"embedding_placement\": \"" << (sm->cfg.host_tables ? "host" : "device") << "\", \"full_updates\": " << sm->full_updates.load() << ", \"delta_updates\": " << sm->delta_updates.load()
     << ", \"gpu_id\": " << sm->cfg.gpu_id << ", \"model_config\": " << drcfg::ToJson(sm->compat) << "}";
  std::string s = os.str();
  *output_size = (int)s.size();
  *output_data = malloc(s.size() + 1);
  memcpy(*output_data, s.c_str(), s.size() + 1);
  return 200;
}

void dr_serving_release(void* model_buf) { delete static_cast<serve::ServingModel*>(model_buf); }
void dr_serving_free(void* p) { free(p); }

}  // extern "C"
