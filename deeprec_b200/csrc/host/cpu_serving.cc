// CPU serving runtime: the Processor for hosts without a GPU (the reference's processor is deployed on CPU boxes first of all:
// serving/processor/, docs/docs_en/Processor.md).  Same saved-model directory, same request encodings (compact "DRRQ" or the
// reference's protobuf PredictRequest), same ModelConfig JSON, same full / delta hot-swap protocol (serving_versions.json) and the
// same four entry points as the GPU runtime in csrc/cuda/serving_runtime.cu -- exported here with a `dr_cpu_` prefix because both
// libraries can live in one process.
//
//   tables      read-only HostEV instances (is_inference: lookups never create keys), looked up with ONE grouped call per chunk
//   dense net   fp32; BatchNorm (moving statistics) of layer l folded into Linear l+1 at load time, weights stored transposed
//               [K][N] so the GEMM vectorises over the outputs; ReLU fused; DLRM dot interaction via the host kernel
//   sessions    N scratch-buffer sets behind mutexes, picked round-robin or by hint / thread id (SessionGroup semantics);
//               the math of one request runs on the process's OpenMP pool
//   updates     a polling thread: newer full version -> load, warm up, atomic swap (in-flight requests keep the old model alive
//               through their shared_ptr); delta for the current version -> rows patched into the live tables, dense block swapped
#include <sched.h>
#if defined(__x86_64__)
#include <immintrin.h>
#endif
#ifdef _OPENMP
#include <omp.h>
#endif

#include <algorithm>
#include <atomic>
#include <cctype>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <mutex>
#include <sstream>
#include <string>
#include <thread>
#include <vector>

#include "../common/bundle.h"
#include "../common/ev_types.h"
#include "../common/mini_json.h"
#include "../common/model_config.h"
#include "../common/predict_pb.h"
#include "../common/saved_model.h"

extern "C" {
void* dr_host_ev_create(const DrEvConfig* cfg);
void dr_host_ev_destroy(void* h);
void dr_host_ev_set_default(void* h, const float* m);
int64_t dr_host_ev_size(void* h);
int64_t dr_host_ev_import(void* h, const int64_t* keys, const float* rows, int64_t ncols, const int64_t* freqs, const int64_t* versions, int64_t n,
                          int part_id, int part_num, int reset_version);
int64_t dr_host_ev_import_cow(void* h, const int64_t* keys, const float* rows, int64_t ncols, int64_t n);
void dr_host_group_lookup(void** hs, int T, const int64_t* keys, int64_t B, float* out);
void dr_host_dot_interaction_fwd(const float* dense, const float* embs, int64_t B, int T, int D, float* out);
void* dr_redis_connect(const char* host, int port, int timeout_ms, const char* password, int db);
int dr_redis_ok(void* h);
const char* dr_redis_last_error(void* h);
void dr_redis_close(void* h);
int64_t dr_redis_mget_rows(void* h, const char* prefix, const int64_t* keys, int64_t n, float* rows, int dim, uint8_t* found);
int64_t dr_redis_get(void* h, const char* key, void* out, int64_t cap);
}

namespace cpusrv {
using drjson::JVal;
using namespace drsm;

struct Config {
  int session_num = 2, max_batch = 4096, select_policy = 0 /*0 RR, 1 MOD*/, update_interval_ms = 1000, intra_threads = 0;
  // Executor policy of op-program models (the reference's ExecutorPolicy {NORMAL, COST_MODEL, INLINE}: core/protobuf/config.proto:19-26,
  // common_runtime/executor.cc:414-478 inline, costmodel*.{h,cc} + kernel_stat.h cost model; env USE_INLINE_EXECUTOR / USE_COST_MODEL_EXECUTOR,
  // START_NODE_STATS_STEP / STOP_NODE_STATS_STEP).  0 = ops in program order, each one spread over the session's threads when the batch is
  // large; 1 = COST_MODEL: per-op times are traced over the requests [stats_start, stats_stop), then small-batch requests run the op DAG
  // critical-path-first on the session's threads (independent towers / experts in parallel, chains of ready ops stay on one thread);
  // 2 = INLINE: the whole request on the caller's thread, no team.
  int executor_policy = 0, stats_start = 2, stats_stop = 34;
  std::string savedmodel_dir, checkpoint_dir, warmup_file_name, timeline_path;
  int64_t timeline_start_step = -1; int timeline_interval_step = 0, timeline_trace_count = 0;
  // feature_store_type "redis" (serving/processor/storage/redis_feature_store.*): embedding rows live in a Redis instance shared by all
  // replicas, key "<redis_prefix>/<model version>/table/<t>:<id>", value = D x fp32; this process keeps only the dense net + default rows
  // SessionGroup CPU placement (docs SessionGroup.md "cpusets" / SESSION_GROUP_CPUSET / SET_SESSION_THREAD_POOL_AFFINITY): session i runs on
  // cpusets[i] -- the caller's thread is moved there for the duration of the request and the session's OpenMP team is pinned core by core
  std::vector<std::vector<int>> cpusets;
  // Request batching (TF-Serving's --enable_batching / batching_parameters: max_batch_size, batch_timeout_micros): concurrent small
  // requests are merged into one forward pass -- the first arrival leads, waits at most batch_timeout_micros for followers, runs the merged
  // rows on one session and hands every caller its slice.  0 = off.
  int batching_max_rows = 0, batching_timeout_us = 200; bool batching_adaptive = true;
  bool remote = false; std::string redis_host = "127.0.0.1", redis_password, redis_prefix = "dlrm"; int redis_port = 6379, redis_db = 0, redis_timeout_ms = 2000;
};

// wt: [K][N] row-major (the batch-1 / tail path streams whole rows); wp: the same weights packed panel-major for the tiled kernels --
// panel p = columns [32p, 32p + 32) stored as K x 32 contiguous floats (zero-padded past N), so a tile's k-loop reads consecutive
// cache lines instead of one line every N floats (the unpacked layout defeated the hardware prefetchers: 2 KB strides, a page every 2 steps)
constexpr int kPanel = 32;
struct Layer {
  int N = 0, K = 0; std::vector<float> wt, bias, wp;
  void Pack() {
    const int np = (N + kPanel - 1) / kPanel;
    wp.assign((size_t)np * K * kPanel, 0.f);
    for (int p = 0; p < np; ++p) for (int k = 0; k < K; ++k) for (int j = 0; j < kPanel && p * kPanel + j < N; ++j)
      wp[((size_t)p * K + k) * kPanel + j] = wt[(size_t)k * N + p * kPanel + j];
  }
};
// Linear from an exported W [N, K] (row stride ldw): transposed to wt [K][N] and packed
static Layer Transposed(int N, int K, const float* W, size_t ldw, std::vector<float> bias) {
  Layer L; L.N = N; L.K = K; L.bias = std::move(bias); L.wt.resize((size_t)K * N);
  for (int n = 0; n < N; ++n) for (int k = 0; k < K; ++k) L.wt[(size_t)k * N + n] = W[(size_t)n * ldw + k];
  L.Pack();
  return L;
}
// weights of one program op: L linear, Gih / Ghh gru, Lq / L1 / L2 din_attention (att: its W1 b1 W2 b2 w3 b3); v0, v1, H1, H2 as in OpTensors
struct PData { Layer L; std::vector<float> v0, v1; std::vector<std::vector<float>> att; int H1 = 0, H2 = 0; Layer Lq, L1, L2; Layer Gih, Ghh; };
struct Dense {
  std::vector<Layer> bot, top; std::vector<float> last_scale, last_shift, head_w; float head_b = 0.f;
  std::vector<PData> pdata; std::vector<int> width;                       // program models: per-op weights, per-buffer widths
  std::shared_ptr<struct ProgPlan> plan;                                  // op DAG + traced cost model (COST_MODEL executor)
};

// Dependency graph of an op program and its cost model.  Built at load (edges from the producer of every input buffer), filled by tracing.
struct ProgPlan {
  std::vector<std::vector<int>> succ; std::vector<int> indeg;
  std::unique_ptr<std::atomic<int64_t>[]> cost_ns;                       // accumulated over the traced runs
  std::atomic<int> traced{0}, seen{0}; std::atomic<bool> ready{false};
  std::vector<double> cost_us, rank_us;                                  // per-op mean cost; rank = cost + longest path below (critical-path priority)
  double total_us = 0, critical_us = 0; int width = 1, team = 1; bool parallel = false;
  std::mutex mu;
  explicit ProgPlan(const std::vector<POp>& ops, int nbuf) {
    const size_t n = ops.size();
    succ.assign(n, {}); indeg.assign(n, 0); cost_ns.reset(new std::atomic<int64_t>[n]);
    for (size_t i = 0; i < n; ++i) cost_ns[i].store(0);
    std::vector<int> producer((size_t)nbuf, -1);
    for (size_t i = 0; i < n; ++i) {
      std::vector<int> deps;
      for (int b : ops[i].in) { const int pr = producer[(size_t)b]; if (pr >= 0 && std::find(deps.begin(), deps.end(), pr) == deps.end()) deps.push_back(pr); }
      for (int pr : deps) { succ[(size_t)pr].push_back((int)i); ++indeg[i]; }
      producer[(size_t)ops[i].out] = (int)i;
    }
  }
  // mean costs -> ranks; parallel execution only when the DAG has real slack (total work well above the critical path) and the critical
  // path is long enough to amortise a team start
  void Finalize() {
    std::lock_guard<std::mutex> l(mu);
    if (ready.load()) return;
    const size_t n = succ.size(); const int runs = std::max(1, traced.load());
    cost_us.assign(n, 0.0); rank_us.assign(n, 0.0); total_us = 0; critical_us = 0;
    for (size_t i = 0; i < n; ++i) { cost_us[i] = (double)cost_ns[i].load() / 1e3 / runs; total_us += cost_us[i]; }
    for (size_t k = n; k-- > 0;) { double below = 0; for (int s2 : succ[k]) below = std::max(below, rank_us[(size_t)s2]); rank_us[k] = cost_us[k] + below; critical_us = std::max(critical_us, rank_us[k]); }
    // width: the largest antichain reachable by level scheduling (how many threads can ever be busy)
    std::vector<int> level(n, 0); std::vector<int> per_level; 
    for (size_t i = 0; i < n; ++i) { for (int s2 : succ[i]) level[(size_t)s2] = std::max(level[(size_t)s2], level[i] + 1); if ((size_t)level[i] >= per_level.size()) per_level.resize((size_t)level[i] + 1, 0); ++per_level[(size_t)level[i]]; }
    width = 1; for (int c : per_level) width = std::max(width, c);
    // decision from the model itself: a scheduled run costs about max(critical path, total / team) stretched by the cores sharing caches,
    // plus the team start and ~0.5 us of list handling per op; it must beat the sequential total by a clear margin (measured on 8 vCPUs:
    // two-tower programs -- ESMM, DSSM: total / critical = 1.5 -- lose to the overheads, expert mixtures -- MMoE 2.3, PLE 3.4 -- win 1.4-1.8x)
    team = std::max(1, std::min(width, (int)std::ceil(total_us / std::max(1e-3, critical_us))));
    const double est = std::max(critical_us, total_us / team) * 1.15 + 12.0 + 0.5 * (double)n / team;
    parallel = team > 1 && est < 0.8 * total_us;
    ready.store(true);
  }
};

struct Model {
  Arch arch; int64_t version = -1; std::string path;
  std::shared_ptr<Dense> dense;
  std::vector<void*> tables;                                   // HostEV handles (owned); empty in remote (Redis) mode
  std::vector<void*> col_handles;                              // tables[col_table[c]] per lookup column (not owned)
  std::vector<std::vector<float>> defaults;                    // remote mode: default-value matrix of every table ([dvd, D])
  std::vector<int64_t> sample_keys;                            // a few stored keys per table for the synthetic warm-up batch, [T][<=64]
  ~Model() { for (void* t : tables) if (t) dr_host_ev_destroy(t); }
};

// program weights in the layout of the CPU kernels: Linear / GRU weights transposed and packed, the DIN attention's first layer split
static bool BuildProgram(dr::BundleReader& r, const Arch& a, std::shared_ptr<Dense>* out) {
  ProgramData p;
  if (!ReadProgram(r, a, &p)) return false;
  auto dp = std::make_shared<Dense>();
  dp->pdata.resize(a.ops.size());
  for (size_t i = 0; i < a.ops.size(); ++i) {
    OpTensors& t = p.ops[i]; PData& d = dp->pdata[i];
    switch (a.ops[i].kind) {
      case P_LINEAR:
      case P_CROSS_LINEAR: d.L = Transposed(t.N, t.K, t.W.data(), (size_t)t.K, t.b); break;
      case P_GRU: d.Gih = Transposed(t.N, t.K, t.W.data(), (size_t)t.K, t.b); d.Ghh = Transposed(t.N, t.H1, t.v0.data(), (size_t)t.H1, t.v1); break;
      case P_DIN_ATT: {
        // first layer split (the algebra of csrc/cuda/attention_kernels.cu): W1 [q | k | q - k | q * k] = (Wa + Wc) q + (Wb - Wc) k + Wd (q * k);
        // the q term is one batched GEMM per request, the per-position work is ONE [rows, 2W] x [2W, H1] GEMM over [k | q * k]
        const int W = p.width[(size_t)a.ops[i].in[0]], H1 = t.H1; const float* W1 = t.att[0].data();
        d.Lq.N = H1; d.Lq.K = W; d.Lq.bias = t.att[1]; d.Lq.wt.assign((size_t)W * H1, 0.f);
        d.L1.N = H1; d.L1.K = 2 * W; d.L1.bias.assign((size_t)H1, 0.f); d.L1.wt.assign((size_t)2 * W * H1, 0.f);
        for (int h = 0; h < H1; ++h) for (int c = 0; c < W; ++c) {
          const float wa = W1[(size_t)h * 4 * W + c], wb = W1[(size_t)h * 4 * W + W + c], wc = W1[(size_t)h * 4 * W + 2 * W + c], wd = W1[(size_t)h * 4 * W + 3 * W + c];
          d.Lq.wt[(size_t)c * H1 + h] = wa + wc; d.L1.wt[(size_t)c * H1 + h] = wb - wc; d.L1.wt[(size_t)(W + c) * H1 + h] = wd;
        }
        d.Lq.Pack(); d.L1.Pack();
        d.L2 = Transposed(t.H2, H1, t.att[2].data(), (size_t)H1, t.att[3]);
        break;
      }
      default: break;
    }
    d.v0 = std::move(t.v0); d.v1 = std::move(t.v1); d.att = std::move(t.att); d.H1 = t.H1; d.H2 = t.H2;
  }
  dp->width = std::move(p.width);
  dp->plan = std::make_shared<ProgPlan>(a.ops, a.nbuf);
  *out = dp;
  return true;
}

// DLRM: the BatchNorm-folded layers transposed and packed
static bool BuildDense(dr::BundleReader& r, const Arch& a, std::shared_ptr<Dense>* out) {
  if (a.program) return BuildProgram(r, a, out);
  DlrmDense t;
  if (!ReadDlrmDense(r, a, &t)) return false;
  auto dp = std::make_shared<Dense>();
  for (const DenseLayer& L : t.bot) dp->bot.push_back(Transposed(L.N, L.K, L.W.data(), (size_t)L.Kp, L.b));
  for (const DenseLayer& L : t.top) dp->top.push_back(Transposed(L.N, L.K, L.W.data(), (size_t)L.Kp, L.b));
  dp->last_scale = std::move(t.last_scale); dp->last_shift = std::move(t.last_shift); dp->head_w = std::move(t.head_w); dp->head_b = t.head_b[0];
  *out = dp;
  return true;
}

static void* BuildTable(const TableData& in, int D) {
  DrEvConfig c{};
  c.dim = D; c.num_slots = 0; c.has_scalars = 0; c.init_capacity = std::max<int64_t>(1024, (int64_t)in.keys.size() * 2);
  c.default_value_dim = (int64_t)in.def.size() / D; c.num_partitions = 16; c.record_freq = 1; c.record_version = 1;
  c.l2_weight_threshold = -1.f;
  void* h = dr_host_ev_create(&c);                            // created writable for the import below; serving only ever calls Lookup
  dr_host_ev_set_default(h, in.def.data());
  if (!in.keys.empty())
    dr_host_ev_import(h, in.keys.data(), in.values.data(), D, in.freqs.empty() ? nullptr : in.freqs.data(), in.versions.empty() ? nullptr : in.versions.data(),
                      (int64_t)in.keys.size(), 0, 1, 0);
  return h;
}

static std::shared_ptr<Model> LoadModel(const std::string& dir, bool remote = false) {
  auto m = std::make_shared<Model>();
  std::string prefix;
  if (!ParseArch(dir, &m->arch, &m->version, &prefix)) { fprintf(stderr, "[deeprec_cpu_serving] bad saved_model.json in %s\n", dir.c_str()); return nullptr; }
  dr::BundleReader r(prefix);
  if (!r.ok()) { fprintf(stderr, "[deeprec_cpu_serving] cannot open bundle %s\n", prefix.c_str()); return nullptr; }
  if (!BuildDense(r, m->arch, &m->dense)) { fprintf(stderr, "[deeprec_cpu_serving] dense parameters incomplete in %s\n", prefix.c_str()); return nullptr; }
  m->sample_keys.assign((size_t)m->arch.T * 64, 0);
  for (int t = 0; t < m->arch.T && remote; ++t) {            // rows are in the feature store: only the default rows are needed here
    std::vector<float> def;
    if (!ReadVec(r, "table/" + std::to_string(t) + "-default", &def) || def.empty() || def.size() % (size_t)m->arch.D) { fprintf(stderr, "[deeprec_cpu_serving] table %d has no default matrix\n", t); return nullptr; }
    m->defaults.push_back(std::move(def));
  }
  for (int t = 0; t < m->arch.T && !remote; ++t) {
    TableData td;
    void* h = ReadTable(r, t, m->arch.D, &td) ? BuildTable(td, m->arch.D) : nullptr;
    if (!h) { fprintf(stderr, "[deeprec_cpu_serving] table %d incomplete\n", t); return nullptr; }
    m->tables.push_back(h);
    const size_t ns = std::min<size_t>(td.keys.size(), 64);
    for (size_t i = 0; i < 64; ++i) m->sample_keys[(size_t)t * 64 + i] = ns ? td.keys[i % ns] : 0;
  }
  for (int c = 0; c < m->arch.C && !remote; ++c) m->col_handles.push_back(m->tables[(size_t)m->arch.col_table[(size_t)c]]);
  m->path = dir;
  return m;
}

// Y[B, N] = act(X[B, K] (ldx) * Wt[K][N] + bias).  Register-blocked micro-kernel: a tile of kMR rows x kNR outputs is accumulated over the
// whole K in registers (8 vector accumulators on AVX2), so per k-step the loop does kMR broadcasts + kNR/8 weight loads for
// kMR * kNR / 8 FMAs and touches Y only once.  The compiler vectorises the fixed-trip inner loops.
constexpr int kMR = 4, kNR = 16;

template <int MR>
static inline void MicroKernel(const float* const* x, int K, const float* __restrict wp /*packed panel + column offset, row stride kPanel*/, int n0, int nr,
                               const float* __restrict bias, float* const* y, bool relu) {
  float acc[MR][kNR];
  for (int r = 0; r < MR; ++r) for (int j = 0; j < kNR; ++j) acc[r][j] = j < nr ? bias[n0 + j] : 0.f;
  for (int k = 0; k < K; ++k) {                                  // columns past N are zero in the packed panel: always the full-width loop
    const float* __restrict w = wp + (size_t)k * kPanel;
    for (int r = 0; r < MR; ++r) { const float a = x[r][k]; for (int j = 0; j < kNR; ++j) acc[r][j] += a * w[j]; }
  }
  for (int r = 0; r < MR; ++r) for (int j = 0; j < nr; ++j) y[r][n0 + j] = relu && acc[r][j] < 0.f ? 0.f : acc[r][j];
}

#if defined(__x86_64__)
// AVX-512 tile: 8 rows x 32 outputs = 16 zmm accumulators, per k-step 2 weight loads + 8 broadcasts for 16 FMAs (the 4 x 16 AVX2 tile
// does 2 loads + 4 broadcasts for 8).  Weights come from the packed panel (zero-padded: no load masks), column tails are masked on
// the store.  Compiled for avx512f regardless of the build flags and selected at run time.
__attribute__((target("avx512f")))
static void MicroKernel512(const float* const* x, int K, const float* __restrict wp /*packed panel: K x 32 contiguous*/, int n0, int nr,
                           const float* __restrict bias, float* const* y, bool relu) {
  constexpr int R = 8;
  const __mmask16 m0 = nr >= 16 ? (__mmask16)0xFFFF : (__mmask16)((1u << nr) - 1);
  const __mmask16 m1 = nr >= 32 ? (__mmask16)0xFFFF : (nr > 16 ? (__mmask16)((1u << (nr - 16)) - 1) : (__mmask16)0);
  const __m512 bias0 = _mm512_maskz_loadu_ps(m0, bias + n0), bias1 = _mm512_maskz_loadu_ps(m1, bias + n0 + 16);
  __m512 a0[R], a1[R];
  for (int r = 0; r < R; ++r) { a0[r] = bias0; a1[r] = bias1; }
  const float* w = wp;
  for (int k = 0; k < K; ++k, w += kPanel) {
    const __m512 w0 = _mm512_loadu_ps(w), w1 = _mm512_loadu_ps(w + 16);
    for (int r = 0; r < R; ++r) {
      const __m512 v = _mm512_set1_ps(x[r][k]);
      a0[r] = _mm512_fmadd_ps(v, w0, a0[r]);
      a1[r] = _mm512_fmadd_ps(v, w1, a1[r]);
    }
  }
  const __m512 zero = _mm512_setzero_ps();
  for (int r = 0; r < R; ++r) {
    if (relu) { a0[r] = _mm512_max_ps(a0[r], zero); a1[r] = _mm512_max_ps(a1[r], zero); }
    _mm512_mask_storeu_ps(y[r] + n0, m0, a0[r]);
    _mm512_mask_storeu_ps(y[r] + n0 + 16, m1, a1[r]);
  }
}
static const bool kHasAvx512 = __builtin_cpu_supports("avx512f") && !(getenv("DEEPREC_CPU_SERVING_NO_AVX512") && atoi(getenv("DEEPREC_CPU_SERVING_NO_AVX512")));
#else
static const bool kHasAvx512 = false;
#endif

// Loop order: rows are cut into groups (<= 64 rows, what a thread owns at a time), and inside a group the weight PANEL (K x 32 columns,
// ~50 KB for K = 429) is the outer loop and the group's row tiles the inner one -- a panel is read from L1/L2 by every tile of the group
// instead of the whole weight matrix (1.7 MB for 429 x 1024) being streamed once per 8-row tile.
// exp / sigmoid the compiler can vectorise (no libm call): 2^f by a degree-5 minimax polynomial on [0, 1) (max relative error 9e-8), the integer
// part through the exponent bits
static inline float FastExp(float x) {
  x = std::min(88.f, std::max(-88.f, x));
  const float t = x * 1.44269504f, fi = std::floor(t), f = t - fi;
  float p = 1.8775767e-3f; p = p * f + 8.9893397e-3f; p = p * f + 5.5826318e-2f; p = p * f + 2.4015361e-1f; p = p * f + 6.9315308e-1f; p = p * f + 9.9999994e-1f;
  const int32_t bits = ((int32_t)fi + 127) << 23;
  float sc; memcpy(&sc, &bits, 4);
  return p * sc;
}
static inline float FastSigmoid(float x) { return 1.f / (1.f + FastExp(-x)); }

static void Linear(const float* X, int64_t ldx, int64_t B, const Layer& L, float* Y, bool relu, int threads) {
  const int N = L.N, K = L.K;
  const float* wt = L.wt.data(); const float* bias = L.bias.data();
  const int64_t tile = kHasAvx512 ? 8 : kMR;
  const int nr_panel = kHasAvx512 ? 32 : kNR;
  const bool par = B >= 64 && threads > 1;
  // a weight matrix that sits comfortably in the per-core L2 is better streamed per row tile (the 8 x K input tile then stays in L1 across
  // all panels): groups of one tile reproduce that order; larger matrices get the panel-outer order described above (measured: DLRM's
  // <= 750 KB layers lose ~10 % with 64-row groups, DeepFM's 1.7 MB first layer gains 25-50 %)
  const bool big_w = (size_t)K * N * sizeof(float) > (size_t(1) << 20);
  int64_t group = big_w ? 64 : tile;
  if (par && big_w) { const int64_t per = (B + threads - 1) / threads; group = std::max<int64_t>(tile, std::min<int64_t>(64, (per + tile - 1) / tile * tile)); }
  const int64_t ngroups = (B + group - 1) / group;
#pragma omp parallel for schedule(static) num_threads(threads) if (par)
  for (int64_t g = 0; g < ngroups; ++g) {
    const int64_t g0 = g * group, g1 = std::min<int64_t>(B, g0 + group);
    const int64_t full_end = g0 + (g1 - g0) / tile * tile;              // rows [g0, full_end) form complete tiles
    for (int n0 = 0; n0 < N && full_end > g0; n0 += nr_panel) {
      const int nr = std::min(nr_panel, N - n0);
      for (int64_t r0 = g0; r0 < full_end; r0 += tile) {
#if defined(__x86_64__)
        if (kHasAvx512) {
          const float* x[8]; float* y[8];
          for (int r = 0; r < 8; ++r) { x[r] = X + (r0 + r) * ldx; y[r] = Y + (r0 + r) * N; }
          MicroKernel512(x, K, L.wp.data() + (size_t)(n0 / kPanel) * K * kPanel, n0, nr, bias, y, relu);
          continue;
        }
#endif
        const float* x[kMR]; float* y[kMR];
        for (int r = 0; r < kMR; ++r) { x[r] = X + (r0 + r) * ldx; y[r] = Y + (r0 + r) * N; }
        MicroKernel<kMR>(x, K, L.wp.data() + (size_t)(n0 / kPanel) * K * kPanel + (n0 % kPanel), n0, nr, bias, y, relu);
      }
    }
    int64_t r0 = full_end;
    for (; g1 - r0 >= kMR; r0 += kMR) {                                   // AVX-512 build: a 4..7-row remainder still gets one 4 x 16 pass
      const float* x[kMR]; float* y[kMR];
      for (int r = 0; r < kMR; ++r) { x[r] = X + (r0 + r) * ldx; y[r] = Y + (r0 + r) * N; }
      for (int n0 = 0; n0 < N; n0 += kNR) MicroKernel<kMR>(x, K, L.wp.data() + (size_t)(n0 / kPanel) * K * kPanel + (n0 % kPanel), n0, std::min(kNR, N - n0), bias, y, relu);
    }
    for (; r0 < g1; ++r0) {          // tail rows (and batch-1 requests): stream whole weight rows -- contiguous reads, the matrix-vector case is bandwidth-bound
      float* __restrict yy = Y + r0 * N; const float* xx = X + r0 * ldx;
      for (int n = 0; n < N; ++n) yy[n] = bias[n];
      for (int k = 0; k < K; ++k) { const float a = xx[k]; const float* __restrict w = wt + (size_t)k * N; for (int n = 0; n < N; ++n) yy[n] += a * w[n]; }
      if (relu) for (int n = 0; n < N; ++n) yy[n] = yy[n] > 0.f ? yy[n] : 0.f;
    }
  }
}

static std::vector<int> ParseCpuList(const std::string& s) {           // "2-4" | "2,3,4" | "0,2-3"
  std::vector<int> out;
  size_t i = 0;
  while (i < s.size()) {
    while (i < s.size() && !isdigit((unsigned char)s[i])) ++i;
    if (i >= s.size()) break;
    int a = 0; while (i < s.size() && isdigit((unsigned char)s[i])) a = a * 10 + (s[i++] - '0');
    int b = a;
    if (i < s.size() && s[i] == '-') { ++i; b = 0; while (i < s.size() && isdigit((unsigned char)s[i])) b = b * 10 + (s[i++] - '0'); }
    for (int c = a; c <= b && c < CPU_SETSIZE; ++c) out.push_back(c);
  }
  return out;
}
static std::vector<std::vector<int>> ParseCpusets(const std::string& s) {   // session groups separated by ';'
  std::vector<std::vector<int>> out;
  size_t b = 0;
  while (b <= s.size()) {
    size_t e = s.find(';', b); if (e == std::string::npos) e = s.size();
    auto l = ParseCpuList(s.substr(b, e - b));
    if (!l.empty()) out.push_back(std::move(l));
    b = e + 1;
  }
  return out;
}
static std::vector<std::vector<int>> AutoCpusets(int sessions) {           // the CPUs this process may use, split evenly and contiguously
  cpu_set_t m; CPU_ZERO(&m);
  std::vector<int> all;
  if (sched_getaffinity(0, sizeof(m), &m) == 0) for (int c = 0; c < CPU_SETSIZE; ++c) if (CPU_ISSET(c, &m)) all.push_back(c);
  std::vector<std::vector<int>> out;
  const int per = (int)all.size() / std::max(1, sessions);
  if (per < 1) return out;
  for (int i = 0; i < sessions; ++i) out.emplace_back(all.begin() + (size_t)i * per, all.begin() + (size_t)(i + 1) * per);
  return out;
}

struct Session {
  std::vector<int> cpus; cpu_set_t mask; std::atomic<int> last_cpu{-1};       // empty cpus = no placement
  std::mutex mu; int max_batch = 0, threads = 1;     // threads: OpenMP team size of this session's GEMMs (cores / sessions)
  std::vector<float> dense, emb, a, b2, z, prob, rrows; std::vector<int64_t> ids; std::vector<uint8_t> found;
  void* redis = nullptr;                                       // remote mode: this session's connection to the feature store
  ~Session() { if (redis) dr_redis_close(redis); }
  void Init(const Arch& ar, int mb, int nthreads) {
    max_batch = mb; threads = std::max(1, nthreads);
    Grow(ar);
  }
  // Scratch buffers must fit EVERY model version this session may still be asked to run: a full hot update can publish a wider
  // architecture (more tables, larger D, wider layers) while requests holding the previous model are queued on the mutex.
  // Grow-only, called with `mu` held (WarmUp of a new version) -- the reference builds fresh sessions per version instead
  // (serving/processor/serving/model_instance.cc:406-427).
  void Grow(const Arch& ar) {
    const size_t mb = (size_t)max_batch;
    int widest = ar.inter;
    for (int n : ar.bot) widest = std::max(widest, n);
    for (int n : ar.top) widest = std::max(widest, n);
    auto grow = [](auto& v, size_t n) { if (v.size() < n) v.resize(n); };
    grow(dense, mb * ar.num_dense); grow(ids, mb * ar.C); grow(emb, mb * ar.C * ar.D);
    grow(a, mb * widest); grow(b2, mb * widest); grow(z, mb * ar.inter); grow(prob, mb * (size_t)ar.n_out);
    grow(rrows, mb * ar.D); grow(found, mb);
  }
  // remote lookup of one chunk: per table ONE pipelined MGET; ids the store does not have read their default row (what a local
  // inference-mode lookup returns)
  bool RemoteLookup(const Model& m, const std::string& prefix, int B) {
    const Arch& ar = m.arch;
    for (int c = 0; c < ar.C; ++c) {
      const int t = ar.col_table[(size_t)c];
      const int64_t* k = ids.data() + (size_t)c * B;
      const std::string p = prefix + "/" + std::to_string(m.version) + "/table/" + std::to_string(t);
      if (!dr_redis_ok(redis) || dr_redis_mget_rows(redis, p.c_str(), k, B, rrows.data(), ar.D, found.data()) < 0) return false;
      const std::vector<float>& def = m.defaults[(size_t)t];
      const int64_t dvd = (int64_t)def.size() / ar.D;
      for (int i = 0; i < B; ++i) {
        const float* src = found[(size_t)i] ? rrows.data() + (size_t)i * ar.D : def.data() + dr_default_row(k[i], dvd) * ar.D;
        memcpy(emb.data() + ((size_t)i * ar.C + c) * ar.D, src, (size_t)ar.D * sizeof(float));
      }
    }
    return true;
  }
  // ---- op-program models: buffers 0 / 1 alias `dense` / `emb`, the others are sized (max_batch x width) on first use of a program ----
  std::vector<std::vector<float>> pbuf; std::vector<int> pbuf_width; std::vector<float> att_hq;
  float* Buf(int id) { return id == 0 ? dense.data() : id == 1 ? emb.data() : pbuf[(size_t)id].data(); }
  // one op of the program on `op_threads` threads (its OpenMP team when the batch is large; 1 under the DAG scheduler)
  void ExecOp(const Arch& ar, const Dense& d, const size_t oi, const int Bfull, const int op_threads) {
      const POp& op = ar.ops[oi]; const PData& pd = d.pdata[oi];
      const int B = op.rows1 ? 1 : Bfull;                          // sample-aware compression: user-side ops once per request (row 0)
      const int threads = op_threads;                              // team size of THIS op (1 when the scheduler runs ops side by side)
      const bool par = B >= 64 && threads > 1;
      float* out = Buf(op.out); const int W = d.width[(size_t)op.out];
      const float* a0 = Buf(op.in[0]); const int w0 = d.width[(size_t)op.in[0]];
      switch (op.kind) {
        case P_LINEAR: {
          const int S = op.len > 0 ? op.len : 1;                     // a sequence buffer [B, S * K] is [B * S, K] in memory
          Linear(a0, w0 / S, (int64_t)B * S, pd.L, out, op.relu, threads); break;
        }
        case P_CONCAT: {
          int off = 0;
          for (int src : op.in) {
            const float* x = Buf(src); const int w = d.width[(size_t)src];
#pragma omp parallel for schedule(static) num_threads(threads) if (par)
            for (int i = 0; i < B; ++i) memcpy(out + (size_t)i * W + off, x + (size_t)i * w, (size_t)w * sizeof(float));
            off += w;
          }
          break;
        }
        case P_AFFINE: {
          const float* sc = pd.v0.data(); const float* sh = pd.v1.data();
#pragma omp parallel for schedule(static) num_threads(threads) if (par)
          for (int i = 0; i < B; ++i) { const float* x = a0 + (size_t)i * W; float* y = out + (size_t)i * W; for (int k = 0; k < W; ++k) y[k] = x[k] * sc[k] + sh[k]; }
          break;
        }
        case P_FM: {                                             // 0.5 ((sum_t v_t)^2 - sum_t v_t^2) per embedding dimension
          const int T = ar.C, D = ar.D;
#pragma omp parallel for schedule(static) num_threads(threads) if (par)
          for (int i = 0; i < B; ++i) {
            const float* e = a0 + (size_t)i * T * D; float* y = out + (size_t)i * D;
            for (int k = 0; k < D; ++k) { float sum = 0.f, sq = 0.f; for (int t = 0; t < T; ++t) { const float v = e[(size_t)t * D + k]; sum += v; sq += v * v; } y[k] = 0.5f * (sum * sum - sq); }
          }
          break;
        }
        case P_CROSS: {                                          // x_{l+1} = x0 (x_l . w) + b + x_l
          const float* xl = Buf(op.in[1]); const float* w = pd.v0.data(); const float* bb = pd.v1.data();
#pragma omp parallel for schedule(static) num_threads(threads) if (par)
          for (int i = 0; i < B; ++i) {
            const float* x0 = a0 + (size_t)i * W; const float* x = xl + (size_t)i * W; float* y = out + (size_t)i * W;
            float dot = 0.f; for (int k = 0; k < W; ++k) dot += x[k] * w[k];
            for (int k = 0; k < W; ++k) y[k] = x0[k] * dot + bb[k] + x[k];
          }
          break;
        }
        case P_CROSS_LINEAR: {                                   // x0 * (t kernel^T + bias) + x_l: the product lands in `out` first
          const float* xl = Buf(op.in[1]); const float* tt = Buf(op.in[2]);
          Linear(tt, d.width[(size_t)op.in[2]], B, pd.L, out, false, threads);
#pragma omp parallel for schedule(static) num_threads(threads) if (par)
          for (int i = 0; i < B; ++i) {
            const float* x0 = a0 + (size_t)i * W; const float* x = xl + (size_t)i * W; float* y = out + (size_t)i * W;
            for (int k = 0; k < W; ++k) y[k] = x0[k] * y[k] + x[k];
          }
          break;
        }
        case P_MUL_ADD: case P_ADD: case P_MUL: {
          const float* b1 = Buf(op.in[1]); const float* c1 = op.kind == P_MUL_ADD ? Buf(op.in[2]) : nullptr;
          const size_t n = (size_t)B * W;
          if (c1) for (size_t k = 0; k < n; ++k) out[k] = a0[k] * b1[k] + c1[k];
          else if (op.kind == P_MUL) for (size_t k = 0; k < n; ++k) out[k] = a0[k] * b1[k];
          else for (size_t k = 0; k < n; ++k) out[k] = a0[k] + b1[k];
          break;
        }
        case P_SLICE: {
          const int st = op.start;
#pragma omp parallel for schedule(static) num_threads(threads) if (par)
          for (int i = 0; i < B; ++i) memcpy(out + (size_t)i * W, a0 + (size_t)i * w0 + st, (size_t)W * sizeof(float));
          break;
        }
        case P_VALID_MASK: {                                     // out[i, l] = ids[column start + l][i] >= 0
          for (int l = 0; l < W; ++l) { const int64_t* k = ids.data() + (size_t)(op.start + l) * Bfull; for (int i = 0; i < B; ++i) out[(size_t)i * W + l] = k[i] >= 0 ? 1.f : 0.f; }
          break;
        }
        case P_GRU: {                                            // r, z, n gates; h' = (1 - z) n + z h; input projection as ONE GEMM over B * L rows
          const int L = op.len, I = w0 / L, H = pd.H1, H3 = 3 * H;
          std::vector<float> gi((size_t)B * L * H3), gh((size_t)B * H3), h((size_t)B * H, 0.f);
          Linear(a0, I, (int64_t)B * L, pd.Gih, gi.data(), false, threads);
          for (int t = 0; t < L; ++t) {
            Linear(h.data(), H, B, pd.Ghh, gh.data(), false, threads);
            for (int i = 0; i < B; ++i) {
              const float* a = gi.data() + ((size_t)i * L + t) * H3; const float* b = gh.data() + (size_t)i * H3;
              float* hh = h.data() + (size_t)i * H; float* y = out + ((size_t)i * L + t) * H;
              for (int j = 0; j < H; ++j) {
                const float rg = 1.f / (1.f + std::exp(-(a[j] + b[j]))), zg = 1.f / (1.f + std::exp(-(a[H + j] + b[H + j])));
                const float ng = std::tanh(a[2 * H + j] + rg * b[2 * H + j]);
                hh[j] = (1.f - zg) * ng + zg * hh[j]; y[j] = hh[j];
              }
            }
          }
          break;
        }
        case P_SEQ_LAST: {                                       // the state at the last valid position: max(sum(mask), 1) - 1
          const float* mk = Buf(op.in[1]); const int L = op.len;
          for (int i = 0; i < B; ++i) {
            int cnt = 0; for (int l = 0; l < L; ++l) cnt += mk[(size_t)i * L + l] > 0.f ? 1 : 0;
            memcpy(out + (size_t)i * W, a0 + (size_t)i * w0 + (size_t)(std::max(cnt, 1) - 1) * W, (size_t)W * sizeof(float));
          }
          break;
        }
        case P_SEQ_MEAN: {                                       // mean over the valid positions (mode 1: sum / sqrt(count))
          const float* mk = Buf(op.in[1]); const int L = op.len;
#pragma omp parallel for schedule(static) num_threads(threads) if (par)
          for (int i = 0; i < B; ++i) {
            float* y = out + (size_t)i * W; for (int k = 0; k < W; ++k) y[k] = 0.f;
            int cnt = 0;
            for (int l = 0; l < L; ++l) if (mk[(size_t)i * L + l] > 0.f) { ++cnt; const float* x = a0 + (size_t)i * w0 + (size_t)l * W; for (int k = 0; k < W; ++k) y[k] += x[k]; }
            const float inv = op.mode == 1 ? 1.f / std::sqrt((float)std::max(cnt, 1)) : 1.f / (float)std::max(cnt, 1);
            for (int k = 0; k < W; ++k) y[k] *= inv;
          }
          break;
        }
        case P_MHA: {                                            // softmax(q k^T / sqrt(dh)) v per head, keys of invalid positions masked
          const float* mk = Buf(op.in[1]); const int S = op.len, E = w0 / (3 * S), nh = op.heads, dh = E / nh; const float scale = 1.f / std::sqrt((float)dh);
#pragma omp parallel for schedule(static) num_threads(threads) if (par)
          for (int i = 0; i < B; ++i) {
            std::vector<float> p((size_t)S);
            const float* x = a0 + (size_t)i * w0; const float* m = mk + (size_t)i * S; float* y = out + (size_t)i * S * E;
            for (int hd = 0; hd < nh; ++hd)
              for (int s1 = 0; s1 < S; ++s1) {
                const float* q = x + (size_t)s1 * 3 * E + hd * dh;
                float mx = -3.4e38f;
                for (int s2 = 0; s2 < S; ++s2) {
                  if (!(m[s2] > 0.f)) { p[(size_t)s2] = -3.4e38f; continue; }
                  const float* k = x + (size_t)s2 * 3 * E + E + hd * dh;
                  float dot = 0.f; for (int c = 0; c < dh; ++c) dot += q[c] * k[c];
                  p[(size_t)s2] = dot * scale; mx = std::max(mx, p[(size_t)s2]);
                }
                float den = 0.f;
                for (int s2 = 0; s2 < S; ++s2) { p[(size_t)s2] = m[s2] > 0.f ? std::exp(p[(size_t)s2] - mx) : 0.f; den += p[(size_t)s2]; }
                float* o = y + (size_t)s1 * E + hd * dh; for (int c = 0; c < dh; ++c) o[c] = 0.f;
                if (den <= 0.f) continue;
                const float inv = 1.f / den;
                for (int s2 = 0; s2 < S; ++s2) { if (p[(size_t)s2] == 0.f) continue; const float wgt = p[(size_t)s2] * inv; const float* v = x + (size_t)s2 * 3 * E + 2 * E + hd * dh; for (int c = 0; c < dh; ++c) o[c] += wgt * v[c]; }
              }
          }
          break;
        }
        case P_TILE: {
#pragma omp parallel for schedule(static) num_threads(threads) if (par)
          for (int i = 0; i < B; ++i) memcpy(out + (size_t)i * W, a0, (size_t)W * sizeof(float));
          break;
        }
        case P_SEQ_ZIP: {                                        // position-wise concat of two [B, L, *] sequences
          const float* b1 = Buf(op.in[1]); const int L = op.len, wa = w0 / L, wb = d.width[(size_t)op.in[1]] / L;
#pragma omp parallel for schedule(static) num_threads(threads) if (par)
          for (int i = 0; i < B; ++i)
            for (int l = 0; l < L; ++l) {
              float* y = out + (size_t)i * W + (size_t)l * (wa + wb);
              memcpy(y, a0 + (size_t)i * w0 + (size_t)l * wa, (size_t)wa * sizeof(float));
              memcpy(y + wa, b1 + (size_t)i * L * wb + (size_t)l * wb, (size_t)wb * sizeof(float));
            }
          break;
        }
        case P_SEQ_MASK: {                                       // x [B, L, w] * mask [B, L]
          const float* mk = Buf(op.in[1]); const int L = op.len, w = W / L;
#pragma omp parallel for schedule(static) num_threads(threads) if (par)
          for (int i = 0; i < B; ++i)
            for (int l = 0; l < L; ++l) { const float f = mk[(size_t)i * L + l]; const float* x = a0 + (size_t)i * W + (size_t)l * w; float* y = out + (size_t)i * W + (size_t)l * w; for (int k = 0; k < w; ++k) y[k] = x[k] * f; }
          break;
        }
        case P_SEQ_SUM: {                                        // sum over the L positions of x [B, L, W]
          const int L = op.len;
#pragma omp parallel for schedule(static) num_threads(threads) if (par)
          for (int i = 0; i < B; ++i) {
            float* y = out + (size_t)i * W; for (int k = 0; k < W; ++k) y[k] = 0.f;
            for (int l = 0; l < L; ++l) { const float* x = a0 + (size_t)i * w0 + (size_t)l * W; for (int k = 0; k < W; ++k) y[k] += x[k]; }
          }
          break;
        }
        case P_PRELU: {
          const float* al = pd.v0.data();
#pragma omp parallel for schedule(static) num_threads(threads) if (par)
          for (int i = 0; i < B; ++i) { const float* x = a0 + (size_t)i * W; float* y = out + (size_t)i * W; for (int k = 0; k < W; ++k) y[k] = x[k] > 0.f ? x[k] : al[k] * x[k]; }
          break;
        }
        case P_SOFTMAX: {
#pragma omp parallel for schedule(static) num_threads(threads) if (par)
          for (int i = 0; i < B; ++i) {
            const float* x = a0 + (size_t)i * W; float* y = out + (size_t)i * W;
            float mx = x[0]; for (int k = 1; k < W; ++k) mx = std::max(mx, x[k]);
            float den = 0.f; for (int k = 0; k < W; ++k) { y[k] = std::exp(x[k] - mx); den += y[k]; }
            for (int k = 0; k < W; ++k) y[k] /= den;
          }
          break;
        }
        case P_COSINE: {                                         // F.cosine_similarity(a, b, eps = 1e-8)
          const float* b1 = Buf(op.in[1]);
#pragma omp parallel for schedule(static) num_threads(threads) if (par)
          for (int i = 0; i < B; ++i) {
            const float* x = a0 + (size_t)i * w0; const float* y = b1 + (size_t)i * w0;
            float xy = 0.f, xx = 0.f, yy = 0.f;
            for (int k = 0; k < w0; ++k) { xy += x[k] * y[k]; xx += x[k] * x[k]; yy += y[k] * y[k]; }
            out[(size_t)i] = xy / (std::max(std::sqrt(xx), 1e-8f) * std::max(std::sqrt(yy), 1e-8f));
          }
          break;
        }
        case P_DIN_ATT: {                                        // DIN attention unit: s_l = MLP([q, k_l, q - k_l, q * k_l]), masked softmax, sum_l w_l k_l
          // blocked: kS samples = kS * L history positions form the rows of two small GEMMs on the packed micro-kernels; sigmoids vectorised
          const float* kk = Buf(op.in[1]); const float* mk = Buf(op.in[2]);
          const int L = d.width[(size_t)op.in[2]], H1 = pd.H1, H2 = pd.H2, Wq = w0; const bool weights_out = op.mode == 1;
          const float* w3 = pd.att[4].data(); const float b3 = pd.att[5][0];
          std::lock_guard<std::mutex> att_lock(att_mu);              // one scratch per session: two attention ops never run side by side
          att_hq.resize((size_t)B * H1);
          Linear(a0, Wq, B, pd.Lq, att_hq.data(), false, threads);                     // (Wa + Wc) q + b1, once per sample
          constexpr int kS = 16;
          const int nblk = (B + kS - 1) / kS;
#pragma omp parallel num_threads(threads) if (par)
          {
            std::vector<float> X((size_t)kS * L * 2 * Wq), h1((size_t)kS * L * H1), h2((size_t)kS * L * H2), sc((size_t)L);
#pragma omp for schedule(static)
            for (int blk = 0; blk < nblk; ++blk) {
              const int s0 = blk * kS, s1 = std::min(B, s0 + kS), rows = (s1 - s0) * L;
              for (int i = s0; i < s1; ++i) {
                const float* q = a0 + (size_t)i * Wq; const float* ks = kk + (size_t)i * L * Wq;
                for (int l = 0; l < L; ++l) {
                  float* x = X.data() + ((size_t)(i - s0) * L + l) * 2 * Wq; const float* k = ks + (size_t)l * Wq;
                  for (int c = 0; c < Wq; ++c) { x[c] = k[c]; x[Wq + c] = q[c] * k[c]; }
                }
              }
              Linear(X.data(), 2 * Wq, rows, pd.L1, h1.data(), false, 1);
              for (int i = s0; i < s1; ++i) {
                const float* hq = att_hq.data() + (size_t)i * H1;
                for (int l = 0; l < L; ++l) {
                  float* h = h1.data() + ((size_t)(i - s0) * L + l) * H1;
#pragma omp simd
                  for (int j2 = 0; j2 < H1; ++j2) h[j2] = FastSigmoid(h[j2] + hq[j2]);
                }
              }
              Linear(h1.data(), H1, rows, pd.L2, h2.data(), false, 1);
              for (int i = s0; i < s1; ++i) {
                const float* m = mk + (size_t)i * L; const float* ks = kk + (size_t)i * L * Wq;
                float mx = -3.4e38f; bool any = false;
                for (int l = 0; l < L; ++l) {
                  const float* h = h2.data() + ((size_t)(i - s0) * L + l) * H2;
                  float s3 = 0.f;
#pragma omp simd reduction(+ : s3)
                  for (int m2 = 0; m2 < H2; ++m2) s3 += w3[m2] * FastSigmoid(h[m2]);
                  sc[(size_t)l] = s3 + b3;
                  if (m[l] > 0.f) { any = true; mx = std::max(mx, sc[(size_t)l]); }
                }
                if (weights_out) {                               // DIEN: softmax(masked_fill(s, -2^31)) -- uniform when nothing is valid
                  float* y = out + (size_t)i * L;
                  if (!any) { for (int l = 0; l < L; ++l) y[l] = 1.f / (float)L; continue; }
                  float den = 0.f;
                  for (int l = 0; l < L; ++l) { y[l] = m[l] > 0.f ? FastExp(sc[(size_t)l] - mx) : 0.f; den += y[l]; }
                  const float inv = 1.f / den;
                  for (int l = 0; l < L; ++l) y[l] *= inv;
                  continue;
                }
                float* y = out + (size_t)i * Wq; for (int c = 0; c < Wq; ++c) y[c] = 0.f;
                if (!any) continue;                              // no valid history position: zero vector (the module multiplies by mask.any())
                float den = 0.f;
                for (int l = 0; l < L; ++l) { sc[(size_t)l] = m[l] > 0.f ? FastExp(sc[(size_t)l] - mx) : 0.f; den += sc[(size_t)l]; }
                const float inv = 1.f / den;
                for (int l = 0; l < L; ++l) {
                  if (sc[(size_t)l] == 0.f) continue;
                  const float wl = sc[(size_t)l] * inv; const float* k = ks + (size_t)l * Wq;
                  for (int c = 0; c < Wq; ++c) y[c] += wl * k[c];
                }
              }
            }
          }
          break;
        }
        case P_LAYERNORM: {                                      // (x - mean) / sqrt(var + eps) * gamma + beta, biased variance, optional ReLU
          const float* g = pd.v0.data(); const float* bt = pd.v1.data(); const float eps = op.eps; const bool relu = op.relu;
          const int S = op.len > 0 ? op.len : 1, W = d.width[(size_t)op.out] / S, B = (op.rows1 ? 1 : Bfull) * S;      // per position of a sequence buffer
#pragma omp parallel for schedule(static) num_threads(threads) if (par)
          for (int i = 0; i < B; ++i) {
            const float* x = a0 + (size_t)i * W; float* y = out + (size_t)i * W;
            float mean = 0.f; for (int k = 0; k < W; ++k) mean += x[k]; mean /= (float)W;
            float var = 0.f; for (int k = 0; k < W; ++k) { const float dlt = x[k] - mean; var += dlt * dlt; } var /= (float)W;
            const float rs = 1.f / std::sqrt(var + eps);
            for (int k = 0; k < W; ++k) { const float v = (x[k] - mean) * rs * g[k] + bt[k]; y[k] = relu && v < 0.f ? 0.f : v; }
          }
          break;
        }
      }
  }

  // COST_MODEL executor, small batches: the op DAG on `team` threads.  Ready ops sit in a rank-ordered list (rank = traced cost + longest
  // path below: critical path first); a thread that finishes an op keeps the best newly-ready successor for itself (chains never leave their
  // thread, cheap glue ops are never queued) and publishes the others.
  void RunScheduled(const Arch& ar, const Dense& d, const ProgPlan& pl, const int Bfull, const int team) {
    const int n = (int)ar.ops.size();
    if ((int)sched_indeg.size() < n) { sched_indeg = std::vector<std::atomic<int>>((size_t)n); }
    for (int i = 0; i < n; ++i) sched_indeg[(size_t)i].store(pl.indeg[(size_t)i], std::memory_order_relaxed);
    sched_ready.clear();
    for (int i = 0; i < n; ++i) if (pl.indeg[(size_t)i] == 0) sched_ready.push_back(i);
    std::atomic<int> remaining{n};
    std::atomic_flag lock = ATOMIC_FLAG_INIT;
    auto pop_best = [&]() -> int {
      while (lock.test_and_set(std::memory_order_acquire)) _mm_pause();
      int best = -1; size_t at = 0;
      for (size_t k = 0; k < sched_ready.size(); ++k) if (best < 0 || pl.rank_us[(size_t)sched_ready[k]] > pl.rank_us[(size_t)best]) { best = sched_ready[k]; at = k; }
      if (best >= 0) { sched_ready[at] = sched_ready.back(); sched_ready.pop_back(); }
      lock.clear(std::memory_order_release);
      return best;
    };
#pragma omp parallel num_threads(team)
    {
      while (remaining.load(std::memory_order_acquire) > 0) {
        int oi = pop_best();
        if (oi < 0) { _mm_pause(); continue; }
        while (oi >= 0) {
          ExecOp(ar, d, (size_t)oi, Bfull, 1);
          int keep = -1;
          for (int s2 : pl.succ[(size_t)oi]) {
            if (sched_indeg[(size_t)s2].fetch_sub(1, std::memory_order_acq_rel) != 1) continue;
            if (keep < 0) { keep = s2; continue; }
            const int other = pl.rank_us[(size_t)s2] > pl.rank_us[(size_t)keep] ? keep : s2;      // the lower-rank one goes to the list
            if (other == keep) keep = s2;
            while (lock.test_and_set(std::memory_order_acquire)) _mm_pause();
            sched_ready.push_back(other);
            lock.clear(std::memory_order_release);
          }
          remaining.fetch_sub(1, std::memory_order_acq_rel);
          oi = keep;
        }
      }
    }
  }

  int exec_policy = 0, stats_start = 2, stats_stop = 34;           // Config::executor_policy & tracing window, copied at Init
  std::mutex att_mu; std::vector<std::atomic<int>> sched_indeg; std::vector<int> sched_ready;
  void RunProgram(const Arch& ar, const Dense& d, const int Bfull) {
    if (pbuf_width != d.width) {
      pbuf.assign(d.width.size(), std::vector<float>());
      for (size_t i = 2; i < d.width.size(); ++i) pbuf[i].resize((size_t)max_batch * d.width[i]);
      pbuf_width = d.width;
    }
    const int nops = (int)ar.ops.size();
    ProgPlan* pl = d.plan.get();
    // the regime of the DAG scheduler: latency-bound requests.  Up to ~16 rows an op streams its weights once and waits on memory -- side-by-side
    // branches overlap those waits (MMoE 1.3-1.4x, PLE 1.7-1.9x at 1-8 rows on 8 vCPUs); at 32 rows the GEMMs are FMA-bound, sibling hyper-threads
    // add nothing and the team start is pure cost (measured: MMoE 0.85x), so those run in program order; from 64 rows every op uses its own team
    const bool small = Bfull <= 16;
    if (exec_policy == 2) {                                          // INLINE: everything on the caller's thread
      for (int oi = 0; oi < nops; ++oi) ExecOp(ar, d, (size_t)oi, Bfull, 1);
    } else if (exec_policy == 1 && pl && small && pl->ready.load(std::memory_order_acquire) && pl->parallel && threads > 1) {
      RunScheduled(ar, d, *pl, Bfull, std::min(threads, pl->team));
    } else if (exec_policy == 1 && pl && small && !pl->ready.load(std::memory_order_acquire)) {
      // tracing window (START / STOP_NODE_STATS_STEP): single-thread op times of the small-batch regime the scheduler will run in
      const int seen = pl->seen.fetch_add(1);
      const bool trace = seen >= stats_start && seen < stats_stop;
      for (int oi = 0; oi < nops; ++oi) {
        if (!trace) { ExecOp(ar, d, (size_t)oi, Bfull, threads); continue; }
        const auto t0 = std::chrono::steady_clock::now();
        ExecOp(ar, d, (size_t)oi, Bfull, 1);
        pl->cost_ns[(size_t)oi].fetch_add(std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count());
      }
      if (trace) pl->traced.fetch_add(1);
      if (seen + 1 >= stats_stop) pl->Finalize();
    } else {
      for (int oi = 0; oi < nops; ++oi) ExecOp(ar, d, (size_t)oi, Bfull, threads);
    }
    const float* lg = Buf(ar.out_buf); const int W = d.width[(size_t)ar.out_buf];
    const int no = ar.n_out;
    for (int i = 0; i < Bfull; ++i) for (int o = 0; o < no; ++o) prob[(size_t)i * no + o] = 1.f / (1.f + std::exp(-lg[(size_t)i * W + o]));
  }

  // dense [B, num_dense], ids [T][B] staged in the session buffers -> prob[B]
  bool Run(const Model& m, const Dense& d, int B, const std::string& remote_prefix = std::string()) {
    const Arch& ar = m.arch;
    if (redis) { if (!RemoteLookup(m, remote_prefix, B)) return false; }
    else dr_host_group_lookup(const_cast<void**>(m.col_handles.data()), ar.C, ids.data(), B, emb.data());    // [B, C, D]
    if (ar.program) { RunProgram(ar, d, B); return true; }
    const float* x = dense.data(); int64_t ldx = ar.num_dense;
    float* cur = a.data(); float* nxt = b2.data();
    for (size_t l = 0; l < d.bot.size(); ++l) { Linear(x, ldx, B, d.bot[l], cur, true, threads); x = cur; ldx = d.bot[l].N; std::swap(cur, nxt); }
    float* y = const_cast<float*>(x);                                                                          // [B, D]: the last BatchNorm, explicit
    for (int64_t i = 0; i < (int64_t)B; ++i) for (int k = 0; k < ar.D; ++k) y[i * ar.D + k] = y[i * ar.D + k] * d.last_scale[k] + d.last_shift[k];
    dr_host_dot_interaction_fwd(y, emb.data(), B, ar.T, ar.D, z.data());                                       // [B, D + F(F-1)/2]
    x = z.data(); ldx = ar.inter;
    for (size_t l = 0; l < d.top.size(); ++l) { Linear(x, ldx, B, d.top[l], cur, true, threads); x = cur; ldx = d.top[l].N; std::swap(cur, nxt); }
    const int K = (int)ldx;
    for (int64_t i = 0; i < (int64_t)B; ++i) {
      float acc = d.head_b; const float* xi = x + i * ldx;
      for (int k = 0; k < K; ++k) acc += xi[k] * d.head_w[k];
      prob[(size_t)i] = 1.f / (1.f + std::exp(-acc));
    }
    return true;
  }
};

// Runs the enclosed request on the session's CPUs: the calling thread takes the session mask (and gets its own mask back afterwards --
// it belongs to the application), team member i of a multi-threaded batch is pinned to cpus[i % n] once (it only ever serves this caller).
struct AffinityScope {
  bool on = false; cpu_set_t saved;
  AffinityScope(Session& s, int batch) {
    if (s.cpus.empty()) return;
    on = sched_getaffinity(0, sizeof(saved), &saved) == 0 && sched_setaffinity(0, sizeof(s.mask), &s.mask) == 0;
    if (!on) return;
#ifdef _OPENMP
    if (batch >= 64 && s.threads > 1) {
      const int n = (int)s.cpus.size();
#pragma omp parallel num_threads(s.threads)
      {
        static thread_local int pinned = -1;
        const int t = omp_get_thread_num(), want = s.cpus[(size_t)(t % n)];
        if (t != 0 && pinned != want) { cpu_set_t one; CPU_ZERO(&one); CPU_SET(want, &one); if (sched_setaffinity(0, sizeof(one), &one) == 0) pinned = want; }
      }
    }
#else
    (void)batch;
#endif
    s.last_cpu.store(sched_getcpu(), std::memory_order_relaxed);
  }
  ~AffinityScope() { if (on) sched_setaffinity(0, sizeof(saved), &saved); }
};

struct Batcher;
struct ServingModel {
  Config cfg;
  drcfg::Compat compat;                            // reference ModelConfig keys without a 1:1 field (csrc/common/model_config.h)
  std::shared_ptr<Batcher> batcher;
  std::atomic<int> busy{0};                        // sessions currently inside a forward pass
  std::shared_ptr<Model> model;                    // atomic_load / atomic_store
  std::vector<std::unique_ptr<Session>> sessions;
  std::atomic<uint64_t> rr{0}, requests{0}, failures{0}, full_updates{0}, delta_updates{0};
  std::atomic<int64_t> delta_version{-1};
  std::thread updater; std::atomic<bool> stop{false};
  std::mutex tmu; std::vector<std::string> trace;
  ~ServingModel() { stop = true; if (updater.joinable()) updater.join(); }
};

static void SessionReleased(ServingModel* sm);

// rows [0, R) given as dense [R, num_dense] and ids [T][R] (table-major, stride ids_stride) -> probs[R] on one session (chunked by max_batch)
// (byte pointers: inside a request buffer the id block follows 24 + 4 * R * num_dense bytes and is not 8-byte aligned in general)
static int RunRows(ServingModel* sm, const std::shared_ptr<Model>& m, const uint8_t* dense_in, const uint8_t* ids_in, size_t ids_stride, uint32_t R,
                   float* probs, int hint) {
  const Arch& a = m->arch;
  const uint64_t pick = sm->cfg.select_policy == 1 ? (hint >= 0 ? (uint64_t)hint : std::hash<std::thread::id>()(std::this_thread::get_id())) : sm->rr.fetch_add(1);
  const size_t ns = sm->sessions.size();
  // declared before the session lock: released (and a waiting batch leader woken) only after the session mutex is free again
  struct Busy { ServingModel* sm; explicit Busy(ServingModel* m) : sm(m) { sm->busy.fetch_add(1); } ~Busy() { SessionReleased(sm); } } busy_mark(sm);
  Session* sp = sm->sessions[pick % ns].get();
  std::unique_lock<std::mutex> l(sp->mu, std::defer_lock);
  if (sm->cfg.select_policy == 1) l.lock();                                       // MOD: the caller / hint owns its session
  else {                                                                           // RR: start at the round-robin slot, take the first idle session
    bool got = false;
    for (size_t i = 0; i < ns && !got; ++i) {
      Session* c = sm->sessions[(pick + i) % ns].get();
      std::unique_lock<std::mutex> t(c->mu, std::try_to_lock);
      if (t.owns_lock()) { l = std::move(t); sp = c; got = true; }
    }
    if (!got) l.lock();                                                            // all busy: queue on the round-robin slot
  }
  Session& s = *sp;
  AffinityScope place(s, (int)std::min<uint32_t>(R, (uint32_t)s.max_batch));
  auto dense = std::atomic_load(&m->dense);
  for (uint32_t off = 0; off < R; off += (uint32_t)s.max_batch) {                  // larger requests are chunked
    const int B = (int)std::min<uint32_t>((uint32_t)s.max_batch, R - off);
    memcpy(s.dense.data(), dense_in + (size_t)off * a.num_dense * 4, (size_t)B * a.num_dense * 4);
    for (int c = 0; c < a.C; ++c) memcpy(s.ids.data() + (size_t)c * B, ids_in + ((size_t)a.id_map[(size_t)c] * ids_stride + off) * 8, (size_t)B * 8);
    if (!s.Run(*m, *dense, B, sm->cfg.redis_prefix)) {
      // feature store hiccup: one reconnect + retry before the request is failed (the next request tries again)
      bool ok = false;
      if (s.redis) {
        dr_redis_close(s.redis);
        s.redis = dr_redis_connect(sm->cfg.redis_host.c_str(), sm->cfg.redis_port, sm->cfg.redis_timeout_ms, sm->cfg.redis_password.c_str(), sm->cfg.redis_db);
        ok = dr_redis_ok(s.redis) && s.Run(*m, *dense, B, sm->cfg.redis_prefix);
      }
      if (!ok) { sm->failures++; return 500; }
    }
    memcpy(probs + (size_t)off * a.n_out, s.prob.data(), (size_t)B * a.n_out * 4);
  }
  return 200;
}

// Leader / follower request batcher (see Config::batching_max_rows)
struct Batcher {
  struct Item { const uint8_t* dense; const uint8_t* ids; uint32_t rows; float* probs; int rc = 0; int64_t version = -1; bool done = false; };
  std::mutex mu; std::condition_variable cv_leader, cv_done;
  std::vector<Item*> pending; uint32_t pending_rows = 0; bool leader_waiting = false;
  std::atomic<uint64_t> merged_batches{0}, merged_requests{0};
};

static int PredictBatched(ServingModel* sm, Batcher& bt, const drpb::WireReq& h, const uint8_t* dense_in, const uint8_t* ids_in, float* probs, int64_t* version) {
  Batcher::Item it{dense_in, ids_in, h.batch, probs};
  std::unique_lock<std::mutex> l(bt.mu);
  bt.pending.push_back(&it); bt.pending_rows += h.batch;
  if (bt.leader_waiting) {                                                        // follower: tell the leader, wait for the slice
    bt.cv_leader.notify_one();
    bt.cv_done.wait(l, [&] { return it.done; });
    *version = it.version;
    return it.rc;
  }
  bt.leader_waiting = true;
  const auto deadline = std::chrono::steady_clock::now() + std::chrono::microseconds(sm->cfg.batching_timeout_us);
  // adaptive: an idle session means there is nothing to wait for (latency of a lone request = the unbatched latency); when every
  // session is busy, requests pile up here until one frees, the row budget is reached or the timeout expires
  const int nsess = (int)sm->sessions.size();
  bt.cv_leader.wait_until(l, deadline, [&] { return bt.pending_rows >= (uint32_t)sm->cfg.batching_max_rows || (sm->cfg.batching_adaptive && sm->busy.load() < nsess); });
  std::vector<Batcher::Item*> mine; mine.swap(bt.pending);                        // everything that arrived: later arrivals elect the next leader
  const uint32_t R = bt.pending_rows; bt.pending_rows = 0; bt.leader_waiting = false;
  l.unlock();
  auto m = std::atomic_load(&sm->model);
  int rc = 500;
  if (m) {
    if (mine.size() == 1) rc = RunRows(sm, m, it.dense, it.ids, it.rows, it.rows, it.probs, -1);
    else {
      const Arch& a = m->arch;
      std::vector<float> dense((size_t)R * a.num_dense), out((size_t)R * a.n_out);
      std::vector<int64_t> ids((size_t)a.R * R);                       // request-shaped: a.R id rows
      uint32_t off = 0;
      for (Batcher::Item* q : mine) {
        memcpy(dense.data() + (size_t)off * a.num_dense, q->dense, (size_t)q->rows * a.num_dense * 4);
        for (int t = 0; t < a.R; ++t) memcpy(ids.data() + (size_t)t * R + off, q->ids + (size_t)t * q->rows * 8, (size_t)q->rows * 8);
        off += q->rows;
      }
      rc = RunRows(sm, m, reinterpret_cast<const uint8_t*>(dense.data()), reinterpret_cast<const uint8_t*>(ids.data()), R, R, out.data(), -1);
      off = 0;
      for (Batcher::Item* q : mine) { if (rc == 200) memcpy(q->probs, out.data() + (size_t)off * a.n_out, (size_t)q->rows * a.n_out * 4); off += q->rows; }
    }
  }
  bt.merged_batches++; bt.merged_requests += mine.size();
  l.lock();
  for (Batcher::Item* q : mine) { q->rc = rc; q->version = m ? m->version : -1; q->done = true; }
  l.unlock();
  bt.cv_done.notify_all();
  *version = it.version;
  return rc;
}

static void SessionReleased(ServingModel* sm) {                                    // wakes a batch leader that is waiting for an idle session
  sm->busy.fetch_sub(1);
  if (Batcher* bt = sm->batcher.get()) { { std::lock_guard<std::mutex> l(bt->mu); } bt->cv_leader.notify_one(); }
}
static Batcher* BatcherOf(ServingModel* sm);

static int Predict(ServingModel* sm, const void* in, int in_size, void** out, int* out_size, int hint) {
  auto m = std::atomic_load(&sm->model);
  if (!m || in_size < (int)sizeof(drpb::WireReq)) return 500;
  drpb::WireReq h; memcpy(&h, in, sizeof(h));
  const Arch& a = m->arch;
  const size_t need = sizeof(h) + (size_t)h.batch * h.num_dense * 4 + (size_t)h.num_sparse * h.batch * 8;
  if (h.magic != drpb::kWireReqMagic || (int)h.num_dense != a.num_dense || (int)h.num_sparse != a.R || h.batch == 0 || (size_t)in_size < need) return 500;
  std::vector<float> probs((size_t)h.batch * a.n_out);
  const auto t0 = std::chrono::steady_clock::now();
  const uint8_t* p = static_cast<const uint8_t*>(in) + sizeof(h);
  const uint8_t* dense_in = p;
  const uint8_t* ids_in = p + (size_t)h.batch * a.num_dense * 4;
  int64_t version = m->version;
  int rc;
  if (sm->cfg.batching_max_rows > 0 && (int)h.batch * 2 <= sm->cfg.batching_max_rows) rc = PredictBatched(sm, *BatcherOf(sm), h, dense_in, ids_in, probs.data(), &version);
  else rc = RunRows(sm, m, dense_in, ids_in, h.batch, h.batch, probs.data(), hint);
  if (rc != 200) return rc;
  const uint64_t rq = ++sm->requests;
  if (sm->cfg.timeline_interval_step > 0 && (int64_t)rq >= sm->cfg.timeline_start_step && (rq % (uint64_t)sm->cfg.timeline_interval_step) == 0) {
    const double us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
    std::lock_guard<std::mutex> l(sm->tmu);
    if ((int)sm->trace.size() < sm->cfg.timeline_trace_count) {
      char line[160]; snprintf(line, sizeof(line), "{\"request\": %llu, \"batch\": %u, \"latency_us\": %.1f, \"model_version\": %lld}", (unsigned long long)rq, h.batch, us, (long long)version);
      sm->trace.emplace_back(line);
      if (!sm->cfg.timeline_path.empty()) { FILE* f = fopen(sm->cfg.timeline_path.c_str(), "a"); if (f) { fprintf(f, "%s\n", line); fclose(f); } }
    }
  }
  drpb::WireResp rh{drpb::kWireRespMagic, h.batch, 200, (uint32_t)(a.n_out > 1 ? a.n_out : 0), version};     // reserved = outputs per row (0: one)
  *out_size = (int)(sizeof(rh) + probs.size() * 4);
  *out = malloc((size_t)*out_size);
  memcpy(*out, &rh, sizeof(rh)); memcpy(static_cast<uint8_t*>(*out) + sizeof(rh), probs.data(), probs.size() * 4);
  return 200;
}

static Batcher* BatcherOf(ServingModel* sm) { return sm->batcher.get(); }

static int PredictAny(ServingModel* sm, const void* in, int in_size, void** out, int* out_size, int hint) {
  if (drpb::IsWireRequest(in, (size_t)std::max(in_size, 0))) return Predict(sm, in, in_size, out, out_size, hint);
  auto m = std::atomic_load(&sm->model);
  if (!m) return 500;
  drpb::Request rq; std::string wire, err, pb;
  if (!drpb::ParseRequest(in, (size_t)std::max(in_size, 0), &rq) || !drpb::RequestToWire(rq, m->arch.num_dense, m->arch.R, &wire, &err)) { sm->failures++; return 500; }
  void* w_out = nullptr; int w_size = 0;
  const int rc = Predict(sm, wire.data(), (int)wire.size(), &w_out, &w_size, hint);
  if (rc != 200) { free(w_out); return rc; }
  const bool ok = drpb::WireToResponse(w_out, (size_t)w_size, rq.output_filter, &pb);
  free(w_out);
  if (!ok) return 500;
  *out_size = (int)pb.size(); *out = malloc(pb.size() ? pb.size() : 1); memcpy(*out, pb.data(), pb.size());
  return 200;
}

// Warm-up: the request stored in warmup_file_name when present, else a synthetic batch cycling over stored keys -- every session runs once
static bool WarmUp(ServingModel* sm, const std::shared_ptr<Model>& m) {
  const Arch& a = m->arch;
  std::string raw;
  const bool from_file = !sm->cfg.warmup_file_name.empty() && drjson::ReadFile(sm->cfg.warmup_file_name, &raw) && drpb::IsWireRequest(raw.data(), raw.size());
  for (auto& sp : sm->sessions) {
    Session& s = *sp;
    std::lock_guard<std::mutex> l(s.mu);
    s.Grow(a);                                   // the new version may be wider than the one the buffers were sized for
    int B = std::min(64, s.max_batch);
    bool filled = false;
    if (from_file) {
      drpb::WireReq h; memcpy(&h, raw.data(), sizeof(h));
      const size_t need = sizeof(h) + (size_t)h.batch * h.num_dense * 4 + (size_t)h.num_sparse * h.batch * 8;
      if ((int)h.num_dense == a.num_dense && (int)h.num_sparse == a.R && h.batch > 0 && raw.size() >= need) {
        B = (int)std::min<uint32_t>(h.batch, (uint32_t)s.max_batch);
        const uint8_t* p = reinterpret_cast<const uint8_t*>(raw.data()) + sizeof(h);
        memcpy(s.dense.data(), p, (size_t)B * a.num_dense * 4);
        const int64_t* ids = reinterpret_cast<const int64_t*>(p + (size_t)h.batch * a.num_dense * 4);
        for (int c = 0; c < a.C; ++c) memcpy(s.ids.data() + (size_t)c * B, ids + (size_t)a.id_map[(size_t)c] * h.batch, (size_t)B * 8);
        filled = true;
      }
    }
    if (!filled) {
      for (int i = 0; i < B * a.num_dense; ++i) s.dense[(size_t)i] = (float)((i * 37) % 100) / 25.f;
      for (int c = 0; c < a.C; ++c) for (int i = 0; i < B; ++i)
        s.ids[(size_t)c * B + i] = m->tables.empty() ? (int64_t)i : m->sample_keys[(size_t)a.col_table[(size_t)c] * 64 + (size_t)(i % 64)];
    }
    auto dense = std::atomic_load(&m->dense);
    if (!s.Run(*m, *dense, B, sm->cfg.redis_prefix)) return false;
    for (int i = 0; i < B * a.n_out; ++i) if (!(s.prob[(size_t)i] >= 0.f && s.prob[(size_t)i] <= 1.f)) return false;       // NaN / garbage -> reject the version
  }
  return true;
}

static bool ApplyDelta(ServingModel* sm, const std::string& prefix, int64_t version) {
  auto m = std::atomic_load(&sm->model);
  if (!m) return false;
  dr::BundleReader r(prefix);
  if (!r.ok()) return false;
  for (int t = 0; t < m->arch.T && !m->tables.empty(); ++t) {      // (remote mode: the trainer inserts delta rows into the feature store itself)
    std::vector<int64_t> keys; std::vector<float> vals;
    if (!ReadDeltaRows(r, t, m->arch.D, &keys, &vals)) return false;
    if (keys.empty()) continue;
    dr_host_ev_import_cow(m->tables[(size_t)t], keys.data(), vals.data(), m->arch.D, (int64_t)keys.size());   // copy-on-write: readers never see a torn row
  }
  std::shared_ptr<Dense> dp;
  if (HasDenseBlock(r, m->arch) && BuildDense(r, m->arch, &dp)) std::atomic_store(&m->dense, dp);
  sm->delta_version = version;
  sm->delta_updates++;
  return true;
}

static void UpdaterLoop(ServingModel* sm) {
  int bad = 0;
#ifdef _OPENMP
  if (sm->compat.update_intra_threads > 0) omp_set_num_threads(sm->compat.update_intra_threads);    // model_update_intra_threads: the hot update's imports / packing run on this thread's team
#endif
  auto load_full = [&](int64_t v, const std::string& dir) {
    auto nm = LoadModel(dir, sm->cfg.remote);
    if (!nm) { if (++bad > 3) fprintf(stderr, "[deeprec_cpu_serving] skipping invalid model version %lld\n", (long long)v); return; }
    bad = 0;
    if (!WarmUp(sm, nm)) return;                  // also grows the sessions to a wider architecture
    std::atomic_store(&sm->model, nm);            // requests in flight keep the old model alive through their shared_ptr
    sm->delta_version = -1;
    sm->full_updates++;
  };
  RunUpdater(sm->cfg.checkpoint_dir.empty() ? sm->cfg.savedmodel_dir : sm->cfg.checkpoint_dir, sm->cfg.update_interval_ms, sm->stop, sm->model, sm->delta_version,
             load_full, [&](int64_t v, const std::string& prefix) { ApplyDelta(sm, prefix, v); });
}

}  // namespace cpusrv

extern "C" {

// model_entry: saved-model directory (may be empty if the JSON config names it).  Returns an opaque model handle; *state = 0 on success.
void* dr_cpu_initialize(const char* model_entry, const char* model_config, int* state) {
  using namespace cpusrv;
  auto* sm = new ServingModel();
  JVal j;
  if (model_config && *model_config && !drjson::ParseJson(model_config, &j)) { *state = -1; delete sm; return nullptr; }
  Config& c = sm->cfg;
  sm->compat = drcfg::ParseCompat(j, "deeprec_cpu_serving");
  if (!sm->compat.error.empty()) { *state = -1; delete sm; return nullptr; }
  c.session_num = (int)j.n("session_num", 2); c.max_batch = (int)j.n("max_batch", 4096);
  c.select_policy = j.s("select_session_policy", "RR") == "MOD" ? 1 : 0;
  c.update_interval_ms = (int)j.n("model_update_interval_ms", 1000);
  if (j.n("enable_batching", 0) != 0) {
    const drjson::JVal* bp = j.get("batching_parameters");
    const drjson::JVal& b = bp && bp->t == drjson::JVal::OBJ ? *bp : j;
    c.batching_max_rows = std::max(2, (int)b.n("max_batch_size", 64));
    c.batching_timeout_us = std::max(0, (int)b.n("batch_timeout_micros", 200));
    c.batching_adaptive = b.n("adaptive", 1) != 0;             // false: always wait for the row budget or the timeout (throughput over latency)
  }
  c.savedmodel_dir = j.s("savedmodel_dir", model_entry ? model_entry : ""); c.checkpoint_dir = j.s("checkpoint_dir", "");
  c.warmup_file_name = j.s("warmup_file_name", ""); c.timeline_path = j.s("timeline_path", "");
  c.timeline_start_step = (int64_t)j.n("timeline_start_step", -1); c.timeline_interval_step = (int)j.n("timeline_interval_step", 0);
  c.timeline_trace_count = (int)j.n("timeline_trace_count", 0);
  c.remote = j.s("feature_store_type", "local") == "redis";
  if (c.remote) {
    const std::string url = j.s("redis_url", "127.0.0.1:6379");
    const size_t colon = url.rfind(':');
    c.redis_host = colon == std::string::npos ? url : url.substr(0, colon);
    c.redis_port = colon == std::string::npos ? 6379 : atoi(url.c_str() + colon + 1);
    c.redis_password = j.s("redis_password", ""); c.redis_db = (int)j.n("redis_db_idx", 0);
    c.redis_prefix = j.s("redis_prefix", "dlrm"); c.redis_timeout_ms = (int)j.n("redis_timeout_ms", 2000);
  }
  auto m = LoadModel(c.savedmodel_dir, c.remote);
  if (!m || c.max_batch <= 0) { *state = -1; delete sm; return nullptr; }
  // sessions run concurrently: each gets cores / sessions OpenMP threads for its GEMMs unless intra_op_parallelism_threads says otherwise
  c.intra_threads = (int)j.n("intra_op_parallelism_threads", sm->compat.omp_num_threads);      // omp_num_threads: the reference's MKL team = a session's OpenMP team here
  {                                                                  // executor policy: ModelConfig first, then the reference's environment switches
    const std::string ep = j.s("executor_policy", "");
    if (ep == "cost_model") c.executor_policy = 1; else if (ep == "inline") c.executor_policy = 2; else if (ep == "normal") c.executor_policy = 0;
    else {
      if (j.n("enable_inline_execute", 0) != 0) c.executor_policy = 2;
      const char* e1 = getenv("USE_COST_MODEL_EXECUTOR"); const char* e2 = getenv("USE_INLINE_EXECUTOR");
      if (e1 && e1[0] == '1') c.executor_policy = 1;
      if (e2 && e2[0] == '1') c.executor_policy = 2;
    }
    const char* s0 = getenv("START_NODE_STATS_STEP"); const char* s1 = getenv("STOP_NODE_STATS_STEP");
    c.stats_start = (int)j.n("start_node_stats_step", s0 ? atoi(s0) : c.stats_start);
    c.stats_stop = (int)j.n("stop_node_stats_step", s1 ? atoi(s1) : c.stats_stop);
    if (c.stats_stop <= c.stats_start) c.stats_stop = c.stats_start + 1;
  }
  const int hw = (int)std::max(1u, std::thread::hardware_concurrency());
  const int per_session = c.intra_threads > 0 ? c.intra_threads : std::max(1, hw / std::max(1, c.session_num));
  {
    std::string sets = j.s("cpusets", "");
    if (sets.empty() && getenv("SESSION_GROUP_CPUSET")) sets = getenv("SESSION_GROUP_CPUSET");
    if (!sets.empty()) c.cpusets = ParseCpusets(sets);
    else if (getenv("SET_SESSION_THREAD_POOL_AFFINITY") && atoi(getenv("SET_SESSION_THREAD_POOL_AFFINITY")) != 0) c.cpusets = AutoCpusets(std::max(1, c.session_num));
  }
  for (int i = 0; i < std::max(1, c.session_num); ++i) {
    sm->sessions.emplace_back(new Session());
    Session& ns = *sm->sessions.back();
    if (!c.cpusets.empty()) {                                   // fewer sets than sessions: the sets are reused round-robin
      ns.cpus = c.cpusets[(size_t)i % c.cpusets.size()];
      CPU_ZERO(&ns.mask); for (int cpu : ns.cpus) CPU_SET(cpu, &ns.mask);
    }
    ns.Init(m->arch, c.max_batch, c.intra_threads > 0 || ns.cpus.empty() ? per_session : (int)ns.cpus.size());
    ns.exec_policy = c.executor_policy; ns.stats_start = c.stats_start; ns.stats_stop = c.stats_stop;
    if (c.remote) {                                             // one connection per session (sessions run concurrently)
      void* conn = dr_redis_connect(c.redis_host.c_str(), c.redis_port, c.redis_timeout_ms, c.redis_password.c_str(), c.redis_db);
      if (!dr_redis_ok(conn)) { fprintf(stderr, "[deeprec_cpu_serving] feature store %s:%d: %s\n", c.redis_host.c_str(), c.redis_port, dr_redis_last_error(conn)); dr_redis_close(conn); *state = -2; delete sm; return nullptr; }
      sm->sessions.back()->redis = conn;
    }
  }
  if (!WarmUp(sm, m)) { *state = -1; delete sm; return nullptr; }
  sm->batcher = std::make_shared<cpusrv::Batcher>();
  std::atomic_store(&sm->model, m);
  if (c.update_interval_ms > 0) sm->updater = std::thread(UpdaterLoop, sm);
  *state = 0;
  return sm;
}

int dr_cpu_process(void* model_buf, const void* input_data, int input_size, void** output_data, int* output_size) {
  if (!model_buf) return 500;
  return cpusrv::PredictAny(static_cast<cpusrv::ServingModel*>(model_buf), input_data, input_size, output_data, output_size, -1);
}

// input_size[0] = number of requests, followed by their sizes (one call, several PredictRequests)
int dr_cpu_batch_process(void* model_buf, const void* input_data[], int* input_size, void* output_data[], int* output_size) {
  if (!model_buf || !input_size) return 500;
  int n = input_size[0], rc = 200;
  for (int i = 0; i < n; ++i) {
    const int r = cpusrv::PredictAny(static_cast<cpusrv::ServingModel*>(model_buf), input_data[i], input_size[i + 1], &output_data[i], &output_size[i], i);
    if (r != 200) rc = r;
  }
  return rc;
}

int dr_cpu_get_serving_model_info(void* model_buf, void** output_data, int* output_size) {
  if (!model_buf) return 500;
  auto* sm = static_cast<cpusrv::ServingModel*>(model_buf);
  auto m = std::atomic_load(&sm->model);
  std::ostringstream os;
  os << "{\"model_version\": " << (m ? m->version : -1) << ", \"delta_version\": " << sm->delta_version.load() << ", \"model_path\": \"" << (m ? m->path : "")
     << "\", \"sessions\": " << sm->sessions.size() << ", \"requests\": " << sm->requests.load() << ", \"failures\": " << sm->failures.load()
     << ", \"mlp_dtype\": \"fp32\", \"device\": \"cpu\", \"model\": \"" << (m ? m->arch.model_name : "") << "\", \"feature_store_type\": \"" << (sm->cfg.remote ? "redis" : "local") << "\", \"full_updates\": " << sm->full_updates.load() << ", \"delta_updates\": " << sm->delta_updates.load()
     << ", \"num_dense\": " << (m ? m->arch.num_dense : 0) << ", \"num_sparse\": " << (m ? m->arch.R : 0) << ", \"num_tables\": " << (m ? m->arch.T : 0);
  os << ", \"batching\": {\"max_batch_size\": " << sm->cfg.batching_max_rows << ", \"batch_timeout_micros\": " << sm->cfg.batching_timeout_us
     << ", \"merged_batches\": " << (sm->batcher ? sm->batcher->merged_batches.load() : 0) << ", \"merged_requests\": " << (sm->batcher ? sm->batcher->merged_requests.load() : 0) << "}";
  {
    static const char* kPol[] = {"normal", "cost_model", "inline"};
    os << ", \"executor\": {\"policy\": \"" << kPol[std::min(2, std::max(0, sm->cfg.executor_policy))] << "\"";
    const cpusrv::ProgPlan* pl = (m && m->dense) ? m->dense->plan.get() : nullptr;
    if (pl) {
      os << ", \"ops\": " << pl->succ.size() << ", \"traced_runs\": " << pl->traced.load() << ", \"cost_model_ready\": " << (pl->ready.load() ? "true" : "false");
      if (pl->ready.load()) os << ", \"total_us\": " << pl->total_us << ", \"critical_path_us\": " << pl->critical_us << ", \"dag_width\": " << pl->width
                               << ", \"team\": " << pl->team << ", \"parallel\": " << (pl->parallel ? "true" : "false");
    }
    os << "}";
  }
  os << ", \"threads_per_session\": " << (sm->sessions.empty() ? 0 : sm->sessions[0]->threads) << ", \"model_config\": " << drcfg::ToJson(sm->compat);
  os << ", \"cpusets\": \"";
  for (size_t i = 0; i < sm->cfg.cpusets.size(); ++i) { if (i) os << ";"; for (size_t k = 0; k < sm->cfg.cpusets[i].size(); ++k) os << (k ? "," : "") << sm->cfg.cpusets[i][k]; }
  os << "\", \"session_last_cpu\": [";
  for (size_t i = 0; i < sm->sessions.size(); ++i) os << (i ? ", " : "") << sm->sessions[i]->last_cpu.load();
  os << "]}";
  const std::string s = os.str();
  *output_size = (int)s.size();
  *output_data = malloc(s.size() + 1);
  memcpy(*output_data, s.c_str(), s.size() + 1);
  return 200;
}

void dr_cpu_serving_release(void* model_buf) { delete static_cast<cpusrv::ServingModel*>(model_buf); }
void dr_cpu_serving_free(void* p) { free(p); }

}  // extern "C"
