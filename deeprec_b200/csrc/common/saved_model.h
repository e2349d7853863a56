// Saved-model format shared by the two native Processors (csrc/cuda/serving_runtime.cu, csrc/host/cpu_serving.cc): saved_model.json, the
// bundle tensors of the dense part and of the tables, delta bundles and serving_versions.json.  Header-only so the host library, the CUDA
// library and its CPU emulation build all compile the one copy.
//
// This module owns what a valid export looks like: every tensor is read as fp32 (through dr::ReadAsFloat, so bf16 / f16 / int8 converted
// models load like the original) and every length is checked against the architecture before a runtime sees it.  The runtimes only turn
// the checked fp32 vectors into their own weight layout and add the conditions of their kernels.
#pragma once
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <memory>
#include <string>
#include <thread>
#include <type_traits>
#include <utility>
#include <vector>

#include "bundle.h"
#include "mini_json.h"

namespace drsm {

inline int pad8(int n) { return (n + 7) / 8 * 8; }

// Op program (saved_model.json "arch": "program", serving/export.py::export_saved_model_program): the inference graph of a model other than
// DLRM as a list of ops over [B, width] buffers; buffer 0 = dense inputs, buffer 1 = embeddings [B, C * D].
enum POpKind { P_CONCAT, P_LINEAR, P_AFFINE, P_FM, P_CROSS, P_MUL_ADD, P_ADD, P_LAYERNORM, P_MUL, P_SLICE,
               P_VALID_MASK, P_SEQ_ZIP, P_SEQ_MASK, P_SEQ_SUM, P_DIN_ATT, P_PRELU, P_SOFTMAX, P_COSINE, P_TILE, P_GRU, P_SEQ_LAST, P_MHA, P_SEQ_MEAN,
               P_CROSS_LINEAR, P_NUM_OPS };
// rows1: sample-aware graph compression (serving/export.py::compress_sample_aware) -- the op depends on user-side features only, which are
// identical for every candidate row of a ranking request: it runs at batch 1 on row 0 of its inputs; a TILE op broadcasts row 0 to the batch
// where a per-candidate op consumes the result (reference: python/graph_optimizer/sample_awared_graph_compression.py:26).
// len on LINEAR / LAYERNORM: the op is applied at each of `len` positions of a [B, len * w] sequence buffer (DIEN / BST); mode: din_attention output
// (0 = weighted sum of the keys, 1 = the softmax weights), seq_mean divisor (0 = count, 1 = sqrt(count): the sqrtn combiner); heads: mha
struct POp { int kind = 0, out = 0; std::vector<int> in; bool relu = false, rows1 = false; float eps = 1e-5f; int start = 0, len = 0, mode = 0, heads = 1; std::string name; };
struct Arch {
  int num_dense = 13, T = 0, D = 16; std::vector<int> bot, top; float bn_eps = 1e-3f; int inter = 0, Zp = 0;     // Zp: interaction width padded to 8
  bool program = false; std::vector<POp> ops; int nbuf = 2, out_buf = -1; std::string model_name = "dlrm";
  // requests carry R id rows; lookup column c reads request row id_map[c] (identity unless several columns share a feature, e.g. the wide
  // and the deep table of one Wide&Deep column) from table col_table[c] (identity unless several columns share a TABLE, e.g. DIN's target
  // item and its L history positions).  C == T and col_table == identity for every model exported before col_table existed.
  int R = 0, C = 0; std::vector<int> id_map, col_table;
  // multi-task programs: the output buffer is [B, n_out] logits, the response carries n_out probabilities per row (sample-major)
  int n_out = 1; std::vector<std::string> out_names;
};

// One tensor of the bundle; float tensors through ReadAsFloat.
template <typename T> inline bool ReadVec(dr::BundleReader& r, const std::string& name, std::vector<T>* out) {
  if constexpr (std::is_same<T, float>::value) {
    return dr::ReadAsFloat(r, name, out);
  } else {
    const dr::BundleEntry* e = r.Find(name);
    if (!e || e->nbytes % (int64_t)sizeof(T)) return false;
    out->resize((size_t)e->nbytes / sizeof(T));
    return r.Read(*e, out->data(), 1) == 0;
  }
}

// <dir>/saved_model.json -> architecture, version and the bundle prefix of the variables
inline bool ParseArch(const std::string& dir, Arch* a, int64_t* version, std::string* prefix) {
  using drjson::JVal;
  std::string txt; JVal j;
  if (!drjson::ReadFile(dir + "/saved_model.json", &txt) || !drjson::ParseJson(txt, &j)) return false;
  a->num_dense = (int)j.n("num_dense", 13); a->D = (int)j.n("embedding_dim", 16); a->bn_eps = (float)j.n("bn_eps", 1e-3);
  a->T = (int)j.n("num_tables", 0);
  if (auto* b = j.get("mlp_bot")) for (auto& v : b->arr) a->bot.push_back((int)v.num);
  if (auto* b = j.get("mlp_top")) for (auto& v : b->arr) a->top.push_back((int)v.num);
  const int F = a->T + 1; a->inter = a->D + F * (F - 1) / 2; a->Zp = pad8(a->inter);
  *version = (int64_t)j.n("version", 0);
  *prefix = dir + "/" + j.s("variables", "variables/variables");
  a->model_name = j.s("model", "dlrm");
  if (a->D <= 0) return false;
  a->C = a->T;
  if (auto* ct = j.get("col_table")) {
    if (ct->t != JVal::ARR || ct->arr.empty()) return false;
    a->C = (int)ct->arr.size();
    for (auto& v : ct->arr) a->col_table.push_back((int)v.num);
  } else for (int t = 0; t < a->T; ++t) a->col_table.push_back(t);
  for (int v : a->col_table) if (v < 0 || v >= a->T) return false;
  a->R = (int)j.n("num_id_rows", a->C);
  a->id_map.resize((size_t)std::max(0, a->C));
  for (int c = 0; c < a->C; ++c) a->id_map[(size_t)c] = c;
  if (auto* im = j.get("id_map")) {
    if (im->t != JVal::ARR || (int)im->arr.size() != a->C) return false;
    for (int c = 0; c < a->C; ++c) a->id_map[(size_t)c] = (int)im->arr[(size_t)c].num;
  }
  for (int v : a->id_map) if (v < 0 || v >= a->R) return false;
  if (a->R <= 0) return false;
  if (j.s("arch", "") != "program") return a->T > 0 && !a->bot.empty() && !a->top.empty() && a->bot.back() == a->D;
  a->program = true;
  std::vector<std::string> names = {"dense", "emb"};
  auto id_of = [&](const std::string& n) { for (size_t i = 0; i < names.size(); ++i) if (names[i] == n) return (int)i; return -1; };
  static const char* kNames[] = {"concat", "linear", "affine", "fm", "cross", "mul_add", "add", "layernorm", "mul", "slice",
                                 "valid_mask", "seq_zip", "seq_mask", "seq_sum", "din_attention", "prelu", "softmax", "cosine", "tile", "gru", "seq_last", "mha", "seq_mean",
                                 "cross_linear"};
  static const int kArity[] = {-1, 1, 1, 1, 2, 3, 2, 1, 2, 1, 1, 2, 2, 1, 3, 1, 1, 2, 1, 1, 2, 2, 2, 3};
  const JVal* pr = j.get("program");
  if (!pr || pr->t != JVal::ARR) return false;
  std::vector<bool> rows1_buf(2, false);
  for (const JVal& o : pr->arr) {
    POp op; op.name = o.s("out", ""); op.relu = o.n("relu", 0) != 0; op.eps = (float)o.n("eps", 1e-5); op.kind = -1;
    op.start = (int)o.n("start", 0); op.len = (int)o.n("len", 0); op.rows1 = o.n("rows1", 0) != 0; op.mode = (int)o.n("mode", 0); op.heads = (int)o.n("heads", 1);
    const std::string kind = o.s("op", "");
    for (int k = 0; k < P_NUM_OPS; ++k) if (kind == kNames[k]) op.kind = k;
    const JVal* in = o.get("in");
    if (op.kind < 0 || op.name.empty() || !in || id_of(op.name) >= 0) return false;
    for (const JVal& v : in->arr) { const int id = id_of(v.str); if (id < 0) return false; op.in.push_back(id); }    // inputs must already exist
    if ((kArity[op.kind] >= 0 && (int)op.in.size() != kArity[op.kind]) || op.in.empty()) return false;
    // a buffer computed at batch 1 holds one valid row: only rows1 ops and TILE may read it
    if (op.kind == P_TILE && op.rows1) return false;
    if (!op.rows1 && op.kind != P_TILE) for (int id : op.in) if (id < (int)rows1_buf.size() && rows1_buf[(size_t)id]) return false;
    op.out = (int)names.size(); names.push_back(op.name);
    rows1_buf.resize(names.size(), false); rows1_buf[(size_t)op.out] = op.rows1;
    a->ops.push_back(std::move(op));
  }
  a->nbuf = (int)names.size();
  a->out_buf = id_of(j.s("output", ""));
  if (a->out_buf >= 0 && a->out_buf < (int)rows1_buf.size() && rows1_buf[(size_t)a->out_buf]) return false;
  a->n_out = (int)j.n("num_outputs", 1);
  if (auto* on = j.get("output_names")) for (auto& v : on->arr) a->out_names.push_back(v.str);
  return a->T > 0 && a->out_buf >= 2 && a->n_out >= 1 && a->n_out <= 16;
}

// fp32 tensors of one program op, row-major as exported
struct OpTensors {
  int N = 0, K = 0;                       // linear: kernel [N, K], K per position of a sequence | gru: w_ih [3H, I] (N = 3H, K = I) | cross_linear: kernel [N, r] (K = r)
  std::vector<float> W, b;                // linear, cross_linear: kernel, bias | gru: w_ih, b_ih
  std::vector<float> v0, v1;              // affine, layernorm: scale, shift | cross: w, b | prelu: alpha | gru: w_hh [3H, H], b_hh
  std::vector<std::vector<float>> att;    // din_attention: w1 [H1, 4W] b1 w2 [H2, H1] b2 w3 [H2] b3 [1]
  int H1 = 0, H2 = 0;                     // gru: H1 = H | din_attention: hidden widths
};
struct ProgramData { std::vector<OpTensors> ops; std::vector<int> width; };

// Weights + buffer widths of a program model; every shape is checked against the widths implied by the op list.
inline bool ReadProgram(dr::BundleReader& r, const Arch& a, ProgramData* out) {
  std::vector<int>& width = out->width;
  width.assign((size_t)a.nbuf, 0); width[0] = a.num_dense; width[1] = a.C * a.D;
  out->ops.assign(a.ops.size(), OpTensors());
  for (size_t i = 0; i < a.ops.size(); ++i) {
    const POp& op = a.ops[i]; OpTensors& t = out->ops[i];
    const int w0 = width[(size_t)op.in[0]];
    const int w1 = op.in.size() > 1 ? width[(size_t)op.in[1]] : 0;
    int w = w0;
    const std::string base = "prog/" + op.name + "/";
    switch (op.kind) {
      case P_CONCAT: w = 0; for (int b : op.in) w += width[(size_t)b]; break;
      case P_LINEAR: {                                               // len > 0: the same Linear at each of len positions ([B, len * K] == [B * len, K])
        const int S = op.len > 0 ? op.len : 1;
        if (w0 % S) return false;
        t.K = w0 / S;
        if (!ReadVec(r, base + "kernel", &t.W) || !ReadVec(r, base + "bias", &t.b) || t.b.empty() || t.W.size() != t.b.size() * (size_t)t.K) return false;
        t.N = (int)t.b.size();
        w = t.N * S; break;
      }
      case P_LAYERNORM: {                                            // len > 0: per position of a [B, len * w] sequence
        const int S = op.len > 0 ? op.len : 1;
        if (w0 % S || !ReadVec(r, base + "scale", &t.v0) || !ReadVec(r, base + "shift", &t.v1) || (int)t.v0.size() != w0 / S || (int)t.v1.size() != w0 / S) return false;
        break;
      }
      case P_AFFINE: if (!ReadVec(r, base + "scale", &t.v0) || !ReadVec(r, base + "shift", &t.v1) || (int)t.v0.size() != w0 || (int)t.v1.size() != w0) return false; break;
      case P_FM: if (op.in[0] != 1) return false; w = a.D; break;
      case P_CROSS: if (!ReadVec(r, base + "w", &t.v0) || !ReadVec(r, base + "b", &t.v1) || (int)t.v0.size() != w0 || (int)t.v1.size() != w0 || w1 != w0) return false; break;
      case P_MUL_ADD: if (w1 != w0 || width[(size_t)op.in[2]] != w0) return false; break;
      case P_MUL:
      case P_ADD: if (w1 != w0) return false; break;
      case P_SLICE: if (op.start < 0 || op.len <= 0 || op.start + op.len > w0) return false; w = op.len; break;
      case P_VALID_MASK: if (op.start < 0 || op.len <= 0 || op.start + op.len > a.C) return false; w = op.len; break;      // [B, len]: 1 where the id of column start + l is >= 0
      case P_SEQ_ZIP: if (op.len <= 0 || w0 % op.len || w1 % op.len) return false; w = w0 + w1; break;                      // position-wise concat of [B, L, *] sequences
      case P_SEQ_MASK: if (op.len <= 0 || w0 % op.len || w1 != op.len) return false; break;                                // x [B, L * W] * mask [B, L]
      case P_SEQ_SUM: if (op.len <= 0 || w0 % op.len) return false; w = w0 / op.len; break;                                // sum over the L positions
      case P_PRELU: if (!ReadVec(r, base + "alpha", &t.v0) || (int)t.v0.size() != w0) return false; break;
      case P_SOFTMAX: break;                                         // row-wise softmax (mixture-of-experts gates)
      case P_TILE: break;                                            // row 0 of a once-per-request buffer -> every row of the batch
      case P_GRU: {                                                  // x [B, L * I] -> every hidden state [B, L * H] (PyTorch gate order r, z, n; h0 = 0)
        if (op.len <= 0 || w0 % op.len || !ReadVec(r, base + "w_ih", &t.W) || !ReadVec(r, base + "w_hh", &t.v0) || !ReadVec(r, base + "b_ih", &t.b) || !ReadVec(r, base + "b_hh", &t.v1)) return false;
        const int I = w0 / op.len, H3 = (int)t.b.size(), H = H3 / 3;
        if (H <= 0 || H3 != 3 * H || (int)t.v1.size() != H3 || (int)t.W.size() != H3 * I || (int)t.v0.size() != H3 * H) return false;
        t.N = H3; t.K = I; t.H1 = H;
        w = op.len * H; break;
      }
      case P_SEQ_MEAN: if (op.mode < 0 || op.mode > 1) return false; [[fallthrough]];                            // mean (mode 1: sum / sqrt(count))
      case P_SEQ_LAST:                                               // the state at the last valid position
        if (op.len <= 0 || w0 % op.len || w1 != op.len) return false;
        w = w0 / op.len; break;
      case P_CROSS_LINEAR: {                                         // x0 [B, N], x_l [B, N], t [B, r]: x0 * (t kernel^T + bias) + x_l, kernel [N, r]
        const int rank = width[(size_t)op.in[2]];
        if (w1 != w0 || !ReadVec(r, base + "kernel", &t.W) || !ReadVec(r, base + "bias", &t.b) || (int)t.b.size() != w0 || t.W.size() != (size_t)w0 * rank) return false;
        t.N = w0; t.K = rank;
        break;
      }
      case P_MHA: {                                                  // qkv [B, S * 3E] (per position [q | k | v]), valid [B, S] -> [B, S * E]
        if (op.len <= 0 || w0 % (3 * op.len) || w1 != op.len) return false;
        const int E = w0 / (3 * op.len);
        if (op.heads <= 0 || E % op.heads) return false;
        w = op.len * E; break;
      }
      case P_COSINE: if (w1 != w0) return false; w = 1; break;      // cosine similarity of two [B, W] towers -> [B, 1]
      case P_DIN_ATT: {                                              // q [B, W], k [B, L * W], mask [B, L] -> [B, W] (mode 0) | [B, L] (mode 1)
        const int L = width[(size_t)op.in[2]];
        if (L <= 0 || w1 != L * w0 || op.mode < 0 || op.mode > 1) return false;
        if (op.mode == 1) w = L;                                     // the softmax weights themselves (DIEN)
        static const char* kT[] = {"w1", "b1", "w2", "b2", "w3", "b3"};
        t.att.resize(6);
        for (int k = 0; k < 6; ++k) if (!ReadVec(r, base + kT[k], &t.att[(size_t)k])) return false;
        t.H1 = (int)t.att[1].size(); t.H2 = (int)t.att[3].size();
        if (t.H1 <= 0 || t.H2 <= 0 || (int)t.att[0].size() != t.H1 * 4 * w0 || (int)t.att[2].size() != t.H2 * t.H1 || (int)t.att[4].size() != t.H2 || t.att[5].size() != 1) return false;
        break;
      }
      default: return false;
    }
    if (w <= 0) return false;
    width[(size_t)op.out] = w;
  }
  return width[(size_t)a.out_buf] >= a.n_out;                        // the output buffer holds n_out logits per row
}

// DLRM dense block.  W [N, Kp = pad8(K)] row-major as exported (columns >= K are padding); the BatchNorm (moving statistics) of bottom layer
// l-1 is folded into Linear l: W' = W diag(s), b' = b + W t, and the last bottom layer's BatchNorm stays explicit as last_scale / last_shift.
struct DenseLayer { int N = 0, K = 0, Kp = 0; std::vector<float> W, b; };
struct DlrmDense { std::vector<DenseLayer> bot, top; std::vector<float> last_scale, last_shift, head_w, head_b; };

inline bool ReadDlrmDense(dr::BundleReader& r, const Arch& a, DlrmDense* out) {
  std::vector<float> s_prev, t_prev;
  int k = a.num_dense;
  for (size_t l = 0; l < a.bot.size(); ++l) {
    const std::string nm = "mlp_bot_" + std::to_string(l);
    DenseLayer L; L.N = a.bot[l]; L.K = k; L.Kp = pad8(k);
    const size_t N = (size_t)std::max(0, L.N);
    std::vector<float> gamma, beta, mean, var;
    if (L.N <= 0 || !ReadVec(r, "dense/" + nm + "/kernel", &L.W) || !ReadVec(r, "dense/" + nm + "/bias", &L.b) || !ReadVec(r, "dense/" + nm + "/bn_gamma", &gamma) ||
        !ReadVec(r, "dense/" + nm + "/bn_beta", &beta) || !ReadVec(r, "bn/" + nm + "/moving_mean", &mean) || !ReadVec(r, "bn/" + nm + "/moving_variance", &var)) return false;
    if (L.W.size() != N * L.Kp || L.b.size() != N || gamma.size() != N || beta.size() != N || mean.size() != N || var.size() != N) return false;
    for (size_t n = 0; n < N && l > 0; ++n) {
      double acc = L.b[n];
      for (int kk = 0; kk < k; ++kk) { float& w = L.W[n * L.Kp + kk]; acc += (double)w * t_prev[(size_t)kk]; w *= s_prev[(size_t)kk]; }
      L.b[n] = (float)acc;
    }
    s_prev.assign(N, 0.f); t_prev.assign(N, 0.f);
    for (size_t n = 0; n < N; ++n) { const float rs = 1.0f / std::sqrt(var[n] + a.bn_eps); s_prev[n] = gamma[n] * rs; t_prev[n] = beta[n] - mean[n] * s_prev[n]; }
    out->bot.push_back(std::move(L));
    k = (int)N;
  }
  out->last_scale = std::move(s_prev); out->last_shift = std::move(t_prev);
  k = a.inter;
  for (size_t l = 0; l < a.top.size(); ++l) {
    const std::string nm = "mlp_top_" + std::to_string(l);
    DenseLayer L; L.N = a.top[l]; L.K = k; L.Kp = pad8(k);
    const size_t N = (size_t)std::max(0, L.N);
    if (L.N <= 0 || !ReadVec(r, "dense/" + nm + "/kernel", &L.W) || !ReadVec(r, "dense/" + nm + "/bias", &L.b) || L.W.size() != N * L.Kp || L.b.size() != N) return false;
    out->top.push_back(std::move(L));
    k = (int)N;
  }
  return ReadVec(r, "dense/logits/kernel", &out->head_w) && ReadVec(r, "dense/logits/bias", &out->head_b) && !out->head_b.empty() && out->head_w.size() >= (size_t)k;
}

// table/<t>-keys, -values [n, D], -default [dvd, D] (required); -freqs, -versions (optional: dropped unless there is one per key)
struct TableData { std::vector<int64_t> keys, freqs, versions; std::vector<float> values, def; };

inline bool ReadTable(dr::BundleReader& r, int t, int D, TableData* d) {
  const std::string base = "table/" + std::to_string(t);
  if (!ReadVec(r, base + "-keys", &d->keys) || !ReadVec(r, base + "-values", &d->values) || !ReadVec(r, base + "-default", &d->def)) return false;
  if (!ReadVec(r, base + "-freqs", &d->freqs) || d->freqs.size() != d->keys.size()) d->freqs.clear();
  if (!ReadVec(r, base + "-versions", &d->versions) || d->versions.size() != d->keys.size()) d->versions.clear();
  return !d->def.empty() && d->def.size() % (size_t)D == 0 && d->values.size() == d->keys.size() * (size_t)D;
}

// Delta rows of table t (table/<t>-sparse_incr_keys / -values): true with no keys when the delta does not touch the table, false when the
// values are missing or do not hold one D-wide row per key.
inline bool ReadDeltaRows(dr::BundleReader& r, int t, int D, std::vector<int64_t>* keys, std::vector<float>* vals) {
  const std::string base = "table/" + std::to_string(t);
  if (!ReadVec(r, base + "-sparse_incr_keys", keys)) keys->clear();
  if (keys->empty()) return true;
  return ReadVec(r, base + "-sparse_incr_values", vals) && vals->size() == keys->size() * (size_t)D;
}

// A delta carries a new dense block when it holds the logits (DLRM) or the kernel of the program's first Linear.
inline bool HasDenseBlock(const dr::BundleReader& r, const Arch& a) {
  if (!a.program) return r.Find("dense/logits/kernel") != nullptr;
  for (const POp& op : a.ops) if (op.kind == P_LINEAR) return r.Find("prog/" + op.name + "/kernel") != nullptr;
  return false;
}

// The model updater's loop.  Every update_interval_ms (in 20 ms ticks, at least one) it rereads <dir>/serving_versions.json =
// {"full": {"version": V, "dir": "..."}, "deltas": [{"version": v, "base": V, "prefix": "..."}]}.  A full version newer than the live model
// goes to load_full(version, dir) and ends the poll; otherwise every delta whose base is the live version and whose version is newer than
// both the live version and the last applied delta goes to apply_delta(version, prefix), in file order.
template <class Model, class LoadFull, class ApplyDelta>
void RunUpdater(const std::string& dir, int update_interval_ms, const std::atomic<bool>& stop, const std::shared_ptr<Model>& live,
                const std::atomic<int64_t>& delta_version, LoadFull load_full, ApplyDelta apply_delta) {
  const std::string path = dir + "/serving_versions.json";
  while (!stop) {
    for (int i = 0; i < std::max(1, update_interval_ms / 20) && !stop; ++i) std::this_thread::sleep_for(std::chrono::milliseconds(20));
    std::string txt; drjson::JVal j;
    if (!drjson::ReadFile(path, &txt) || !drjson::ParseJson(txt, &j)) continue;
    const auto cur = std::atomic_load(&live);
    if (!cur) continue;
    if (auto* f = j.get("full")) {
      const int64_t v = (int64_t)f->n("version", -1); const std::string d = f->s("dir", "");
      if (v > cur->version && !d.empty()) { load_full(v, d); continue; }
    }
    if (auto* d = j.get("deltas"))
      for (auto& e : d->arr) {
        const int64_t v = (int64_t)e.n("version", -1), base = (int64_t)e.n("base", -1);
        if (base == cur->version && v > std::max<int64_t>(cur->version, delta_version.load())) apply_delta(v, e.s("prefix", ""));
      }
  }
}

}  // namespace drsm
