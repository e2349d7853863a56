// ModelConfig compatibility: every key of the reference Processor's JSON configuration (serving/processor/serving/model_config.{h,cc},
// docs/docs_en/Processor.md "Configure file") is classified ONCE here for both native runtimes (csrc/host/cpu_serving.cc, csrc/cuda/serving_runtime.cu):
//   * keys a runtime implements are read by that runtime (session_num, select_session_policy, cpusets, checkpoint_dir, warmup_file_name, timeline_*,
//     feature_store_type / redis_*, enable_inline_execute, enable_device_placement_optimization, intra_op_parallelism_threads, ...);
//   * keys with a direct equivalent are mapped (omp_num_threads -> the per-session team when intra_op_parallelism_threads is absent,
//     model_update_intra_threads -> the updater thread's OpenMP team, gpu_ids_list -> the first id when gpu_id is absent: one native instance serves
//     one GPU, serving.ProcessorGroup fans a list out);
//   * keys whose behaviour is structural here are accepted and reported (use_per_session_threads: every session always owns its team;
//     use_multi_stream: every GPU session always owns its stream; inter_op_parallelism_threads / model_update_inter_threads: no inter-op pools;
//     kmp_blocktime: no Intel OpenMP runtime; init_timeout_minutes, signature_name: reserved / single-signature models);
//   * values this build cannot honour are an initialisation ERROR with the reason (model_store_type oss / hdfs and oss:// hdfs:// paths: no remote
//     filesystem plugins -- SURVEY 2.10 n/a; serialize_protocol other than protobuf);
//   * anything else is reported as unknown (a typo would otherwise silently fall back to a default).
#pragma once
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "mini_json.h"

namespace drcfg {

struct Compat {
  int omp_num_threads = 0, update_intra_threads = 0, first_gpu = -1;
  std::string signature_name = "serving_default";
  std::vector<std::string> structural, unknown;      // accepted-by-construction keys present in the config; keys nobody knows
  std::string error;                                 // non-empty: initialize() must fail
};

inline bool Known(const std::string& k) {
  static const char* kKeys[] = {
      // reference keys
      "session_num", "select_session_policy", "use_per_session_threads", "cpusets", "gpu_ids_list", "use_multi_stream", "enable_device_placement_optimization",
      "enable_inline_execute", "omp_num_threads", "kmp_blocktime", "feature_store_type", "redis_url", "redis_password", "redis_db_idx", "read_thread_num",
      "update_thread_num", "serialize_protocol", "inter_op_parallelism_threads", "intra_op_parallelism_threads", "model_update_inter_threads",
      "model_update_intra_threads", "init_timeout_minutes", "signature_name", "warmup_file_name", "model_store_type", "checkpoint_dir", "savedmodel_dir",
      "oss_endpoint", "oss_access_id", "oss_access_key", "timeline_start_step", "timeline_interval_step", "timeline_trace_count", "timeline_path",
      "lock_file", "shard_embedding", "shard_embedding_names", "ev_storage_type", "ev_storage_path", "ev_storage_size",
      // keys of this build
      "max_batch", "model_update_interval_ms", "gpu_id", "mlp_dtype", "embedding_placement", "delta_extra_rows", "executor_policy", "start_node_stats_step",
      "stop_node_stats_step", "enable_batching", "batching_parameters", "max_batch_size", "batch_timeout_micros", "adaptive", "redis_prefix", "redis_timeout_ms",
      "device"};
  for (const char* x : kKeys) if (k == x) return true;
  return false;
}

inline Compat ParseCompat(const drjson::JVal& j, const char* who) {
  Compat c;
  for (const auto& kv : j.obj) if (!Known(kv.first)) c.unknown.push_back(kv.first);
  static const char* kStructural[] = {"use_per_session_threads", "use_multi_stream", "inter_op_parallelism_threads", "model_update_inter_threads", "kmp_blocktime",
                                      "init_timeout_minutes", "read_thread_num", "update_thread_num", "lock_file"};
  for (const char* k : kStructural) if (j.get(k)) c.structural.push_back(k);
  c.omp_num_threads = (int)j.n("omp_num_threads", 0);
  c.update_intra_threads = (int)j.n("model_update_intra_threads", 0);
  c.signature_name = j.s("signature_name", "serving_default");
  const std::string ids = j.s("gpu_ids_list", "");
  if (!ids.empty()) c.first_gpu = atoi(ids.c_str());
  const std::string store = j.s("model_store_type", "local");
  auto remote = [](const std::string& p) { return p.rfind("oss://", 0) == 0 || p.rfind("hdfs://", 0) == 0; };
  if (store != "local" && store != "")
    c.error = "model_store_type \"" + store + "\": this build has no OSS / HDFS filesystem plugin -- sync or mount the bucket and give local paths";
  else if (remote(j.s("savedmodel_dir", "")) || remote(j.s("checkpoint_dir", "")))
    c.error = "savedmodel_dir / checkpoint_dir name a remote filesystem (oss:// / hdfs://): only local paths are supported";
  const std::string proto = j.s("serialize_protocol", "protobuf");
  if (c.error.empty() && proto != "protobuf" && proto != "")
    c.error = "serialize_protocol \"" + proto + "\": requests are PredictRequest protobufs (or the compact DRRQ encoding) only";
  if (!c.error.empty()) fprintf(stderr, "[%s] ModelConfig: %s\n", who, c.error.c_str());
  if (!c.unknown.empty()) {
    std::string u;
    for (auto& k : c.unknown) u += (u.empty() ? "" : ", ") + k;
    fprintf(stderr, "[%s] ModelConfig: unknown key(s) ignored: %s\n", who, u.c_str());
  }
  return c;
}

inline std::string ToJson(const Compat& c) {
  auto list = [](const std::vector<std::string>& v) { std::string s = "["; for (size_t i = 0; i < v.size(); ++i) s += (i ? ", \"" : "\"") + v[i] + "\""; return s + "]"; };
  return "{\"signature_name\": \"" + c.signature_name + "\", \"omp_num_threads\": " + std::to_string(c.omp_num_threads) + ", \"model_update_intra_threads\": " +
         std::to_string(c.update_intra_threads) + ", \"structural\": " + list(c.structural) + ", \"unknown\": " + list(c.unknown) + "}";
}

}  // namespace drcfg
