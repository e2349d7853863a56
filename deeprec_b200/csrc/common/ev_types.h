// Shared POD types for the host (C++) and device (CUDA sm_90a) embedding engines.
//
// Behavioural parity targets in the reference (DeepRec):
//   EmbeddingConfig            tensorflow/core/framework/embedding/embedding_config.h:12-127
//   FeatureDescriptor layout   tensorflow/core/framework/embedding/feature_descriptor_impl.h:212-304
//   sparse apply math          tensorflow/core/kernels/training_ali_ops.cc:73-210,431,1203,1396,2298,2871,3016
//
// Layout decision (GPU-first, not a translation): one row per admitted key,
//   [ emb(dim) | slot0(dim) | ... | slotS-1(dim) | scalars(4) ]   (fp32, 16-byte aligned)
// so one hash probe serves the variable and all of its optimizer slots; frequency /
// version / row-index metadata live in SoA arrays indexed by the key's table position
// so that un-admitted keys cost 16 bytes, not a row.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define DR_HD __host__ __device__ __forceinline__
#else
#define DR_HD inline
#endif

extern "C" {

enum DrFilterType { DR_FILTER_NONE = 0, DR_FILTER_COUNTER = 1, DR_FILTER_BLOOM = 2 };

enum DrOptKind {
  DR_OPT_SGD = 0,
  DR_OPT_ADAGRAD = 1,
  DR_OPT_ADAGRAD_DECAY = 2,
  DR_OPT_ADAM = 3,
  DR_OPT_ADAM_ASYNC = 4,
  DR_OPT_ADAMW = 5,
  DR_OPT_FTRL = 6,
  DR_OPT_ADAM_ASYNC_RMSPROP = 7,  // AdamAsync with apply_sparse_rmsprop=True
};

enum DrStorageType {
  DR_STORAGE_DRAM = 0,
  DR_STORAGE_HBM = 1,
  DR_STORAGE_HBM_DRAM = 2,
  DR_STORAGE_DRAM_SSDHASH = 3,
};

// Plain struct mirrored by ctypes in deeprec_b200/_native.py (keep field order in sync).
struct DrEvConfig {
  int64_t dim;                      // embedding dimension
  int32_t num_slots;                // optimizer slots sharing the row (0..3)
  int32_t has_scalars;              // 1 => 4 trailing per-row scalars (AdagradDecay power, ...)
  int64_t init_capacity;            // initial key capacity (grows)
  int32_t filter_type;              // DrFilterType
  int32_t bloom_counter_bits;       // 8/16/32/64
  int64_t filter_freq;              // admission threshold (0 = admit at first sight)
  int64_t bloom_max_elements;       // CBF sizing: n
  double  bloom_fpp;                // CBF sizing: p
  int64_t steps_to_live;            // GlobalStepEvict (0 = off)
  float   l2_weight_threshold;      // L2WeightEvict   (<0 = off)
  float   default_value_no_permission;
  int64_t default_value_dim;        // rows in the default-value matrix (4096)
  int32_t record_freq;
  int32_t record_version;
  int32_t is_inference;             // INFERENCE_MODE: never create
  int32_t storage_type;             // DrStorageType
  int64_t hbm_cache_rows;           // multi-tier: rows resident in HBM tier
  int32_t cache_strategy;           // 0 = LFU, 1 = LRU
  int32_t num_partitions;           // host KV partitions
  float   slot_init[4];             // initial value of each optimizer slot row
};

struct DrOptHyper {
  int32_t kind;                     // DrOptKind
  int32_t apply_sparse_rmsprop;
  float lr, beta1, beta2, epsilon;
  float beta1_power, beta2_power;   // running powers (Adam family)
  float weight_decay;               // AdamW
  float l1, l2, l2_shrinkage, lr_power;  // Ftrl
  float decay_rate, decay_baseline; // AdagradDecay
  float init_accum;
  int64_t decay_step;               // AdagradDecay
  int64_t global_step;
};

}  // extern "C"

// ---------------------------------------------------------------------------------------
// Row geometry helpers
// ---------------------------------------------------------------------------------------
DR_HD int64_t dr_row_stride(int64_t dim, int num_slots, int has_scalars) {
  int64_t n = dim * (1 + num_slots) + (has_scalars ? 4 : 0);
  return (n + 3) & ~int64_t(3);   // 16-byte aligned rows (reference: EV_DATA_ALIGNED)
}

DR_HD int dr_opt_num_slots(int kind) {
  switch (kind) {
    case DR_OPT_SGD: return 0;
    case DR_OPT_ADAGRAD: return 1;
    case DR_OPT_ADAGRAD_DECAY: return 1;
    case DR_OPT_ADAM: case DR_OPT_ADAMW: case DR_OPT_ADAM_ASYNC:
    case DR_OPT_ADAM_ASYNC_RMSPROP: case DR_OPT_FTRL: return 2;
  }
  return 0;
}

// ---------------------------------------------------------------------------------------
// Element-wise optimizer rules (identical expressions on host and device so the CPU
// engine is the numerics oracle for the CUDA kernels). `w` is the embedding element,
// `s0`/`s1` the two slot elements, `g` the (already de-duplicated, summed) gradient.
// Adam-family `alpha` = lr*sqrt(1-b2^t)/(1-b1^t) is precomputed by the caller.
// FTRL is row-coupled (group-lasso on ||linear||) and handled by dr_ftrl_* below.
// ---------------------------------------------------------------------------------------
DR_HD float dr_rsqrtf(float x) {
#if defined(__CUDA_ARCH__)
  return rsqrtf(x);
#else
  return 1.0f / __builtin_sqrtf(x);
#endif
}
DR_HD float dr_sqrtf(float x) {
#if defined(__CUDA_ARCH__)
  return sqrtf(x);
#else
  return __builtin_sqrtf(x);
#endif
}

DR_HD void dr_apply_elem(int kind, const DrOptHyper& hp, float alpha, bool decay_now,
                         float g, float& w, float& s0, float& s1) {
  switch (kind) {
    case DR_OPT_SGD:
      w -= hp.lr * g;
      break;
    case DR_OPT_ADAGRAD:
      // training_ali_ops.cc:152-156   a += g^2 ; v -= lr * g * rsqrt(a)
      s0 += g * g;
      w -= hp.lr * g * dr_rsqrtf(s0);
      break;
    case DR_OPT_ADAGRAD_DECAY:
      // training_ali_ops.cc:1316-1323
      if (decay_now) {
        s0 *= hp.decay_rate;
        s0 = s0 > hp.decay_baseline ? s0 : hp.decay_baseline;
      }
      s0 += g * g;
      w -= hp.lr * g * dr_rsqrtf(s0);
      break;
    case DR_OPT_ADAM:
      // training_ali_ops.cc:1521-1523
      s0 += (g - s0) * (1.0f - hp.beta1);
      s1 += (g * g - s1) * (1.0f - hp.beta2);
      w -= (s0 * alpha) / (dr_sqrtf(s1) + hp.epsilon);
      break;
    case DR_OPT_ADAMW:
      // training_ali_ops.cc:3149-3153
      s0 += (g - s0) * (1.0f - hp.beta1);
      s1 += (g * g - s1) * (1.0f - hp.beta2);
      w -= (s0 * alpha) / (dr_sqrtf(s1) + hp.epsilon) + hp.weight_decay * w;
      break;
    case DR_OPT_ADAM_ASYNC:
      // training_ali_ops.cc:2475-2477
      s0 = s0 * hp.beta1 + g * (1.0f - hp.beta1);
      s1 = s1 * hp.beta2 + g * g * (1.0f - hp.beta2);
      w -= (s0 * alpha) / (dr_sqrtf(s1) + hp.epsilon);
      break;
    case DR_OPT_ADAM_ASYNC_RMSPROP:
      // training_ali_ops.cc:2425-2432  (v first, then momentum of the scaled grad)
      s1 = s1 * hp.beta2 + g * g * (1.0f - hp.beta2);
      s0 = s0 * hp.beta1 + dr_rsqrtf(s1 + hp.epsilon) * hp.lr * g;
      w -= s0;
      break;
    default:
      break;
  }
}

DR_HD float dr_adam_alpha(const DrOptHyper& hp) {
  return hp.lr * dr_sqrtf(1.0f - hp.beta2_power) / (1.0f - hp.beta1_power);
}

DR_HD float dr_powf(float a, float b) {
#if defined(__CUDA_ARCH__)
  return powf(a, b);
#else
  return __builtin_powf(a, b);
#endif
}

// FTRL phase 1: update `linear` (slot1) for one element, return its new value; accum (slot0)
// is NOT yet advanced (phase 2 needs the old value only through new_accum which we return).
DR_HD float dr_ftrl_linear(const DrOptHyper& hp, float g_in, float w, float accum, float& linear,
                           float& new_accum_out) {
  float g = g_in + 2.0f * hp.l2_shrinkage * w;
  float new_accum = accum + g * g;
  if (hp.lr_power == -0.5f) {
    linear += g - (dr_sqrtf(new_accum) - dr_sqrtf(accum)) / hp.lr * w;
  } else {
    linear += g - (dr_powf(new_accum, -hp.lr_power) - dr_powf(accum, -hp.lr_power)) / hp.lr * w;
  }
  new_accum_out = new_accum;
  return linear;
}
// FTRL phase 2: given the row norm of linear, produce the new weight.
DR_HD float dr_ftrl_weight(const DrOptHyper& hp, float linear, float new_accum, float linear_norm) {
  if (linear_norm > hp.l1) {
    float eta_rec = (hp.lr_power == -0.5f ? dr_sqrtf(new_accum) : dr_powf(new_accum, -hp.lr_power)) / hp.lr;
    float coef = (hp.l1 - linear_norm) / ((eta_rec + 2.0f * hp.l2) * linear_norm);
    return coef * linear;
  }
  return 0.0f;
}

// 64-bit mix (splitmix64 finaliser) used by the host KV, the device cuckoo table and the
// counting-Bloom filter (seeded variants).
DR_HD uint64_t dr_mix64(uint64_t x) {
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ULL;
  x ^= x >> 27; x *= 0x94d049bb133111ebULL;
  x ^= x >> 31;
  return x;
}
DR_HD uint64_t dr_hash_seed(uint64_t key, uint64_t seed) {
  return dr_mix64(key + 0x9e3779b97f4a7c15ULL * (seed + 1));
}

// Rank that owns `key` under row-wise model parallelism (every table sharded hash(key) % W): the ONE definition shared by the sparse pipeline's
// requester-side bucketing (sparse_pipeline.cu), the multi-tier prefetch of an owner (tier_kernels.cu) and host-side tools (checkpoint re-sharding).
DR_HD int dr_sp_owner(int64_t key, int W) {
  return W == 1 ? 0 : (int)((dr_mix64((uint64_t)key ^ 0x5bd1e9955bd1e995ULL) >> 33) % (uint64_t)W);
}

// Row of the default-value matrix a fresh key is initialised from (embedding_var.h:207-209).
DR_HD int64_t dr_default_row(int64_t key, int64_t default_value_dim) {
  int64_t r = key % default_value_dim;
  return r < 0 ? r + default_value_dim : r;
}

// Logical checkpoint bucket (kSavedPartitionNum = 1000, kv_interface.h:26).
DR_HD int dr_ckpt_bucket(int64_t key) {
  int64_t r = key % 1000;
  return (int)(r < 0 ? r + 1000 : r);
}
