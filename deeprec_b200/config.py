"""Typed option objects (one config layer instead of the reference's protobuf + python options +
~40 env vars, SURVEY §5.6).  Names and defaults follow ``python/ops/variables.py:179-302``.

Environment overrides kept for parity/debugging (read once, at object construction):
``INFERENCE_MODE``, ``TF_EV_SAVE_FILTERED_FEATURES``, ``TF_EV_RESET_VERSION``,
``COLLECTIVE_STRATEGY``, ``DEEPREC_HOST_THREADS``.
"""
from __future__ import annotations

import enum
import os
from dataclasses import dataclass, field
from typing import Callable, Optional, Sequence

import torch


class StorageType(enum.IntEnum):
    """storage_config.h:22-47 (tiers that make sense on an H100 box)."""
    DRAM = 0
    HBM = 1
    HBM_DRAM = 2
    DRAM_SSDHASH = 3
    HBM_DRAM_SSDHASH = 4


class CacheStrategy(enum.IntEnum):
    LFU = 0
    LRU = 1


class FilterType(enum.IntEnum):
    NONE = 0
    COUNTER = 1
    BLOOM = 2


@dataclass
class InitializerOption:
    """variables.py:179 -- new key ``k`` starts from row ``k % default_value_dim`` of a
    pre-generated matrix drawn from ``initializer``."""
    initializer: Optional[Callable[[torch.Tensor], None]] = None
    default_value_dim: int = 4096
    default_value_no_permission: float = 0.0


@dataclass
class GlobalStepEvict:
    steps_to_live: int = 0


@dataclass
class L2WeightEvict:
    l2_weight_threshold: float = -1.0


@dataclass
class CounterFilter:
    filter_freq: int = 0

    def __post_init__(self):
        if self.filter_freq >= 4096:
            # counter_filter_descriptor_impl.h:43 -- un-admitted keys keep freq in 12 bits
            raise ValueError("CounterFilter.filter_freq must be < 4096")


@dataclass
class CBFFilter:
    filter_freq: int = 0
    max_element_size: int = 0
    false_positive_probability: float = -1.0
    counter_type: torch.dtype = torch.int64

    def counter_bits(self) -> int:
        return {torch.uint8: 8, torch.int8: 8, torch.int16: 16, torch.int32: 32, torch.int64: 64}[self.counter_type]


@dataclass
class StorageOption:
    storage_type: StorageType = StorageType.DRAM
    storage_path: Optional[str] = None
    storage_size: Sequence[int] = (1 << 30,)       # bytes per tier (tier 0 first)
    cache_strategy: CacheStrategy = CacheStrategy.LFU
    layout: Optional[str] = None


@dataclass
class CheckpointOption:
    ckpt_to_load_from: Optional[str] = None
    tensor_name_in_ckpt: Optional[str] = None
    always_load_from_specific_ckpt: bool = False
    init_data_source: Optional[str] = None


@dataclass
class EmbeddingVariableOption:
    ht_type: str = ""
    ht_partition_num: int = 16
    evict_option: Optional[object] = None            # GlobalStepEvict | L2WeightEvict
    ckpt: Optional[CheckpointOption] = None
    filter_option: Optional[object] = None           # CounterFilter | CBFFilter
    storage_option: StorageOption = field(default_factory=StorageOption)
    init_option: InitializerOption = field(default_factory=InitializerOption)
    init_capacity: int = 1 << 16                     # initial key capacity (grows)
    # accepted for API parity (TF_RECORD_FREQ / TF_RECORD_VERSION): both engines keep freq / version in the key's metadata slot
    # (same cache line / DRAM sector as the key), so they are always maintained and these switches save nothing
    record_freq: bool = True
    record_version: bool = True


# The one int64 value that is never a key (the hash tables' empty-slot marker).  Host tables treat it as PADDING: a lookup returns a zero
# row, nothing is created / counted / updated for it -- so a dense ``[B, L]`` history tensor can mark its unused positions with it instead
# of looking up (and polluting the statistics of) a real id.
PAD_KEY = -(1 << 63)


def env_flag(name: str, default: bool = False) -> bool:
    v = os.environ.get(name)
    if v is None:
        return default
    return v.strip().lower() in ("1", "true", "yes", "on")


def inference_mode() -> bool:
    """``INFERENCE_MODE`` env (kv_variable_ops.cc:200-204): EV lookups never create keys."""
    return env_flag("INFERENCE_MODE")


# ---- the reference's environment switches (SURVEY §2.11 "Env-var flags"): what each one does HERE ---------------------------------------
# status: "honoured" = read by this framework with the reference's meaning; "always" = the behaviour it enables is unconditional here (the
# switch is accepted and ignored); "n/a" = tied to a component this design does not have (setting it has no effect; env_report() says so).
REFERENCE_ENV_FLAGS = {
    "INFERENCE_MODE": ("honoured", "EmbeddingVariable lookups never create keys (config.inference_mode)"),
    "TF_EV_SAVE_FILTERED_FEATURES": ("honoured", "checkpoints include / omit the un-admitted keys and their counters (checkpoint/saver.py)"),
    "TF_EV_RESET_VERSION": ("honoured", "restore resets the version (last-update step) of every key (checkpoint/saver.py)"),
    "TF_SSDHASH_ASYNC_COMPACTION": ("honoured", "SSD tier compaction on a background thread (also DEEPREC_SSDHASH_ASYNC_COMPACTION)"),
    "COLLECTIVE_STRATEGY": ("honoured", "sok | hb | hvd select the CollectiveStrategy flavour name (parallel/collective.py)"),
    "TF_GPU_ALLOCATOR": ("honoured", "tensorpool | cuda_malloc_async (utils/memory.maybe_enable_from_env; also DEEPREC_GPU_ALLOCATOR)"),
    "TF_GPU_VMEM": ("honoured", "managed-memory fallback of the pool allocator on OOM (also DEEPREC_GPU_VMEM)"),
    "ENABLE_MEMORY_OPTIMIZATION": ("honoured", "host TensorPool planning on / off (utils/memory.HostTensorPool.from_env)"),
    "START_STATISTIC_STEP": ("honoured", "TensorPool: first step whose allocation sizes are recorded"),
    "STABLE_STATISTIC_STEP": ("honoured", "TensorPool: steps after which the plan is frozen"),
    "MAX_STATISTIC_STEP": ("honoured", "TensorPool: re-plan horizon"),
    "STOP_STATISTIC_STEP": ("honoured", "TensorPool: last recorded step"),
    "SESSION_GROUP_CPUSET": ("honoured", "per-session CPU sets of the CPU Processor (also ModelConfig cpusets)"),
    "SET_SESSION_THREAD_POOL_AFFINITY": ("honoured", "automatic even split of the cores over the serving sessions"),
    "EV_DATA_ALIGNED": ("always", "rows are 16-byte aligned by construction on both engines"),
    "TF_EMBEDDING_FBJ_OPT": ("always", "lookup and apply share the probed positions by construction (no graph pass to enable)"),
    "PER_SESSION_HOSTALLOC": ("always", "every serving session owns its pinned staging buffers"),
    "MERGE_COMPUTE_COPY_STREAM": ("always", "a serving session runs copies and kernels on its ONE stream; training forks explicit side streams inside the CUDA graph"),
    "USE_INLINE_EXECUTOR": ("always", "sessions execute inline on the caller's thread; there is no op scheduler"),
    "TF_MULTI_TIER_EV_EVICTION_THREADS": ("n/a", "the device tier manager runs one migration thread per table (ops/tier_manager.py); host tiers demote inline"),
    "USE_COST_MODEL_EXECUTOR": ("n/a", "no per-op executor: a training step is one CUDA graph"),
    "START_NODE_STATS_STEP": ("n/a", "cost-model executor tracing"),
    "STOP_NODE_STATS_STEP": ("n/a", "cost-model executor tracing"),
    "ENABLE_MPS": ("n/a", "multi-context SessionGroup over MPS: sessions share one context and use one stream each"),
    "CONTEXTS_COUNT_PER_GPU": ("n/a", "see ENABLE_MPS"),
    "TARGET_NODES_NAME": ("n/a", "graph-node names: the cut of smart_stage() is the loader boundary; use mark_target_node() for explicit targets"),
}


def env_report(warn: bool = True) -> dict:
    """The reference switches present in the environment and how this framework treats them; ``warn`` logs the ones without effect."""
    import logging
    out = {}
    for name, (status, note) in REFERENCE_ENV_FLAGS.items():
        if name in os.environ:
            out[name] = {"value": os.environ[name], "status": status, "note": note}
            if warn and status == "n/a":
                logging.getLogger("deeprec_b200").warning("%s=%s has no effect here: %s", name, os.environ[name], note)
    return out
