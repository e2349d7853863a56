"""deeprec_b200 -- a Hopper (H100)-native sparse-recommender training & serving engine with the
capabilities of DeepRec (EmbeddingVariable, admission/eviction, multi-tier storage, GroupEmbedding,
model-parallel embeddings + data-parallel dense, SmartStage, incremental checkpoint, SessionGroup serving).

Layers (see DESIGN.md):
  csrc/host   C++17 host engine        (CPU EV, ckpt bundle, staging queue, work queue, serving C ABI)
  csrc/cuda   sm_90a CUDA kernels     (hash table, fused lookup, sparse optimizers, wgmma MLP, P2P collectives)
  python      framework layer          (this package)
"""
from .config import (CacheStrategy, CBFFilter, CheckpointOption, CounterFilter, EmbeddingVariableOption,
                     GlobalStepEvict, InitializerOption, L2WeightEvict, StorageOption, StorageType)
from .embedding_variable import (DynamicEmbeddingVariable, EmbeddingVariable, MultiHashVariable,
                                 PartitionedEmbeddingVariable, fixed_size_partitioner,
                                 get_dynamic_dimension_embedding_variable, get_embedding_variable,
                                 get_multihash_variable)
from . import ops, optim  # noqa: E402
from .ops.embedding_ops import (SparseIds, adaptive_embedding_lookup_sparse, embedding_lookup,
                                embedding_lookup_sparse, embedding_lookup_sparse_multi_dim,
                                fused_embedding_lookup_sparse, fused_safe_embedding_lookup_sparse,
                                group_embedding_lookup, group_embedding_lookup_sparse,
                                safe_embedding_lookup_sparse)
from .ops.sparse_ops import (sparse_fill_empty_rows, sparse_prune_fill, sparse_reshape, sparse_segment_mean,  # noqa: E402,F401
                             sparse_segment_sqrt_n, sparse_segment_sum, sparse_slice)
from .optim.optimizers import get_or_create_global_step
from . import graph_optimizer  # noqa: E402,F401
from . import feature_column  # noqa: E402,F401
from .config import PAD_KEY  # noqa: E402,F401
# top-level spellings of the reference's tf.* additions (tf.staged, tf.make_prefetch_hook, tf.SmartStageOptions, tf.stream,
# tf.train.mark_target_node, tf.config.experimental.enable_distributed_strategy)
from .data.staged import SmartStageOptions, make_prefetch_hook, smart_stage, staged  # noqa: E402,F401
from .parallel.collective import CollectiveStrategy, enable_distributed_strategy  # noqa: E402,F401
from .utils.streams import mark_target_node, stream  # noqa: E402,F401

__version__ = "0.1.0"
