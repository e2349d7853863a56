"""DLRMEngine -- the fused H100 training/inference step for DLRM (the flagship benchmark path).

Model (modelzoo/dlrm/train.py:68-243): bottom MLP [512,256,64,16] (Dense+ReLU+BatchNorm each), 26
EmbeddingVariable tables of dim 16, 'dot' interaction (strict lower triangle of the 27x27 Gram
matrix, concatenated with the bottom output), top MLP [512,256] (Dense+ReLU), logits Dense(1),
sigmoid + binary cross-entropy, one optimizer for dense and sparse parameters.

Execution design (GPU-first; nothing here is a translation of the TF graph):
  * static buffers + ONE CUDA graph per step (~75 kernel nodes), embedding branch forked onto a
    second stream inside the graph so probes/gathers overlap the bottom MLP;
  * every GEMM is the hand-written wgmma/TMA kernel (csrc/cuda/gemm_wgmma.cu) with bias,
    ReLU and ReLU-backward masks fused in the epilogue; weight gradients are split-K wgmma GEMMs
    reading both operands MN-major straight from the activations (no transposes);
  * embeddings are model-parallel (every table row-sharded by hash(key) % world) and the dense net
    data-parallel.  The sparse path is "unique-first" (parallel/sparse_pipeline.py): the requester
    dedups its ids in an L2-resident scratch hash, owners probe only distinct keys and push bf16
    rows straight into the requester's unique-row buffer over NVLink, the interaction kernels gather
    through the inverse index, the backward pre-reduces gradients per distinct key in fp32 and the
    owners pull one row per key; ranks synchronise with in-kernel release/acquire flags, never with
    a barrier kernel or an NCCL call.  The same kernels run at world_size 1.  An NCCL
    implementation of the reference (SOK) dataflow is kept as the measured baseline
    (parallel/nccl_baseline.py, table-wise sharding, no requester-side dedup);
  * hyper-parameters / global step live in device memory and are advanced by a device kernel, so
    the captured graph needs no per-step host work besides the input H2D copy.
"""
from __future__ import annotations

import ctypes as C
import math
from contextlib import nullcontext
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import torch

from .. import _native
from .._native import OptHyper, check, ptr, stream_ptr
from ..checkpoint.engine_ckpt import restore_engine, save_engine
from ..ops.device_table import DeviceTable
from ..optim.optimizers import OPT_KIND, OPT_SLOTS, slot0_init
from . import embedding_group as _eg
from .embedding_group import EmbeddingGroup

# Criteo-Terabyte cardinalities (MLPerf DLRM preprocessing, 40M cap) -- used only to shape the
# synthetic id distributions and pre-size the tables; EmbeddingVariables are hash tables and grow.
CRITEO_TB_CARDINALITIES = [39884406, 39043, 17289, 7420, 20263, 3, 7120, 1543, 63, 38532951, 2953546, 403346, 10, 2208, 11938,
                           155, 4, 976, 14, 39979771, 25641295, 39664984, 585935, 12972, 108, 36]
# Criteo-Kaggle cardinalities used by the modelzoo (modelzoo/dlrm/train.py:33-66)
CRITEO_KAGGLE_CARDINALITIES = [1460, 583, 10131227, 2202608, 305, 24, 12517, 633, 3, 93145, 5683, 8351593, 3194, 27, 14992,
                               5461306, 10, 5652, 2173, 4, 7046547, 18, 15, 286181, 105, 142572]

@dataclass
class DLRMConfig:
    batch_size: int = 8192                      # per-rank batch
    num_dense: int = 13
    cardinalities: Sequence[int] = field(default_factory=lambda: list(CRITEO_TB_CARDINALITIES))
    embedding_dim: int = 16
    mlp_bot: Sequence[int] = (512, 256, 64, 16)
    mlp_top: Sequence[int] = (512, 256)
    optimizer: str = "adagrad"
    learning_rate: float = 0.01
    initial_accumulator_value: float = 0.1
    bn_eps: float = 1e-3                        # tf.layers.batch_normalization defaults
    bn_momentum: float = 0.99
    max_rows_per_table: int = 1 << 24           # row-slab pre-size cap per table (grows past it at a step boundary)
    filter_freq: int = 0                        # CounterFilter threshold (0 = admit at first sight)
    steps_to_live: int = 0
    seed: int = 1234
    overlap_embedding: bool = True              # fork the embedding branch onto a side stream inside the graph
    sparse_blocks_per_sm: int = 4               # resident-block budget of the side-stream sparse kernels
    # SMs of the green context the embedding branch runs in during the two overlap windows; the bottom MLP gets the rest (csrc/cuda/
    # sm_partition.cu).  Rounded by the driver (multiples of 8 on Hopper).  0 = both branches share every SM as two streams of one context.
    # 40 balances both windows at the bench shapes on an H100 SXM (DESIGN.md: SM partition).
    sparse_sms: int = 40
    gemm_v1: bool = False                       # A/B switch: separate statistics passes instead of the statistics fused into the GEMM epilogue
    # combine + dot interaction + top-MLP layer 0 in ONE tensor-core kernel (csrc/cuda/fused_interaction_gemm.cu).  Opt-in: the builder
    # phase and the GEMM phase of a tile share one 96 KB Z tile in shared memory and run one after the other, so the default step keeps
    # the two kernels.
    fuse_interaction_gemm: bool = False
    # "dot": the DLRM interaction above.  "dcnv2": DLRM-DCNv2 (modelzoo/mlperf/train.py): x0 = [bottom | emb_0 .. emb_{T-1}] through
    # dcn_num_layers low-rank cross layers x_{l+1} = x0 * (x_l V_l W_l + b_l) + x_l of rank dcn_low_rank_dim, then the top MLP
    interaction_op: str = "dot"
    dcn_num_layers: int = 3
    dcn_low_rank_dim: int = 512

# MLPerf DLRM-DCNv2 shapes (modelzoo/mlperf/train.py): DLRMConfig(**MLPERF_DCNV2, ...)
MLPERF_DCNV2 = dict(embedding_dim=128, mlp_bot=(512, 256, 128), mlp_top=(1024, 1024, 512, 256), interaction_op="dcnv2", dcn_num_layers=3,
                    dcn_low_rank_dim=512)


def _check_interaction(cfg: DLRMConfig, comm) -> None:
    if cfg.interaction_op == "dot":
        return
    if cfg.interaction_op != "dcnv2":
        raise ValueError(f"interaction_op must be 'dot' or 'dcnv2', got {cfg.interaction_op!r}")
    if cfg.embedding_dim not in (16, 32, 64, 128):
        raise ValueError(f"dcnv2: embedding_dim must be 16, 32, 64 or 128, got {cfg.embedding_dim}")
    if cfg.mlp_bot[-1] != cfg.embedding_dim:
        raise ValueError("dcnv2: the bottom MLP output must equal embedding_dim (it is column block 0 of x0)")
    if cfg.fuse_interaction_gemm:
        raise ValueError("dcnv2: fuse_interaction_gemm fuses the dot interaction only")
    if comm is not None and not getattr(comm, "unique_first", False):
        raise ValueError("dcnv2: needs the unique-first sparse pipeline (the NCCL baseline comm runs the dot interaction only)")
    if cfg.dcn_num_layers < 1 or cfg.dcn_low_rank_dim <= 0 or cfg.dcn_low_rank_dim % 8:
        raise ValueError("dcnv2: dcn_num_layers >= 1 and dcn_low_rank_dim a positive multiple of 8")


def _pad8(n: int) -> int:
    return (n + 7) // 8 * 8


class _Layer:
    """One Linear layer's views into the flat parameter / gradient buffers + bf16 shadows."""

    def __init__(self, name: str, n_out: int, k_in: int, has_bn: bool):
        self.name, self.N, self.K, self.Kp, self.Np, self.has_bn = name, n_out, k_in, _pad8(k_in), _pad8(n_out), has_bn


class DLRMEngine:
    def __init__(self, cfg: DLRMConfig, device: Optional[torch.device] = None, rank: int = 0, world_size: int = 1, comm=None):
        _check_interaction(cfg, comm)
        self.cfg = cfg
        self.dcn = cfg.interaction_op == "dcnv2"
        self.rank, self.world = rank, world_size
        self.emu = _native.emu_active()          # CPU CI: the same launch sequence on the CUDA-on-CPU emulation (eager, one stream, no CUDA graph)
        self.dev = torch.device("cpu") if self.emu else (torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device()))
        self.lib = _native.cuda()
        if not self.emu:
            _native.set_device(self.dev.index)
        self.lib.dr_cuda_set_sparse_blocks_per_sm(int(cfg.sparse_blocks_per_sm if cfg.overlap_embedding else 16))
        self.comm = comm                           # parallel.p2p.P2PComm or parallel.nccl_baseline.NcclComm (world_size > 1)
        self.B, self.T, self.D = cfg.batch_size, len(cfg.cardinalities), cfg.embedding_dim
        self.kind = OPT_KIND[cfg.optimizer.lower()]
        self._launches = 0
        self._graph = None
        import os as _os
        self._timing, self._events = _os.environ.get("DEEPREC_STEP_TIMING") == "1", {}
        self._side = None if self.emu else torch.cuda.Stream(device=self.dev)
        self._dense, self._ctas = None, 0          # dense-partition stream, persistent GEMM grid cap (0 = every SM)
        self.partition_sms = None                  # (sparse, dense) SMs the driver provisioned when sparse_sms > 0
        if cfg.sparse_sms > 0 and cfg.overlap_embedding and not self.emu and (comm is None or getattr(comm, "unique_first", False)):
            info, h = (C.c_int * 2)(), (C.c_void_p * 5)()
            check(self.lib.dr_cuda_sm_partition(self.dev.index, int(cfg.sparse_sms), info, h), f"SM partition ({cfg.sparse_sms} sparse SMs)")
            self.partition_sms = (info[0], info[1])
            self._side = torch.cuda.ExternalStream(h[0], device=self.dev)
            self._dense = torch.cuda.ExternalStream(h[1], device=self.dev)
        self._build_params()
        self._build_tables()
        self._build_buffers()
        self._pack_weights()
        _native.device_sync(self.dev)

    # ------------------------------------------------------------------------------------------------
    # parameters
    # ------------------------------------------------------------------------------------------------
    def _build_params(self) -> None:
        cfg, dev = self.cfg, self.dev
        self.bot: List[_Layer] = []
        k = cfg.num_dense
        for i, n in enumerate(cfg.mlp_bot):
            self.bot.append(_Layer(f"mlp_bot_{i}", n, k, True)); k = n
        F = self.T + 1
        self.inter_dim = F * cfg.embedding_dim if self.dcn else cfg.embedding_dim + F * (F - 1) // 2
        self.Zp = _pad8(self.inter_dim)
        self.top: List[_Layer] = []
        k = self.inter_dim
        for i, n in enumerate(cfg.mlp_top):
            self.top.append(_Layer(f"mlp_top_{i}", n, k, False)); k = n
        self.head_K = k
        if cfg.mlp_bot[-1] != cfg.embedding_dim:
            raise ValueError("bottom MLP output must equal embedding_dim for the dot interaction")
        # low-rank cross layers (dcnv2): V_l [rank, inter_dim] (no bias) and W_l [inter_dim, rank] + b_l, stored [N_out, K_in] like every Linear
        self.cross: List[tuple] = []
        for l in range(cfg.dcn_num_layers if self.dcn else 0):
            self.cross.append((_Layer(f"low_rank_cross_net_{l}_v", cfg.dcn_low_rank_dim, self.inter_dim, False),
                               _Layer(f"low_rank_cross_net_{l}_w", self.inter_dim, cfg.dcn_low_rank_dim, False)))
        self.xlayers: List[_Layer] = [L for pair in self.cross for L in pair]
        off = 0
        self.views: Dict[str, tuple] = {}

        def take(name, numel):
            nonlocal off
            self.views[name] = (off, numel)
            off += (numel + 63) // 64 * 64

        for L in self.bot + self.top:
            take(L.name + "/kernel", L.N * L.Kp); take(L.name + "/bias", L.N)
            if L.has_bn:
                take(L.name + "/bn_gamma", L.N); take(L.name + "/bn_beta", L.N)
        for V, W in self.cross:
            take(V.name + "/kernel", V.N * V.Kp); take(W.name + "/kernel", W.N * W.Kp); take(W.name + "/bias", W.N)
        take("logits/kernel", self.head_K); take("logits/bias", 4)
        self.P = off
        g = torch.Generator(device="cpu").manual_seed(cfg.seed)
        flat = torch.zeros(self.P, dtype=torch.float32)
        for L in self.bot + self.top + self.xlayers:
            o, n = self.views[L.name + "/kernel"]
            lim = math.sqrt(6.0 / (L.K + L.N))                      # glorot_uniform (tf.layers.dense default)
            w = torch.zeros(L.N, L.Kp)
            w[:, : L.K] = (torch.rand(L.N, L.K, generator=g) * 2 - 1) * lim
            flat[o:o + n] = w.view(-1)
            if L.has_bn:
                o, n = self.views[L.name + "/bn_gamma"]; flat[o:o + n] = 1.0
        o, n = self.views["logits/kernel"]
        flat[o:o + n] = (torch.rand(n, generator=g) * 2 - 1) * math.sqrt(6.0 / (self.head_K + 1))
        self.params = flat.to(dev)
        self.grads = torch.zeros(self.P, dtype=torch.float32, device=dev) if self.comm is None else self.comm.alloc_grads(self.P)
        ns = OPT_SLOTS[self.kind]
        self.s0 = torch.full((self.P,), slot0_init(self.kind, cfg.initial_accumulator_value), dtype=torch.float32, device=dev) if ns > 0 else None
        self.s1 = torch.zeros(self.P, dtype=torch.float32, device=dev) if ns > 1 else None
        # bf16 shadows for the wgmma GEMMs: W [N, Kp] and W^T [Kp, Np]
        for L in self.bot + self.top + self.xlayers:
            L.w_bf16 = torch.zeros(L.N, L.Kp, dtype=torch.bfloat16, device=dev)
            L.wt_bf16 = torch.zeros(L.Kp, L.Np, dtype=torch.bfloat16, device=dev)
            if L.has_bn:
                for nm in ("mean", "rstd", "scale", "shift", "c1", "c2"):
                    setattr(L, nm, torch.zeros(L.N, dtype=torch.float32, device=dev))
                L.running_mean = torch.zeros(L.N, dtype=torch.float32, device=dev)
                L.running_var = torch.ones(L.N, dtype=torch.float32, device=dev)
        # one arena for every per-step column statistic (BatchNorm fwd sums, BatchNorm bwd sums): ONE memset per step
        tot = sum(4 * ((L.N + 63) // 64 * 64) for L in self.bot)
        self.stats = torch.zeros(max(tot, 64), dtype=torch.float32, device=dev)
        o = 0
        for L in self.bot:
            n64 = (L.N + 63) // 64 * 64
            L.S1, L.S2, L.S1b, L.S2b = (self.stats[o + i * n64: o + i * n64 + L.N] for i in range(4))
            o += 4 * n64
        # BatchNorm folding: layer l >= 1 consumes the un-normalised activation a_{l-1} with W' = W diag(s), b' = b + W t
        for L in self.bot[1:]:
            L.wf_bf16 = torch.zeros(L.N, L.Kp, dtype=torch.bfloat16, device=dev)
            L.bf = torch.zeros(L.N, dtype=torch.float32, device=dev)

    def p(self, name: str) -> torch.Tensor:
        o, n = self.views[name]
        return self.params[o:o + n]

    def g(self, name: str) -> torch.Tensor:
        o, n = self.views[name]
        return self.grads[o:o + n]

    # ------------------------------------------------------------------------------------------------
    # embedding tables.  unique-first mode: every rank owns the hash(key) % world shard of EVERY table;
    # legacy mode (NCCL baseline arm): table t lives on rank t % world (SOK "localized" placement).
    # ------------------------------------------------------------------------------------------------
    def _build_tables(self) -> None:
        cfg = self.cfg
        W = self.world
        self.uf = self.comm is None or getattr(self.comm, "unique_first", False)
        if self.uf:
            self.owner_of = [-1] * self.T
            self.local_tables = list(range(self.T))
        else:
            self.owner_of = [t % W for t in range(self.T)]
            self.local_tables = [t for t in range(self.T) if self.owner_of[t] == self.rank]
        self.group = EmbeddingGroup(self.dev, self.D, self.kind, cfg.learning_rate, cfg.initial_accumulator_value, id(self) & 0x7FFFFFFF,
                                    cfg.seed + 17, self.local_tables, cfg.cardinalities, self.B, col_table=list(range(self.T)) if self.uf else None,
                                    rank=self.rank, world=W, comm=self.comm, filter_freq=cfg.filter_freq, steps_to_live=cfg.steps_to_live,
                                    max_rows_per_table=cfg.max_rows_per_table)
        self.groups = [self.group]
        self.tables: Dict[int, DeviceTable] = self.group.tables
        self.sp, self.hp_dev = self.group.sp, self.group.hp_dev

    # ------------------------------------------------------------------------------------------------
    # static activations
    # ------------------------------------------------------------------------------------------------
    def _build_buffers(self) -> None:
        B, T, D, dev = self.B, self.T, self.D, self.dev
        bf, f32 = torch.bfloat16, torch.float32
        z = lambda *s, dt=bf: torch.zeros(*s, dtype=dt, device=dev)
        self.dense_in = z(B, self.cfg.num_dense, dt=f32)
        self.labels = z(B, dt=f32)
        if self.uf:
            self.ids = torch.zeros(T, B, dtype=torch.int64, device=dev)          # feature-major id columns (local: never leave the GPU)
            self.emb = self.pos = None
            self.demb = z(T, B, D)                                               # per-sample gradient rows, feature-major (local)
        else:
            self.ids, self.emb, self.demb = self.comm.alloc_exchange(T, B, D)
            self.pos = torch.zeros(max(1, len(self.local_tables) * self.world * B), dtype=torch.int32, device=dev)   # probe results for owned (table, src, sample)
        self.x0 = z(B, _pad8(self.cfg.num_dense))
        for L in self.bot:
            L.a = z(B, L.N); L.y = z(B, L.N); L.dy = z(B, L.N); L.da = z(B, L.N)
        if self.dcn:
            # x_0 .. x_L [B, (T + 1) D]: x_0 is assembled in place (bottom output | gathered rows), x_L feeds the top MLP.  u_l = x_l V_l W_l + b_l
            # and t_l = x_l V_l are kept for the backward; g ping-pongs dL/dx_l, dx0 accumulates the x0-factor gradients in fp32.
            N, r, nl = self.inter_dim, self.cfg.dcn_low_rank_dim, len(self.cross)
            self.xs = [z(B, N) for _ in range(nl + 1)]
            self.us = [z(B, N) for _ in range(nl)]
            self.ts = [z(B, r) for _ in range(nl)]
            self.gbuf = [z(B, N), z(B, N)]
            self.du, self.dt, self.dx0 = z(B, N), z(B, r), z(B, N, dt=f32)
            self.Z = self.xs[-1]; self.dZ = z(B, self.Zp)
        else:
            self.Z = z(B, self.Zp); self.dZ = z(B, self.Zp)
        for L in self.top:
            L.a = z(B, L.N); L.da = z(B, L.N)
        self.prob = z(B, dt=f32)
        self.loss = z(1, dt=f32)
        self.dx = z(B, D)
        self._l2_scratch = None

    # ------------------------------------------------------------------------------------------------
    # kernel-call helpers (every call is one launch of one of OUR kernels; counted for gpu_launches)
    # ------------------------------------------------------------------------------------------------
    launches = property(_eg.engine_launches)
    loss_value = _eg.loss_value
    save, restore = save_engine, restore_engine      # training-state checkpoints: full / incremental save, restore under any world size

    # ---- optional per-phase CUDA-event timing of EAGER steps (DEEPREC_STEP_TIMING=1; never inside a captured graph) ------------
    def _tick(self, name: str) -> None:
        if self._timing and not self.emu and not torch.cuda.is_current_stream_capturing():
            e = torch.cuda.Event(enable_timing=True)
            e.record(torch.cuda.current_stream(self.dev))
            self._events.setdefault(name, []).append(e)

    def timing_report(self, skip: int = 2) -> Dict[str, float]:
        """Mean milliseconds per phase over the eager steps recorded so far (first `skip` steps dropped)."""
        torch.cuda.synchronize(self.dev)
        pairs = [("dedup", "e0", "e_dedup"), ("lookup", "e_dedup", "f_emb"), ("segsum", "g0", "g_segsum"), ("reset", "g_segsum", "g_reset"),
                 ("grad_pull", "g_reset", "g_grad"), ("apply", "g_grad", "b_emb"),
                 ("emb_fwd(side)", "f0", "f_emb"), ("bot_fwd", "f0", "f_bot"), ("dot_fwd", "f_join", "f_dot"), ("top_fwd", "f_dot", "f_top"),
                 ("head", "f_top", "h1"), ("top_bwd", "h1", "b_top"), ("dot_bwd", "b_top", "b_dot"), ("emb_bwd(side)", "b_dot", "b_emb"),
                 ("bot_bwd", "b_dot", "b_bot"), ("dense_update", "b_join", "u1"), ("step", "f0", "u1")]
        out = {}
        for nm, a, b in pairs:
            if a in self._events and b in self._events:
                ts = [x.elapsed_time(y) for x, y in zip(self._events[a], self._events[b])][skip:]
                if ts:
                    out[nm] = sum(ts) / len(ts)
        return out

    def _call(self, fn, *args):
        check(fn(*args, stream_ptr(self.dev)), fn.__name__)
        self._launches += 1

    def _gemm(self, A, lda, Bm, ldb, M, N, K, bias, relu, mask, ldm, out, ldc, aux_mode=None, S1=None, S2=None):
        """out[M,N] = A[M,K] Bm[N,K]^T (+bias)(relu); aux ``mask`` with aux_mode 1 = ReLU-backward mask, 2 = S2 partner;
        S1/S2 = column statistics fused into the epilogue (fused GEMM epilogue)."""
        mode = aux_mode if aux_mode is not None else (1 if mask is not None else 0)
        self._call(self.lib.dr_cuda_gemm_tn_ex, ptr(A), lda, ptr(Bm), ldb, M, N, K, ptr(bias) if bias is not None else None, int(relu),
                   ptr(mask) if mask is not None else None, ldm, mode, ptr(out), ldc, None, ptr(S1) if S1 is not None else None,
                   ptr(S2) if S2 is not None else None, self._ctas, int(self.cfg.gemm_v1))

    def _gemm_dw(self, dY, ldy, X, ldx, n_out, k_in, dW, ldw):
        self._call(self.lib.dr_cuda_gemm_dw, ptr(dY), ldy, ptr(X), ldx, self.B, n_out, k_in, ptr(dW), ldw, 0)

    def _pack_weights(self) -> None:
        for L in self.bot + self.top + self.xlayers:
            self._call(self.lib.dr_cuda_pack_weights, ptr(self.p(L.name + "/kernel")), L.N, L.Kp, ptr(L.w_bf16), ptr(L.wt_bf16), L.Np)

    # ------------------------------------------------------------------------------------------------
    # the step
    # ------------------------------------------------------------------------------------------------
    def _embedding_forward(self, train: bool) -> None:
        """Requester: dedup + bucket the local ids.  Owner: probe (+admit/claim) the distinct keys of every source and push rows."""
        if not self.uf:
            self.comm.lookup_forward(self, train)
            return
        self._tick("e0")
        self.group.forward(self.ids, train, self._tick)

    def _embedding_backward(self) -> None:
        """Owner: pull the sources' pre-reduced gradient rows, then the row-wise optimizer over this step's distinct keys."""
        if not self.uf:
            self.comm.sparse_backward(self)
            return
        self._tick("g0")
        self.group.backward(self.demb, self._tick)

    def _bn_fold(self, L, Ln, train: bool) -> None:
        """finalize BatchNorm(L) from the fused epilogue statistics and fold it into the next Linear (Ln)."""
        cfg = self.cfg
        self._call(self.lib.dr_cuda_bn_fold, ptr(L.S1), ptr(L.S2), L.N, self.B, ptr(self.p(L.name + "/bn_gamma")), ptr(self.p(L.name + "/bn_beta")),
                   cfg.bn_eps, cfg.bn_momentum, ptr(L.running_mean), ptr(L.running_var), ptr(L.mean), ptr(L.rstd), ptr(L.scale), ptr(L.shift),
                   int(train), ptr(self.p(Ln.name + "/kernel")), ptr(self.p(Ln.name + "/bias")), Ln.N, Ln.Kp, ptr(Ln.wf_bf16), ptr(Ln.bf))

    # ---- the two overlap windows.  With an SM partition the main-stream work of a window runs on the dense green context's stream, with
    #      persistent GEMM grids sized to that context's SMs (a grid sized to the whole GPU would run as two waves there)
    def _fork(self, main) -> None:
        self._side.wait_stream(main)
        if self._dense is not None:
            self._dense.wait_stream(main)
            self.lib.dr_cuda_set_sparse_sms(self.partition_sms[0])     # side-stream grids: one wave on the sparse partition

    def _dense_window(self):
        if self._dense is None:
            return nullcontext()
        self._ctas = self.partition_sms[1]
        return torch.cuda.stream(self._dense)

    def _join(self, main) -> None:
        main.wait_stream(self._side)
        if self._dense is not None:
            main.wait_stream(self._dense)
            self._ctas = 0
            self.lib.dr_cuda_set_sparse_sms(0)

    def _forward(self, train: bool) -> None:
        cfg = self.cfg
        main = None if self.emu else torch.cuda.current_stream(self.dev)
        fork = cfg.overlap_embedding and not self.emu
        self._tick("f0")
        if fork:
            self._fork(main)
            with torch.cuda.stream(self._side):
                self._embedding_forward(train)
                self._tick("f_emb")
        with self._dense_window() if fork else nullcontext():
            x, ldx = self._bottom_forward(train)
        if fork:
            self._join(main)
        else:
            self._embedding_forward(train)
            self._tick("f_emb")
        self._tick("f_join")
        self._top_forward(train, x, ldx)

    def _bottom_forward(self, train: bool):
        lib, B, cfg = self.lib, self.B, self.cfg
        # ---- bottom MLP.  Layer l: a_l = relu(a_{l-1} W_l'^T + b_l') with BatchNorm_{l-1} folded into (W', b'); the batch
        #      statistics of a_l come out of the GEMM epilogue, so no activation is read twice and y_l is never written.
        self._call(lib.dr_cuda_cast_pad, ptr(self.dense_in), B, cfg.num_dense, ptr(self.x0), self.x0.shape[1])
        x, ldx = self.x0, self.x0.shape[1]
        nb = len(self.bot)
        for i, L in enumerate(self.bot):
            w, bias = (L.w_bf16, self.p(L.name + "/bias")) if i == 0 else (L.wf_bf16, L.bf)
            fused = train and L.N > 32 and not cfg.gemm_v1
            self._gemm(x, ldx, w, L.Kp, B, L.N, L.Kp, bias, True, None, 0, L.a, L.N, S1=L.S1 if fused else None, S2=L.S2 if fused else None)
            if train and not fused:
                self._call(lib.dr_cuda_colstats, ptr(L.a), ptr(L.a), B, L.N, L.N, L.N, ptr(L.S1), ptr(L.S2))
            if i + 1 < nb:
                self._bn_fold(L, self.bot[i + 1], train)
                x, ldx = L.a, L.N
            else:   # last bottom layer: its normalised output feeds the interaction, materialise it ([B, D] only; dcnv2: columns [0, D) of x0)
                self._call(lib.dr_cuda_bn_finalize, ptr(L.S1), ptr(L.S2), L.N, B, ptr(self.p(L.name + "/bn_gamma")), ptr(self.p(L.name + "/bn_beta")),
                           cfg.bn_eps, cfg.bn_momentum, ptr(L.running_mean), ptr(L.running_var), ptr(L.mean), ptr(L.rstd), ptr(L.scale),
                           ptr(L.shift), int(train))
                y, ldy = (self.xs[0], self.inter_dim) if self.dcn else (L.y, L.N)
                self._call(lib.dr_cuda_bn_apply, ptr(L.a), B, L.N, L.N, ptr(L.scale), ptr(L.shift), ptr(y), ldy)
                x, ldx = y, ldy
        self._tick("f_bot")
        return x, ldx

    def _top_forward(self, train: bool, x, ldx) -> None:
        lib, B, cfg = self.lib, self.B, self.cfg
        # ---- interaction + top MLP
        fused0 = self.uf and cfg.fuse_interaction_gemm and self.D == 16 and self.top[0].N <= 512 and self.inter_dim <= 384 and not self.emu
        if self.dcn:  # the gathered rows complete x0 (the kernel waits for every owner's ROWS flag), then the cross layers
            self.sp.gather_pitched(self.xs[0][:, self.D:])
            self._cross_forward(train)
        elif fused0:    # gather + Gram + lower-triangle pack + Linear(512) + ReLU in one kernel; Z only leaves the SM as a TMA store for the backward
            L0 = self.top[0]
            self._call(lib.dr_cuda_dlrm_inter_gemm, ptr(x), ldx, ptr(self.sp.urow), ptr(self.sp.inv), self.sp.ldinv, self.T, self.D, B, ptr(L0.w_bf16), L0.Kp,
                       L0.N, ptr(self.p(L0.name + "/bias")), ptr(L0.a), L0.N, ptr(self.Z) if train else None, self.Zp, self.sp.sync_ref())
        elif self.uf and self.emu:   # emulation: the indirect kernels are mma code -> k_sp_gather (waits for the ROWS flags) + the SIMT interaction kernel
            if getattr(self, "_emb_g", None) is None:
                self._emb_g = torch.zeros(B, self.T, self.D, dtype=torch.bfloat16, device=self.dev)
            self.sp.gather(self._emb_g)
            self._call(lib.dr_cuda_dot_interaction_fwd, ptr(x), ldx, ptr(self._emb_g), self.D, self.T * self.D, self.T, self.D, B, ptr(self.Z), self.Zp)
        elif self.uf:   # gathers urow[inv[b][t]]; the kernel itself waits for every owner's ROWS flag
            self._call(lib.dr_cuda_dot_interaction_fwd_u, ptr(x), ldx, ptr(self.sp.urow), ptr(self.sp.inv), self.sp.ldinv, self.T, self.D, B, ptr(self.Z),
                       self.Zp, self.sp.sync_ref())
        else:
            self._call(lib.dr_cuda_dot_interaction_fwd, ptr(x), ldx, ptr(self.emb), B * self.D, self.D, self.T, self.D, B, ptr(self.Z), self.Zp)
        self._tick("f_dot")
        if train:
            # every owner's ROWS flag of this step has been seen => every peer finished last step's all-reduce reads of this buffer
            self.grads.zero_()
        x, ldx = self.Z, self.Zp
        for li, L in enumerate(self.top):
            if not (fused0 and li == 0):
                self._gemm(x, ldx, L.w_bf16, L.Kp, B, L.N, L.Kp, self.p(L.name + "/bias"), True, None, 0, L.a, L.N)
            x, ldx = L.a, L.N
        self._tick("f_top")

    def _cross_forward(self, train: bool) -> None:
        """x_{l+1} = x0 * (t_l W_l^T + b_l) + x_l with t_l = x_l V_l^T: a plain GEMM, then a GEMM whose epilogue applies the cross (and keeps u_l)."""
        B, N, x0 = self.B, self.inter_dim, self.xs[0]
        for l, (V, W) in enumerate(self.cross):
            self._gemm(self.xs[l], N, V.w_bf16, V.Kp, B, V.N, V.Kp, None, False, None, 0, self.ts[l], V.N)
            self._call(self.lib.dr_cuda_gemm_tn_cross, ptr(self.ts[l]), V.N, ptr(W.w_bf16), W.Kp, B, N, W.Kp, ptr(self.p(W.name + "/bias")), 1,
                       ptr(x0), N, ptr(self.xs[l]), N, ptr(self.xs[l + 1]), N, ptr(self.us[l]) if train else None, N, self._ctas)

    def _cross_backward(self) -> None:
        """dL/dx_L (dZ) back through the cross layers -> dy of the last bottom layer and the feature-major demb."""
        lib, B, N, x0 = self.lib, self.B, self.inter_dim, self.xs[0]
        g, nl = self.dZ, len(self.cross)
        for l in range(nl - 1, -1, -1):
            V, W = self.cross[l]
            # du = g * x0, dx0 (+)= g * u_l, db_l += column sums of du
            self._call(lib.dr_cuda_cross_bwd, ptr(g), N, ptr(x0), N, ptr(self.us[l]), N, B, N, ptr(self.du), N, ptr(self.dx0), N, int(l == nl - 1),
                       ptr(self.g(W.name + "/bias")))
            self._gemm_dw(self.du, N, self.ts[l], V.N, W.N, W.Kp, self.g(W.name + "/kernel"), W.Kp)          # dW_l += du^T t_l
            self._gemm(self.du, N, W.wt_bf16, W.Np, B, V.N, N, None, False, None, 0, self.dt, V.N)            # dt = du W_l
            self._gemm_dw(self.dt, V.N, self.xs[l], N, V.N, V.Kp, self.g(V.name + "/kernel"), V.Kp)         # dV_l += dt^T x_l
            gn = self.gbuf[l % 2]                                                                             # dx_l = g + dt V_l
            self._call(lib.dr_cuda_gemm_tn_cross, ptr(self.dt), V.N, ptr(V.wt_bf16), V.Np, B, N, V.N, None, 2, None, 0, ptr(g), N, ptr(gn), N, None, 0,
                       self._ctas)
            g = gn
        last = self.bot[-1]
        self._call(lib.dr_cuda_cross_split, ptr(self.dx0), N, ptr(g), N, B, self.T, self.D, ptr(last.dy), last.N, ptr(self.demb))

    def _head(self, train: bool) -> None:
        h = self.top[-1]
        inv = 1.0 / float(self.B * self.world)
        self._call(self.lib.dr_cuda_head, ptr(h.a), h.N, self.B, self.head_K, ptr(self.p("logits/kernel")), ptr(self.p("logits/bias")),
                   ptr(self.labels), inv, ptr(self.prob), ptr(self.loss), ptr(h.da), ptr(self.g("logits/kernel")),
                   ptr(self.g("logits/bias")), 1, int(train), ptr(self.g(h.name + "/bias")) if train else None)

    def _backward(self) -> None:
        lib, B, cfg = self.lib, self.B, self.cfg
        v2 = not cfg.gemm_v1
        self._tick("h1")
        # ---- top MLP (da of the last hidden layer and its bias gradient were produced by the head kernel)
        for i in range(len(self.top) - 1, -1, -1):
            L = self.top[i]
            x, ldx = (self.top[i - 1].a, self.top[i - 1].N) if i > 0 else (self.Z, self.Zp)
            self._gemm_dw(L.da, L.N, x, ldx, L.N, L.Kp, self.g(L.name + "/kernel"), L.Kp)
            if i > 0:
                P = self.top[i - 1]       # dX epilogue: * relu'(h_{i-1}) and bias gradient of layer i-1 (column sums) fused
                self._gemm(L.da, L.N, L.wt_bf16, L.Np, B, P.N, L.N, None, False, P.a, P.N, P.da, P.N, aux_mode=1,
                           S1=self.g(P.name + "/bias") if v2 else None)
                if not v2:
                    self._call(lib.dr_cuda_colstats, ptr(P.da), None, B, P.N, P.N, P.N, ptr(self.g(P.name + "/bias")), None)
            else:
                self._gemm(L.da, L.N, L.wt_bf16, L.Np, B, self.Zp, L.N, None, False, None, 0, self.dZ, self.Zp)
        self._tick("b_top")
        # ---- interaction backward -> dy of the last bottom layer, demb (feature-major)
        last = self.bot[-1]
        if self.dcn:
            self._cross_backward()
        elif self.uf and self.emu:
            self._call(lib.dr_cuda_dot_interaction_bwd, ptr(self.dZ), self.Zp, ptr(last.y), last.N, ptr(self._emb_g), self.D, self.T * self.D, self.T, self.D, B,
                       ptr(last.dy), last.N, ptr(self.demb), B * self.D, self.D)
        elif self.uf:   # features gathered through inv; per-sample gradient rows -> demb (pre-reduced per key by k_sp_segsum on the side stream)
            self._call(lib.dr_cuda_dot_interaction_bwd_u, ptr(self.dZ), self.Zp, ptr(last.y), last.N, ptr(self.sp.urow), ptr(self.sp.inv), self.sp.ldinv,
                       self.T, self.D, B, ptr(last.dy), last.N, ptr(self.demb), B * self.D, self.D)
        else:
            self._call(lib.dr_cuda_dot_interaction_bwd, ptr(self.dZ), self.Zp, ptr(last.y), last.N, ptr(self.emb), B * self.D, self.D, self.T, self.D, B,
                       ptr(last.dy), last.N, ptr(self.demb), B * self.D, self.D)
        main = None if self.emu else torch.cuda.current_stream(self.dev)
        fork = cfg.overlap_embedding and not self.emu
        self._tick("b_dot")
        if fork:
            self._fork(main)
            with torch.cuda.stream(self._side):
                self._embedding_backward()
                self._tick("b_emb")
        with self._dense_window() if fork else nullcontext():
            self._bottom_backward()
        if fork:
            self._join(main)
        else:
            self._embedding_backward()
            self._tick("b_emb")
        self._tick("b_join")

    def _bottom_backward(self) -> None:
        lib, B, cfg = self.lib, self.B, self.cfg
        v2 = not cfg.gemm_v1
        # ---- bottom MLP backward
        for i in range(len(self.bot) - 1, -1, -1):
            L = self.bot[i]
            if i == len(self.bot) - 1 or not v2:      # statistics of dy not produced by a v2 GEMM epilogue
                self._call(lib.dr_cuda_colstats, ptr(L.dy), ptr(L.a), B, L.N, L.N, L.N, ptr(L.S1b), ptr(L.S2b))
            self._call(lib.dr_cuda_bn_bwd_finalize, ptr(L.S1b), ptr(L.S2b), L.N, B, ptr(L.mean), ptr(L.rstd), ptr(self.g(L.name + "/bn_gamma")),
                       ptr(self.g(L.name + "/bn_beta")), ptr(L.c1), ptr(L.c2), 1.0)
            # da = relu'(a) * BN'(dy)  (+ bias gradient = column sums of da, fused)
            self._call(lib.dr_cuda_bn_bwd_apply_v2, ptr(L.dy), ptr(L.a), B, L.N, L.N, ptr(L.scale), ptr(L.mean), ptr(L.rstd), ptr(L.c1), ptr(L.c2),
                       ptr(L.da), 1, ptr(self.g(L.name + "/bias")))
            if i > 0:
                P = self.bot[i - 1]
                # dW = (da^T a_{l-1}) diag(s_{l-1}) + db t_{l-1}^T  : GEMM on the un-normalised activation + tiny fix-up
                self._gemm_dw(L.da, L.N, P.a, P.N, L.N, L.Kp, self.g(L.name + "/kernel"), L.Kp)
                self._call(lib.dr_cuda_dw_fixup, ptr(self.g(L.name + "/kernel")), ptr(self.g(L.name + "/bias")), ptr(P.scale), ptr(P.shift), L.N, L.K, L.Kp)
                # dy_{l-1} = da W  with BatchNorm-backward statistics (sum dy, sum dy * a_{l-1}) fused into the epilogue
                fused = v2 and P.N > 32
                self._gemm(L.da, L.N, L.wt_bf16, L.Np, B, P.N, L.N, None, False, P.a if fused else None, P.N, P.dy, P.N, aux_mode=2 if fused else 0,
                           S1=P.S1b if fused else None, S2=P.S2b if fused else None)
                if v2 and not fused:
                    self._call(lib.dr_cuda_colstats, ptr(P.dy), ptr(P.a), B, P.N, P.N, P.N, ptr(P.S1b), ptr(P.S2b))
            else:
                self._gemm_dw(L.da, L.N, self.x0, self.x0.shape[1], L.N, L.Kp, self.g(L.name + "/kernel"), L.Kp)
        self._tick("b_bot")

    def _dense_update(self) -> None:
        lib = self.lib
        if self.comm is not None:
            self.comm.dense_allreduce_update(self)
        else:
            self._call(lib.dr_cuda_dense_apply, ptr(self.params), ptr(self.grads), ptr(self.s0) if self.s0 is not None else None,
                       ptr(self.s1) if self.s1 is not None else None, self.P, ptr(self.hp_dev), 1.0, None)
        self._pack_weights()
        self.group.end_step()
        self._tick("u1")

    def _step_body(self) -> None:
        self.loss.zero_()
        self.stats.zero_()
        self._forward(True)
        self._head(True)
        self._backward()
        self._dense_update()

    # ------------------------------------------------------------------------------------------------
    # public API
    # ------------------------------------------------------------------------------------------------
    def load_batch(self, dense: torch.Tensor, ids: torch.Tensor, labels: torch.Tensor, non_blocking: bool = True) -> None:
        """Copy one batch (host pinned or device tensors) into the static input buffers.  ids: [T, B] feature-major."""
        self.dense_in.copy_(dense, non_blocking=non_blocking)
        self.ids.copy_(ids, non_blocking=non_blocking)
        self.labels.copy_(labels, non_blocking=non_blocking)

    def capture(self) -> None:
        """Warm up eagerly (loads modules, sizes everything) then capture the whole step into one CUDA graph."""
        self.train_step_eager()
        if self.emu:                                # kernels run synchronously on the host: the eager step IS the step
            return
        torch.cuda.synchronize(self.dev)
        n0 = self.launches
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=torch.cuda.Stream(device=self.dev)):
            self._step_body()
        self.launches_per_step = self.launches - n0
        self._graph = g

    def train_step_eager(self) -> None:
        n0 = self.launches
        self._step_body()
        self.launches_per_step = self.launches - n0

    def train_step(self) -> None:
        """One optimizer step on the batch currently in the input buffers (graph replay when captured)."""
        if self._graph is not None:
            self._graph.replay()
            self._launches += self.launches_per_step
        else:
            self.train_step_eager()

    def predict(self) -> torch.Tensor:
        """Forward only (BatchNorm uses running statistics, tables are read-only)."""
        self.loss.zero_()
        self._forward(False)
        self._head(False)
        if self.uf:
            self.group.forward_only_tail()
        return self.prob

    def global_step(self) -> int:
        raw = bytes(self.hp_dev.cpu().numpy().tobytes())
        return int(OptHyper.from_buffer_copy(raw).global_step)

    def l2_flush(self) -> None:
        if self._l2_scratch is None:
            self._l2_scratch = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=self.dev)   # 256 MB > 50 MB L2
        self._call(self.lib.dr_cuda_l2_flush, ptr(self._l2_scratch), self._l2_scratch.numel(), 0.0)

    def state_dict(self) -> Dict[str, torch.Tensor]:
        out = {k: self.params[o:o + n].clone() for k, (o, n) in self.views.items()}
        for L in self.bot:
            out[L.name + "/bn_moving_mean"] = L.running_mean.clone()
            out[L.name + "/bn_moving_variance"] = L.running_var.clone()
        return out
