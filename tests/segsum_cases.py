"""k_sp_segsum (csrc/cuda/sparse_pipeline.cu) bit for bit against a numpy model of its exact semantics, shared by the GPU test
(test_gpu_segsum_flush.py) and its CUDA-on-CPU emulation twin (test_cuda_emu_segsum_flush.py).

The semantics: id column c is cut into 32-sample tiles; inside a tile the samples holding the same key (invT[c][b] = gs >= 0) form one group,
whose rows are added in fp32 from 0 in ascending sample order; every element of that sum is converted once to 64-bit fixed point (x 2^40,
clamped to +-2^62, NaN -> 0, rounded to nearest even) and the groups' integers are added into ugrad[gs] (wrapping, so in any order)."""
import numpy as np
import torch

SCALE = np.float32(2.0 ** 40)
FIX_MAX = np.float32(2.0 ** 62)


def ugrad_fix(x: np.ndarray) -> np.ndarray:
    """float32 -> int64 bits (as uint64) the way ugrad_fix does it."""
    y = x.astype(np.float32) * SCALE
    y = np.where(np.isnan(y), np.float32(0), np.where(np.abs(y) <= FIX_MAX, y, np.copysign(FIX_MAX, y))).astype(np.float32)
    return np.rint(y).astype(np.int64).view(np.uint64)


def reference(invT: np.ndarray, demb_f32: np.ndarray, rows: int) -> np.ndarray:
    """ugrad contributions [rows, dim] (uint64) of one segsum over invT [C][B] and the bf16 gradient rows demb [C][B][dim] (as float32)."""
    C, B, dim = demb_f32.shape
    tiles = (B + 31) // 32
    pad = tiles * 32 - B
    gs = np.concatenate([invT, np.full((C, pad), -1, invT.dtype)], axis=1).reshape(C, tiles, 32)
    x = np.concatenate([demb_f32, np.zeros((C, pad, dim), np.float32)], axis=1).reshape(C, tiles, 32, dim)
    # leader[c, t, l] = the first lane of tile (c, t) holding the same key as lane l
    eq = gs[:, :, :, None] == gs[:, :, None, :]
    leader = eq.argmax(axis=3)
    acc = np.zeros((C, tiles, 32, dim), np.float32)
    ci, ti = np.meshgrid(np.arange(C), np.arange(tiles), indexing="ij")
    for lane in range(32):                      # ascending lane order: one member per group and step, so the fp32 adds are the kernel's
        live = gs[:, :, lane] >= 0
        ld = leader[:, :, lane]
        acc[ci[live], ti[live], ld[live]] += x[ci[live], ti[live], lane]
    is_leader = (leader == np.arange(32)) & (gs >= 0)
    out = np.zeros((rows, dim), np.uint64)
    np.add.at(out, gs[is_leader], ugrad_fix(acc[is_leader]))
    return out


def cases(small: bool):
    """(name, ids [C][B] int64 with -1 = padding, demb bf16 [C][B][dim]).  small: sizes the emulation runs in seconds."""
    out = []
    g = torch.Generator().manual_seed(11)

    def grad(C, B, dim, lo=-8.0, hi=2.0):
        mag = 10.0 ** (torch.rand(C, B, dim, generator=g) * (hi - lo) + lo)            # |g| over ten decades: the add order shows in the bits
        sign = torch.where(torch.rand(C, B, dim, generator=g) < 0.5, -1.0, 1.0)
        return (mag * sign).bfloat16()

    B = 300 if small else 4133                                                          # not a multiple of 32 or of 256
    dims = [8, 16, 64, 128]
    for dim in dims:
        C = 3
        ids = torch.full((C, B), 7, dtype=torch.int64)                                  # all samples on one key
        out.append((f"one_key_d{dim}", ids, grad(C, B, dim)))
        ids = torch.arange(C * B, dtype=torch.int64).reshape(C, B)                      # all keys distinct
        out.append((f"distinct_d{dim}", ids, grad(C, B, dim)))
        u = torch.rand(C, B, generator=g, dtype=torch.float64)                          # power law: P(k) ~ k^-1.05 over 5000 ids
        ids = (torch.pow(5000.0, u) - 1.0).long()
        ids[1, ::5] = -1                                                                # padding rows (gs = -1)
        ids[2, 100:180] = -1                                                            # and a fully padded tile
        out.append((f"powerlaw_pad_d{dim}", ids, grad(C, B, dim)))
    # one key hot across every block of a column, mixed with distinct keys
    C, dim = 2, 16
    ids = torch.randint(0, 1 << 20, (C, B), generator=g)
    ids[:, ::3] = 42
    out.append(("hot_across_blocks_d16", ids, grad(C, B, dim)))
    # saturation: groups whose fp32 sum lies beyond +-2^22 are clamped to +-2^62 (and their 64-bit sum wraps)
    ids = torch.randint(0, 4, (C, B), generator=g)
    demb = grad(C, B, dim)
    demb[0, :, :4] = 3.0e5                                                              # 32 x 3e5 > 2^22 = 4.19e6
    demb[1, :, 4:8] = -1.0e7
    demb[1, :64, 8] = 2.0 ** 22                                                         # one such element alone lands exactly on the bound
    out.append(("saturate_d16", ids, demb))
    return out


def check(sp, ids: torch.Tensor, demb: torch.Tensor, sync=lambda: None) -> None:
    """dedup + segsum on the pipeline `sp`, then every touched ugrad row against the model, bit for bit; leaves the scratch clean."""
    sp.dedup(ids)
    sync()
    invT = sp.invT[:, : ids.shape[1]].cpu().numpy()
    ref = reference(invT, demb.float().cpu().numpy(), sp.Htot)
    sp.segsum(demb)
    sync()
    got = sp.ugrad.cpu().numpy().view(np.uint64)
    sp.reset(); sp.step_end()
    sync()
    touched = np.unique(invT[invT >= 0])
    bad = np.nonzero((got[touched] != ref[touched]).any(axis=1))[0]
    assert bad.size == 0, f"{bad.size} of {touched.size} keys differ, first gs {touched[bad[0]]}: {got[touched[bad[0]]]} vs {ref[touched[bad[0]]]}"
