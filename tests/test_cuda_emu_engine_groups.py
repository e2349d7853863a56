"""FusedRecEngine's launch count against the CUDA-on-CPU emulation's own counter: every kernel a training step launches is counted exactly once,
by the code that launches it (the embedding groups and their pipelines, the dense optimizer, the communicator's all-reduce), without and with the
linear group, at world 1 and with 2 ranks as threads.  ``capture()`` reports the same count per step."""
import ctypes
import threading

import pytest
import torch

from deeprec_b200 import _native

pytestmark = [pytest.mark.timeout(900)]
CARDS = [50, 1000, 7, 300] + [97] * 22
B = 64


def _batch(step: int, rank: int):
    g = torch.Generator().manual_seed(1000 * step + rank)
    ids = torch.stack([torch.randint(0, c, (B,), generator=g) for c in CARDS])
    return ids, (torch.rand(B, generator=g) < 0.3).float(), {"dense": torch.rand(B, 13, generator=g)}


def _fwd(net, dense, emb, ids, linear=None):
    out = net(torch.cat([dense["dense"], emb.float().flatten(1)], 1)).squeeze(-1)
    return out if linear is None else out + linear


def _rank(rank, world, linear, comm, sync, seen, reported):
    """Two train steps, then capture() (one warm-up step); the emulator's counter is read by rank 0 between barriers."""
    from deeprec_b200.models.rec_engine import FusedRecEngine
    with _native.cuda_emulation():
        lib = _native.cuda()
        lib.dr_cuda_emu_launch_count.restype = ctypes.c_int64
        eng = FusedRecEngine(torch.nn.Linear(26 * 16 + 13, 1), _fwd, list(range(26)), CARDS, B, dense_inputs={"dense": ((B, 13), torch.float32)},
                             rank=rank, world_size=world, comm=comm, linear=linear, linear_optimizer="ftrl" if linear else None)
        for step in range(3):
            eng.load_batch(*_batch(step, rank))
            sync()
            c0 = lib.dr_cuda_emu_launch_count()
            sync()
            if step < 2:
                n0 = eng.launches
                eng.train_step()
                reported[rank].append(eng.launches - n0)
            else:
                eng.capture(warmup=1)
                reported[rank].append(eng.launches_per_step)
            sync()
            if rank == 0:
                seen.append(lib.dr_cuda_emu_launch_count() - c0)


@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("linear", [False, True], ids=["deep", "linear_ftrl"])
def test_step_launches_match_the_emulator(linear, world):
    with _native.cuda_emulation():          # build + load the library on the main thread (the rank threads must not fork a compiler)
        pass
    seen, reported = [], {r: [] for r in range(world)}
    if world == 1:
        _rank(0, 1, linear, None, lambda: None, seen, reported)
    else:
        from deeprec_b200.parallel.emu_comm import EmuComm, EmuWorld
        shared, errors = EmuWorld(world), []

        def run(rank):
            try:
                _rank(rank, world, linear, EmuComm(shared, rank), shared.barrier.wait, seen, reported)
            except BaseException as e:                          # noqa: BLE001
                errors.append((rank, repr(e)))
                shared.barrier.abort()

        threads = [threading.Thread(target=run, args=(r,), daemon=True) for r in range(world)]
        for t in threads:
            t.start()
        for t in threads:
            t.join(timeout=600)
        assert not errors, errors
    counted = [sum(reported[r][s] for r in range(world)) for s in range(3)]
    assert counted == seen and min(seen) > 0, (counted, seen)
