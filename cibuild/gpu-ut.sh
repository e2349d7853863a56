#!/usr/bin/env bash
# GPU unit tests (needs an H100; multi-GPU parts need >= 2).  Mirrors the reference's cibuild/gpu-ut/*.sh shards.
#   bash cibuild/gpu-ut.sh            # pytest -m gpu
#   bash cibuild/gpu-ut.sh sanitize   # + compute-sanitizer memcheck / racecheck over the sparse pipeline and the flag protocol
set -euo pipefail
cd "$(dirname "$0")/.."
python -c "import __graft_entry__ as g; g.build()"
python -m pytest tests/ -x -q -m gpu --timeout 600
if [ "${1:-}" = "sanitize" ]; then
  # shared-memory hazards of the dedup / segsum / lookup kernels and the fused engines (single GPU)
  compute-sanitizer --tool racecheck --error-exitcode 1 python -m pytest tests/test_gpu_sparse_pipeline.py -q -m gpu -x -k "dedup or lookup_rows"
  compute-sanitizer --tool memcheck --error-exitcode 1 python -m pytest tests/test_gpu_sparse_pipeline.py tests/test_gpu_tier.py -q -m gpu -x
  # the release/acquire flag protocol + peer loads / stores under memcheck on 2 ranks (racecheck does not model cross-device accesses)
  if [ "$(python -c 'import torch; print(torch.cuda.device_count())')" -ge 2 ]; then
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29655 \
      --no-python compute-sanitizer --tool memcheck --error-exitcode 1 python tests/mp_check.py
  fi
fi
