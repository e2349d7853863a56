# Developer entry points (the CI scripts under cibuild/ call the same targets).
PY ?= python
GPUS ?= 1

.PHONY: build test test-gpu sanitize model-test bench bench-cpu clean

build:            ## both native libraries, in-tree (nvcc cross-compiles sm_90a without a GPU)
	$(PY) -c "import __graft_entry__ as g; g.build()"

test: build       ## everything that runs without a GPU (multi-process paths on gloo)
	$(PY) -m pytest tests/ -x -q -m "not gpu"

test-gpu: build   ## needs an H100
	$(PY) -m pytest tests/ -x -q -m gpu

sanitize:         ## TSAN / ASAN / UBSAN builds of the host runtime + fuzzers
	$(PY) -m pytest tests/test_native_stress.py tests/test_cpu_serving.py -x -q -k "sanitizer or fuzz or stress"
	DEEPREC_EMU_SANITIZE_FULL=1 $(PY) -m pytest tests/test_cuda_emu_sanitizers.py -x -q      # the CUDA kernels under ASAN / TSAN (CPU emulation)

model-test: build ## smoke-train every zoo model for a few steps (cibuild/model-test.sh)
	bash cibuild/model-test.sh

bench: build      ## the headline benchmark (bench.py contract)
	@if [ "$(GPUS)" = "1" ]; then $(PY) bench.py; else $(PY) -m torch.distributed.run --nnodes=1 --nproc-per-node $(GPUS) --master-addr 127.0.0.1 --master-port 29517 bench.py --gpus $(GPUS); fi

bench-cpu: build  ## CPU training / serving / storage-engine benchmarks
	$(PY) benchmarks/cpu_zoo_bench.py --dtype both
	$(PY) benchmarks/cpu_serving_bench.py
	$(PY) benchmarks/ev_bench.py --keys 10000000

clean:
	rm -rf deeprec_b200/lib build *.egg-info
