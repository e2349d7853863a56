"""In-tree native build: g++ for the host engine, nvcc (sm_90a only) for the device engine.

Both libraries are plain C-ABI shared objects loaded with ctypes (no torch headers, so a full
rebuild takes seconds and cross-compiles on a box without a GPU).  The .so files land in
``deeprec_b200/lib``, so the package imports straight from the source tree.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.abspath(__file__))
CSRC = os.environ.get("DEEPREC_CSRC") or os.path.join(ROOT, "csrc")           # overridable: build a scratch copy of the sources next to a running test suite
LIB = os.environ.get("DEEPREC_LIB") or os.path.join(ROOT, "lib")
OBJ = os.path.join(LIB, "obj")

HOST_SOURCES = ["host/host_engine.cc", "host/io_runtime.cc", "host/ssd_store.cc", "host/predict_codec.cc", "host/redis_store.cc", "host/tensor_pool.cc", "host/cpu_serving.cc", "host/ps_server.cc", "host/csv_ops.cc"]
CUDA_SOURCES = [
    "cuda/table_kernels.cu",
    "cuda/embedding_kernels.cu",
    "cuda/optimizer_kernels.cu",
    "cuda/dense_kernels.cu",
    "cuda/gemm_fp8.cu",
    "cuda/gemm_mxfp8.cu",
    "cuda/gemm_wgmma.cu",
    "cuda/interaction_kernels.cu",
    "cuda/comm_kernels.cu",
    "cuda/sparse_pipeline.cu",
    "cuda/ag_embedding.cu",
    "cuda/fused_interaction_gemm.cu",
    "cuda/tier_kernels.cu",
    "cuda/nvls.cu",
    "cuda/program_kernels.cu",
    "cuda/sparse_utils.cu",
    "cuda/serving_runtime.cu",
    "cuda/fused_ops.cu",
    "cuda/allocator.cu",
    "cuda/attention_kernels.cu",
]

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _stamp(srcs: list[str], flags: list[str]) -> str:
    h = hashlib.sha1()
    for f in flags:
        h.update(f.encode())
    deps = list(srcs)
    for d in ("common", "cuda", "host"):
        dd = os.path.join(CSRC, d)
        if os.path.isdir(dd):
            for fn in sorted(os.listdir(dd)):
                if fn.endswith((".h", ".cuh")):
                    deps.append(os.path.join(dd, fn))
    for s in deps:
        with open(s, "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()


def _run(cmd: list[str]) -> None:
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError("native build failed: " + " ".join(cmd[:3]))
    if os.environ.get("DEEPREC_BUILD_VERBOSE"):
        sys.stderr.write(r.stdout + r.stderr)


def _up_to_date(out: str, stamp: str) -> bool:
    sf = out + ".stamp"
    return os.path.exists(out) and os.path.exists(sf) and open(sf).read() == stamp


def build_host(force: bool = False) -> str:
    os.makedirs(LIB, exist_ok=True)
    out = os.path.join(LIB, "libdeeprec_host.so")
    srcs = [os.path.join(CSRC, s) for s in HOST_SOURCES if os.path.exists(os.path.join(CSRC, s))]
    # -fopenmp + DR_USE_OPENMP: the host engine's parallel loops share PyTorch's libgomp pool (see ThreadPool in host_engine.cc)
    flags = ["-O3", "-std=c++17", "-fPIC", "-shared", "-pthread", "-march=x86-64-v3", "-fno-math-errno", "-fopenmp", "-DDR_USE_OPENMP"]
    stamp = _stamp(srcs, flags)
    if not force and _up_to_date(out, stamp):
        return out
    _run(["g++"] + flags + srcs + ["-o", out, "-ldl"])
    open(out + ".stamp", "w").write(stamp)
    return out


def build_cuda(force: bool = False, verbose_ptxas: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    out = os.path.join(LIB, "libdeeprec_cuda.so")
    srcs = [os.path.join(CSRC, s) for s in CUDA_SOURCES if os.path.exists(os.path.join(CSRC, s))]
    flags = ARCH_FLAGS + ["-O3", "-std=c++17", "-lineinfo", "--use_fast_math", "-Xcompiler", "-fPIC",
                          "--expt-relaxed-constexpr", "-I" + os.path.join(CSRC)]
    if verbose_ptxas:
        flags += ["-Xptxas", "-v"]
    stamp = _stamp(srcs, flags)
    if not force and _up_to_date(out, stamp):
        return out

    def compile_one(src: str) -> str:
        obj = os.path.join(OBJ, os.path.basename(src) + ".o")
        ostamp = _stamp([src], flags)
        if not force and _up_to_date(obj, ostamp):
            return obj
        _run([NVCC] + flags + ["-c", src, "-o", obj])
        open(obj + ".stamp", "w").write(ostamp)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(compile_one, srcs))
    _run([NVCC] + ARCH_FLAGS + ["-shared", "-Xcompiler", "-fPIC", "-cudart", "static"] + objs + ["-o", out])
    open(out + ".stamp", "w").write(stamp)
    return out


# ---- CUDA-on-CPU emulation build (csrc/cuda/emu/cuda_emu.h): the SIMT kernels compiled by g++, one host thread per CUDA thread -----------------
# Sources without wgmma / TMA / mbarrier code.  The library exports the same dr_* C entry points as libdeeprec_cuda.so, taking host pointers.
EMU_SOURCES = [
    "cuda/table_kernels.cu",
    "cuda/embedding_kernels.cu",
    "cuda/optimizer_kernels.cu",
    "cuda/dense_kernels.cu",
    "cuda/interaction_kernels.cu",      # SIMT variants only (the tensor-core kernels are compiled out)
    "cuda/fused_ops.cu",
    "cuda/program_kernels.cu",
    "cuda/sparse_utils.cu",
    "cuda/attention_kernels.cu",
    "cuda/serving_runtime.cu",
    "cuda/sparse_pipeline.cu",          # unique-first model-parallel pipeline: ranks = host threads, peer memory = the shared address space
    "cuda/comm_kernels.cu",
    "cuda/ag_embedding.cu",             # all-gather -> lookup -> reduce-scatter embedding (SOK DistributedEmbedding dataflow) over peer memory
    "cuda/tier_kernels.cu",             # multi-tier: miss list / histogram eviction kernels + the manager's background thread
    "cuda/emu/emu_stubs.cu",            # host-loop stand-ins for the wgmma GEMM entry points
]


def _split_top_level(text: str) -> list[str]:
    parts, depth, cur = [], 0, ""
    for ch in text:
        if ch in "([{":
            depth += 1
        elif ch in ")]}":
            depth -= 1
        if ch == "," and depth == 0:
            parts.append(cur.strip())
            cur = ""
        else:
            cur += ch
    if cur.strip():
        parts.append(cur.strip())
    return parts


def _emu_shared_decls(text: str) -> str:
    """``__shared__ T name[dims];`` -> a reference into per-BLOCK storage (``emu::shared_var``): function-level statics would be shared by every
    kernel running in the process (two serving sessions, the rank threads of a multi-rank emulation)."""
    import re
    import zlib
    seed = zlib.crc32(text[:4096].encode()) % 30000
    counter = [0]

    def repl(m):
        counter[0] += 1
        uid = seed * 1000 + counter[0]
        ty, name, dims = m.group(2), m.group(3), m.group(4) or ""
        return (f"{m.group(1)}using emu_sh_{uid} = {ty}{dims}; "
                f"emu_sh_{uid}& {name} = *reinterpret_cast<emu_sh_{uid}*>(emu::shared_var({uid}, sizeof(emu_sh_{uid})));")

    return re.sub(r"(^|[;{}\s])(?<!extern )__shared__\s+(?:__align__\(\d+\)\s+)?([\w:]+(?:<[^<>;]*>)?)\s+(\w+)((?:\[[^\];]*\])*)\s*;",
                  lambda m: repl(m) if "extern" not in text[max(0, m.start() - 8):m.start() + 1] else m.group(0), text)


def emu_translate(src: str) -> str:
    """``kernel<T><<<grid, block, smem, stream>>>(args);`` -> ``emu::launch(grid, block, smem, stream, [&] { kernel<T>(args); });`` and
    ``extern __shared__ T name[];`` -> a pointer into the block's dynamic shared memory.  Everything else is handled by macros / inline functions."""
    import re
    out, pos = [], 0
    launch = re.compile(r"([A-Za-z_][\w:]*(?:<[^<>;(){}]*>)?)\s*<<<")
    while True:
        m = launch.search(src, pos)
        if not m:
            out.append(src[pos:])
            break
        end_cfg = src.index(">>>", m.end())
        cfg = _split_top_level(src[m.end():end_cfg])
        cfg += ["0"] * (4 - len(cfg))
        i = end_cfg + 3
        while src[i].isspace():
            i += 1
        assert src[i] == "(", "kernel launch without an argument list"
        depth, j = 0, i
        while True:
            depth += src[j] == "("
            depth -= src[j] == ")"
            if depth == 0:
                break
            j += 1
        out.append(src[pos:m.start()])
        out.append(f"emu::launch(dim3({cfg[0]}), dim3({cfg[1]}), (size_t)({cfg[2]}), (cudaStream_t)({cfg[3]}), [&] {{ {m.group(1)}{src[i:j + 1]}; }})")
        pos = j + 1
    text = "".join(out)
    text = _emu_shared_decls(text)
    text = re.sub(r"extern\s+__shared__\s+((?:__align__\(\d+\)\s+)?)([\w:<> ]+?)\s+(\w+)\[\];",
                  lambda m: f"{m.group(2)}* {m.group(3)} = ({m.group(2)}*)emu::dyn_smem();", text)
    return text


def build_cuda_emu(sanitize: str | None = None, force: bool = False, sources: list[str] | None = None) -> str:
    """g++ build of the SIMT kernels (``-DDR_CUDA_EMU``).  ``sanitize`` = ``"address"`` / ``"thread"`` / ``"undefined"`` instruments the kernels
    themselves: the library then has to be loaded by a process that preloads the sanitizer runtime (tests/native/emu_driver.py does)."""
    emu_dir = os.path.join(OBJ, "emu" + ("_" + sanitize if sanitize else ""))
    os.makedirs(os.path.join(emu_dir, "cuda", "emu"), exist_ok=True)
    out = os.path.join(LIB, "libdeeprec_cuda_emu" + ("_" + sanitize.replace(",", "_") if sanitize else "") + ".so")
    names = sources or EMU_SOURCES
    srcs = [os.path.join(CSRC, s) for s in names]
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(NVCC)), "include")
    flags = ["-O1" if sanitize else "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-DDR_CUDA_EMU", "-x", "c++", "-I" + cuda_inc, "-I" + CSRC,
             "-Wno-attributes", "-Wno-unknown-pragmas", "-Wno-deprecated-declarations"]
    if sanitize:
        flags += ["-fsanitize=" + sanitize, "-fno-omit-frame-pointer"]
    stamp = _stamp(srcs + [os.path.join(CSRC, "cuda", "emu", "cuda_emu.h")], flags + names)
    if not force and _up_to_date(out, stamp):
        return out
    # translated copies keep the csrc layout so that "common.cuh" / "../common/ev_types.h" resolve next to them
    for d in ("common", "cuda", os.path.join("cuda", "emu")):
        os.makedirs(os.path.join(emu_dir, d), exist_ok=True)
        for fn in os.listdir(os.path.join(CSRC, d)):
            if fn.endswith((".h", ".cuh")):
                with open(os.path.join(CSRC, d, fn)) as fh:
                    text = fh.read()
                with open(os.path.join(emu_dir, d, fn), "w") as fh:
                    fh.write(emu_translate(text) if fn.endswith(".cuh") else text)
    tus = []
    for s in srcs:
        tu = os.path.join(emu_dir, os.path.relpath(s, CSRC) + ".cc")
        with open(s) as fh:
            text = fh.read()
        with open(tu, "w") as fh:
            fh.write(f'#line 1 "{s}"\n' + emu_translate(text))
        tus.append(tu)
    cflags = [f for f in flags if f != "-shared"]

    def compile_one(tu: str) -> str:
        obj = tu + ".o"
        _run(["g++"] + cflags + ["-c", tu, "-o", obj])
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(tus))) as ex:
        objs = list(ex.map(compile_one, tus))
    _run(["g++", "-shared", "-pthread"] + (["-fsanitize=" + sanitize] if sanitize else []) + objs + ["-o", out])
    open(out + ".stamp", "w").write(stamp)
    return out


def build_all(force: bool = False) -> None:
    build_host(force)
    build_cuda(force)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv)
    print("built:", os.listdir(LIB))
