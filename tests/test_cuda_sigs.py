"""The ctypes table of libdeeprec_cuda.so (deeprec_b200/_cuda_sigs.py) against the extern "C" definitions under csrc/cuda, and the binding of
the CUDA-on-CPU emulation build when it loads.  A wrong argument type is silent in ctypes and a fault on the device, so it is caught here."""
import ctypes as C
import glob
import os
import re

import pytest

from deeprec_b200 import _cuda_sigs, _native
from deeprec_b200 import build as _build

PKG = os.path.dirname(os.path.abspath(_cuda_sigs.__file__))
CUDA_DIR = os.path.join(_build.CSRC, "cuda")

# dr_* entry points of csrc/cuda that keep bindings of their own, outside the table
BOUND_ELSEWHERE = {
    "dr_serving_release": "serving/processor.py (_Abi: the serving runtime ABI, shared with the CPU runtime's dr_cpu_* names)",
    "dr_serving_free": "serving/processor.py (_Abi)",
    "dr_tp_cuda_stats": "utils/memory.py (tensor-pool allocator, loaded before the first CUDA allocation)",
    "dr_tp_cuda_step_end": "utils/memory.py",
}

_DEF = re.compile(r"^(int|int64_t|void\s*\*|void)\s+(dr_\w+)\s*\(([^()]*)\)\s*\{", re.M)
_C_CLASS = {"int": "int", "int32_t": "int", "int64_t": "int64_t", "uint32_t": "uint32_t", "float": "float", "cudaStream_t": "pointer"}
_PY_CLASS = {C.c_int: "int", C.c_int64: "int64_t", C.c_uint32: "uint32_t", C.c_float: "float", C.c_void_p: "pointer"}


def _definitions():
    """name -> [(source relative to csrc, return class, [argument classes])] of every dr_* function defined in csrc/cuda."""
    out = {}
    for path in sorted(glob.glob(os.path.join(CUDA_DIR, "*.cu")) + glob.glob(os.path.join(CUDA_DIR, "emu", "*.cu"))):
        text = open(path).read()
        text = re.sub(r"//[^\n]*", "", re.sub(r"/\*.*?\*/", " ", text, flags=re.S))
        for m in _DEF.finditer(text):
            params = [p.strip() for p in m.group(3).split(",") if p.strip() not in ("", "void")]
            out.setdefault(m.group(2), []).append((os.path.relpath(path, _build.CSRC), _c_class(m.group(1)), [_c_class(p) for p in params]))
    return out


def _c_class(decl):
    """pointer / int / int64_t / uint32_t / float / void for one C parameter (named or not) or return type."""
    if "*" in decl:
        return "pointer"
    ty = decl.split()[1] if decl.startswith("const ") else decl.split()[0]
    return _C_CLASS.get(ty, ty)


def _py_class(t):
    if t is None:
        return "void"
    if issubclass(t, C._Pointer):
        return "pointer"
    return _PY_CLASS[t]


def test_every_table_entry_matches_its_c_definition():
    defs = _definitions()
    assert len(defs) > 100, "the extern \"C\" definitions were not found"
    bad = []
    for name, (argtypes, restype) in _cuda_sigs.SIGNATURES.items():
        assert name in defs, f"{name} is declared but not defined in csrc/cuda"
        want = ([_py_class(t) for t in argtypes], _py_class(restype))
        for src, ret, args in defs[name]:
            if (args, ret) != want:
                bad.append(f"{name} ({src}): C ({', '.join(args)}) -> {ret}, table ({', '.join(want[0])}) -> {want[1]}")
    assert not bad, "\n".join(bad)


def test_every_called_entry_point_is_in_the_table():
    defined = set(_definitions())
    called = set()
    for path in glob.glob(os.path.join(PKG, "**", "*.py"), recursive=True):
        called |= set(re.findall(r"\.(dr_\w+)\(", open(path).read()))
    missing = sorted((called & defined) - set(_cuda_sigs.SIGNATURES) - set(BOUND_ELSEWHERE))
    assert not missing, f"called but not declared in _cuda_sigs.py: {missing}"


@pytest.fixture
def fresh_emulation(monkeypatch):
    """Enter the emulation as the first thing a process does: a new library object that nothing has touched yet."""
    monkeypatch.setattr(_native, "_EMU", None)
    with _native.cuda_emulation() as lib:
        yield lib


def test_emulation_library_is_bound_when_it_loads(fresh_emulation):
    lib = fresh_emulation
    unbound = [name for name, (argtypes, restype) in _cuda_sigs.SIGNATURES.items()
               if hasattr(lib, name) and (tuple(getattr(lib, name).argtypes or ()) != tuple(argtypes) or getattr(lib, name).restype != restype)]
    assert not unbound, f"not bound by cuda_emulation(): {unbound}"
    assert _native.cuda() is lib


def test_entry_points_missing_from_the_emulation_are_hardware_only(fresh_emulation):
    defs = _definitions()
    wrong = {}
    for name in _cuda_sigs.SIGNATURES:
        if not hasattr(fresh_emulation, name):
            srcs = {src for src, _, _ in defs[name]}
            if not srcs <= set(_build.CUDA_SOURCES) or srcs & set(_build.EMU_SOURCES):
                wrong[name] = sorted(srcs)
    assert not wrong, f"missing from the emulation build although defined in its sources: {wrong}"
