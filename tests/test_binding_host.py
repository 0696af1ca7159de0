"""CPU: the ctypes binding against include/dmnerf_b200.h, without loading the library.  ctypes passes whatever it is given,
so a prototype that disagrees with the header, or a tensor of the wrong dtype or layout, would reach a kernel unnoticed."""
import ctypes as C
import os
import re

import pytest
import torch

from dmnerf_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "dm-nerf_b200")

_C_KINDS = {"int": "int", "int32_t": "int", "int64_t": "int64_t", "uint64_t": "uint64_t", "uint32_t": "uint32_t",
            "float": "float", "double": "double"}
_PY_KINDS = {C.c_int: "int", C.c_int64: "int64_t", C.c_uint64: "uint64_t", C.c_uint32: "uint32_t", C.c_float: "float",
             C.c_double: "double"}


def _c_kind(decl):
    """Kind of a C return type or parameter declaration ("const float* x" -> pointer, "int64_t n" -> int64_t)."""
    if "*" in decl:
        return "pointer"
    return _C_KINDS[[w for w in re.findall(r"\w+", decl) if w != "const"][0]]


def _py_kind(t):
    if t in (C.c_void_p, C.c_char_p) or issubclass(t, C._Pointer):
        return "pointer"
    return _PY_KINDS[t]


def _header_signatures():
    src = open(os.path.join(ROOT, "include", "dmnerf_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    src = "\n".join(line for line in src.splitlines() if not line.lstrip().startswith("#"))
    sigs = {}
    for ret, name, params in re.findall(r"DMNERF_API\s+([^;(]*?)\b(dmnerf_\w+)\s*\(([^)]*)\)\s*;", src):
        params = params.strip()
        args = [] if params in ("", "void") else [_c_kind(p) for p in params.split(",")]
        sigs[name] = (_c_kind(ret), args)
    return sigs


def test_prototypes_match_the_header_argument_kinds():
    header = _header_signatures()
    assert set(header) == set(_lib.PROTOTYPES), set(header) ^ set(_lib.PROTOTYPES)
    for name, (res, args) in _lib.PROTOTYPES.items():
        assert (_py_kind(res), [_py_kind(a) for a in args]) == header[name], name


def test_ptr_checks_dtype_and_layout():
    t = torch.zeros(4, 3)
    assert _lib.ptr(t).value == t.data_ptr() and _lib.ptr(None) is None
    i = torch.zeros(5, dtype=torch.int32)
    assert _lib.ptr(i, torch.int32).value == i.data_ptr()
    for bad, dtype in ((t.double(), torch.float32), (t.t(), torch.float32), (t, torch.int32), (i, torch.int64)):
        with pytest.raises(RuntimeError, match="contiguous"):
            _lib.ptr(bad, dtype)
    assert _lib.ptr(t.t(), strided=True).value == t.data_ptr()
    with pytest.raises(RuntimeError):
        _lib.ptr(t.t().double(), strided=True)
    assert list(_lib.ptrs([t, t[1:]])) == [t.data_ptr(), t[1:].data_ptr()]
    with pytest.raises(RuntimeError):
        _lib.ptrs([t, t.t()])


def test_camera_takes_a_3x3_intrinsics_and_the_top_3x4_of_the_pose():
    K = [[500.0, 0.0, 320.0], [0.0, 500.0, 240.0], [0.0, 0.0, 1.0]]
    c2w = torch.arange(16, dtype=torch.float64).reshape(4, 4) / 7
    k9, p12 = _lib.camera(K, c2w)
    assert list(k9) == [v for row in K for v in row]
    assert list(p12) == c2w[:3, :4].float().reshape(-1).tolist()
    assert list(_lib.camera(torch.tensor(K), c2w[:3].numpy())[1]) == list(p12)
    with pytest.raises(ValueError):
        _lib.camera(torch.eye(4), c2w)


def test_only_the_binding_hands_tensor_addresses_to_the_library():
    """Every pointer goes through _lib.ptr / ptrs; engine.py reads data_ptr() only for its binding key."""
    offenders = []
    for dp, _, files in os.walk(PKG):
        for f in files:
            path = os.path.join(dp, f)
            if f.endswith(".py") and path not in (os.path.join(PKG, "_lib.py"), os.path.join(PKG, "engine.py")):
                if ".data_ptr()" in open(path).read():
                    offenders.append(os.path.relpath(path, ROOT))
    assert not offenders, offenders
