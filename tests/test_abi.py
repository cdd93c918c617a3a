"""CPU-side checks of the C-ABI boundary: the library loads without a GPU and exports every symbol
include/atomai_b200.h declares; the ctypes table mirrors the header; no compute is launched."""
import ctypes
import os
import re

from atomai_b200 import _C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "atomai_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(atomai_b200_\w+)\s*\(", src)))


def test_library_builds_and_loads():
    path = _C.build()
    assert os.path.exists(path)
    lib = _C.lib()
    assert b"sm_90a" in lib.atomai_b200_version()


def test_every_declared_symbol_is_exported_and_bound():
    lib = _C.lib()
    syms = header_symbols()
    assert len(syms) >= 25
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in the header but not exported"
        assert s in _C.SIGNATURES, f"{s} has no ctypes signature"
    for s in _C.SIGNATURES:
        assert s in syms, f"{s} bound in _C.py but not declared in the header"


def test_struct_layouts_match_header():
    # ab_src_t: 3 pointers + 4 int32; ab_conv_t: 8 int32 + 2 ab_src_t + float + 3 int32
    assert ctypes.sizeof(_C.Src) == 3 * 8 + 4 * 4
    assert ctypes.sizeof(_C.Conv) == 8 * 4 + 2 * ctypes.sizeof(_C.Src) + 4 * 4
    assert ctypes.sizeof(_C.CoordLat) == 6 * 4 + 6 * 8


def test_error_convention_without_gpu():
    """Bad arguments return a non-zero status + message; nothing throws across the ABI."""
    lib = _C.lib()
    d = _C.Conv()
    d.N, d.H, d.W, d.Cout, d.ks_h, d.ks_w, d.dil, d.nsrc = 1, 8, 8, 16, 5, 5, 1, 1
    rc = lib.atomai_b200_conv_fwd(ctypes.byref(d), 1, None, 1, 16, None, None)
    assert rc != 0
    assert b"conv" in lib.atomai_b200_last_error()
    assert lib.atomai_b200_gram(None, None, None, 1.0, 1, 1, 1, 0, 2, None, 1, None, 0, None) != 0
    assert lib.atomai_b200_gram_workspace_bytes(1000, 500, 128) >= (1000 + 500) * 160 * 4
