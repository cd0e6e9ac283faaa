"""CPU-side checks of the drop-in boundary: the shared library builds, loads, and exports every
symbol include/ptranking_b200.h declares; the ctypes prototypes cover the same set."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    text = open(os.path.join(ROOT, "include", "ptranking_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(ptrb200_[a-z0-9_]+)\s*\(", text)))


@pytest.fixture(scope="module")
def lib_path():
    from ptranking_b200 import build
    return build.build()


def test_header_declares_entry_points():
    syms = header_symbols()
    assert "ptrb200_lambdarank_fwd_bwd" in syms and "ptrb200_ffnet_forward" in syms
    assert len(syms) >= 16


def test_library_exports_every_declared_symbol(lib_path):
    lib = ctypes.CDLL(lib_path)
    for s in header_symbols():
        assert hasattr(lib, s), f"{s} declared in the header but not exported"


def test_ctypes_prototypes_match_header(lib_path):
    from ptranking_b200 import _lib
    assert sorted(_lib.SIGNATURES) == header_symbols()
    lib = _lib.load()
    assert lib.ptrb200_version() >= 101
    assert isinstance(lib.ptrb200_launch_count(), int)


def test_standard_scale_refuses_unknown_dtype_and_aliased_bf16_output(lib_path):
    """The output element type is checked with the arguments, before anything reaches the device."""
    from ptranking_b200 import _lib
    lib = _lib.load()
    buf = (ctypes.c_float * 16)()
    p = ctypes.addressof(buf)          # never dereferenced: the call returns at the argument check
    assert lib.ptrb200_standard_scale(p, None, p, 7, 1, 4, 4, 0, 0.0, None) == -1
    assert b"out_dtype" in lib.ptrb200_last_error()
    assert lib.ptrb200_standard_scale(p, None, p, _lib.DTYPE_BF16, 1, 4, 4, 0, 0.0, None) == -1
    assert b"alias" in lib.ptrb200_last_error()


def test_no_cpu_fallback():
    import torch
    import ptranking_b200
    from ptranking_b200 import ops, _lib
    sf = dict(sf_id="pointsf", opt="Adam", lr=1e-4, pointsf=dict(num_features=4))
    with pytest.raises(RuntimeError):
        ptranking_b200.ListNet(sf_para_dict=sf, gpu=False, device="cpu")
    with pytest.raises(_lib.B200LibraryError):
        ops.rank_loss_and_grad("ListNet", torch.zeros(1, 4), torch.zeros(1, 4))


def test_product_never_imports_oracle():
    """The shipped package must not import, call or link anything under oracle/."""
    pkg = os.path.join(ROOT, "ptranking_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f
                assert not re.search(r"\boracle\b", src), f
