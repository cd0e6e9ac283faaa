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
    assert lib.ptrb200_version() >= 100
    assert isinstance(lib.ptrb200_launch_count(), int)


def test_attention_tc_entry_points_reject_passes_other_than_3(lib_path):
    """The attention calls keep their `passes` argument for ABI stability; only 3 (3xTF32) is implemented, and any other
    value is refused while the arguments are checked, before anything reaches the device."""
    from ptranking_b200 import _lib
    lib = _lib.load()
    buf = (ctypes.c_float * 16)()
    p = ctypes.addressof(buf)          # never dereferenced: the call returns at the argument check
    B, n, H, D = 1, 4, 1, 4
    calls = {
        "attention_tc_fwd": lambda: lib.ptrb200_attention_tc_fwd(*[p] * 6, B, n, H, D, 0.0, 0, 0, 1, None),
        "attention_tc_bwd": lambda: lib.ptrb200_attention_tc_bwd(*[p] * 9, B, n, H, D, 0.0, 0, 0, 1, None),
        "attention_tc_fwd_ld": lambda: lib.ptrb200_attention_tc_fwd_ld(*[p] * 6, B, n, H, D, 0, 0, None, 0.0, 0, 0, 1, None),
        "attention_tc_bwd_ld": lambda: lib.ptrb200_attention_tc_bwd_ld(*[p] * 9, B, n, H, D, 0, 0, 0.0, 0, 0, 1, None),
    }
    for name, call in calls.items():
        with pytest.raises(_lib.B200LibraryError, match="passes must be 3"):
            _lib.check(call(), name)


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
