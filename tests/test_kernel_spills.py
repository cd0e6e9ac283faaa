"""The persistent row kernel (rows_gemm_ws_kernel) must compile without local-memory spills.

Its consumer and producer warpgroups run on separate register budgets (setmaxnreg); a spill in either role puts
local-memory traffic on the scorer's hot path.  The check reads ptxas's report (-Xptxas -v) of ffnet.cu from the build
log that `python -m ptranking_b200.build` writes; it skips when that log is missing or older than the sources (compiling
ffnet.cu here would take minutes).
"""
from __future__ import annotations

import glob
import os
import re

import pytest

from ptranking_b200 import build as b

BUILD_LOG = os.path.join(b.LIB_DIR, "build.log")


def _ffnet_report():
    """ptxas's report for ffnet.cu from an up-to-date build log, or None."""
    deps = b.sources() + glob.glob(os.path.join(b.CSRC, "*.cuh")) + [b.HEADER]
    if not os.path.exists(BUILD_LOG) or any(os.path.getmtime(d) > os.path.getmtime(BUILD_LOG) for d in deps):
        return None
    text = open(BUILD_LOG).read()
    start = text.find("== ffnet.cu")
    if start < 0:
        return None
    end = text.find("\n== ", start + 1)
    return text[start:end if end >= 0 else None]


def ws_kernel_spills(report: str) -> dict:
    """{mangled rows_gemm_ws_kernel name: (spill store bytes, spill load bytes)} from a ptxas -v report."""
    out, cur = {}, None
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1) if "rows_gemm_ws_kernel" in m.group(1) else None
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and m:
            out[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    return out


def test_rows_gemm_ws_kernel_does_not_spill():
    report = _ffnet_report()
    if report is None:
        pytest.skip("no up-to-date build log: run `python -m ptranking_b200.build` first")
    spills = ws_kernel_spills(report)
    # every instantiation the host launcher selects: 2 modes x 2 pass counts x activations, K-specialised, bf16 input
    assert len(spills) >= 20, f"expected every rows_gemm_ws_kernel instantiation in the ptxas report, found {len(spills)}"
    bad = {k: v for k, v in spills.items() if v != (0, 0)}
    assert not bad, "rows_gemm_ws_kernel instantiations spill (stores, loads bytes):\n" + "\n".join(
        f"  {k}: {v}" for k, v in sorted(bad.items()))


TILE_CASES = [
    # B, n, dims, AF, TL_AF, norm, affine, dropout (as tests/test_gpu_scorer.py TC_CASES).  More row tiles than the H100's
    # 132 SMs, so the persistent CTAs own different numbers of tiles, with a ragged last tile; the producers prefetch
    # across tile boundaries from inputs of 5, 4, 1 and 2 K-chunks.
    (100, 181, [136, 100, 24, 40, 100, 1], "GE", "S", "BN", True, 0.1),
    (80, 300, [136, 100, 100, 1], "GE", "S", "BN2", False, 0.1),          # per-query groups: 128 + 128 + 44 rows
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", TILE_CASES, ids=[f"tiles{i}" for i in range(len(TILE_CASES))])
def test_row_kernel_tile_boundaries_match_simt(case):
    from tests import test_gpu_scorer
    test_gpu_scorer.test_tensor_core_path_matches_simt_path(case)
