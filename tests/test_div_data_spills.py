"""The device DIVDataset's kernels (csrc/div_data.cu) must compile without local-memory spills.  The check reads
ptxas's report (-Xptxas -v) from the build log that `python -m ptranking_b200.build` writes; it skips when that log is
missing or older than the sources."""
import glob
import os
import re

import pytest

from ptranking_b200 import build as b

BUILD_LOG = os.path.join(b.LIB_DIR, "build.log")


def test_div_data_kernels_do_not_spill():
    deps = b.sources() + glob.glob(os.path.join(b.CSRC, "*.cuh")) + [b.HEADER]
    if not os.path.exists(BUILD_LOG) or any(os.path.getmtime(d) > os.path.getmtime(BUILD_LOG) for d in deps):
        pytest.skip("no up-to-date build log: run `python -m ptranking_b200.build` first")
    text = open(BUILD_LOG).read()
    start = text.find("== div_data.cu")
    assert start >= 0, "div_data.cu missing from the build log"
    end = text.find("\n== ", start + 1)
    report = text[start:end if end >= 0 else None]
    found, cur = {}, None
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and m:
            found[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    assert any("div_ideal_order_kernel" in k for k in found) and any("div_pack_kernel" in k for k in found), found
    assert all(v == (0, 0) for v in found.values()), found
