"""The host replica of the dropout stream (tests/dropout_ref.py) against common.cuh itself, bit for bit.

A small host-only program includes common.cuh and prints make_drop / make_drop_call, dropout_key, dropout_draw4 and
dropout_keep for a list of (seed, offset, element, p) cases; the replica must print the same.  These functions are
__host__ __device__, so a host build checks the exact code the kernels inline.  Needs nvcc, no GPU."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests import dropout_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "ptranking_b200", "csrc")

PROGRAM = r"""
#include "common.cuh"
#include <stdio.h>
#include <string.h>
using namespace ptrb200;
int main() {
    unsigned long long seed, offset, elem;
    float p;
    while (scanf("%llu %llu %llu %a", &seed, &offset, &elem, &p) == 4) {
        const DropCfg d = make_drop(p, seed, offset);
        const DropCfg c = make_drop_call(p, seed, offset);
        uint32_t sb;
        memcpy(&sb, &d.scale, 4);
        printf("%u %u %llu %llu %llu %d %llu\n", d.thr, sb, (unsigned long long)d.key,
               (unsigned long long)dropout_draw4(d.key, elem >> 2), (unsigned long long)dropout_key(seed, offset),
               (int)dropout_keep(d.key, elem, d.thr), (unsigned long long)c.key);
    }
    return 0;
}
"""

PS = [1e-6, 0.1, 0.25, 0.5, 0.9, 0.99999]


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module")
def stream_program(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found: the host build of common.cuh cannot be made")
    d = tmp_path_factory.mktemp("dropout_stream")
    src, exe = d / "stream.cu", d / "stream"
    src.write_text(PROGRAM)
    r = subprocess.run([nvcc, "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a", "-I", CSRC, str(src), "-o", str(exe)],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    return str(exe)


def _cases():
    rng = np.random.default_rng(2024)
    seeds = [0, 1, 1234, 2 ** 63, 2 ** 64 - 1] + [int(s) for s in rng.integers(0, 2 ** 63, 4, dtype=np.int64)] + [2 ** 63 + 12345]
    offsets = [0, 1, 7, 2 ** 32 + 3, 2 ** 58 - 1] + [o * 64 + l for o in (1, 5, 1000) for l in (0, 1, 15, 63)]
    elems = [0, 1, 2, 3, 4, 5, 7, 8, 135, 136, 137, 262144 * 136 - 1, 2 ** 32 - 1, 2 ** 32, 2 ** 40 - 4, 2 ** 40 - 1, 2 ** 40, 2 ** 40 + 3]
    elems += [int(e) for e in rng.integers(0, 2 ** 40, 6, dtype=np.int64)]
    out = []
    for i, s in enumerate(seeds):
        for j, o in enumerate(offsets):
            for k, e in enumerate(elems):
                if (i + j + k) % 3 == 0:            # a third of the grid; every seed, offset and element still appears
                    out.append((s, o, e, PS[(i * 7 + j * 3 + k) % len(PS)]))
    for p in PS:                                    # every p with every extreme seed
        for s in (0, 2 ** 63, 2 ** 64 - 1):
            out.append((s, 64 * 3 + 15, 2 ** 40 + 1, p))
    return out


def _expected(seed, offset, elem, p):
    thr = ref.threshold(p)
    sc = ref.scale(p)
    key = ref.dropout_key(seed, offset)
    return (thr, int(np.float32(sc).view(np.uint32)), int(key), int(ref.dropout_draw4(key, elem >> 2)), int(key),
            int(bool(ref.keep(key, elem, thr))), int(ref.dropout_key(seed, ref.call_index(offset))))


def test_replica_matches_common_cuh_bit_for_bit(stream_program):
    cases = _cases()
    stdin = "".join(f"{s} {o} {e} {float(np.float32(p)).hex()}\n" for s, o, e, p in cases)
    r = subprocess.run([stream_program], input=stdin, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, check=True)
    lines = r.stdout.splitlines()
    assert len(lines) == len(cases)
    names = ("thr", "scale bits", "key", "draw4", "dropout_key", "keep", "call key")
    for case, line in zip(cases, lines):
        got = tuple(int(v) for v in line.split())
        want = _expected(*case)
        for nm, g, w in zip(names, got, want):
            assert g == w, (case, nm, g, w)


def test_threshold_and_scale_of_the_documented_rates():
    assert ref.threshold(0.0) == 0 and ref.threshold(1e-6) == 0 and ref.scale(1e-6) == np.float32(1.0)
    assert ref.threshold(0.1) == 6554 and ref.threshold(0.25) == 16384 and ref.threshold(0.5) == 32768
    assert ref.threshold(0.99999) == 65535 and ref.scale(0.99999) == np.float32(65536.0)
    # the kernels' 65536 / (65536 - thr), not 1 / (1 - p): at p = 0.1 that is 6.8e-6 relative
    assert ref.scale(0.1) == np.float32(65536.0 / 58982.0)
    assert abs(float(ref.scale(0.1)) * 0.9 - 1.0 - 6.8e-6) < 1e-7


def test_keep_stream_equals_per_element_keep():
    """The vectorised mask (one draw per quad, lanes low bits first) equals keep() element by element, and a quad's four
    lanes come from one draw."""
    key = ref.dropout_key(99, ref.ff_index(3, 2))
    thr = ref.threshold(0.5)
    m = ref.keep_stream(key, 1001, thr)
    e = np.arange(1001, dtype=np.uint64)
    assert np.array_equal(m, ref.keep(key, e, thr))
    draws = ref.dropout_draw4(key, np.arange(251, dtype=np.uint64))
    lanes = np.stack([(draws >> np.uint64(16 * i)) & np.uint64(0xFFFF) for i in range(4)], 1).reshape(-1)[:1001]
    assert np.array_equal(m, lanes >= thr)
    assert 0.45 < 1.0 - m.mean() < 0.55


def test_key_domains_are_disjoint():
    """An FF call owns key indices o*64 + l for its layers l < PTRB200_MAX_FF_LAYERS - 1; a one-mask call owns o*64 + 63.
    No index of one kind can equal an index of the other, for any pair of offsets."""
    ff = {ref.ff_index(o, l) for o in range(1, 300) for l in range(ref.MAX_FF_LAYERS - 1)}
    calls = {ref.call_index(o) for o in range(1, 20000)}
    assert not ff & calls
    assert len(calls) == 19999
