"""The LETOR reader's host-side ground: the device decimal parser against Python's float(), the golden fixture's
coverage, and the refusals of ``read_letor`` -- all without a GPU.

letor_float.cuh's parse_decimal is __host__ __device__; a host build of the same source prints the float64 bit
pattern of each token it reads, and Python's float() must produce the same bits (float() is correctly rounded, as the
parser must be).  Needs nvcc, no GPU."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "ptranking_b200", "csrc")
GOLDEN = os.path.join(ROOT, "tests", "golden", "letor.npz")

PROGRAM = r"""
#include "letor_float.cuh"
#include <stdio.h>
using namespace ptrb200;
int main() {
    static char buf[1 << 16];
    while (fgets(buf, sizeof buf, stdin)) {
        size_t n = strlen(buf);
        while (n && buf[n - 1] == '\n') --n;
        const DecResult d = parse_decimal(buf, buf + n);
        unsigned long long b;
        memcpy(&b, &d.value, 8);
        printf("%d %016llx\n", d.status, b);
    }
    return 0;
}
"""

HARD = [
    "9007199254740993", "9007199254740992", "9007199254740994", "9007199254740995", "-9007199254740993",
    "2.2250738585072011e-308", "2.2250738585072012e-308", "2.2250738585072014e-308", "2.225073858507201136057409796709131975934819546351645648e-308",
    "1.7976931348623157e308", "1.7976931348623158e308", "1.7976931348623159e308", "1.79769313486e+308", "-1.79769313486e+308",
    "0.1", "0.2", "0.3", "-0.1", ".1", "1.", "+1", "-0", "0", "00000", "0.000", "0e0", "0e-999999", "1e400", "-1e400", "1e-400",
    "5e-324", "4.9406564584124654e-324", "2.4703282292062327e-324", "2.4703282292062328e-324", "2.4703282292062327208828e-324",
    "3e-324", "7.4109846876186982e-324", "1e-320", "1e23", "8.98846567431158e307", "123456789012345678901234567890",
    "0.30000000000000001665334536937734810635447502136230468750", "0.3000000000000000166533453693773481063544750213623046875",
    "0.30000000000000001665334536937734810635447502136230468751", "1.00000000000000011102230246251565404236316680908203125",
    "1.00000000000000011102230246251565404236316680908203124", "1.00000000000000011102230246251565404236316680908203126",
    "9007199254740993.0000000000000000000000000001", "4503599627370496.5", "4503599627370497.5", "1.0000000000000002",
    "1e22", "1e-22", "1234567890123456789", "12345678901234567890", "99999999999999999999", "1.E5", "1e+5", "1E-5",
    "0.0000000000000000000000000000000000000000000000000000001", "3.141592653589793238462643383279502884197",
    "7.2057594037927933e16", "2.0000000000000004440892098500626161694526672363281250", "0.017453292519943295769236907684886",
    "1448997445238699", "5708990770823839524233143877797980545530986496", "6.6e-309", "1e-308", "1.8e308",
]
BAD = ["", "+", "-", ".", "e5", "1e", "1e+", "1x", "--1", "1.2.3", "inf", "nan", "1_0", "0x10", " 1", "1 ", "1e5.5", "+-1"]


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module")
def parser_program(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found: the host build of letor_float.cuh cannot be made")
    d = tmp_path_factory.mktemp("letor_float")
    src, exe = d / "parse.cu", d / "parse"
    src.write_text(PROGRAM)
    r = subprocess.run([nvcc, "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a", "-I", CSRC, str(src), "-o", str(exe)],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    return str(exe)


def _run(exe, tokens):
    r = subprocess.run([exe], input="".join(t + "\n" for t in tokens), stdout=subprocess.PIPE, text=True, check=True)
    out = [line.split() for line in r.stdout.splitlines()]
    assert len(out) == len(tokens)
    return [(int(s), int(b, 16)) for s, b in out]


def _bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def _seeded_tokens(count: int, seed: int = 2025):
    """Tokens shaped like LETOR values and beyond: %g / %.17g / repr of doubles over the full exponent range, short
    fixed-point decimals, integers, long mantissas (up to 30 digits), exact halfway points of adjacent doubles, signs and
    exponent spellings."""
    rng = np.random.default_rng(seed)
    toks = []
    per = count // 8
    # 1. random doubles over the whole range, printed shortest-repr, %.17g and %.15g
    bits = rng.integers(0, 0x7FF0000000000000, per, dtype=np.int64).view(np.float64)
    for i, v in enumerate(bits):
        toks.append((repr, "%.17g", "%.15g")[i % 3] % v if i % 3 else repr(float(v)))
    # 2. LETOR-typical: fixed-point values with up to 6 decimals, scaled normals, integers
    vals = np.round(rng.standard_normal(per) * 10.0 ** rng.integers(-3, 7, per), 6)
    toks += ["%g" % v if i % 2 else "%.6f" % v for i, v in enumerate(vals)]
    toks += [str(int(v)) for v in rng.integers(-10 ** 12, 10 ** 12, per)]
    # 3. long mantissas: 17..30 random digits with a decimal point and an exponent
    for _ in range(per):
        nd = int(rng.integers(17, 31))
        digits = "".join(rng.choice(list("0123456789"), nd))
        dot = int(rng.integers(0, nd + 1))
        e = int(rng.integers(-330, 310))
        toks.append(("-" if rng.random() < 0.3 else "") + digits[:dot] + "." + digits[dot:] + "e%d" % e)
    # 4. exact halfway points between adjacent doubles (round-half-even decides), and one digit either side
    base = rng.integers(1, 0x7FE0000000000000, per, dtype=np.int64)
    from decimal import Decimal, getcontext
    getcontext().prec = 800
    for b in base[: per // 4]:
        lo = float(np.int64(b).view(np.float64))
        hi = float(np.int64(b + 1).view(np.float64))
        mid = (Decimal(lo) + Decimal(hi)) / 2
        s = format(mid, "e")
        toks.append(s)
        toks.append(format(mid.next_plus() if False else mid * (1 + Decimal(10) ** -40), ".40e"))
        toks.append(format(mid * (1 - Decimal(10) ** -40), ".40e"))
    # 5. subnormals and the extremes
    sub = rng.integers(1, 1 << 52, per, dtype=np.int64).view(np.float64)
    toks += [repr(float(v)) for v in sub]
    toks += ["%.20e" % v for v in sub[: per // 4]]
    # 6. spellings: leading '+', '.5', '5.', 'E', zero padding
    for v in rng.standard_normal(count - len(toks)):
        k = int(rng.integers(0, 5))
        s = repr(float(v))
        toks.append(["+" + s.lstrip("-"), s.replace("0.", "."), "%.3E" % v, "000" + "%.4f" % abs(v), "%d." % int(v * 1000)][k])
    return toks


def test_hard_cases_bit_equal_python_float(parser_program):
    got = _run(parser_program, HARD)
    undecided = []
    for tok, (st, b) in zip(HARD, got):
        if st == 2:
            undecided.append(tok)
            continue
        assert st == 0, tok
        assert b == _bits(float(tok)), (tok, hex(b), float(tok).hex())
    # handed to float(): only tokens with more than 19 significant digits that sit on a rounding boundary
    assert all(_significant_digits(t) > 19 for t in undecided), undecided
    assert "9007199254740993" not in undecided and "2.2250738585072011e-308" not in undecided


def _significant_digits(tok: str) -> int:
    m = tok.lstrip("+-").lower().split("e")[0].replace(".", "").lstrip("0")
    return len(m)


def test_malformed_tokens_are_rejected(parser_program):
    for tok, (st, _) in zip(BAD, _run(parser_program, BAD)):
        assert st == 1, tok


def test_a_million_seeded_tokens_bit_equal_python_float(parser_program):
    toks = _seeded_tokens(1_000_000)
    got = _run(parser_program, toks)
    undecided = []
    for tok, (st, b) in zip(toks, got):
        if st == 2:                       # > 19 significant digits on a rounding boundary: the reader asks float()
            undecided.append(tok)
            continue
        assert st == 0, tok
        assert b == _bits(float(tok)), (tok, hex(b), float(tok).hex())
    assert all(_significant_digits(t) > 19 for t in undecided)
    # the constructed halfway points (3 * 31250 tokens of 40+ digits) are undecided by design; the random long
    # mantissas almost never are
    assert len(undecided) <= 3 * (1_000_000 // 8 // 4) + 100, len(undecided)


def test_pow5_table_matches_its_generator():
    r = subprocess.run(["python", os.path.join(ROOT, "tools", "gen_letor_pow5.py"), "--check"])
    assert r.returncode == 0, "letor_pow5.cuh differs from tools/gen_letor_pow5.py's output"


def test_fixture_covers_the_awkward_inputs():
    z = np.load(GOLDEN)
    mslr = z["mslr/file"].tobytes().decode()
    assert "qid:010 " in mslr and "qid:10 " in mslr
    qids = [line.split()[1] for line in mslr.splitlines()]
    first = {q: qids.index(q) for q in qids}
    assert any(qids[i] != qids[i - 1] and first[qids[i]] < i for i in range(1, len(qids)))     # non-contiguous recurrence
    assert any(len([t for t in line.split()[2:] if t.startswith("5:")]) > 1 for line in mslr.splitlines())
    toks = [t.split(":", 1)[1] for line in mslr.splitlines() for t in line.split()[2:]]
    assert any(_significant_digits(t) >= 17 for t in toks) and any("e" in t.lower() for t in toks)
    assert any(t.startswith(("-", "+")) for t in toks) and "9007199254740993" in toks
    assert b"\r\n" in z["mq2008/file"].tobytes() and b"#docid" in z["mq2008/file"].tobytes()
    assert not z["yahoo/file"].tobytes().endswith(b"\n") and b" 699:" in z["yahoo/file"].tobytes()
    assert b"1.79769313486e+308" in z["istella/file"].tobytes()
    assert str(z["mqlist/data_id"]) == "MQ2008_List"
    names = {k.split("/")[1] for k in z.files if k.count("/") == 2}
    for s in ("none", "StandardScaler", "MinMaxScaler"):
        for p in (0, 1):
            assert any(n.startswith(s + "_md3_mr1") and n.endswith("_p%d" % p) for n in names)


@pytest.mark.parametrize("dd,kw", [
    (dict(data_id="MSLRWEB30K", scale_data=True, scaler_id="RobustScaler", scaler_level="QUERY"), {}),
    (dict(data_id="MSLRWEB30K", scale_data=True, scaler_id="SLog1P", scaler_level="QUERY"), {}),
    (dict(data_id="MSLRWEB30K", scale_data=True, scaler_id="StandardScaler", scaler_level="DATASET"), {}),
])
def test_refusals_raise_before_any_device_work(dd, kw, monkeypatch):
    from ptranking_b200 import _lib
    from ptranking_b200.letor import read_letor

    def no_device(*a, **k):
        raise AssertionError("the device was touched")
    monkeypatch.setattr(_lib, "load", no_device)
    with pytest.raises(NotImplementedError):
        read_letor("/nonexistent.txt", dd, presort=False, **kw)


def test_dataset_refusals_raise_before_any_device_work(monkeypatch):
    from ptranking_b200 import _lib
    from ptranking_b200.letor import LTRDataset

    monkeypatch.setattr(_lib, "load", lambda *a, **k: (_ for _ in ()).throw(AssertionError("the device was touched")))
    with pytest.raises(NotImplementedError):
        LTRDataset(None, "/nonexistent.txt", data_id="MSLRWEB30K", hot=True)
    with pytest.raises(NotImplementedError):
        LTRDataset(None, "/nonexistent.txt", data_id="MSLRWEB30K", eval_dict=dict(mask_label=True, mask_ratio=0.1, mask_type="rand_mask_all"))
