"""read_letor on the device against the reference loader's output (tests/golden/letor.npz, made by
tests/golden/make_golden_letor.py from the unmodified reference on the CPU)."""
import os

import numpy as np
import pytest
import torch

from ptranking_b200 import _lib
from ptranking_b200.data import LengthBucketedBatches, RaggedBatches
from ptranking_b200.letor import LTRDataset, read_letor

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "letor.npz")
FORMATS = ("mslr", "mq2008", "yahoo", "istella", "mqlist")
SCALERS = (None, "StandardScaler", "MinMaxScaler")
LABEL_CFGS = ((0, 0, False, False), (3, 1, True, False), (0, 2, False, True), (4, 0, True, True))


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLDEN))


@pytest.fixture(scope="module")
def files(gold, tmp_path_factory):
    d = tmp_path_factory.mktemp("letor")
    out = {}
    for fmt in FORMATS:
        p = d / (fmt + ".txt")
        p.write_bytes(gold[f"{fmt}/file"].tobytes())
        out[fmt] = (str(p), str(gold[f"{fmt}/data_id"]))
    return out


def _name(s, md, mr, b, u, p):
    return "%s_md%d_mr%d_b%d_u%d_p%d" % (s or "none", md, mr, int(b), int(u), int(p))


def _dd(data_id, s, md, mr, b, u):
    return dict(data_id=data_id, scale_data=s is not None, scaler_id=s, scaler_level="QUERY" if s else None,
                min_docs=md, min_rele=mr, binary_rele=b, unknown_as_zero=u)


def _long_tokens(raw: bytes) -> int:
    toks = [t.split(b":", 1)[-1] for line in raw.split(b"\n") for t in line.split(b"#")[0].split()]
    return sum(len(t.lstrip(b"+-").lower().split(b"e")[0].replace(b".", b"").lstrip(b"0")) > 19 for t in toks)


def _ulp_diff(a, b):
    ai = a.view(np.int32).astype(np.int64)
    bi = b.view(np.int32).astype(np.int64)
    ai = np.where(ai < 0, -(ai & 0x7fffffff), ai)
    bi = np.where(bi < 0, -(bi & 0x7fffffff), bi)
    return np.abs(ai - bi)


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("scaler", SCALERS)
def test_presort_off_matches_reference(gold, files, fmt, scaler):
    path, data_id = files[fmt]
    base = _name(scaler, 0, 0, False, False, False)
    Xb, ob, qb = gold[f"{fmt}/{base}/X"], gold[f"{fmt}/{base}/offsets"], list(gold[f"{fmt}/{base}/qids"])
    rows = {q: Xb[ob[i]:ob[i + 1]] for i, q in enumerate(qb)}
    for md, mr, b, u in LABEL_CFGS:
        key = f"{fmt}/{_name(scaler, md, mr, b, u, False)}"
        sp = read_letor(path, _dd(data_id, scaler, md, mr, b, u), presort=False)
        assert sp.qids == list(gold[key + "/qids"])
        assert np.array_equal(sp.offsets_host, gold[key + "/offsets"])
        assert np.array_equal(sp.offsets.cpu().numpy(), gold[key + "/offsets"])
        assert np.array_equal(sp.y.cpu().numpy().view(np.int32), gold[key + "/y"].view(np.int32))
        want = np.concatenate([rows[q] for q in sp.qids]) if sp.qids else np.zeros((0, Xb.shape[1]), np.float32)
        got = sp.X.cpu().numpy()
        assert got.shape == want.shape
        if scaler is None:
            assert np.array_equal(got.view(np.int32), want.view(np.int32))
        else:
            # float64 sums in another order than numpy's: within 1 fp32 ulp
            d = _ulp_diff(got, want)
            assert d.max() <= 1, (key, d.max())
            print(f"{key}: {100.0 * np.mean(d == 0):.2f}% bit-equal")
        # tokens handed to float(): only ones with more than 19 significant digits (the fixture has a few on purpose)
        assert sp.host_tokens <= _long_tokens(gold[f"{fmt}/file"].tobytes())


@pytest.mark.parametrize("fmt", FORMATS)
def test_presort_on(gold, files, fmt):
    path, data_id = files[fmt]
    for scaler in SCALERS:
        for md, mr, b, u in LABEL_CFGS:
            dd = _dd(data_id, scaler, md, mr, b, u)
            off = read_letor(path, dd, presort=False)
            on = read_letor(path, dd, presort=True, seed=7)
            again = read_letor(path, dd, presort=True, seed=7)
            # bit patterns: a 1.8e308 column standard-scales to NaN, in the reference as here
            assert torch.equal(on.X.view(torch.int32), again.X.view(torch.int32)) and torch.equal(on.y, again.y)
            assert on.qids == off.qids and np.array_equal(on.offsets_host, off.offsets_host)
            key = f"{fmt}/{_name(scaler, md, mr, b, u, True)}"
            assert np.array_equal(on.y.cpu().numpy(), gold[key + "/y"])       # same labels, in the reference's order
            Xo, yo, Xn, yn = off.X.cpu().numpy(), off.y.cpu().numpy(), on.X.cpu().numpy(), on.y.cpu().numpy()
            for i in range(len(on)):
                a, e = on.offsets_host[i], on.offsets_host[i + 1]
                assert np.all(np.diff(yn[a:e]) <= 0)
                ka = sorted(map(tuple, np.column_stack([yo[a:e, None], Xo[a:e]]).view(np.int32).tolist()))
                kb = sorted(map(tuple, np.column_stack([yn[a:e, None], Xn[a:e]]).view(np.int32).tolist()))
                assert ka == kb


def test_bf16_is_the_rounded_fp32(files):
    path, data_id = files["mslr"]
    dd = _dd(data_id, "StandardScaler", 0, 0, False, False)
    a = read_letor(path, dd, presort=True, seed=3)
    b = read_letor(path, dd, presort=True, seed=3, feature_dtype=torch.bfloat16)
    assert b.X.dtype == torch.bfloat16
    assert torch.equal(a.X.to(torch.bfloat16).view(torch.int16), b.X.view(torch.int16))
    assert torch.equal(a.y, b.y)


BAD = [
    (b"1 qid:1 1:0.5\n\n2 qid:1 1:0.25\n", 2, "empty line"),
    (b"1 qid:1 1:0.5\r\n   \r\n", 2, "empty line"),
    (b"1 qid:1 1:0.5\nx qid:1 1:0.25\n", 2, "label"),
    (b"1 qid:1 1:0.5\n1 q:1 1:0.25\n", 2, "qid"),
    (b"1 qid:1 1:0.5\n1\n", 2, "qid"),
    (b"1 qid:1 1:0.5\n1 qid:1 1:abc\n", 2, "feature token"),
    (b"1 qid:1 1:0.5\n1 qid:1 1-0.5\n", 2, "feature token"),
    (b"1 qid:1 1:0.5\n1 qid:2 0:0.5\n", 2, "below the first index"),
    (b"1 qid:1 1:0.5\n1 qid:1 99999999999999999999:0.5\n", 2, "above PTRB200_LETOR_MAX_FEATURES"),
    (b"1 qid:1 1:0.5\n1 qid:3\n", 2, "no features"),
    (b"1 qid:1 1:0.5\n1 qid:1 1:0.5\n1 qid:1 1:0.5\n1 qid:1 1:1e\n", 4, "feature token"),
]


@pytest.mark.parametrize("text,line,what", BAD)
def test_malformed_lines_are_errors_naming_the_line(tmp_path, text, line, what):
    p = tmp_path / "bad.txt"
    p.write_bytes(text)
    with pytest.raises(_lib.B200LibraryError, match=f"line {line}: .*{what}"):
        read_letor(str(p), _dd("MSLRWEB30K", None, 0, 0, False, False), presort=False)


def test_query_over_the_list_limit_is_an_error(tmp_path):
    p = tmp_path / "long.txt"
    p.write_bytes(b"".join(b"1 qid:9 1:%d\n" % i for i in range(_lib.MAX_LIST_LEN + 1)))
    with pytest.raises(_lib.B200LibraryError, match="PTRB200_MAX_LIST_LEN"):
        read_letor(str(p), _dd("MSLRWEB30K", None, 0, 0, False, False), presort=False)


@pytest.mark.parametrize("dtype", (torch.float32, torch.bfloat16))
def test_batches_from_split_equal_host_batches(files, dtype):
    path, data_id = files["mq2008"]
    sp = read_letor(path, _dd(data_id, "StandardScaler", 0, 0, False, False), presort=True, seed=1, feature_dtype=torch.float32)
    spd = read_letor(path, _dd(data_id, "StandardScaler", 0, 0, False, False), presort=True, seed=1, feature_dtype=dtype)
    host = [(q, X.cpu().numpy(), y.cpu().numpy()) for q, X, y in (sp.query(b) for b in range(len(sp)))]
    for a, b in ((RaggedBatches(host, docs_per_batch=12, presort=False, feature_dtype=dtype, shuffle_seed=4),
                  RaggedBatches.from_split(spd, docs_per_batch=12, shuffle_seed=4)),
                 (LengthBucketedBatches(host, docs_per_batch=12, presort=False, feature_dtype=dtype, shuffle_seed=4),
                  LengthBucketedBatches.from_split(spd, docs_per_batch=12, shuffle_seed=4))):
        ba, bb = list(a), list(b)
        assert len(ba) == len(bb) > 1
        for x, z in zip(ba, bb):
            assert x[0] == z[0]
            assert z[1].is_cuda and z[1].dtype == dtype
            for u, v in zip(x[1:], z[1:]):
                if isinstance(u, torch.Tensor):
                    assert torch.equal(u, v.cpu())
                else:
                    assert u == v


def test_ltrdataset_drop_in(gold, files):
    path, data_id = files["mslr"]
    dd = _dd(data_id, None, 0, 0, False, False)
    ds = LTRDataset(split_type=None, file=path, data_dict=dd, presort=False)
    key = f"mslr/{_name(None, 0, 0, False, False, False)}"
    assert len(ds) == len(gold[key + "/qids"])
    # the LETORSampler contract: iterate (qid, X, y), then collate same-length queries with the default collate
    lens = {}
    for i, (qid, X, y) in enumerate(ds):
        assert X.is_cuda and X.shape[0] == y.shape[0]
        lens.setdefault(y.shape[0], []).append(i)
    loader = torch.utils.data.DataLoader(ds, batch_sampler=list(lens.values()), num_workers=0)
    seen = 0
    for qids, X, y in loader:
        assert X.is_cuda and X.dim() == 3
        seen += len(qids)
    assert seen == len(ds)
    Xall = torch.cat([ds[i][1] for i in range(len(ds))]).cpu().numpy()
    assert np.array_equal(Xall.view(np.int32), gold[key + "/X"].view(np.int32))
    with pytest.raises(NotImplementedError):
        LTRDataset(split_type=None, file=path, data_dict=dd, hot=True)
