"""Host-side bf16 feature batches of the two loaders (no device needed)."""
import numpy as np
import pytest
import torch

from ptranking_b200 import data


def _queries(nq=40, F=46, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for q in range(nq):
        n = int(rng.integers(1, 90))
        out.append((f"q{q}", rng.standard_normal((n, F)).astype(np.float32) * 3.0, rng.integers(0, 5, n).astype(np.float32)))
    return out


def _rounded(qs):
    """the queries after the loader's presort, features rounded to bf16 by torch"""
    out = {}
    for qid, X, y in qs:
        Xs, ys = data.presort_query(X, y)
        out[qid] = (torch.from_numpy(Xs).to(torch.bfloat16), torch.from_numpy(ys))
    return out


def test_ragged_batches_bf16_features():
    qs = _queries()
    ref = _rounded(qs)
    a = list(data.RaggedBatches(qs, docs_per_batch=500, shuffle_seed=3, pin_memory=False))
    b = list(data.RaggedBatches(qs, docs_per_batch=500, shuffle_seed=3, pin_memory=False, feature_dtype=torch.bfloat16))
    assert len(a) == len(b) > 1
    for (ia, Xa, ya, oa, ma, ba), (ib, Xb, yb, ob, mb, bb) in zip(a, b):
        assert ia == ib and ma == mb and ba == bb
        assert torch.equal(oa, ob) and torch.equal(ya, yb)
        assert Xa.dtype == torch.float32 and Xb.dtype == torch.bfloat16
        assert torch.equal(Xb, Xa.to(torch.bfloat16))
        offs = ob.tolist()
        for k, qid in enumerate(ib):
            assert torch.equal(Xb[offs[k]: offs[k + 1]], ref[qid][0])


def test_length_bucketed_batches_bf16_features():
    qs = _queries(seed=1)
    ref = _rounded(qs)
    a = list(data.LengthBucketedBatches(qs, docs_per_batch=300, pin_memory=False))
    b = list(data.LengthBucketedBatches(qs, docs_per_batch=300, pin_memory=False, feature_dtype=torch.bfloat16))
    assert len(a) == len(b) > 1
    for (ia, Xa, ya), (ib, Xb, yb) in zip(a, b):
        assert ia == ib and torch.equal(ya, yb) and Xb.dtype == torch.bfloat16
        for k, qid in enumerate(ib):
            assert torch.equal(Xb[k], ref[qid][0])


def test_fp32_default_keeps_numpy_storage():
    qs = _queries(nq=3)
    loader = data.RaggedBatches(qs, pin_memory=False)
    assert loader.feature_dtype == torch.float32 and isinstance(loader.queries[0][1], np.ndarray)


@pytest.mark.parametrize("cls", [data.RaggedBatches, data.LengthBucketedBatches])
def test_unsupported_feature_dtype_is_refused(cls):
    with pytest.raises(ValueError):
        cls(_queries(nq=2), pin_memory=False, feature_dtype=torch.float16)
