"""One training epoch fed from a device LetorSplit equals, bit for bit, the same epoch fed from host arrays in the same
order: RaggedBatches.from_split hands the ranker the values, batches and order that RaggedBatches builds on the host."""
import numpy as np
import pytest
import torch

import ptranking_b200
from ptranking_b200 import LABEL_TYPE, ops
from ptranking_b200.data import RaggedBatches
from ptranking_b200.letor import read_letor

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F = 46


@pytest.fixture(scope="module")
def split(tmp_path_factory):
    rng = np.random.default_rng(31)
    lines = []
    for q in range(60):
        n = int(rng.integers(5, 41))
        lab = rng.choice(5, n, p=[.5, .3, .12, .05, .03])
        lab[0] = max(lab[0], 1)
        for i in range(n):
            vals = np.round(rng.standard_normal(F) * 10 ** rng.integers(0, 3, F), 6)
            lines.append(f"{lab[i]} qid:{q + 1} " + " ".join(f"{j + 1}:{v:g}" for j, v in enumerate(vals)))
    p = tmp_path_factory.mktemp("letor_train") / "train.txt"
    p.write_text("\n".join(lines) + "\n")
    dd = dict(data_id="MSLRWEB30K", scale_data=True, scaler_id="StandardScaler", scaler_level="QUERY",
              min_docs=1, min_rele=1, binary_rele=False, unknown_as_zero=False)
    return read_letor(str(p), dd, presort=True, seed=2)


def _epoch(model, sf, paras, loader):
    torch.manual_seed(5)
    ops._tie_offset, ops._dropout_offset = 0, 0          # same dropout and tie streams in both runs
    cls = getattr(ptranking_b200, model)
    r = cls(sf_para_dict=sf, model_para_dict=paras, gpu=True, device=DEV)
    r.init()
    loss, stop = r.train(loader, epoch_k=1, presort=True, label_type=LABEL_TYPE.MultiLabel)
    torch.cuda.synchronize()
    assert not stop
    return float(loss), [p.detach().cpu().clone() for p in r.get_parameters()]


POINT = dict(sf_id="pointsf", opt="Adam", lr=1e-3,
             pointsf=dict(num_features=F, num_layers=3, AF="GE", TL_AF="S", apply_tl_af=True, BN=True, bn_type="BN",
                          bn_affine=True, dropout=0.1))
LIST = dict(sf_id="listsf", opt="Adagrad", lr=1e-3,
            listsf=dict(num_features=F, ff_dims=[32, 32, 16], AF="R", TL_AF="GE", apply_tl_af=False, BN=False,
                        bn_type="BN2", bn_affine=False, n_heads=2, encoder_layers=2, encoder_type="DASALC", dropout=0.1))


@pytest.mark.parametrize("model,sf,paras", [
    ("LambdaRank", POINT, dict(model_id="LambdaRank", sigma=1.0)),
    ("ApproxNDCG", LIST, dict(model_id="ApproxNDCG", alpha=10.0)),
])
def test_epoch_from_split_equals_epoch_from_host_arrays(split, model, sf, paras):
    host = [(q, X.cpu().numpy(), y.cpu().numpy()) for q, X, y in (split.query(b) for b in range(len(split)))]
    kw = dict(docs_per_batch=300, bucket_edges=(16, 32))
    from_host = RaggedBatches(host, presort=False, pin_memory=True, **kw)
    from_split = RaggedBatches.from_split(split, **kw)
    assert len(from_host) == len(from_split) > 1
    loss_h, params_h = _epoch(model, sf, paras, from_host)
    loss_d, params_d = _epoch(model, sf, paras, from_split)
    assert np.isfinite(loss_h)
    assert loss_d == loss_h
    for a, b in zip(params_d, params_h):
        assert torch.equal(a, b)
    assert any(not torch.equal(a, b) for a, b in zip(params_h, _epoch_init(model, sf, paras)))    # the epoch trained


def _epoch_init(model, sf, paras):
    torch.manual_seed(5)
    r = getattr(ptranking_b200, model)(sf_para_dict=sf, model_para_dict=paras, gpu=True, device=DEV)
    r.init()
    return [p.detach().cpu().clone() for p in r.get_parameters()]
