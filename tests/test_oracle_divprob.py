"""CPU checks of DivProbRanker's oracle and class: the fp32 ATen port against the unmodified reference's fixtures
(tests/golden/divprob.npz), the float64 closed form against float64 autograd, the construction-time refusals and the
DiversityNeuralRanker hooks' defaults."""
import os

import numpy as np
import pytest
import torch

from tests import divprob_oracle as dpo

pytestmark = pytest.mark.filterwarnings("ignore")
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "divprob.npz"))


def _parse(name):
    """'loss_<i>_<loss>_k<top_k>_<norm|raw>_<bin|flt>' -> dict of the case."""
    _, i, loss, k, norm, tag = name.split("_")
    n, m, K, ld = GOLD[f"list_{i}__meta"]
    pair = loss in ("PairCLS", "LambdaPairCLS")
    return dict(loss=loss, top_k=None if k == "kNone" else int(k[1:]), norm=norm == "norm", K=int(K),
                limit_delta=None if ld == 0 else float(ld), raw=GOLD[f"list_{i}__raw_{'pair' if pair else 'free'}"],
                rele=GOLD[f"list_{i}__rele_{tag}"], ref_loss=float(GOLD[name + "__loss"]), ref_grad=GOLD[name + "__grad"])


LOSS = sorted({k[:-len("__loss")] for k in GOLD.files if k.startswith("loss_") and k.endswith("__loss")})
CASES = [(c, _parse(c)) for c in LOSS]
KEYS = sorted({k.split("__")[0] for k in GOLD.files if k.startswith("key_")})


def _kw(d):
    return dict(K=d["K"], limit_delta=d["limit_delta"], top_k=d["top_k"], norm=d["norm"])


def test_fixture_coverage():
    losses = {d["loss"] for _, d in CASES}
    assert losses == set(dpo.LOSSES)
    assert {(d["K"], d["limit_delta"]) for _, d in CASES} == {(1, None), (5, None), (1, 0.01), (5, 0.1), (1, 0.1), (5, 0.01)}
    assert {d["top_k"] for _, d in CASES if d["loss"] == "aNDCG"} == {None, 1, 10}
    assert {d["norm"] for _, d in CASES if d["loss"] == "LambdaPairCLS"} == {True, False}
    assert {d["raw"].shape[0] for _, d in CASES} == {1, 2, 7, 50, 300}
    assert {d["rele"].shape[0] for _, d in CASES} == {1, 3, 8, 32}


@pytest.mark.parametrize("case,d", CASES, ids=[c for c, _ in CASES])
def test_port_matches_reference_fixture(case, d):
    L, g = dpo.port_loss_and_grad(d["raw"], d["rele"], d["loss"], **_kw(d))
    if np.isnan(d["ref_loss"]):      # LambdaPairCLS with norm on a query without relevance: 0 / 0 in the reference
        assert np.isnan(L)
        return
    assert abs(L - d["ref_loss"]) <= 1e-5 * max(1.0, abs(d["ref_loss"]))
    sc = max(float(np.abs(d["ref_grad"]).max()), 1.0)
    assert float(np.abs(g - d["ref_grad"]).max()) <= 1e-5 * sc


@pytest.mark.parametrize("key", KEYS)
def test_port_sort_keys_match_reference_fixture(key):
    _, _, K, ld = GOLD[key + "__meta"]
    for sort_id in ("ExpRele", "RERAR", "RiskAware"):
        got = dpo.port_sort_key(GOLD[key + "__raw"], sort_id, int(K), None if ld == 0 else float(ld))
        np.testing.assert_allclose(got, GOLD[f"{key}__{sort_id}"], rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("loss", dpo.LOSSES)
@pytest.mark.parametrize("K,limit_delta", [(1, None), (1, 0.1), (5, None), (5, 0.01)])
@pytest.mark.parametrize("top_k", [None, 1, 3])
def test_closed_form_matches_float64_autograd(loss, K, limit_delta, top_k):
    rng = np.random.default_rng([K, top_k or 0, dpo.LOSSES.index(loss)])
    for n, m, pair_safe in ((1, 2, False), (6, 3, False), (9, 4, True), (13, 1, False)):
        u = dpo.draw_raw(rng, n, K, limit_delta, pair_safe)
        R = (rng.random((m, n)) < 0.4).astype(np.float64) * rng.choice([1.0, 1.6])
        if m >= 3:
            R[1] = 0.0
        for norm in (True, False) if loss == "LambdaPairCLS" else (True,):
            L, g = dpo.closed_form(u, R, loss, K, limit_delta, top_k, norm)
            La, ga = dpo.autograd64(u, R, loss, K, limit_delta, top_k, norm)
            # the port's discounts / 2^r are fp32 constants (torch.arange(dtype=float), torch.tensor([2.0])): 1e-7
            assert abs(L - La) <= 1e-7 * max(1.0, abs(La))
            assert float(np.abs(g - ga).max()) <= 1e-7 * max(1.0, float(np.abs(ga).max()))


def _sf(sf_id="pointsf"):
    if sf_id == "pointsf":
        return dict(sf_id="pointsf", opt="Adagrad", lr=0.01, pointsf=dict(num_features=6, h_dim=8, num_layers=2, AF="R",
                                                                          TL_AF="S", apply_tl_af=False, BN=False,
                                                                          bn_type=None, bn_affine=False, dropout=0.0))
    return dict(sf_id=sf_id, opt="Adagrad", lr=0.01, **{sf_id: dict(num_features=6, encoder_type="AttnDIN", n_heads=2,
                                                                    encoder_layers=1, ff_dims=[8], BN=False)})


def _mp(**kw):
    d = dict(model_id="DivProbRanker", K=1, cluster=False, sort_id="ExpRele", top_k=None, opt_id="SuperSoft",
             limit_delta=0.01, metric="nERR-IA", opt_ideal=True, norm=True)
    d.update(kw)
    return d


@pytest.mark.parametrize("kw,sf_id,word", [
    (dict(opt_id="Portfolio"), "pointsf", "cvxpy"),
    (dict(cluster=True, K=3), "pointsf", "separate scorers"),
    ({}, "listsf_co", "listsf_co"),
    (dict(opt_ideal=False), "pointsf", "opt_ideal"),
    (dict(opt_ideal=False, opt_id="LambdaPairCLS"), "pointsf", "opt_ideal"),
])
def test_refused_configurations(kw, sf_id, word):
    from ptranking_b200 import DivProbRanker
    with pytest.raises(NotImplementedError, match=word):
        DivProbRanker(sf_para_dict=_sf(sf_id), model_para_dict=_mp(**kw), gpu=False, device="cpu")


@pytest.mark.parametrize("sf_id", ["pointsf", "listsf"])
def test_hook_defaults_leave_daletor_unchanged(sf_id):
    """DALETOR keeps the base class's hooks: [q, q*d, d] for pointsf, [q, d, q*d] for listsf, the scores as sort keys
    (rankers need a device to be built, so the hooks are called on a stand-in)."""
    from types import SimpleNamespace
    from ptranking_b200 import DALETOR, DivProbRanker
    assert DALETOR.split_list_order is DALETOR.__mro__[1].split_list_order
    assert DALETOR.split_sort_keys is DALETOR.__mro__[1].split_sort_keys
    me = SimpleNamespace(sf_id=sf_id)
    assert DALETOR.split_list_order(me) is (sf_id == "listsf")
    preds = torch.arange(5.0)
    assert DALETOR.split_sort_keys(me, preds, None) is preds
    assert DivProbRanker.split_list_order(me) is True


def test_registered_for_the_driver():
    import ptranking_b200
    assert ptranking_b200.DIV_MODELS["DivProbRanker"] is ptranking_b200.DivProbRanker

    class Driver:
        pass
    ptranking_b200.install_diversification(Driver)
    assert Driver.DivProbRanker is ptranking_b200.DivProbRanker and Driver.DALETOR is ptranking_b200.DALETOR
