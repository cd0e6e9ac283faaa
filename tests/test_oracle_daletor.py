"""Pin the two restatements of the diversification path in tests/daletor_oracle.py -- the ATen port and the float64
closed form -- against outputs of the unmodified reference (tests/golden/daletor.npz, made by
tests/golden/make_golden_daletor.py), and check the drop-in classes' settings and registration without a GPU."""
import types

import numpy as np
import pytest
import torch

from tests import daletor_oracle as do
from tests.helpers import load

KS = [1, 3, 5, 10, 20]


def _groups(prefix):
    z = load("daletor.npz")
    out = {}
    for k in z.files:
        if k.startswith(prefix):
            case, field = k[len(prefix):].split("__")
            out.setdefault(case, {})[field] = z[k]
    return out


def loss_cases():
    """-> sorted [(case, dict(scores, rele, loss, grad, rt, top_k))]."""
    lists = _groups("list_")
    out = []
    for case, d in sorted(_groups("loss_").items()):
        n, m, k, rt, tag = case.split("_")
        src = lists[f"{n}_{m}"]
        out.append((case, dict(scores=src["scores"], rele=src["rele_" + tag], loss=float(d["loss"]), grad=d["grad"],
                               rt=float(rt[2:]), top_k=None if k == "kNone" else int(k[1:]))))
    return out


def metric_cases():
    return sorted(_groups("met_").items())


LOSS = loss_cases()
METRICS = metric_cases()


def scale(d):
    return max(float(np.abs(d["grad"]).max()), abs(d["loss"]), 1.0)


def test_fixture_covers_the_grid():
    names = {c for c, _ in LOSS}
    for n in (1, 2, 7, 50, 300):
        for m in (1, 3, 8, 20):
            for k in (None, 1, 2, 10):
                for rt in (1, 10, 50):
                    assert f"n{n}_m{m}_k{k}_rt{rt}_bin" in names
                assert f"n{n}_m{m}_k{k}_rt10_flt" in names
    assert len(METRICS) == 7
    # rows without relevance, and a list shorter than max(ks)
    assert any((d["rele"].sum(axis=1) == 0).any() for _, d in LOSS)
    assert any(d["scores"].shape[1] < max(KS) for _, d in METRICS)


def test_top_k_slices_subtopic_rows():
    """The reference's top_k keeps the first top_k rows of R, not the first top_k documents (daletor.py:30-35)."""
    by = dict(LOSS)
    d7 = by["n7_m3_k1_rt10_bin"]
    R = d7["rele"]
    row0, _ = do.closed_form(d7["scores"], R[:1], 10.0, None)
    assert abs(d7["loss"] - row0) <= 1e-6 * max(1.0, abs(row0))
    full = by["n7_m3_kNone_rt10_bin"]["loss"]
    assert by["n7_m3_k10_rt10_bin"]["loss"] == full


@pytest.mark.parametrize("case,d", LOSS, ids=[c for c, _ in LOSS])
def test_port_matches_reference(case, d):
    loss, grad = do.port_loss_and_grad(d["scores"], d["rele"], d["rt"], d["top_k"])
    assert loss == pytest.approx(d["loss"], rel=1e-6, abs=1e-6)
    assert np.abs(grad - d["grad"][0]).max() <= 1e-6 * scale(d)


@pytest.mark.parametrize("case,d", LOSS, ids=[c for c, _ in LOSS])
def test_closed_form_matches_reference(case, d):
    loss, grad = do.closed_form(d["scores"], d["rele"], d["rt"], d["top_k"])
    assert abs(loss - d["loss"]) <= 2e-6 * max(1.0, abs(d["loss"]))
    assert np.abs(grad - d["grad"][0]).max() <= 2e-6 * scale(d)


@pytest.mark.parametrize("case,d", METRICS, ids=[c for c, _ in METRICS])
def test_metric_restatements_match_reference(case, d):
    s, R, ml = d["scores"], d["rele"], float(d["max_label"])
    n = s.shape[1]
    # the reference's alpha-nDCG@ks for a list shorter than max(ks) is an [m, len(ks)] matrix of identical rows
    want_a = np.atleast_2d(d["andcg_ks"])
    assert (want_a == want_a[0]).all()
    for fn, tol in ((do.port_metrics, 1e-6), (do.closed_form_metrics, 1e-6)):
        a, e, ne, order = fn(s, R, KS, ml)
        assert np.array_equal(np.asarray(order), d["order"])
        assert np.abs(a - want_a[0]).max() <= tol
        assert np.abs(e - d["err_ia_ks"]).max() <= tol
        assert np.abs(ne - d["nerr_ia_ks"]).max() <= tol
        if n >= 5:
            c = KS.index(5)
            assert abs(a[c] - float(d["andcg_k5"])) <= tol
            assert abs(e[c] - float(d["err_ia_k5"])) <= tol
            assert abs(ne[c] - float(d["nerr_ia_k5"])) <= tol


def test_srd_metric_zero_beyond_the_list():
    """Cutoffs beyond a list's length give 0 for all three metrics (one vector per query, DESIGN §2)."""
    d = dict(METRICS)["n3_m5"]
    for fn in (do.port_metrics, do.closed_form_metrics):
        a, e, ne, _ = fn(d["scores"], d["rele"], KS, 1.0)
        assert (a[2:] == 0).all() and (e[2:] == 0).all() and (ne[2:] == 0).all()      # ks 5, 10, 20 > n = 3
        assert a[1] > 0


def _sf(F=4, **over):
    d = dict(num_features=F, num_layers=5, AF="GE", TL_AF="GE", apply_tl_af=False, BN=True, bn_type="BN",
             bn_affine=True, dropout=0.0)
    d.update(over)
    return dict(sf_id="pointsf", opt="Adagrad", lr=0.001, pointsf=d)


def test_daletor_settings_and_cuda_only():
    from ptranking_b200 import DALETOR
    with pytest.raises(RuntimeError):
        DALETOR(sf_para_dict=_sf(), model_para_dict=dict(model_id="DALETOR", rt=10.0, top_k=10), gpu=False, device="cpu")
    with pytest.raises(NotImplementedError, match="list scorer"):
        DALETOR(sf_para_dict=dict(sf_id="listsf", opt="Adagrad", lr=0.01, listsf={}),
                model_para_dict=dict(model_id="DALETOR", rt=10.0, top_k=10), gpu=True, device="cuda:0")
    sf = _sf(F=100)
    r = DALETOR(sf_para_dict=sf, model_para_dict=dict(model_id="DALETOR", rt=50.0, top_k=None), gpu=True,
                device="cuda:0")
    assert (r.rt, r.top_k, r.id, r.queries_per_step) == (50.0, None, "DALETOR", 1)
    assert sf["pointsf"]["num_features"] == 300            # [q, q*d, d], as the reference widens it


def test_per_query_bn_keeps_checkpoint_keys():
    """The per-query BN scorer has the reference's state_dict keys (LTRBatchNorm's bn.weight / bn.bias)."""
    from ptranking_b200.base.utils import StackedFFNet, get_stacked_FFNet
    dims = [12, 8, 8, 1]
    for affine in (True, False):
        a = StackedFFNet(dims, AF="GE", BN=True, bn_type="BN", bn_affine=affine, bn_per_query=True)
        b = get_stacked_FFNet(dims, AF="GE", BN=True, bn_type="BN", bn_affine=affine)
        assert list(a.state_dict()) == list(b.state_dict())
        assert a.spec.norm == "BN2" and not a.spec.norm_affine
        ps = a.ordered_parameters()
        assert len(ps) == 3 * 2 + 2 * 2
        if affine:
            assert ps[2] is a.bn_2.bn.weight and ps[3] is a.bn_2.bn.bias
        else:
            assert torch.equal(ps[2], torch.ones(8)) and torch.equal(ps[3], torch.zeros(8))
    with pytest.raises(ValueError):
        StackedFFNet(dims, AF="GE", BN=True, bn_type="BN2", bn_per_query=True)


def test_install_diversification_registers_daletor():
    import ptranking_b200
    mod = types.ModuleType("fake_ltr_diversification")
    mod.DALETOR = object
    prev = ptranking_b200.install_diversification(mod)
    assert mod.DALETOR is ptranking_b200.DALETOR and prev == {"DALETOR": object}
    assert "DALETOR" not in ptranking_b200.MODELS           # install() of the ad-hoc driver is unchanged


def test_install_diversification_into_the_reference_driver():
    ref = pytest.importorskip("ptranking.ltr_diversification.eval.ltr_diversification")
    import ptranking_b200
    prev = ptranking_b200.install_diversification()
    try:
        assert ref.DALETOR is ptranking_b200.DALETOR
    finally:
        ref.DALETOR = prev["DALETOR"]
