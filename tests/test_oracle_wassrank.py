"""Pin the two WassRank restatements of tests/wassrank_oracle.py -- the K-matrix ATen port and the float64
log-domain form -- against outputs of the unmodified reference (tests/golden/wassrank.npz, made by
tests/golden/make_golden_wassrank.py), and check the drop-in class's settings and registration without a GPU."""
import types

import numpy as np
import pytest
import torch

from tests import wassrank_oracle as wo
from tests.helpers import load, rel_err

COSTS = ["p1", "p2", "eg", "dg", "ddg"]


def wass_cases():
    """tests/golden/wassrank.npz -> sorted list of (case, dict)."""
    z = load("wassrank.npz")
    groups = {}
    for k in z.files:
        case, field = k.split("__")
        groups.setdefault(case, {})[field] = z[k]
    return sorted(groups.items())


def wass_params(d):
    return dict(cost_type=COSTS[int(d["cost"])], lam=float(d["lam"]), sh_itr=int(d["sh_itr"]))


CASES = wass_cases()
IDS = [c for c, _ in CASES]


def test_fixture_covers_the_grid():
    names = set(IDS)
    for cost in COSTS:
        for n in (1, 2, 8, 50, 256, 1024):
            for tag in ("sig", "wide"):
                for lam, it in ((0.1, 20), (1.0, 5)):
                    assert f"{cost}_lam{lam}_it{it}_n{n}_{tag}" in names
        assert f"{cost}_lam0.1_it20_n50_unsorted" in names and f"{cost}_lam0.1_it20_n64_real" in names
    # the reference's fp32 breakdown is part of what the fixtures record
    assert any(not np.isfinite(float(d["loss"])) for _, d in CASES)


@pytest.mark.parametrize("case,d", CASES, ids=IDS)
def test_port_matches_reference(case, d):
    loss, grad = wo.port_loss_and_grad(torch.from_numpy(d["scores"]), torch.from_numpy(d["labels"]), **wass_params(d))
    loss, grad = float(loss), grad.numpy()
    want, want_g = float(d["loss"]), d["grad"]
    assert np.isnan(loss) == np.isnan(want)
    assert np.array_equal(np.isnan(grad), np.isnan(want_g))
    if np.isfinite(want):
        assert abs(loss - want) <= 1e-6 * max(abs(want), 1e-30)
    ok = ~np.isnan(want_g)
    if ok.any():
        assert np.abs(grad[ok] - want_g[ok]).max() <= 1e-6 * max(np.abs(want_g[ok]).max(), 1e-30)


@pytest.mark.parametrize("case,d", [(c, d) for c, d in CASES if "loss64" in d], ids=[c for c, d in CASES if "loss64" in d])
def test_closed_form_matches_float64_reference(case, d):
    loss, grad = wo.closed_form(d["scores"], d["labels"], **wass_params(d))
    assert np.isfinite(loss) and np.isfinite(grad).all()
    want, want_g = float(d["loss64"]), d["grad64"]
    if np.isfinite(want):
        assert abs(loss - want) <= 1e-9 * max(abs(want), 1e-30), (loss, want)
    if np.isfinite(want_g).all():
        assert rel_err(grad, want_g) <= 1e-9 or np.abs(grad - want_g).max() <= 1e-15


P_CASES = [(c, d) for c, d in CASES if COSTS[int(d["cost"])] in ("p1", "p2") and float(d["lam"]) == 1.0]


@pytest.mark.parametrize("case,d", P_CASES, ids=[c for c, _ in P_CASES])
def test_closed_form_matches_fp32_reference_p1_p2(case, d):
    """p1 / p2 have fp32 runs only; at lam = 1 the fp32 reference is accurate enough to pin the float64 form."""
    loss, grad = wo.closed_form(d["scores"], d["labels"], **wass_params(d))
    want, want_g = float(d["loss"]), d["grad"]
    assert abs(loss - want) <= 1e-5 * max(abs(want), 1e-30)
    assert np.abs(grad - want_g).max() <= 1e-5 * max(np.abs(want_g).max(), 1e-30) + 1e-12


def test_closed_form_is_finite_where_the_reference_is_not():
    bad = [(c, d) for c, d in CASES if not np.isfinite(float(d["loss"]))]
    assert bad
    for _, d in bad:
        loss, grad = wo.closed_form(d["scores"], d["labels"], **wass_params(d))
        assert np.isfinite(loss) and np.isfinite(grad).all()


def _sf():
    return dict(sf_id="pointsf", opt="Adam", lr=1e-4, pointsf=dict(num_features=4))


@pytest.mark.parametrize("over,word", [(dict(mode="EntropicOT"), "EntropicOT"), (dict(smooth_type="NG"), "NG"),
                                       (dict(cost_type="Group"), "Group")])
def test_constructor_rejects_unsupported_settings(over, word):
    """Settings are checked before the device: the error names the setting even without a GPU."""
    import ptranking_b200
    para = dict(model_id="WassRank", mode="SinkhornOT", sh_itr=20, lam=0.1, smooth_type="ST", norm_type="BothST",
                cost_type="eg", non_rele_gap=100, var_penalty=np.e, gain_base=4)
    para.update(over)
    with pytest.raises(NotImplementedError, match=word):
        ptranking_b200.WassRank(sf_para_dict=_sf(), wass_para_dict=para, dict_cost_mats={}, dict_std_dists={},
                                gpu=False, device="cpu")


def test_constructor_without_cuda_is_refused():
    import ptranking_b200
    with pytest.raises(RuntimeError):
        ptranking_b200.WassRank(sf_para_dict=_sf(), wass_para_dict=None, dict_cost_mats=None, dict_std_dists=None,
                                gpu=False, device="cpu")


def test_install_registers_wassrank():
    import ptranking_b200
    stand_in = types.ModuleType("stand_in_ltr")
    prev = ptranking_b200.install(module=stand_in)
    assert stand_in.WassRank is ptranking_b200.WassRank and prev["WassRank"] is None
    assert ptranking_b200.MODELS["WassRank"] is ptranking_b200.WassRank
