"""Pin the two MDPRank restatements of tests/mdprank_oracle.py -- the ATen port and the float64 closed form -- against
outputs of the unmodified reference (tests/golden/mdprank.npz, made by tests/golden/make_golden_mdprank.py), and check
the drop-in class's settings and registration without a GPU."""
import types

import numpy as np
import pytest
import torch

from tests import mdprank_oracle as mo
from tests.helpers import load, rel_err


def mdp_cases():
    """tests/golden/mdprank.npz -> sorted list of (case, dict) with the list's scores and labels merged in."""
    z = load("mdprank.npz")
    groups = {}
    for k in z.files:
        case, field = k.split("__")
        groups.setdefault(case, {})[field] = z[k]
    lists = {c: d for c, d in groups.items() if "loss" not in d}
    out = []
    for case, d in sorted(groups.items()):
        if "loss" in d:
            d.update(lists["_".join(case.split("_")[4:])])
            d["perm"] = d["perm"].astype(np.int64)
            out.append((case, d))
    return out


def mdp_params(case):
    """'STPL_k10_g0.9_T0.5_n50_sig' -> dict(distribution, top_k, gamma, temperature)."""
    dist, k, g, T = case.split("_")[:4]
    return dict(distribution=dist, top_k=None if k == "kNone" else int(k[1:]), gamma=float(g[1:]), temperature=float(T[1:]))


CASES = mdp_cases()
IDS = [c for c, _ in CASES]


def draws(case, d):
    """The reference's draw as the port and the kernel take it: the PL ordering or the STPL uniforms."""
    return dict(perm=d["perm"]) if case.startswith("PL_") else dict(unif=d["unif"])


def test_fixture_covers_the_grid():
    names = set(IDS)
    for dist in ("PL", "STPL"):
        for n in (1, 2, 8, 50, 256, 1024):
            for tag in ("sig", "wide"):
                for k in (None, 1, 10):
                    for g in (1.0, 0.9):
                        for T in (1.0, 0.5, 0.1):
                            assert (f"{dist}_k{k}_g{g}_T{T}_n{n}_{tag}" in names) == (k is None or k <= n)


@pytest.mark.parametrize("case,d", CASES, ids=IDS)
def test_port_matches_reference(case, d):
    p = mdp_params(case)
    dr = {k: torch.from_numpy(v) for k, v in draws(case, d).items()}
    loss, grad, order = mo.port_loss_and_grad(torch.from_numpy(d["scores"]), torch.from_numpy(d["labels"]), **p, **dr)
    assert np.array_equal(order.numpy(), d["perm"])
    want, want_g = float(d["loss"]), d["grad"]
    assert np.isnan(float(loss)) == np.isnan(want)
    if np.isfinite(want):
        assert abs(float(loss) - want) <= 1e-6 * max(abs(want), 1e-30)
    grad = grad.numpy()
    ok = np.isfinite(want_g)
    assert np.array_equal(np.isnan(grad), np.isnan(want_g)) and np.array_equal(np.isinf(grad), np.isinf(want_g))
    if ok.any():
        assert np.abs(grad[ok] - want_g[ok]).max() <= 1e-6 * max(np.abs(want_g[ok]).max(), 1e-30)


def fp32_tolerances(n, loss_scale, grad_scale):
    """What fp32 rounding allows between the reference and float64: a relative 2e-5 plus the rounding of the action
    values (one ulp of the largest |a|, carried by each term of the loss) and of the length-n sums behind each gradient
    entry."""
    tol_l = 2e-5 + 2.0 ** -22 * loss_scale
    tol_g = (2e-5 + 2.0 * n * 2.0 ** -24) * grad_scale
    return tol_l, tol_g


@pytest.mark.parametrize("case,d", CASES, ids=IDS)
def test_closed_form_matches_reference(case, d):
    p = mdp_params(case)
    loss, grad, ls, gs = mo.closed_form(d["scores"], d["labels"], d["perm"], unif=d.get("unif"), with_scales=True, **p)
    assert np.isfinite(loss) and np.isfinite(grad).all()
    want, want_g = float(d["loss"]), d["grad"]
    tol_l, tol_g = fp32_tolerances(want_g.size, ls, gs)
    if np.isfinite(want):
        assert abs(loss - want) <= tol_l * max(abs(want), 1.0), (loss, want)
    ok = np.isfinite(want_g)
    if ok.any():
        assert np.abs(grad[ok] - want_g[ok]).max() <= tol_g, (np.abs(grad[ok] - want_g[ok]).max(), tol_g)


def test_reference_breakdowns_are_recorded():
    """Where exp(a - max a) underflows in fp32 (STPL at T = 0.1 on widely spread scores), the reference takes the log of
    a zero tail sum: 0 * inf = NaN in the gradient of every document from that position on, or a NaN loss when the zero
    sum lies inside the top-k window; a denormal sum instead overflows its reciprocal to an infinite gradient.  The
    fixtures record all three; the closed form (like the kernel) is finite on every case."""
    nan_loss = [d for _, d in CASES if np.isnan(float(d["loss"]))]
    broken = [(c, d) for c, d in CASES if not np.isfinite(d["grad"]).all()]
    assert nan_loss and len(broken) > len(nan_loss) and any(np.isinf(d["grad"]).any() for _, d in CASES)
    for case, d in broken:
        loss, grad = mo.closed_form(d["scores"], d["labels"], d["perm"], unif=d.get("unif"), **mdp_params(case))
        assert np.isfinite(loss) and np.isfinite(grad).all()


@pytest.mark.parametrize("case,d", [(c, d) for c, d in CASES if c.startswith("STPL_")],
                         ids=[c for c in IDS if c.startswith("STPL_")])
def test_stpl_order_follows_from_the_uniforms(case, d):
    order, z = mo.stpl_order(d["scores"], d["unif"], mdp_params(case)["temperature"])
    assert np.array_equal(order, d["perm"])


def test_gradient_sums_to_zero():
    """The loss depends on differences of the action values only."""
    rng = np.random.default_rng(0)
    s = rng.standard_normal((3, 40)); y = rng.integers(0, 5, (3, 40)).astype(np.float64)
    order = np.stack([rng.permutation(40) for _ in range(3)])
    for top_k, gamma in ((None, 1.0), (7, 0.9), (100, 0.5)):
        _, g = mo.closed_form(s, y, order, top_k=top_k, gamma=gamma)
        assert np.abs(g.sum(1)).max() <= 1e-12 * np.abs(g).max()


def _sf():
    return dict(sf_id="pointsf", opt="Adam", lr=1e-4, pointsf=dict(num_features=4))


def _para(**over):
    p = dict(model_id="MDPRank", temperature=1.0, gamma=1.0, top_k=10, distribution="PL")
    p.update(over)
    return p


def test_constructor_rejects_unknown_distribution():
    """The distribution is checked before the device: the error names it even without a GPU."""
    import ptranking_b200
    with pytest.raises(NotImplementedError, match="Gumbel"):
        ptranking_b200.MDPRank(sf_para_dict=_sf(), model_para_dict=_para(distribution="Gumbel"), gpu=False, device="cpu")


def test_constructor_without_cuda_is_refused():
    import ptranking_b200
    for dist in ("PL", "STPL"):
        with pytest.raises(RuntimeError):
            ptranking_b200.MDPRank(sf_para_dict=_sf(), model_para_dict=_para(distribution=dist), gpu=False, device="cpu")


def test_install_registers_mdprank_and_its_parameter_class():
    import ptranking_b200
    stand_in = types.ModuleType("stand_in_ltr")
    prev = ptranking_b200.install(module=stand_in)
    assert stand_in.MDPRank is ptranking_b200.MDPRank and prev["MDPRank"] is None
    assert ptranking_b200.MODELS["MDPRank"] is ptranking_b200.MDPRank
    try:
        from ptranking.ltr_adhoc.listwise.mdprank import MDPRankParameter
    except ImportError:
        assert not hasattr(stand_in, "MDPRankParameter") and "MDPRankParameter" not in prev
    else:
        assert stand_in.MDPRankParameter is MDPRankParameter and prev["MDPRankParameter"] is None
    # a module that already has the parameter class keeps it
    own = types.ModuleType("stand_in_ltr_2")
    own.MDPRankParameter = object
    prev = ptranking_b200.install(module=own)
    assert own.MDPRankParameter is object and "MDPRankParameter" not in prev


def test_install_supplies_the_reference_parameter_class(monkeypatch):
    """With a module standing in for the reference's mdprank.py importable, install() takes its MDPRankParameter."""
    import sys
    import ptranking_b200
    fake = types.ModuleType("ptranking.ltr_adhoc.listwise.mdprank")
    fake.MDPRankParameter = type("MDPRankParameter", (), {})
    for name in ("ptranking", "ptranking.ltr_adhoc", "ptranking.ltr_adhoc.listwise"):
        if name not in sys.modules:
            monkeypatch.setitem(sys.modules, name, types.ModuleType(name))
    monkeypatch.setitem(sys.modules, "ptranking.ltr_adhoc.listwise.mdprank", fake)
    monkeypatch.setattr(sys.modules["ptranking.ltr_adhoc.listwise"], "mdprank", fake, raising=False)
    stand_in = types.ModuleType("stand_in_ltr")
    prev = ptranking_b200.install(module=stand_in)
    assert stand_in.MDPRankParameter is fake.MDPRankParameter and prev["MDPRankParameter"] is None
