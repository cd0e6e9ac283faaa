"""GPU parity of the fused MDPRank kernel (ptrb200_mdprank_fwd_bwd): against the unmodified reference's runs
(tests/golden/mdprank.npz) with its draws injected, against the ATen port and the float64 closed form on fresh inputs,
batch and ragged-batch semantics, the distribution of the device's own samples, full-size properties and the drop-in
class's train step."""
import itertools

import numpy as np
import pytest
import torch
from scipy import stats

from tests import mdprank_oracle as mo
from tests.test_oracle_mdprank import CASES, IDS, draws, fp32_tolerances, mdp_params

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-5


def _run(s, y, sample=False, **params):
    """-> (loss, per-query losses, grad, sampled orderings or None) through ops."""
    from ptranking_b200 import ops
    st = torch.as_tensor(np.ascontiguousarray(s, dtype=np.float32)).to(DEV)
    yt = torch.as_tensor(np.ascontiguousarray(y, dtype=np.float32)).to(DEV)
    kw = dict(params)
    for f in ("perm", "unif"):
        if kw.get(f) is not None:
            kw[f] = torch.as_tensor(np.ascontiguousarray(kw[f])).to(DEV)
    if kw.get("offsets") is not None:
        kw["offsets"] = torch.as_tensor(kw["offsets"]).to(DEV)
    out = torch.empty(st.shape, dtype=torch.int32, device=DEV) if sample else None
    loss, lq, g = ops.rank_loss_and_grad("MDPRank", st, yt, sample_out=out, **kw)
    torch.cuda.synchronize()
    return float(loss.cpu()), lq.cpu().numpy(), g.cpu().numpy(), None if out is None else out.cpu().numpy()


def _check(loss, grad, ref_loss, ref_grad, fl, fg, loss_scale, grad_scale):
    """The kernel within TOL of the fp32 reference, or within twice the reference's own distance from float64 where
    that is larger (the sibling tests' rule).  Losses are compared on the scale max(|loss|, 1) and gradients on the size
    of the returns (an entry differences two terms of that size; closed_form's grad scale).  Where the reference broke
    down in fp32 (NaN or inf), the kernel is held to float64 within the fp32 rounding bound the reference meets
    elsewhere (tests/test_oracle_mdprank.py::fp32_tolerances)."""
    assert np.isfinite(loss) and np.isfinite(grad).all()
    n = grad.shape[-1]
    scale = max(np.abs(fg).max(), grad_scale, 1e-30)
    tol_l32, tol_g32 = fp32_tolerances(n, loss_scale, grad_scale)
    if np.isfinite(ref_loss):
        tol_l = max(TOL, 2.0 * abs(ref_loss - fl) / max(abs(fl), 1.0))
        assert abs(loss - ref_loss) <= tol_l * max(abs(ref_loss), 1.0), (loss, ref_loss, fl)
    else:
        assert abs(loss - fl) <= tol_l32 * max(abs(fl), 1.0), (loss, fl)
    ok = np.isfinite(ref_grad)
    tol_g = max(TOL, 2.0 * np.abs(ref_grad[ok] - fg[ok]).max() / scale) if ok.any() else TOL
    assert np.abs(np.where(ok, grad - ref_grad, 0.0)).max() <= tol_g * scale, (np.abs(grad[ok] - ref_grad[ok]).max() / scale, tol_g)
    assert np.abs(np.where(ok, 0.0, grad - fg)).max() <= max(tol_g32, TOL * scale)


def _stpl_order_ok(s, unif, T, order):
    """``order`` is a permutation of each list that takes the fp32 perturbed logits in descending order, up to the
    last-bit difference between the device's logf and the host's log: a few ulps of s and of the Gumbel noise
    (|g| < 17 for 24-bit uniforms), divided by T."""
    _, z = mo.stpl_order(s, unif, T)
    zo = np.take_along_axis(z, order.astype(np.int64), 1)
    assert np.array_equal(np.sort(order, 1), np.tile(np.arange(order.shape[1]), (order.shape[0], 1)))
    assert (np.diff(zo, axis=1) <= 2.0 ** -20 * (np.abs(s).max() + 17.0) / T).all()


@pytest.mark.parametrize("case,d", CASES, ids=IDS)
def test_kernel_matches_reference_fixture(case, d):
    p = mdp_params(case)
    dr = draws(case, d)
    loss, lq, grad, order = _run(d["scores"], d["labels"], sample=True, **p, **dr)
    if case.startswith("PL_"):
        assert np.array_equal(order, d["perm"])
    else:   # the ordering follows from the uniforms
        _stpl_order_ok(d["scores"], d["unif"], p["temperature"], order)
    fl, fg, ls, gs = mo.closed_form(d["scores"], d["labels"], d["perm"], unif=d.get("unif"), with_scales=True, **p)
    if np.array_equal(order, d["perm"]):
        _check(loss, grad, float(d["loss"]), d["grad"], fl, fg, ls, gs)
    else:   # a near-tie of the perturbed logits went the other way on the device: float64 on the device's ordering
        _check_own_order(loss, grad, d["scores"], d["labels"], order, float(d["loss"]), d["grad"], fl, fg, p, d["unif"])
    assert abs(float(lq.sum()) - loss) <= 1e-5 * max(abs(loss), 1.0)


def _check_own_order(loss, grad, s, y, order, ref_loss, ref_grad, fl, fg, p, unif):
    """Against float64 on the kernel's ordering, as close as the fp32 result on its own ordering is to float64 on that."""
    kl, kg, ls, gs = mo.closed_form(s, y, order, unif=unif, with_scales=True, **p)
    scale = max(np.abs(kg).max(), gs, 1e-30)
    tol_l32, tol_g32 = fp32_tolerances(grad.shape[-1], ls, gs)
    tol_l = max(TOL, 2.0 * abs(ref_loss - fl) / max(abs(fl), 1.0)) if np.isfinite(ref_loss) else tol_l32
    ok = np.isfinite(ref_grad)
    tol_g = max(TOL, 2.0 * np.abs(ref_grad[ok] - fg[ok]).max() / scale) if ok.all() else tol_g32 / scale
    assert abs(loss - kl) <= tol_l * max(abs(kl), 1.0), (loss, kl)
    assert np.abs(grad - kg).max() <= tol_g * scale, (np.abs(grad - kg).max() / scale, tol_g)


def _fresh(B, n, seed):
    rng = np.random.default_rng(seed)
    s = (2.5 * rng.standard_normal((B, n)) if seed % 2 else 1.0 / (1.0 + np.exp(-rng.standard_normal((B, n))))).astype(np.float32)
    p = np.array([1940952, 1225770, 504958, 69010, 30435], dtype=np.float64)
    y = -np.sort(-rng.choice(5, size=(B, n), p=p / p.sum()).astype(np.float32), axis=1)
    return s, y


@pytest.mark.parametrize("dist", ["PL", "STPL"])
@pytest.mark.parametrize("T", [1.0, 0.3])
@pytest.mark.parametrize("gamma", [1.0, 0.9])
@pytest.mark.parametrize("top_k", [None, 1, 10, "n+5"])
@pytest.mark.parametrize("n", [1, 2, 33, 50, 256, 1024, 2000, 4096])
def test_kernel_matches_port_and_float64_fresh_inputs(n, top_k, gamma, T, dist):
    """PL: the device draws the ordering itself and reports it; the port and the closed form take that ordering.  STPL:
    the uniforms are injected so that the port can replay them."""
    B = 2 if n <= 1024 else 1
    s, y = _fresh(B, n, seed=n * 7 + (top_k if isinstance(top_k, int) else 3) + int(gamma * 10) + int(T * 10))
    k = n + 5 if top_k == "n+5" else top_k
    p = dict(distribution=dist, top_k=k, gamma=gamma, temperature=T)
    unif = np.random.default_rng(n).random((B, n), dtype=np.float32) if dist == "STPL" else None
    loss, _, grad, order = _run(s, y, sample=True, unif=unif, seed=5, offset=n, **p)
    dr = dict(perm=torch.from_numpy(order)) if dist == "PL" else dict(unif=torch.from_numpy(unif))
    o_loss, o_grad, o_order = mo.port_loss_and_grad(torch.from_numpy(s), torch.from_numpy(y), **p, **dr)
    o_order = o_order.numpy()
    if dist == "STPL":
        _stpl_order_ok(s, unif, T, order)
    fl, fg, ls, gs = mo.closed_form(s, y, o_order, unif=unif, with_scales=True, **p)
    if np.array_equal(o_order, order):
        _check(loss, grad, float(o_loss), o_grad.numpy(), fl, fg, ls, gs)
    else:   # STPL near-ties of the perturbed logits ordered differently by the device's logf and the host's log
        _check_own_order(loss, grad, s, y, order, float(o_loss), o_grad.numpy(), fl, fg, p, unif)


def test_batch_equals_single_queries_bit_for_bit():
    B, n = 5, 100
    s, y = _fresh(B, n, seed=3)
    rng = np.random.default_rng(1)
    perm = np.stack([rng.permutation(n) for _ in range(B)]).astype(np.int32)
    unif = rng.random((B, n), dtype=np.float32)
    for p in (dict(distribution="PL", perm=perm, top_k=10, gamma=0.9, temperature=0.5),
              dict(distribution="STPL", unif=unif, top_k=None, gamma=1.0, temperature=0.3)):
        loss, lq, g, o = _run(s, y, sample=True, **p)
        for b in range(B):
            q = {f: (v[b:b + 1] if f in ("perm", "unif") else v) for f, v in p.items()}
            _, lq1, g1, o1 = _run(s[b:b + 1], y[b:b + 1], sample=True, **q)
            assert lq1[0] == lq[b] and np.array_equal(g1[0], g[b]) and np.array_equal(o1[0], o[b])


def _ragged(lens, seed):
    S, Y = [], []
    for i, n in enumerate(lens):
        s, y = _fresh(1, n, seed=seed + i)
        S.append(s[0]); Y.append(y[0])
    off = np.zeros(len(lens) + 1, dtype=np.int32)
    off[1:] = np.cumsum(lens)
    return np.concatenate(S).astype(np.float32), np.concatenate(Y).astype(np.float32), off


@pytest.mark.parametrize("dist", ["PL", "STPL"])
def test_ragged_batch_matches_per_query(dist):
    lens = [300, 64, 37, 5, 2, 1, 0, 4096, 0, 130, 1024]
    s, y, off = _ragged(lens, seed=11)
    rng = np.random.default_rng(2)
    perm = np.concatenate([rng.permutation(n) for n in lens]).astype(np.int32)
    unif = rng.random(s.shape, dtype=np.float32)
    inj = dict(perm=perm) if dist == "PL" else dict(unif=unif)
    p = dict(distribution=dist, top_k=10, gamma=0.9, temperature=0.5)
    _, lq, g, o = _run(s, y, sample=True, offsets=off, max_len=max(lens), **p, **inj)
    for b, n in enumerate(lens):
        if n == 0:
            assert lq[b] == 0.0
            continue
        sl = slice(off[b], off[b + 1])
        l1, _, g1, o1 = _run(s[sl][None], y[sl][None], sample=True, **p, **{f: v[sl][None] for f, v in inj.items()})
        assert np.array_equal(o[sl], o1[0])
        assert abs(lq[b] - l1) <= 2e-6 * max(abs(l1), 1.0), (b, n)
        assert np.abs(g[sl] - g1[0]).max() <= 2e-6 * max(np.abs(g1).max(), 1e-30), (b, n)


def test_dense_and_ragged_layouts_draw_the_same_noise():
    B, n = 6, 77
    s, y = _fresh(B, n, seed=4)
    off = (np.arange(B + 1) * n).astype(np.int32)
    for dist in ("PL", "STPL"):
        p = dict(distribution=dist, top_k=10, temperature=0.7, seed=9, offset=4)
        _, lq, g, o = _run(s, y, sample=True, **p)
        _, lqr, gr, orr = _run(s.reshape(-1), y.reshape(-1), sample=True, offsets=off, max_len=n, **p)
        assert np.array_equal(lq, lqr) and np.array_equal(g.reshape(-1), gr) and np.array_equal(o.reshape(-1), orr)


def test_argument_checks():
    from ptranking_b200 import ops, _lib
    lib = _lib.load()
    st = torch.zeros(2, 4097, device=DEV)
    g, lq = torch.empty_like(st), torch.empty(2, device=DEV)
    stream = torch.cuda.current_stream().cuda_stream
    args = lambda perm, n, T, dist: (st.data_ptr(), st.data_ptr(), None, perm, None, None, g.data_ptr(), lq.data_ptr(), 2, n,
                                     10, 1.0, T, dist, 1, 1, stream)
    assert lib.ptrb200_mdprank_fwd_bwd(*args(None, 4097, 1.0, 0)) == -2          # PTRB200_ERR_UNSUPPORTED
    assert lib.ptrb200_mdprank_fwd_bwd(*args(None, 64, 0.0, 0)) == -1           # temperature <= 0
    assert lib.ptrb200_mdprank_fwd_bwd(*args(None, 64, 1.0, 2)) == -1           # unknown distribution
    pm = torch.zeros(2, 64, dtype=torch.int32, device=DEV)
    assert lib.ptrb200_mdprank_fwd_bwd(*args(pm.data_ptr(), 64, 1.0, 1)) == -1  # an injected ordering under STPL
    torch.cuda.synchronize()
    with pytest.raises(ValueError):
        ops.rank_loss_and_grad("MDPRank", st[:, :8], st[:, :8], distribution="Gumbel")


@pytest.mark.parametrize("dist", ["PL", "STPL"])
def test_sampler_distribution(dist):
    """2^16 copies of one 5-document list in one launch, the device's own draws: first-position frequencies against
    softmax(s / T) (PL) or softmax(s) (STPL, whose ordering of s + g does not depend on T), and the frequencies of all
    120 orderings against their Plackett-Luce probabilities (chi-square)."""
    N, T = 1 << 16, 0.7
    s1 = np.array([0.9, 0.4, 0.0, -0.3, -0.8], dtype=np.float32)
    s = np.tile(s1, (N, 1)); y = np.tile(np.array([2, 1, 1, 0, 0], dtype=np.float32), (N, 1))
    _, _, _, o = _run(s, y, sample=True, distribution=dist, temperature=T, seed=1234, offset=77)
    assert np.array_equal(np.sort(o, 1), np.tile(np.arange(5), (N, 1)))
    w = np.exp(s1.astype(np.float64) / (T if dist == "PL" else 1.0))
    p1 = w / w.sum()
    f1 = np.bincount(o[:, 0], minlength=5) / N
    assert (np.abs(f1 - p1) <= 5 * np.sqrt(p1 * (1 - p1) / N)).all(), (f1, p1)
    perms = list(itertools.permutations(range(5)))
    probs = np.array([np.prod([w[q[i]] / w[list(q[i:])].sum() for i in range(5)]) for q in perms])
    index = {q: i for i, q in enumerate(perms)}
    counts = np.bincount([index[tuple(r)] for r in o.tolist()], minlength=len(perms))
    assert abs(probs.sum() - 1.0) < 1e-12 and (probs * N >= 5).all()
    assert stats.chisquare(counts, probs * N).pvalue > 1e-6


def test_device_draws_are_keyed():
    s, y = _fresh(64, 50, seed=6)
    for dist in ("PL", "STPL"):
        _, lq1, g1, o1 = _run(s, y, sample=True, distribution=dist, seed=7, offset=1)
        _, lq2, g2, o2 = _run(s, y, sample=True, distribution=dist, seed=7, offset=1)
        _, _, _, o3 = _run(s, y, sample=True, distribution=dist, seed=7, offset=2)
        assert np.array_equal(o1, o2) and np.array_equal(g1, g2) and np.array_equal(lq1, lq2)
        assert not np.array_equal(o1, o3)


@pytest.mark.parametrize("dist", ["PL", "STPL"])
def test_full_size_properties(dist):
    for (B, n) in [(1024, 256), (16, 4096)]:
        s, y = _fresh(B, n, seed=B + n)
        for top_k in (10, None):
            p = dict(distribution=dist, top_k=top_k, gamma=0.9, temperature=0.5, seed=3, offset=9)
            loss, lq, g, o = _run(s, y, sample=True, **p)
            _, lq2, g2, o2 = _run(s, y, sample=True, **p)
            assert np.array_equal(g, g2) and np.array_equal(lq, lq2) and np.array_equal(o, o2)   # bit for bit
            assert np.isfinite(g).all() and np.isfinite(lq).all() and np.isfinite(loss)
            assert np.abs(g.astype(np.float64).sum(1)).max() <= 2e-4 * np.abs(g).max() * np.sqrt(n)


def test_drop_in_class_train_step():
    import ptranking_b200
    from ptranking_b200 import LABEL_TYPE
    from tests.test_oracle_vs_golden import point_cfg
    F = 46
    sf = dict(sf_id="pointsf", opt="Adam", lr=1e-3, pointsf=point_cfg(F, num_layers=2))
    para = dict(model_id="MDPRank", temperature=1.0, gamma=1.0, top_k=10, distribution="PL")
    torch.manual_seed(3)
    r = ptranking_b200.MDPRank(sf_para_dict=sf, model_para_dict=para, gpu=True, device=DEV)
    r.init()
    _, y = _fresh(6, 40, seed=8)
    X = torch.randn(6, 40, F, generator=torch.Generator().manual_seed(1)).to(DEV)
    perm = torch.stack([torch.randperm(40, generator=torch.Generator().manual_seed(i)) for i in range(6)])
    before = r.grad_bucket.flat_param.clone()
    with torch.no_grad():
        scores = r.predict(X).detach().cpu()
    loss, stop = r.train_op(X, torch.from_numpy(y).to(DEV), presort=True, label_type=LABEL_TYPE.MultiLabel,
                            perm=perm.to(DEV))
    want, _, _ = mo.port_loss_and_grad(scores, torch.from_numpy(y), distribution="PL", top_k=10, perm=perm)
    assert not stop and abs(float(loss) - float(want)) <= 2e-5 * max(abs(float(want)), 1.0)
    assert not torch.equal(before, r.grad_bucket.flat_param)
    with pytest.raises(AssertionError):
        r.train_op(X, torch.from_numpy(y).to(DEV), presort=False, label_type=LABEL_TYPE.MultiLabel)
