"""GPU parity of the fused WassRank kernel (ptrb200_wassrank_fwd_bwd), through the C ABI: against the float64 log-domain
form on every reference fixture (tests/golden/wassrank.npz, including the cases where the fp32 reference returns NaN),
against the fp32 reference where it is finite, against the float64 form on fresh inputs of both schedules, batch and
ragged-batch semantics, full-size properties and the drop-in class's train step."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import wassrank_oracle as wo
from tests.helpers import rel_err
from tests.test_oracle_wassrank import CASES, COSTS, IDS, wass_params

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL64 = 5e-5
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(s, y, **params):
    from ptranking_b200 import ops
    st = torch.from_numpy(np.ascontiguousarray(s, dtype=np.float32)).to(DEV)
    yt = torch.from_numpy(np.ascontiguousarray(y, dtype=np.float32)).to(DEV)
    loss, lq, g = ops.rank_loss_and_grad("WassRank", st, yt, **params)
    torch.cuda.synchronize()
    return float(loss.cpu()), lq.cpu().numpy(), g.cpu().numpy()


def _check_f64(loss, grad, fl, fg):
    assert np.isfinite(loss) and np.isfinite(grad).all()
    assert abs(loss - fl) <= TOL64 * max(abs(fl), 1e-30), (loss, fl)
    assert np.abs(grad - fg).max() <= TOL64 * max(np.abs(fg).max(), 1e-30), (np.abs(grad - fg).max(), np.abs(fg).max())


@pytest.mark.parametrize("case,d", CASES, ids=IDS)
def test_kernel_matches_float64_on_fixtures(case, d):
    p = wass_params(d)
    loss, lq, grad = _run(d["scores"], d["labels"], **p)
    fl, fg = wo.closed_form(d["scores"], d["labels"], **p)
    _check_f64(loss, grad, fl, fg)
    assert abs(float(lq.sum()) - loss) <= 1e-6 * max(abs(loss), 1e-30)


FINITE = [(c, d) for c, d in CASES if np.isfinite(float(d["loss"])) and np.isfinite(d["grad"]).all()]


@pytest.mark.parametrize("case,d", FINITE, ids=[c for c, _ in FINITE])
def test_kernel_matches_fp32_reference_where_finite(case, d):
    """Where the fp32 reference is itself further from float64 than 1e-5, the kernel only has to be as close to the
    reference as twice the reference's own error; losses below 1 are compared on the scale 1 (the rule of
    test_gpu_siblings.py).  The float64 bar above holds on every case."""
    p = wass_params(d)
    loss, _, grad = _run(d["scores"], d["labels"], **p)
    fl, fg = wo.closed_form(d["scores"], d["labels"], **p)
    ref, ref_g = float(d["loss"]), d["grad"]
    tol_l = max(1e-5, 2.0 * abs(ref - fl) / max(abs(fl), 1e-30))
    tol_g = max(1e-5, 2.0 * rel_err(ref_g, fg))
    assert abs(loss - ref) <= tol_l * max(abs(ref), 1.0), (loss, ref, fl)
    assert rel_err(grad, ref_g) <= tol_g, (rel_err(grad, ref_g), rel_err(ref_g, fg))


def _fresh(B, n, seed, real_labels):
    rng = np.random.default_rng(seed)
    s = (2.5 * rng.standard_normal((B, n)) if seed % 2 else 1.0 / (1.0 + np.exp(-rng.standard_normal((B, n))))).astype(np.float32)
    if real_labels:       # more distinct values than the kernel's label-group table: the general schedule for eg / dg too
        y = np.round(4.0 * rng.random((B, n)), 3).astype(np.float32)
    else:
        p = np.array([1940952, 1225770, 504958, 69010, 30435], dtype=np.float64)
        y = rng.choice(5, size=(B, n), p=p / p.sum()).astype(np.float32)     # unsorted integer grades
    return s, y


@pytest.mark.parametrize("real_labels", [False, True], ids=["int_labels", "real_labels"])
@pytest.mark.parametrize("lam", [0.1, 1.0])
@pytest.mark.parametrize("cost", COSTS)
@pytest.mark.parametrize("shape", [(8, 256), (4, 50), (2, 1024), (3, 33), (5, 1), (2, 2), (1, 2000)])
def test_kernel_matches_float64_fresh_inputs(shape, cost, lam, real_labels):
    B, n = shape
    s, y = _fresh(B, n, seed=31 * B + n + int(real_labels), real_labels=real_labels)
    p = dict(cost_type=cost, lam=lam, sh_itr=20)
    loss, lq, grad = _run(s, y, **p)
    fl, fg = wo.closed_form(s, y, **p)
    _check_f64(loss, grad, fl, fg)


@pytest.mark.parametrize("cost", COSTS)
def test_batch_is_the_mean_of_single_queries(cost):
    B, n = 5, 40
    s, y = _fresh(B, n, seed=5, real_labels=False)
    loss, lq, g = _run(s, y, cost_type=cost)
    for b in range(B):
        l1, _, g1 = _run(s[b:b + 1], y[b:b + 1], cost_type=cost)
        # equal up to the rounding of the extra 1/B factor inside the kernel
        assert abs(lq[b] * B - l1) <= 4e-6 * abs(l1)
        assert np.abs(g[b] * B - g1[0]).max() <= 4e-6 * np.abs(g1).max()
    assert abs(loss - lq.sum()) <= 1e-6 * abs(loss)


def _ragged(lens, seed, real_labels=False):
    S, Y = [], []
    for k, n in enumerate(lens):
        s, y = _fresh(1, n, seed=seed + k, real_labels=real_labels)
        S.append(s[0]); Y.append(y[0])
    off = np.zeros(len(lens) + 1, dtype=np.int32)
    off[1:] = np.cumsum(lens)
    return np.concatenate(S).astype(np.float32), np.concatenate(Y).astype(np.float32), off


@pytest.mark.parametrize("cost", COSTS)
def test_ragged_batch_matches_dense_queries(cost):
    from ptranking_b200 import ops
    lens = [300, 64, 37, 5, 2, 1, 0, 1024, 0, 130]
    s, y, off = _ragged(lens, seed=11)
    B = len(lens)
    st, yt, od = torch.from_numpy(s).to(DEV), torch.from_numpy(y).to(DEV), torch.from_numpy(off).to(DEV)
    loss, lq, g = ops.rank_loss_and_grad("WassRank", st, yt, offsets=od, max_len=max(lens), cost_type=cost)
    lq, g = lq.cpu().numpy(), g.cpu().numpy()
    for b, n in enumerate(lens):
        if n == 0:
            assert lq[b] == 0.0
            continue
        l1, _, g1 = _run(s[off[b]:off[b + 1]][None], y[off[b]:off[b + 1]][None], cost_type=cost)
        assert abs(lq[b] * B - l1) <= 1e-6 * max(abs(l1), 1e-30), (b, n)
        assert np.abs(g[off[b]:off[b + 1]] * B - g1[0]).max() <= 1e-6 * max(np.abs(g1).max(), 1e-30), (b, n)


@pytest.mark.parametrize("cost", COSTS)
def test_bucketed_and_single_launches_are_bit_identical(cost):
    """Length buckets launch CTAs sized for their own lists; every launch divides by the whole batch's query count and
    the CTA size is fixed, so each query's result does not depend on the launch it was part of."""
    from ptranking_b200 import ops, _lib
    from ptranking_b200.data import length_buckets
    rng = np.random.default_rng(7)
    # three length classes of at least 8 lists each (length_buckets merges smaller ones), plus short and empty lists
    lens = np.concatenate([rng.integers(513, 1100, 8), rng.integers(129, 512, 10), rng.integers(2, 128, 30), [1, 0, 0]])
    lens = np.sort(lens)[::-1].copy()
    s, y, off = _ragged(list(lens), seed=23)
    st, yt, od = torch.from_numpy(s).to(DEV), torch.from_numpy(y).to(DEV), torch.from_numpy(off).to(DEV)
    B, ml = len(lens), int(lens.max())
    buckets = length_buckets(lens)
    assert len(buckets) >= 2
    l0, q0, g0 = ops.rank_loss_and_grad("WassRank", st, yt, offsets=od, max_len=ml, cost_type=cost)
    l1, q1, g1 = ops.rank_loss_and_grad("WassRank", st, yt, offsets=od, max_len=ml, buckets=buckets, cost_type=cost)
    assert torch.equal(q0, q1) and torch.equal(g0, g1)
    # the same through the C ABI directly, one launch per bucket (ops keeps the label-group costs in one launch)
    lib = _lib.load()
    g2, q2 = torch.empty_like(st), torch.empty(B, dtype=torch.float32, device=DEV)
    stream = torch.cuda.current_stream().cuda_stream
    for b0, b1, mlen in buckets:
        _lib.check(lib.ptrb200_wassrank_fwd_bwd(st.data_ptr(), yt.data_ptr(), od.data_ptr() + 4 * b0, g2.data_ptr(),
                                                q2.data_ptr() + 4 * b0, b1 - b0, max(int(mlen), 1), B,
                                                _lib.WASS_COST_TYPES[cost], 0.1, 20, 100.0, float(np.e), 4.0, stream), "wassrank")
    torch.cuda.synchronize()
    assert torch.equal(q0, q2) and torch.equal(g0, g2)


@pytest.mark.parametrize("cost", ["eg", "ddg"])
def test_full_size_properties(cost):
    for (B, n) in [(1024, 256), (16, 1024)]:
        s, y = _fresh(B, n, seed=B + n, real_labels=False)
        y = -np.sort(-y, axis=1)
        loss, lq, g = _run(s, y, cost_type=cost)
        _, lq2, g2 = _run(s, y, cost_type=cost)
        assert np.array_equal(g, g2) and np.array_equal(lq, lq2)            # deterministic, bit for bit
        assert np.isfinite(g).all() and np.isfinite(lq).all() and np.isfinite(loss)
        # softmax's backward: every query's gradient sums to zero
        assert np.abs(g.astype(np.float64).sum(1)).max() <= 1e-5 * np.abs(g).max() * np.sqrt(n)


def test_zero_iterations_and_argument_checks():
    from ptranking_b200 import ops, _lib
    s, y = _fresh(3, 20, seed=3, real_labels=False)
    for cost in COSTS:
        loss, _, g = _run(s, y, cost_type=cost, sh_itr=0)
        fl, fg = wo.closed_form(s, y, cost_type=cost, sh_itr=0)
        _check_f64(loss, g, fl, fg)
    st, yt = torch.from_numpy(s).to(DEV), torch.from_numpy(y).to(DEV)
    with pytest.raises(ValueError):
        ops.rank_loss_and_grad("WassRank", st, yt, cost_type="Group")
    with pytest.raises(_lib.B200LibraryError):
        ops.rank_loss_and_grad("WassRank", st, yt, lam=0.0)
    with pytest.raises(_lib.B200LibraryError):
        ops.rank_loss_and_grad("WassRank", st, yt, sh_itr=-1)


def test_drop_in_class_train_step():
    """Built with the keywords the reference evaluator passes (ltr.py:174) and the default pointsf scorer: one train_op
    returns the float64 form's loss on the scores the scorer produced, and the optimizer moves the weights."""
    import ptranking_b200
    from ptranking_b200 import LABEL_TYPE
    from tests.test_oracle_vs_golden import point_cfg
    F = 46
    sf = dict(sf_id="pointsf", opt="Adam", lr=1e-3, pointsf=point_cfg(F, num_layers=5))
    para = dict(model_id="WassRank", mode="SinkhornOT", sh_itr=20, lam=0.1, smooth_type="ST", norm_type="BothST",
                cost_type="eg", non_rele_gap=100, var_penalty=np.e, gain_base=4)
    torch.manual_seed(3)
    r = ptranking_b200.WassRank(sf_para_dict=sf, wass_para_dict=para, dict_cost_mats={}, dict_std_dists={}, gpu=True, device=DEV)
    r.init()
    _, y = _fresh(6, 40, seed=8, real_labels=False)
    y = -np.sort(-y, axis=1)
    X = torch.randn(6, 40, F, generator=torch.Generator().manual_seed(1)).to(DEV)
    before = r.grad_bucket.flat_param.clone()
    with torch.no_grad():
        scores = r.predict(X).detach().cpu().numpy()
    loss, stop = r.train_op(X, torch.from_numpy(y).to(DEV), batch_ids=[str(i) for i in range(6)], presort=True,
                            label_type=LABEL_TYPE.MultiLabel)
    want, _ = wo.closed_form(scores, y, cost_type="eg", lam=0.1, sh_itr=20)
    assert not stop and abs(float(loss) - want) <= TOL64 * abs(want)
    assert not torch.equal(before, r.grad_bucket.flat_param)


@pytest.mark.skipif(not os.path.isdir(os.path.join(ROOT, "baseline", "_ref", "ptranking")),
                    reason="the reference package (baseline/_ref) is not installed next to this GPU")
def test_reference_driver_runs_wassrank():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "dropin_run.py"), "--impl", "b200", "--model", "WassRank",
                        "--queries", "48"], cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
