"""GPU parity of the diversification path: the fused DALETOR loss kernel (ptrb200_daletor_fwd_bwd), the alpha-nDCG /
ERR-IA / nERR-IA kernel (ptrb200_srd_metrics_at_ks), the [q, q*d, d] input kernel, the scorer's per-query BN mode and
the drop-in DALETOR ranker -- against the unmodified reference's outputs (tests/golden/daletor.npz), the ATen port and
the float64 closed form of tests/daletor_oracle.py."""
import numpy as np
import pytest
import torch

from oracle import ref_port as rp
from tests import daletor_oracle as do
from tests.helpers import load, rel_err
from tests.test_oracle_daletor import KS, LOSS, METRICS

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-5


def _rele(mats):
    from ptranking_b200 import ops
    return ops.SubtopicRele.pack([torch.as_tensor(np.asarray(r, dtype=np.float32)) for r in mats], DEV)


def _loss(s_list, mats, rt=10.0, top_k=10, ragged=True):
    """-> (per-query losses, per-query gradients) of one launch over the queries."""
    from ptranking_b200 import ops
    lens = [len(s) for s in s_list]
    if ragged:
        off = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=DEV)
        s = torch.from_numpy(np.concatenate(s_list).astype(np.float32)).to(DEV)
        _, lq, g = ops.daletor_loss_and_grad(s, _rele(mats), rt=rt, top_k=top_k, offsets=off, max_len=max(max(lens), 1))
        g = g.cpu().numpy()
        o = np.concatenate([[0], np.cumsum(lens)])
        return lq.cpu().numpy(), [g[o[i]:o[i + 1]] for i in range(len(lens))]
    s = torch.from_numpy(np.stack(s_list).astype(np.float32)).to(DEV)
    _, lq, g = ops.daletor_loss_and_grad(s, _rele(mats), rt=rt, top_k=top_k)
    return lq.cpu().numpy(), list(g.cpu().numpy())


def _check(loss, grad, ref_loss, ref_grad, fl, fg, tol=TOL):
    """Within ``tol`` of the fp32 reference, or within twice the reference's own distance from float64 where that is
    larger (the sibling tests' rule); losses on the scale max(|loss|, 1), gradients on max(|grad|, |loss|, 1)."""
    sc = max(float(np.abs(fg).max()) if fg.size else 0.0, abs(fl), 1.0)
    tol_l = max(tol, 2.0 * abs(ref_loss - fl) / max(abs(fl), 1.0))
    assert abs(loss - ref_loss) <= tol_l * max(abs(ref_loss), 1.0), (loss, ref_loss, fl)
    if grad.size:
        tol_g = max(tol, 2.0 * float(np.abs(ref_grad - fg).max()) / sc)
        assert float(np.abs(grad - ref_grad).max()) <= tol_g * sc, (float(np.abs(grad - ref_grad).max()) / sc, tol_g)


@pytest.mark.parametrize("case,d", LOSS, ids=[c for c, _ in LOSS])
def test_kernel_matches_reference_fixture(case, d):
    lq, g = _loss([d["scores"][0]], [d["rele"]], d["rt"], d["top_k"])
    fl, fg = do.closed_form(d["scores"], d["rele"], d["rt"], d["top_k"])
    _check(float(lq[0]), g[0], d["loss"], d["grad"][0], fl, fg)


def _fresh(rng, n, m, graded=False):
    s = (rng.standard_normal(n) * rng.choice([0.1, 1.0, 3.0])).astype(np.float32)
    R = do_rele(rng, m, n, graded)
    return s, R


def do_rele(rng, m, n, graded):
    R = (rng.random((m, n)) < 0.25).astype(np.float32)
    if graded:
        R *= rng.uniform(0.0, 2.0, (m, n)).astype(np.float32)
    if m >= 3:
        R[rng.integers(m)] = 0.0
    return R


@pytest.mark.parametrize("n,m,top_k,rt", [(1, 3, 10, 10.0), (2, 1, None, 1.0), (33, 5, 2, 10.0), (256, 8, 10, 10.0),
                                          (256, 32, None, 50.0), (1024, 8, 10, 10.0), (1024, 4, 3, 1.0)])
def test_fresh_inputs_against_port_and_float64(n, m, top_k, rt):
    rng = np.random.default_rng(n * 131 + m)
    for graded in (False, True):
        s, R = _fresh(rng, n, m, graded)
        lq, g = _loss([s], [R], rt, top_k)
        pl, pg = do.port_loss_and_grad(s, R, rt, top_k)
        fl, fg = do.closed_form(s, R, rt, top_k)
        _check(float(lq[0]), g[0], pl, pg, fl, fg)


@pytest.mark.parametrize("n", [2048, 4096])
def test_long_lists_against_float64(n):
    """Beyond what the [m, n, n] port can hold on the host: float64 only, on fp32's summation bound over n partners."""
    rng = np.random.default_rng(n)
    s, R = _fresh(rng, n, 8)
    lq, g = _loss([s], [R], 10.0, 10)
    fl, fg = do.closed_form(s, R, 10.0, 10)
    sc = max(float(np.abs(fg).max()), abs(fl), 1.0)
    assert abs(float(lq[0]) - fl) <= 2e-5 * max(abs(fl), 1.0)
    assert float(np.abs(g[0] - fg).max()) <= 1e-4 * sc


def test_ragged_batch_bit_equal_to_single_queries_and_reruns():
    rng = np.random.default_rng(7)
    lens = [0, 1, 5, 300, 64, 2049, 17]
    ms = [3, 1, 2, 8, 32, 6, 5]
    qs = [_fresh(rng, n, m) for n, m in zip(lens, ms)]
    lq, g = _loss([s for s, _ in qs], [R for _, R in qs], 10.0, None)
    lq2, g2 = _loss([s for s, _ in qs], [R for _, R in qs], 10.0, None)
    assert np.array_equal(lq, lq2) and all(np.array_equal(a, b) for a, b in zip(g, g2))     # bit-identical reruns
    assert lq[0] == 0.0 and g[0].size == 0                                                 # empty list
    for i, (s, R) in enumerate(qs):
        if not len(s):
            continue
        l1, g1 = _loss([s], [R], 10.0, None)
        assert l1[0] == lq[i] and np.array_equal(g1[0], g[i]), i                           # same bits alone
    # a dense [B, n] batch takes the same path
    same = [_fresh(rng, 40, 4) for _ in range(5)]
    ld, gd = _loss([s for s, _ in same], [R for _, R in same], 10.0, 10, ragged=False)
    for i, (s, R) in enumerate(same):
        l1, g1 = _loss([s], [R], 10.0, 10)
        assert l1[0] == ld[i] and np.array_equal(g1[0], gd[i])


def test_full_size_determinism_and_zero_sum_gradient():
    from ptranking_b200 import ops
    rng = np.random.default_rng(11)
    B, n, m = 64, 1024, 8
    s = torch.from_numpy(rng.standard_normal((B, n)).astype(np.float32)).to(DEV)
    rele = _rele([do_rele(rng, m, n, False) for _ in range(B)])
    a = ops.daletor_loss_and_grad(s, rele, rt=10.0, top_k=10)
    b = ops.daletor_loss_and_grad(s, rele, rt=10.0, top_k=10)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    g = a[2].double()
    # the loss depends on score differences only
    assert float(g.sum(dim=1).abs().max()) <= 1e-4 * float(g.abs().max())


def test_error_codes_at_the_limits():
    from ptranking_b200 import ops, _lib
    rng = np.random.default_rng(3)
    s = torch.zeros(1, 4097, device=DEV)
    with pytest.raises(_lib.B200LibraryError, match="MAX_LIST_LEN"):
        ops.daletor_loss_and_grad(s, _rele([np.ones((2, 4097), np.float32)]))
    s = torch.zeros(1, 8, device=DEV)
    with pytest.raises(_lib.B200LibraryError, match="MAX_SUBTOPICS"):
        ops.daletor_loss_and_grad(s, _rele([np.ones((33, 8), np.float32)]))
    with pytest.raises(_lib.B200LibraryError, match="MAX_SUBTOPICS"):
        ops.srd_metrics_at_ks(s, _rele([np.ones((33, 8), np.float32)]), [1], max_label=1.0)
    with pytest.raises(_lib.B200LibraryError):           # an empty batch
        ops.daletor_loss_and_grad(torch.zeros(1, 0, device=DEV), _rele([np.ones((2, 0), np.float32)]))
    lq, g = _loss([np.arange(8, dtype=np.float32)], [np.ones((0, 8), np.float32)])   # a query without subtopic rows
    assert lq[0] == 0.0 and (g[0] == 0).all()
    with pytest.raises(_lib.B200LibraryError):           # alpha outside [0, 1)
        ops.daletor_loss_and_grad(s, _rele([np.ones((2, 8), np.float32)]), alpha=1.0)
    # exactly at the limits it runs
    s32, R32 = _fresh(rng, 4096, 32)
    lq, g = _loss([s32], [R32], 10.0, None)
    assert np.isfinite(lq).all() and np.isfinite(g[0]).all()


# ---- metrics ------------------------------------------------------------------------------------------------------- #
@pytest.mark.parametrize("case,d", METRICS, ids=[c for c, _ in METRICS])
def test_metrics_match_reference_fixture(case, d):
    from ptranking_b200 import ops
    s = torch.from_numpy(d["scores"]).to(DEV)
    a, e, ne, flags, order = ops.srd_metrics_at_ks(s, _rele([d["rele"]]), KS, max_label=float(d["max_label"]),
                                                   return_order=True)
    assert np.array_equal(order.cpu().numpy()[0], d["order"])                 # orders exact
    want_a = np.atleast_2d(d["andcg_ks"])[0]
    assert np.abs(a.cpu().numpy()[0] - want_a).max() <= 1e-6
    assert np.abs(e.cpu().numpy()[0] - d["err_ia_ks"]).max() <= 1e-6
    assert np.abs(ne.cpu().numpy()[0] - d["nerr_ia_ks"]).max() <= 1e-6
    tot = float(d["rele"].sum())
    assert int(flags[0]) == (1 if tot >= 1 else 0) | (2 if tot > 0 else 0)


def test_metrics_ragged_batch_against_port_and_float64():
    from ptranking_b200 import ops
    rng = np.random.default_rng(5)
    lens = [3, 0, 50, 4096, 1, 700, 20]
    ms = [2, 4, 8, 5, 1, 32, 3]
    ks = [20, 1, 5, 10, 4096, 3]
    qs = []
    for n, m in zip(lens, ms):
        s = np.round(rng.standard_normal(n) * 4).astype(np.float32) / 4       # ties: index order breaks them
        qs.append((s, do_rele(rng, m, n, graded=(m == 8))))
    off = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=DEV)
    st = torch.from_numpy(np.concatenate([s for s, _ in qs])).to(DEV)
    a, e, ne, flags, order = ops.srd_metrics_at_ks(st, _rele([R for _, R in qs]), ks, max_label=2.0, offsets=off,
                                                   max_len=max(lens), return_order=True)
    a, e, ne, order = a.cpu().numpy(), e.cpu().numpy(), ne.cpu().numpy(), order.cpu().numpy()
    o = np.concatenate([[0], np.cumsum(lens)])
    for q, (s, R) in enumerate(qs):
        if not len(s):
            assert (a[q] == 0).all() and (e[q] == 0).all() and (ne[q] == 0).all()
            continue
        pa, pe, pne, porder = do.port_metrics(s, R, ks, 2.0)
        fa, fe, fne, forder = do.closed_form_metrics(s, R, ks, 2.0)
        assert np.array_equal(order[o[q]:o[q + 1]], porder) and np.array_equal(porder, forder)
        for got, port, f64 in ((a[q], pa, fa), (e[q], pe, fe), (ne[q], pne, fne)):
            tol = np.maximum(TOL, 2.0 * np.abs(port - f64))
            assert (np.abs(got - port) <= tol).all(), (q, got, port, f64)


def test_div_features():
    from ptranking_b200 import ops
    rng = np.random.default_rng(9)
    F, lens = 100, [5, 0, 17]
    q = torch.from_numpy(rng.standard_normal((3, F)).astype(np.float32))
    d = torch.from_numpy(rng.standard_normal((sum(lens), F)).astype(np.float32))
    off = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=DEV)
    X = ops.div_features(q.to(DEV), d.to(DEV), offsets=off, max_len=max(lens)).cpu()
    o = np.concatenate([[0], np.cumsum(lens)])
    for i in range(3):
        dq = d[o[i]:o[i + 1]]
        want = torch.cat((q[i:i + 1].expand(dq.size(0), -1), q[i:i + 1] * dq, dq), 1)   # div_point_ranker.py:14-19
        assert torch.equal(X[o[i]:o[i + 1]], want)
    Xd = ops.div_features(q[:1].to(DEV), d[:5].unsqueeze(0).to(DEV)).cpu()
    assert torch.equal(Xd[0], X[:5])


# ---- scorer: per-query BN ------------------------------------------------------------------------------------------- #
@pytest.mark.parametrize("affine", [True, False])
@pytest.mark.parametrize("F", [300, 46])
def test_per_query_bn_ragged_equals_per_query_dense_reference(F, affine):
    """One ragged launch of the per-query BN scorer = the reference's BN applied to each query alone, forward and
    backward (300 = the default diversification input width, a first-layer K the tensor-core kernels take)."""
    from ptranking_b200.base.utils import StackedFFNet
    torch.manual_seed(F)
    dims = [F, 100, 100, 100, 100, 100, 1]
    net = StackedFFNet(dims, AF="GE", TL_AF="GE", apply_tl_af=False, dropout=0.0, BN=True, bn_type="BN",
                       bn_affine=affine, bn_per_query=True).to(DEV)
    ref = rp.stacked_ffnet(dims, "GE", "GE", False, 0.0, True, "BN", affine)
    ref.load_state_dict({k: v.cpu() for k, v in net.state_dict().items()})
    if affine:
        with torch.no_grad():
            for p in list(net.parameters()):
                if p.dim() == 1 and p.numel() == 100:
                    p.add_(0.1 * torch.randn_like(p))
        ref.load_state_dict({k: v.cpu() for k, v in net.state_dict().items()})
    rng = np.random.default_rng(F)
    lens = [40, 7, 129, 64]
    X = torch.from_numpy(rng.standard_normal((sum(lens), F)).astype(np.float32))
    w = torch.from_numpy(rng.standard_normal(sum(lens)).astype(np.float32))
    off = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=DEV)
    out = net(X.to(DEV), offsets=off, max_len=max(lens)).view(-1)
    (out * w.to(DEV)).sum().backward()
    o = np.concatenate([[0], np.cumsum(lens)])
    outs = []
    for i in range(len(lens)):
        y = ref(X[o[i]:o[i + 1]].unsqueeze(0)).view(-1)
        outs.append(y)
    ref_out = torch.cat(outs)
    (ref_out * w).sum().backward()
    assert rel_err(out.detach().cpu().numpy(), ref_out.detach().numpy()) <= 2e-5
    ref_grads = dict(ref.named_parameters())
    for name, p in net.named_parameters():
        g, rg = p.grad.cpu().numpy(), ref_grads[name].grad.numpy()
        bias_into_bn = name.endswith(".bias") and name.startswith("ff_") and name != f"ff_{len(dims)}.bias"
        if bias_into_bn:
            assert np.abs(g).max() == 0.0          # exactly zero (DESIGN §2); the reference returns rounding noise
            continue
        assert np.abs(g - rg).max() <= 5e-5 * np.abs(rg).max() + 1e-7, name
    # the same query alone as a dense [1, n, F] batch
    net.zero_grad()
    d0 = net(X[:40].unsqueeze(0).to(DEV)).view(-1)
    assert rel_err(d0.detach().cpu().numpy(), outs[0].detach().numpy()) <= 2e-5


def _div_data(z):
    return [(f"q{i}", torch.from_numpy(z[f"train__q{i}_q_repr"]), [f"d{j}" for j in range(z[f"train__q{i}_doc_reprs"].shape[0])],
             torch.from_numpy(z[f"train__q{i}_doc_reprs"]), None, None, torch.from_numpy(z[f"train__q{i}_rele"]))
            for i in range(3)]


def _daletor(z, **over):
    from ptranking_b200 import DALETOR
    sf = dict(sf_id="pointsf", opt="Adagrad", lr=0.001,
              pointsf=dict(num_features=100, num_layers=5, AF="GE", TL_AF="GE", apply_tl_af=False,
                           BN=True, bn_type="BN", bn_affine=True, dropout=0.0))
    r = DALETOR(sf_para_dict=sf, model_para_dict=dict(model_id="DALETOR", rt=10.0, top_k=10), gpu=True, device=DEV)
    r.init()
    init = do.seeded_state({k: tuple(v.shape) for k, v in r.point_sf.state_dict().items()})
    with torch.no_grad():
        for k, v in r.point_sf.state_dict().items():
            v.copy_(torch.from_numpy(init[k]))
    return r


def _pre_bn_bias(name):
    """A Linear bias that feeds a BN (every one but the output layer's, ff_7, in these 5-hidden-layer nets): its exact
    gradient is 0, which the kernels return (DESIGN §2); the reference's autograd returns rounding noise."""
    return name.startswith("ff_") and name.endswith(".bias") and name != "ff_7.bias"


def test_div_train_matches_reference_train_steps():
    z = load("daletor.npz")
    data = _div_data(z)
    r = _daletor(z)
    r.train_mode()
    with torch.no_grad():
        pred0 = r.div_forward(data[0][1].to(DEV), data[0][3].to(DEV)).cpu().numpy()
    assert rel_err(pred0, z["train__pred0"]) <= 2e-5
    # first step's gradients, through the per-query entry
    r0 = _daletor(z)
    loss0, stop = r0.div_train_op(data[0][1], data[0][3], data[0][6], presort=True, epoch_k=1)
    assert not stop and abs(float(loss0.detach()) - z["train__losses"][0]) <= 2e-5 * max(1.0, abs(z["train__losses"][0]))
    gscale = max(np.abs(z["train__grad0__" + k]).max() for k, _ in r0.point_sf.named_parameters())
    for name, p in r0.point_sf.named_parameters():
        ref = z["train__grad0__" + name]
        got = p.grad.cpu().numpy()
        if _pre_bn_bias(name):
            assert np.abs(got).max() == 0.0
        else:
            assert np.abs(got - ref).max() <= 3e-5 * np.abs(ref).max() + 2e-6 * gscale, name
    # one epoch of div_train: three queries, three Adagrad steps
    epoch_loss, stop = r.div_train(data, epoch_k=1)
    assert not stop
    want = float(np.sum(z["train__losses"])) / 3
    assert abs(float(epoch_loss) - want) <= 3e-5 * max(1.0, abs(want))
    # the trained scorer against the reference's after the same three steps, scored on each query (parameters are not
    # compared entry by entry: Adagrad's first steps are ~lr * sign(g), which turns rounding-level gradients into lr)
    for i, (_, q, _, dr, _, _, _) in enumerate(data):
        with torch.no_grad():
            got = r.div_forward(q.to(DEV), dr.to(DEV)).cpu().numpy()
        assert rel_err(got, z[f"train__final_scores_q{i}"]) <= 5e-5


def test_queries_per_step_equals_sum_of_per_query_gradients():
    """One ragged step over several queries (per-query BN, one loss launch) = the per-query steps' gradients summed, both
    held to the reference semantics (each query scored and differentiated alone by the CPU oracle)."""
    from ptranking_b200 import ops
    from ptranking_b200.base.utils import StackedFFNet
    torch.manual_seed(1)
    rng = np.random.default_rng(1)
    F = 30
    dims = [3 * F, 100, 100, 100, 100, 100, 1]
    net = StackedFFNet(dims, AF="GE", TL_AF="GE", dropout=0.0, BN=True, bn_type="BN", bn_affine=True,
                       bn_per_query=True).to(DEV)
    ref = rp.stacked_ffnet(dims, "GE", "GE", False, 0.0, True, "BN", True)
    ref.load_state_dict({k: v.cpu() for k, v in net.state_dict().items()})
    lens, ms = [12, 40, 9, 77], [3, 5, 1, 8]
    q = torch.from_numpy(rng.standard_normal((4, F)).astype(np.float32))
    d = torch.from_numpy(rng.standard_normal((sum(lens), F)).astype(np.float32))
    mats = [do_rele(rng, m, n, False) for n, m in zip(lens, ms)]
    for R in mats:
        R[0, 0] = 1.0
    off = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=DEV)
    X = ops.div_features(q.to(DEV), d.to(DEV), offsets=off, max_len=max(lens))
    s = net(X, offsets=off, max_len=max(lens)).view(-1)
    loss, lq = ops.daletor_loss(s, _rele(mats), rt=10.0, top_k=10, offsets=off, max_len=max(lens))
    loss.backward()
    batch = {k: p.grad.clone() for k, p in net.named_parameters()}
    o = np.concatenate([[0], np.cumsum(lens)])
    total = {k: torch.zeros_like(p) for k, p in net.named_parameters()}
    losses, ref_losses = [], []
    for i in range(4):
        net.zero_grad()
        si = net(X[o[i]:o[i + 1]].unsqueeze(0)).view(1, -1)
        li, _ = ops.daletor_loss(si, _rele([mats[i]]), rt=10.0, top_k=10)
        li.backward()
        losses.append(float(li.detach()))
        for k, p in net.named_parameters():
            total[k] += p.grad
        dq = d[o[i]:o[i + 1]]
        xi = torch.cat((q[i:i + 1].expand(dq.size(0), -1), q[i:i + 1] * dq, dq), 1)
        lr_ = do.port_loss(ref(xi.unsqueeze(0)).view(1, -1), torch.from_numpy(mats[i]), 10.0, 10)
        lr_.backward()                          # the oracle's parameter gradients accumulate over the queries
        ref_losses.append(float(lr_.detach()))
    assert abs(float(loss.detach()) - sum(losses)) <= 1e-5 * max(1.0, abs(sum(losses)))
    assert np.allclose(lq.cpu().numpy(), losses, rtol=1e-5, atol=1e-6)
    assert np.allclose(losses, ref_losses, rtol=2e-5, atol=1e-6)
    ref_grads = dict(ref.named_parameters())
    gscale = max(float(p.grad.abs().max()) for p in ref.parameters())
    for k in batch:
        want = ref_grads[k].grad.numpy()
        for got in (batch[k].cpu().numpy(), total[k].cpu().numpy()):
            if _pre_bn_bias(k):
                assert np.abs(got).max() == 0.0
                continue
            err = float(np.abs(got - want).max())
            assert err <= 1e-4 * gscale, (k, err, gscale)       # scale: the net's largest gradient entry


def test_ranker_evaluation_and_batched_training():
    """div_train with queries_per_step > 1, and the evaluation methods against the port on the ranker's own scores."""
    z = load("daletor.npz")
    data = _div_data(z)
    rng = np.random.default_rng(4)
    data.append(("q_none", data[0][1], ["x"] * 9, torch.from_numpy(rng.standard_normal((9, 100)).astype(np.float32)),
                 None, None, torch.zeros(2, 9)))                     # no relevance: skipped everywhere
    data.append(("q_short", data[1][1], ["y"] * 4, torch.from_numpy(rng.standard_normal((4, 100)).astype(np.float32)),
                 None, None, torch.ones(3, 4)))                      # shorter than k = 5
    r = _daletor(z)
    loss, stop = r.div_train(data, epoch_k=10, queries_per_step=2)
    assert not stop and np.isfinite(float(loss))
    r.eval_mode()
    with torch.no_grad():
        preds = [r.div_predict(q.to(DEV), dr.to(DEV)).cpu().numpy()[0] for _, q, _, dr, _, _, _ in data]
    ks = [1, 3, 5, 10, 20]
    per = [do.port_metrics(p, R.numpy(), ks, 1.0) for p, (*_, R) in zip(preds, data)]
    sums = [float(R.sum()) for *_, R in data]
    lens = [len(p) for p in preds]
    cnt = [i for i in range(len(data)) if sums[i] >= 1 and lens[i] >= 5]
    assert float(r.alpha_ndcg_at_k(test_data=data, k=5)) == pytest.approx(np.mean([per[i][0][2] for i in cnt]), abs=2e-5)
    assert float(r.err_ia_at_k(test_data=data, k=5, max_label=1.0)) == pytest.approx(np.mean([per[i][1][2] for i in cnt]), abs=2e-5)
    assert float(r.nerr_ia_at_k(test_data=data, k=5, max_label=1.0)) == pytest.approx(np.mean([per[i][2][2] for i in cnt]), abs=2e-5)
    cnt1 = [i for i in range(len(data)) if sums[i] >= 1]
    got = r.alpha_ndcg_at_ks(test_data=data, ks=ks).numpy()
    assert np.abs(got - np.mean([per[i][0] for i in cnt1], axis=0)).max() <= 2e-5
    cnt0 = [i for i in range(len(data)) if sums[i] > 0]
    a, e, ne, per_q = r.srd_performance_at_ks(test_data=data, ks=ks, max_label=1.0, need_per_q_andcg=True)
    for j, got in enumerate((a, e, ne)):
        assert np.abs(got.numpy() - np.mean([per[i][j] for i in cnt0], axis=0)).max() <= 2e-5
    assert len(per_q) == len(cnt0) and tuple(per_q[0].shape) == (1, len(ks))
    v = r.div_validation(vali_data=data, vali_metric="nERR-IA", k=5, max_label=1.0)
    assert float(v) == pytest.approx(np.mean([per[i][2][2] for i in cnt]), abs=2e-5)
