"""GPU parity of DivProbRanker: the fused loss kernel (ptrb200_divprob_fwd_bwd), the sort keys
(ptrb200_divprob_sort_key), the head (ptrb200_divprob_head), the scorer at out_dim 2 / 15 and the drop-in ranker --
against the unmodified reference's outputs (tests/golden/divprob.npz), the ATen port and the float64 closed form of
tests/divprob_oracle.py."""
import copy

import numpy as np
import pytest
import torch

from tests import daletor_oracle as do
from tests import divlist_oracle as dl
from tests import divprob_oracle as dpo
from tests.helpers import load, rel_err
from tests.test_gpu_daletor import _check
from tests.test_oracle_divprob import CASES, KEYS, GOLD

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rele(mats):
    from ptranking_b200 import ops
    return ops.SubtopicRele.pack([torch.as_tensor(np.asarray(r, dtype=np.float32)) for r in mats], DEV)


def _run(raws, mats, loss, K=1, limit_delta=None, top_k=None, norm=True):
    """One ragged launch over the queries -> (per-query losses, per-query d loss / d raw)."""
    from ptranking_b200 import ops
    lens = [r.shape[0] for r in raws]
    o = np.concatenate([[0], np.cumsum(lens)])
    off = torch.tensor(o, dtype=torch.int32, device=DEV)
    u = torch.from_numpy(np.concatenate(raws).astype(np.float32)).to(DEV)
    opt_id, metric = ("SuperSoft", loss) if loss in ("aNDCG", "nERR-IA") else (loss, None)
    _, lq, g = ops.divprob_loss_and_grad(u, _rele(mats), opt_id=opt_id, metric=metric, K=K, limit_delta=limit_delta,
                                         top_k=top_k, norm=norm, offsets=off, max_len=max(max(lens), 1))
    g = g.cpu().numpy()
    return lq.cpu().numpy(), [g[o[i]:o[i + 1]] for i in range(len(lens))]


def _kw(d):
    return dict(K=d["K"], limit_delta=d["limit_delta"], top_k=d["top_k"], norm=d["norm"])


@pytest.mark.parametrize("case,d", CASES, ids=[c for c, _ in CASES])
def test_kernel_matches_reference_fixture(case, d):
    lq, g = _run([d["raw"]], [d["rele"]], d["loss"], **_kw(d))
    if np.isnan(d["ref_loss"]):       # LambdaPairCLS norm over a query without relevance: 0 / 0, as the reference
        assert np.isnan(lq[0])
        return
    fl, fg = dpo.closed_form(d["raw"], d["rele"], d["loss"], **_kw(d))
    _check(float(lq[0]), g[0], d["ref_loss"], d["ref_grad"], fl, fg)


def _fresh(rng, n, m, loss, K=1, limit_delta=None):
    u = dpo.draw_raw(rng, n, K, limit_delta, loss in ("PairCLS", "LambdaPairCLS"))
    R = (rng.random((m, n)) < 0.2).astype(np.float32)
    R[0, 0] = 1.0
    return u, R


@pytest.mark.parametrize("loss,n,m,K,ld,top_k", [
    ("aNDCG", 4096, 32, 1, None, None), ("aNDCG", 2048, 8, 5, 0.1, 10), ("nERR-IA", 4096, 32, 5, None, None),
    ("nERR-IA", 1025, 3, 1, 0.01, 10), ("PairCLS", 1025, 8, 1, 0.1, None), ("LambdaPairCLS", 2048, 4, 5, 0.01, None),
    ("LambdaPairCLS", 1025, 32, 1, None, None)])
def test_long_lists_match_float64(loss, n, m, K, ld, top_k):
    rng = np.random.default_rng([n, m, K])
    u, R = _fresh(rng, n, m, loss, K, ld)
    lq, g = _run([u], [R], loss, K, ld, top_k)
    fl, fg = dpo.closed_form(u, R, loss, K, ld, top_k, True)
    assert abs(float(lq[0]) - fl) <= 1e-4 * max(1.0, abs(fl)), (float(lq[0]), fl)
    assert float(np.abs(g[0] - fg).max()) <= 1e-4 * max(float(np.abs(fg).max()), 1.0)


@pytest.mark.parametrize("loss", dpo.LOSSES)
def test_ragged_launch_is_bitwise_per_query(loss):
    rng = np.random.default_rng(7)
    lens, ms = [0, 37, 1, 300, 0, 2, 129], [3, 5, 2, 8, 1, 32, 4]
    raws, mats = [], []
    for n, m in zip(lens, ms):
        u = dpo.draw_raw(rng, n, 5, 0.1, loss in ("PairCLS", "LambdaPairCLS")) if n else np.zeros((0, 15), np.float32)
        R = (rng.random((m, n)) < 0.3).astype(np.float32)
        if n:
            R[0, 0] = 1.0
        raws.append(u)
        mats.append(R)
    lq, g = _run(raws, mats, loss, 5, 0.1, 10)
    for i in range(len(lens)):
        if lens[i] == 0:
            assert lq[i] == 0.0
            continue
        a, ga = _run([raws[i]], [mats[i]], loss, 5, 0.1, 10)
        assert lq[i].tobytes() == a[0].tobytes() and g[i].tobytes() == ga[0].tobytes(), i


@pytest.mark.parametrize("ld", [None, 0.1])
def test_head_and_its_gradient_k5(ld):
    from ptranking_b200 import ops
    rng = np.random.default_rng(11)
    u = dpo.draw_raw(rng, 60, 5, ld, False)
    mu, var = ops.divprob_head(torch.from_numpy(u).to(DEV), K=5, limit_delta=ld)
    m64, v64 = dpo.head64(u, 5, ld)
    assert rel_err(mu.cpu().numpy(), m64) <= 1e-6 and rel_err(var.cpu().numpy(), v64) <= 1e-6
    R = (rng.random((4, 60)) < 0.3).astype(np.float32)
    up = dpo.draw_raw(rng, 60, 5, ld, True)      # the pair losses away from fp32 saturation of 1 - erfc / 2
    for loss in dpo.LOSSES:
        if loss in ("PairCLS", "LambdaPairCLS"):
            u = up
        lq, g = _run([u], [R], loss, 5, ld, None)
        fl, fg = dpo.closed_form(u, R, loss, 5, ld, None, True)
        assert abs(float(lq[0]) - fl) <= 2e-5 * max(1.0, abs(fl))
        assert float(np.abs(g[0] - fg).max()) <= 2e-5 * max(float(np.abs(fg).max()), 1.0), loss


@pytest.mark.parametrize("key", KEYS)
def test_sort_keys_match_reference_fixture_and_feed_the_metrics(key):
    from ptranking_b200 import ops
    _, _, K, ld = GOLD[key + "__meta"]
    K, ld = int(K), (None if ld == 0 else float(ld))
    u = GOLD[key + "__raw"]
    n = u.shape[0]
    rng = np.random.default_rng(n)
    R = (rng.random((5, n)) < 0.3).astype(np.float32)
    ks = [1, 3, 5, 10, 20]
    for sort_id in ("ExpRele", "RERAR", "RiskAware"):
        got = ops.divprob_sort_key(torch.from_numpy(u).to(DEV).unsqueeze(0), sort_id, K=K, limit_delta=ld)[0]
        np.testing.assert_allclose(got.cpu().numpy(), GOLD[f"{key}__{sort_id}"], rtol=2e-6, atol=1e-7)
        port = dpo.port_sort_key(u, sort_id, K, ld)
        # the kernel's ranking is a ranking by the port's keys (up to ties within the keys' tolerance) ...
        order = np.argsort(-got.cpu().numpy(), kind="stable")
        assert np.all(np.diff(port[order]) <= 2e-6 * max(1.0, float(np.abs(port).max()))), sort_id
        # ... and the metrics of the kernel's keys are the port's evaluator on those keys
        a, e, ne, _ = ops.srd_metrics_at_ks(got.view(1, -1), _rele([R]), ks, max_label=1.0)
        pa, pe, pne, _ = do.port_metrics(got.cpu().numpy(), R, ks, 1.0)
        for x, y in ((a, pa), (e, pe), (ne, pne)):
            assert np.abs(x.cpu().numpy()[0] - y).max() <= 2e-6


def _point_ranker(K, ld, opt_id="SuperSoft", metric="nERR-IA", top_k=None, F=20, BN=True, lr=0.01, seeded=False,
                  tail=False):
    from ptranking_b200 import DivProbRanker
    sf = dict(sf_id="pointsf", opt="Adagrad", lr=lr,
              pointsf=dict(num_features=F, h_dim=16, num_layers=3, AF="GE", TL_AF="S" if tail else "GE", apply_tl_af=tail,
                           BN=BN, bn_type="BN", bn_affine=True, dropout=0.0))
    r = DivProbRanker(sf_para_dict=sf, model_para_dict=dict(model_id="DivProbRanker", K=K, cluster=False,
                                                            sort_id="ExpRele", top_k=top_k, opt_id=opt_id,
                                                            limit_delta=ld, metric=metric, opt_ideal=True, norm=True),
                      gpu=True, device=DEV)
    r.init()
    if seeded:
        init = do.seeded_state({k: tuple(v.shape) for k, v in r.point_sf.state_dict().items()})
        with torch.no_grad():
            for k, v in r.point_sf.state_dict().items():
                v.copy_(torch.from_numpy(init[k]))
    return r


@pytest.mark.parametrize("K,out_dim,tail,BN", [(1, 2, False, True), (5, 15, False, True), (5, 15, True, True),
                                              (5, 15, False, False), (5, 15, True, False)])
def test_scorer_output_width_with_per_query_bn(K, out_dim, tail, BN):
    """The scorer's last layer at 2 and 15 outputs (not a multiple of 4), with and without the tail BN + activation the
    reference's grid sets (apply_tl_af with BN), and without BN: a ragged batch with per-query BN statistics equals each
    query scored alone and the fp32 port of the scorer, and the gradient reaches the output layer's own parameters."""
    from oracle import ref_port as rp
    from ptranking_b200 import ops
    r = _point_ranker(K, None, tail=tail, BN=BN)
    assert r.sf_para_dict["pointsf"]["out_dim"] == out_dim
    r.train_mode()
    rng = np.random.default_rng(K)
    lens = [17, 1, 64, 5]
    q = torch.from_numpy(rng.standard_normal((4, 20)).astype(np.float32)).to(DEV)
    d = torch.from_numpy(rng.standard_normal((sum(lens), 20)).astype(np.float32)).to(DEV)
    o = np.concatenate([[0], np.cumsum(lens)])
    off = torch.tensor(o, dtype=torch.int32, device=DEV)
    X = ops.div_list_features(q, d, offsets=off, max_len=max(lens))
    with torch.no_grad():
        raw = r.div_forward_ragged(X, off, max(lens)).view(-1, out_dim).cpu().numpy()
    dims = [60, 16, 16, 16, out_dim]
    ref = rp.stacked_ffnet(dims, "GE", "S" if tail else "GE", tail, 0.0, BN, "BN", True)
    ref.load_state_dict({k: v.cpu() for k, v in r.point_sf.state_dict().items()})
    for i in range(4):
        with torch.no_grad():
            alone = r.point_sf(X[o[i]:o[i + 1]].unsqueeze(0)).view(-1, out_dim).cpu().numpy()
        assert np.abs(raw[o[i]:o[i + 1]] - alone).max() <= 1e-5 * max(1.0, np.abs(alone).max())
        if lens[i] > 2 or not BN:          # torch's BN refuses a one-document batch in training mode
            with torch.no_grad():
                want = ref(X[o[i]:o[i + 1]].cpu().unsqueeze(0)).view(-1, out_dim).numpy()
            assert np.abs(alone - want).max() <= 1e-4 * max(1.0, np.abs(want).max()), i
    # the gradient reaches the output layer's own [out_dim, h] parameters through the ragged path, for the last column
    # only (the padded columns never leak into the real ones); random row weights, since a BN'd column sums to a constant
    r.point_sf.zero_grad()
    wts = torch.from_numpy(rng.standard_normal(sum(lens)).astype(np.float32)).to(DEV)
    (r.div_forward_ragged(X, off, max(lens)).view(-1, out_dim)[:, -1] * wts).sum().backward()
    w = r.point_sf.state_dict()
    last = max(int(k[3:].split(".")[0]) for k in w if k.startswith("ff_"))
    g = getattr(r.point_sf, f"ff_{last}").weight.grad
    assert g.shape == (out_dim, 16) and torch.count_nonzero(g[:-1]) == 0 and torch.count_nonzero(g[-1]) > 0
    if tail and BN:
        bn = getattr(r.point_sf, f"bn_{last}").bn
        assert bn.weight.grad.shape == (out_dim,) and torch.count_nonzero(bn.weight.grad[:-1]) == 0
        assert torch.count_nonzero(bn.weight.grad[-1]) > 0


# the reference's grid (div_parameter.py: pointsf 5 layers, listsf DASALC 3 x 2 heads, [128, 256, 512]; R hidden,
# apply_tl_af with BN 'BN' affine; Adam 0.001) with DivProbRanker's grid K = 5, SuperSoft aNDCG at top_k 10
GRID_POINTSF = dict(sf_id="pointsf", opt="Adam", lr=0.001,
                    pointsf=dict(num_features=20, h_dim=100, num_layers=5, AF="R", TL_AF="S", apply_tl_af=True, BN=True,
                                 bn_type="BN", bn_affine=True, dropout=0.0))
GRID_LISTSF = dict(sf_id="listsf", opt="Adam", lr=0.001,
                   listsf=dict(num_features=20, ff_dims=[128, 256, 512], AF="R", TL_AF="S", apply_tl_af=True, BN=True,
                               bn_type="BN", bn_affine=True, n_heads=2, encoder_type="DASALC", encoder_layers=3))


@pytest.mark.parametrize("sf", [GRID_POINTSF, GRID_LISTSF], ids=["pointsf", "listsf"])
@pytest.mark.parametrize("limit_delta", [None, 0.1])
def test_reference_grid_configuration_trains_and_evaluates(sf, limit_delta):
    """K = 5 with a BN'd 15-wide output layer: one ragged step equals the sum of the per-query losses with each query's
    raw output equal to its own, div_train with 1 and 2 queries per step, and the split's evaluation."""
    from ptranking_b200 import DivProbRanker, ops
    r = DivProbRanker(sf_para_dict=copy.deepcopy(sf),
                      model_para_dict=dict(model_id="DivProbRanker", K=5, cluster=False, sort_id="ExpRele", top_k=10,
                                           opt_id="SuperSoft", limit_delta=limit_delta, metric="aNDCG",
                                           opt_ideal=True, norm=True), gpu=True, device=DEV)
    r.init()
    r.eval_mode()              # dropout off (the list scorer's uni_sf keeps a fixed 0.1); BN keeps per-call statistics
    rng = np.random.default_rng(3)
    data = []
    for i, (n, m) in enumerate(((40, 5), (9, 3), (130, 8), (23, 2))):
        R = (rng.random((m, n)) < 0.3).astype(np.float32)
        R[0, 0] = 1.0
        data.append((f"q{i}", torch.from_numpy(rng.standard_normal((1, 20)).astype(np.float32)), [f"d{j}" for j in range(n)],
                     torch.from_numpy(rng.standard_normal((n, 20)).astype(np.float32)), None, None, torch.from_numpy(R)))
    sp = r._split(data)
    with torch.no_grad():
        if sf["sf_id"] == "listsf":
            raw = r.list_scores(sp.X, sp.plan(0, len(sp), r))
        else:
            raw = r.div_forward_ragged(sp.X, sp.offsets, sp.max_len)
        raw = raw.view(-1, 15)
        o = sp.offsets_host
        for i, (_, q, _, d, _, _, _) in enumerate(data):
            alone = r._raw(q.to(DEV), d.to(DEV))
            assert torch.allclose(raw[o[i]:o[i + 1]], alone, rtol=1e-5, atol=1e-5), i
    batch, lq, _ = ops.divprob_loss_and_grad(raw, sp.rele, opt_id="SuperSoft", metric="aNDCG", K=5,
                                             limit_delta=limit_delta, top_k=10, offsets=sp.offsets, max_len=sp.max_len)
    for i in range(len(data)):
        _, li, _ = ops.divprob_loss_and_grad(raw[o[i]:o[i + 1]].unsqueeze(0), sp.rele.select(i, i + 1),
                                             opt_id="SuperSoft", metric="aNDCG", K=5, limit_delta=limit_delta, top_k=10)
        assert lq[i].item() == li[0].item()
    r.train_mode()
    for qps in (1, 2):
        loss, stop = r.div_train(data, epoch_k=10, queries_per_step=qps)
        assert stop is False and np.isfinite(float(loss))
    a, e, ne = r.srd_performance_at_ks(test_data=data, ks=[1, 5, 10], max_label=1.0)
    assert all(np.isfinite(x.numpy()).all() for x in (a, e, ne))


def _train_data(z, name):
    return [(f"q{i}", torch.from_numpy(z[f"train_{name}__q{i}_q_repr"]),
             [f"d{j}" for j in range(z[f"train_{name}__q{i}_doc_reprs"].shape[0])],
             torch.from_numpy(z[f"train_{name}__q{i}_doc_reprs"]), None, None,
             torch.from_numpy(z[f"train_{name}__q{i}_rele"])) for i in range(3)]


def _fixture_ranker(name):
    from ptranking_b200 import DivProbRanker
    mp, sf = dpo.TRAIN[name]
    r = DivProbRanker(sf_para_dict=copy.deepcopy(sf), model_para_dict=dict(model_id="DivProbRanker", cluster=False,
                                                                          sort_id="ExpRele", opt_ideal=True, **mp),
                      gpu=True, device=DEV)
    r.init()
    if name == "pointsf":
        init = do.seeded_state({k: tuple(v.shape) for k, v in r.point_sf.state_dict().items()})
        with torch.no_grad():
            for k, v in r.point_sf.state_dict().items():
                v.copy_(torch.from_numpy(init[k]))
        r.train_mode()
        named = [("point_sf", k, p) for k, p in r.point_sf.named_parameters()]
    else:
        init = dl.seeded_state(dl.state_shapes(r.list_sf["encoder"], r.list_sf["uni_sf"]))
        with torch.no_grad():
            for part in ("encoder", "uni_sf"):
                for k, v in r.list_sf[part].state_dict().items():
                    v.copy_(torch.from_numpy(init[part][k]))
        r.eval_mode()
        named = [(part, k, p) for part in ("encoder", "uni_sf") for k, p in r.list_sf[part].named_parameters()]
    return r, named


@pytest.mark.parametrize("name", ["pointsf", "listsf"])
def test_training_fixture(name):
    z = load("divprob.npz")
    data = _train_data(z, name)
    r, named = _fixture_ranker(name)
    want = z[f"train_{name}__losses"]
    for i, (_, q, _, d, _, _, R) in enumerate(data):
        loss, stop = r.div_train_op(q, d, R, presort=True, epoch_k=10)
        assert stop is False
        assert abs(float(loss.detach()) - want[i]) <= 1e-4 * max(1.0, abs(want[i])), (i, float(loss), want[i])
        if i == 0:
            gscale = max(float(np.abs(z[f"train_{name}__grad0__{part}__{k}"]).max()) for part, k, _ in named)
            for part, k, p in named:
                ref = z[f"train_{name}__grad0__{part}__{k}"]
                got = p.grad.cpu().numpy()
                assert np.abs(got - ref).max() <= 1e-4 * np.abs(ref).max() + 2e-5 * gscale, (part, k)
    for i, (_, q, _, d, _, _, _) in enumerate(data):
        with torch.no_grad():
            mu, var = r.div_forward(q.to(DEV), d.to(DEV))
        assert rel_err(mu.cpu().numpy(), z[f"train_{name}__final_mu_q{i}"]) <= 2e-3
        assert rel_err(var.cpu().numpy(), z[f"train_{name}__final_var_q{i}"]) <= 2e-3


@pytest.mark.parametrize("sort_id", ["ExpRele", "RERAR", "RiskAware"])
def test_div_train_epoch_evaluation_and_checkpoint(sort_id, tmp_path):
    z = load("divprob.npz")
    data = _train_data(z, "pointsf")
    rng = np.random.default_rng(5)
    data.append(("q_none", data[0][1], ["x"] * 9, torch.from_numpy(rng.standard_normal((9, 20)).astype(np.float32)),
                 None, None, torch.zeros(2, 9)))
    data.append(("q_short", data[1][1], ["y"] * 4, torch.from_numpy(rng.standard_normal((4, 20)).astype(np.float32)),
                 None, None, torch.ones(3, 4)))
    for qps in (1, 2):
        r = _point_ranker(1, 0.01, seeded=True)
        r.sort_id = sort_id
        loss, stop = r.div_train(data, epoch_k=10, queries_per_step=qps)
        assert stop is False and np.isfinite(float(loss))
    r.eval_mode()
    with torch.no_grad():
        keys = [r.div_predict(q.to(DEV), d.to(DEV)).cpu().numpy()[0] for _, q, _, d, _, _, _ in data]
    ks = [1, 3, 5, 10]
    per = [do.port_metrics(k, R.numpy(), ks, 1.0) for k, (*_, R) in zip(keys, data)]
    counted = [i for i, (*_, R) in enumerate(data) if float(R.sum()) > 0]
    a, e, ne = r.srd_performance_at_ks(test_data=data, ks=ks, max_label=1.0)
    for j, got in enumerate((a, e, ne)):
        assert np.abs(got.numpy() - np.mean([per[i][j] for i in counted], axis=0)).max() <= 2e-5
    r.save(str(tmp_path) + "/", "m.pt")
    r2 = _point_ranker(1, 0.01)
    r2.sort_id = sort_id
    r2.load(str(tmp_path) + "/m.pt")
    assert set(torch.load(str(tmp_path) + "/m.pt").keys()) == set(r.point_sf.state_dict().keys())
    a2, e2, ne2 = r2.srd_performance_at_ks(test_data=data, ks=ks, max_label=1.0)
    assert torch.equal(a, a2) and torch.equal(e, e2) and torch.equal(ne, ne2)


def test_listsf_ragged_step_and_checkpoint(tmp_path):
    z = load("divprob.npz")
    data = _train_data(z, "listsf")
    r, _ = _fixture_ranker("listsf")
    loss, stop = r.div_train(data, epoch_k=10, queries_per_step=3)
    assert stop is False and np.isfinite(float(loss))
    res = r.srd_performance_at_ks(test_data=data, ks=[1, 5], max_label=1.0)
    r.save(str(tmp_path) + "/", "l.pt")
    assert set(torch.load(str(tmp_path) + "/l.pt").keys()) == {"encoder", "uni_sf"}
    r2, _ = _fixture_ranker("listsf")
    r2.load(str(tmp_path) + "/l.pt")
    res2 = r2.srd_performance_at_ks(test_data=data, ks=[1, 5], max_label=1.0)
    for x, y in zip(res, res2):
        assert torch.equal(x, y)


def test_bad_arguments_are_refused_before_launch():
    from ptranking_b200 import ops, _lib
    u = torch.zeros(1, 5, 3, device=DEV)
    with pytest.raises(ValueError):
        ops.divprob_loss_and_grad(u, _rele([np.ones((2, 5))]), K=1)
    lib = _lib.load()
    R = _rele([np.ones((2, 5))])
    rp, rop, scp = R._ptrs(torch.device(DEV))
    g = torch.empty(1, 5, 2, device=DEV)
    lq = torch.empty(1, device=DEV)
    n0 = lib.ptrb200_launch_count()
    # out_dim / K mismatch, unknown loss, missing workspace, m over the limit
    assert lib.ptrb200_divprob_fwd_bwd(g.data_ptr(), 3, None, rp, rop, scp, None, g.data_ptr(), lq.data_ptr(), 1, 5, 2, 1,
                                       0.0, 2, 0, 1, None) != 0
    assert lib.ptrb200_divprob_fwd_bwd(g.data_ptr(), 2, None, rp, rop, scp, None, g.data_ptr(), lq.data_ptr(), 1, 5, 2, 1,
                                       0.0, 7, 0, 1, None) != 0
    assert lib.ptrb200_divprob_fwd_bwd(g.data_ptr(), 2, None, rp, rop, scp, None, g.data_ptr(), lq.data_ptr(), 1, 5, 2, 1,
                                       0.0, 0, 0, 1, None) != 0
    assert lib.ptrb200_divprob_fwd_bwd(g.data_ptr(), 2, None, rp, rop, scp, None, g.data_ptr(), lq.data_ptr(), 1, 5, 33, 1,
                                       0.0, 2, 0, 1, None) != 0
    assert lib.ptrb200_divprob_sort_key(g.data_ptr(), 2, None, lq.data_ptr(), 1, 5, 1, 0.0, 9, None) != 0
    assert lib.ptrb200_launch_count() == n0
