"""Ragged batches inside one launch (SURVEY 8f-2): every loss kernel, the metric kernels, the per-query StandardScaler
and a full training step on variable-length lists, checked against the oracle run query by query."""
import numpy as np
import pytest
import torch

from oracle import ref_port as rp
from tests.helpers import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MSLR_P = np.array([1940952, 1225770, 504958, 69010, 30435], dtype=np.float64)
MSLR_P /= MSLR_P.sum()


def _ragged(lens, seed, sigmoid=False):
    rng = np.random.default_rng(seed)
    S, Y = [], []
    for n in lens:
        y = rng.choice(5, size=n, p=MSLR_P).astype(np.float32)
        if n:
            y[0] = max(y[0], 1.0)
        y = -np.sort(-y)
        s = rng.standard_normal(n).astype(np.float32)
        if sigmoid:
            s = (1.0 / (1.0 + np.exp(-s))).astype(np.float32)
        S.append(s); Y.append(y)
    off = np.zeros(len(lens) + 1, dtype=np.int32)
    off[1:] = np.cumsum(lens)
    return S, Y, off


LENS = [37, 1, 256, 2, 120, 5, 64, 1024, 33, 8]
LOSSES = [("RankNet", dict(sigma=1.0)), ("LambdaRank", dict(sigma=1.0)),
          ("LambdaLoss", dict(k=5, sigma=1.0, mu=5.0, loss_type="NDCG_Loss2++", presort=True)),
          ("LambdaLoss", dict(k=40, sigma=1.0, mu=5.0, loss_type="NDCG_Loss2", presort=True)),
          ("ListNet", {}), ("ListMLE", {}), ("RankCosine", {}), ("STListNet", dict(temperature=1.0)),
          ("SoftRank", dict(delta=2.0, top_k=None)), ("SoftRank", dict(delta=1.0, top_k=10))]


@pytest.mark.parametrize("name,params", LOSSES, ids=[f"{n}-{i}" for i, (n, _) in enumerate(LOSSES)])
@pytest.mark.parametrize("lens", [LENS, [3, 0, 7, 1251, 0, 12]], ids=["mixed", "with_empty_and_long"])
def test_ragged_loss_equals_per_query_oracle(name, params, lens):
    """One ragged launch == the oracle (the reference's ATen ops) run on every query alone, summed."""
    from ptranking_b200 import ops
    S, Y, off = _ragged(lens, seed=len(lens) * 31 + max(lens), sigmoid=(name != "RankNet"))
    s = torch.from_numpy(np.concatenate(S)).to(DEV)
    y = torch.from_numpy(np.concatenate(Y)).to(DEV)
    offd = torch.from_numpy(off).to(DEV)
    kw = dict(params)
    perms, unifs = [], []
    if name == "ListMLE":
        g = torch.Generator().manual_seed(7)
        perms = [rp.shuffle_ties_perm(torch.from_numpy(yq)[None], generator=g)[0] if len(yq) else torch.zeros(0, dtype=torch.long) for yq in Y]
        kw["perm"] = torch.cat(perms).to(torch.int32).to(DEV)
    if name == "STListNet":
        unifs = [torch.rand(len(sq), generator=torch.Generator().manual_seed(11 + i)) for i, sq in enumerate(S)]
        kw["unif"] = torch.cat(unifs).to(DEV)
    loss, loss_q, grad = ops.rank_loss_and_grad(name, s, y, offsets=offd, max_len=max(lens), **kw)
    loss_q, grad = loss_q.cpu().numpy(), grad.cpu().numpy()
    want_total = 0.0
    for b, (sq, yq) in enumerate(zip(S, Y)):
        if len(sq) == 0:
            assert loss_q[b] == 0.0
            continue
        okw = dict(params)
        if name == "ListMLE":
            okw["perm"] = perms[b][None]
        if name == "STListNet":
            okw["unif"] = unifs[b][None]
        ol, og = rp.loss_and_grad(name, torch.from_numpy(sq)[None], torch.from_numpy(yq)[None], **okw)
        ol, og = float(ol), og.numpy()[0]
        got = grad[off[b]: off[b + 1]]
        tol = 2e-5 if len(sq) <= 256 else 1e-4           # the fp32 reference's own O(n^2) rounding grows with n
        assert abs(loss_q[b] - ol) <= tol * max(abs(ol), 1.0), (b, len(sq), loss_q[b], ol)
        assert rel_err(got, og) <= tol or np.abs(got - og).max() <= 1e-7, (b, len(sq), rel_err(got, og))
        want_total += ol
    assert abs(float(loss) - want_total) <= 1e-4 * max(abs(want_total), 1.0)


def test_ragged_equals_dense_when_lengths_are_uniform():
    """With equal lengths the ragged launch reproduces the dense [B,n] launch bit for bit."""
    from ptranking_b200 import ops
    B, n = 12, 96
    S, Y, off = _ragged([n] * B, seed=5)
    s = torch.from_numpy(np.stack(S)).to(DEV); y = torch.from_numpy(np.stack(Y)).to(DEV)
    offd = torch.from_numpy(off).to(DEV)
    for name, kw in [("LambdaRank", dict(sigma=1.0)), ("RankNet", dict(sigma=1.0)), ("ListNet", {}),
                     ("LambdaLoss", dict(k=5)), ("SoftRank", dict(delta=2.0)), ("RankCosine", {}), ("RankMSE", {}),
                     ("ApproxNDCG", dict(alpha=10.0))]:
        l0, q0, g0 = ops.rank_loss_and_grad(name, s, y, **kw)
        l1, q1, g1 = ops.rank_loss_and_grad(name, s.reshape(-1), y.reshape(-1), offsets=offd, max_len=n, **kw)
        assert torch.equal(q0, q1) and torch.equal(g0.reshape(-1), g1) and torch.equal(l0, l1), name


def test_ragged_approxndcg_and_rankmse_batch_coupling():
    """ApproxNDCG keeps the reference's [B]/[B,1] coupling (every query scaled by sum_a 1/iDCG_a) and RankMSE its mean
    over queries -- both defined over the ragged batch exactly as over a dense one."""
    from ptranking_b200 import ops
    from oracle import closed_form as cf
    lens = [20, 7, 64, 33]
    S, Y, off = _ragged(lens, seed=3, sigmoid=True)
    s = torch.from_numpy(np.concatenate(S)).to(DEV); y = torch.from_numpy(np.concatenate(Y)).to(DEV)
    offd = torch.from_numpy(off).to(DEV)
    _, lq, g = ops.rank_loss_and_grad("ApproxNDCG", s, y, offsets=offd, max_len=max(lens), alpha=10.0, presort=True)
    inv = sum(1.0 / float(cf._idcg(yq[None].astype(np.float64))[0]) for yq in Y)
    for b, (sq, yq) in enumerate(zip(S, Y)):
        l1, g1 = cf.approxndcg(sq[None], yq[None], alpha=10.0, batch_coupled=False)
        scale = inv * float(cf._idcg(yq[None].astype(np.float64))[0])
        assert abs(lq[b].item() - l1 * scale) <= 5e-5 * abs(l1 * scale)
        assert rel_err(g[off[b]: off[b + 1]].cpu().numpy(), g1[0] * scale) <= 5e-5
    _, lq, g = ops.rank_loss_and_grad("RankMSE", s, y, offsets=offd, max_len=max(lens))
    want = np.concatenate([2.0 * (sq - yq) / len(lens) for sq, yq in zip(S, Y)])
    assert rel_err(g.cpu().numpy(), want) <= 1e-6
    assert abs(float(lq.sum()) - sum(((sq - yq) ** 2).sum() for sq, yq in zip(S, Y)) / len(lens)) <= 1e-4


def test_ragged_metrics_equal_per_query_oracle():
    from ptranking_b200 import ops
    lens = [37, 1, 256, 2, 120, 5, 0, 1024]
    S, Y, off = _ragged(lens, seed=17)
    rng = np.random.default_rng(2)
    Y = [rng.permutation(yq) for yq in Y]                     # unsorted labels: presort=False path
    s = torch.from_numpy(np.concatenate(S)).to(DEV); y = torch.from_numpy(np.concatenate(Y)).to(DEV)
    offd = torch.from_numpy(off).to(DEV)
    ks = [1, 3, 5, 10, 50]
    nd, order = ops.ndcg_at_ks(s, y, ks, presort=False, return_order=True, offsets=offd, max_len=max(lens))
    m = ops.adhoc_metrics_at_ks(s, y, ks, presort=False, max_label=4.0, offsets=offd, max_len=max(lens))
    nd, order = nd.cpu().numpy(), order.cpu().numpy()
    for b, (sq, yq) in enumerate(zip(S, Y)):
        if len(sq) == 0:
            assert not nd[b].any()
            continue
        st, yt = torch.from_numpy(sq)[None], torch.from_numpy(yq)[None]
        want = rp.evaluator_ndcg_at_ks(st, yt, ks, presort=False).numpy()[0]
        assert np.abs(nd[b] - want).max() <= 1e-6
        want_order = torch.sort(st, dim=1, descending=True, stable=True)[1][0].numpy()
        assert np.array_equal(order[off[b]: off[b + 1]], want_order)          # integer ranks bit-exact
        wm = rp.evaluator_metrics_at_ks(st, yt, ks, presort=False, max_label=4.0)
        for got, w in zip(m, wm):
            assert np.abs(got[b].cpu().numpy() - w.numpy()[0]).max() <= 1e-6


@pytest.mark.parametrize("dense", [True, False])
def test_standard_scaler_matches_sklearn_per_query(dense):
    """ops.standard_scale against the loader's sklearn StandardScaler().fit_transform per query (data_utils.py:482-487),
    including a constant column (scale 1), heavy-tailed columns and the ISTELLA clip."""
    from ptranking_b200 import ops
    rng = np.random.default_rng(0)
    F = 136
    lens = [50] * 6 if dense else [37, 1, 256, 2, 120, 1251]
    Xs = []
    for n in lens:
        x = rng.standard_normal((n, F)) * rng.lognormal(0, 2, F) + rng.standard_normal(F) * 50
        x[:, 3] = 7.25                                        # constant feature
        x[:, 5] = np.exp(rng.standard_normal(n) * 4)          # heavy tail (raw counts)
        Xs.append(x.astype(np.float32))
    off = np.zeros(len(lens) + 1, dtype=np.int32); off[1:] = np.cumsum(lens)
    for clip in (None, 50.0):
        if dense:
            got = ops.standard_scale(torch.from_numpy(np.stack(Xs)).to(DEV), clip_max=clip).cpu().numpy().reshape(-1, F)
        else:
            got = ops.standard_scale(torch.from_numpy(np.concatenate(Xs)).to(DEV), offsets=torch.from_numpy(off).to(DEV),
                                     max_len=max(lens), clip_max=clip).cpu().numpy()
        want = np.concatenate([rp.per_query_standard_scale(x, clip_max=clip) for x in Xs]).astype(np.float32)
        assert np.abs(got - want).max() <= 2e-6 * max(np.abs(want).max(), 1.0)
        assert np.array_equal(got[:, 3], np.zeros_like(got[:, 3]))


@pytest.mark.parametrize("model,paras", [("LambdaRank", dict(model_id="LambdaRank", sigma=1.0)), ("ListNet", None),
                                         ("ApproxNDCG", dict(model_id="ApproxNDCG", alpha=10.0))])
def test_ragged_train_step_matches_oracle(model, paras):
    """RaggedBatches -> ranker.train(): scorer (batch-level BN: one statistics group over every document of the ragged
    batch), ragged loss kernel, backward, optimizer -- against the oracle stepping the same ragged batch with the loss
    evaluated query by query."""
    import ptranking_b200
    from ptranking_b200 import LABEL_TYPE
    from ptranking_b200.data import RaggedBatches
    from tests.test_oracle_vs_golden import point_cfg
    F = 46
    lens = [50, 7, 120, 33, 64, 12]
    rng = np.random.default_rng(4)
    S, Y, off = _ragged(lens, seed=9)
    queries = [(f"q{i}", rng.standard_normal((n, F)).astype(np.float32), Y[i]) for i, n in enumerate(lens)]
    sf = dict(sf_id="pointsf", opt="Adam", lr=1e-3, pointsf=point_cfg(F, num_layers=3))
    cls = getattr(ptranking_b200, model)
    torch.manual_seed(1)
    r = cls(sf_para_dict=sf, gpu=True, device=DEV) if paras is None else cls(sf_para_dict=sf, model_para_dict=paras, gpu=True, device=DEV)
    r.init()
    net = rp.point_scorer(**sf["pointsf"])
    net.load_state_dict({k: v.cpu() for k, v in r.point_sf.state_dict().items()})
    opt, _ = rp.make_optimizer(net.parameters(), "Adam", 1e-3)
    loader = RaggedBatches(queries, docs_per_batch=10 ** 6, presort=False, pin_memory=False)
    ep_loss, stop = r.train(loader, epoch_k=1, presort=True, label_type=LABEL_TYPE.MultiLabel)
    # oracle: one forward over all documents (BN couples them), loss = sum over queries of the per-query loss
    X = torch.from_numpy(np.concatenate([q[1] for q in queries]))[None]
    net.train()
    scores = rp.point_forward(net, X).view(-1)
    lname = {"LambdaRank": rp.lambdarank_loss, "ListNet": rp.listnet_loss, "ApproxNDCG": rp.approxndcg_loss}[model]
    if model == "ApproxNDCG":       # batch-coupled: sum_b DCG_b * sum_a 1/iDCG_a
        inv = sum(1.0 / rp.dcg_at_k(torch.from_numpy(yq)[None]) for yq in Y)
        dcgs = [-(rp.approxndcg_loss(scores[off[b]: off[b + 1]][None], torch.from_numpy(Y[b])[None], alpha=10.0) *
                  rp.dcg_at_k(torch.from_numpy(Y[b])[None])) for b in range(len(lens))]
        loss = -(torch.stack([d.reshape(()) for d in dcgs]).sum() * inv.reshape(()))
    else:
        kw = dict(sigma=1.0) if model == "LambdaRank" else {}
        loss = sum(lname(scores[off[b]: off[b + 1]][None], torch.from_numpy(Y[b])[None], **kw) for b in range(len(lens)))
    opt.zero_grad(); loss.backward(); opt.step()
    assert not stop
    assert abs(float(ep_loss) * len(lens) - float(loss)) <= 2e-5 * max(abs(float(loss)), 1.0)
    for (k, v), (_, w) in zip(r.point_sf.state_dict().items(), net.state_dict().items()):
        assert rel_err(v.cpu().numpy(), w.numpy()) <= 2e-2, k             # one Adam step: sign-dominated update
    # evaluation over the same ragged loader, both sides on the oracle's weights (rank flips cannot enter)
    r.point_sf.load_state_dict({k: v.clone() for k, v in net.state_dict().items()})
    nd = r.ndcg_at_ks(test_data=loader, ks=[1, 5, 10], label_type=LABEL_TYPE.MultiLabel, presort=True)
    net.eval()
    with torch.no_grad():
        sc = rp.point_forward(net, X).view(-1)
    want = torch.stack([rp.evaluator_ndcg_at_ks(sc[off[b]: off[b + 1]][None], torch.from_numpy(Y[b])[None], [1, 5, 10], presort=True)[0]
                        for b in range(len(lens))]).mean(0)
    assert np.abs(nd.numpy() - want.numpy()).max() <= 1e-5
    nd10 = r.ndcg_at_k(test_data=loader, k=10, label_type=LABEL_TYPE.MultiLabel, presort=True)
    assert np.isfinite(nd10.numpy()).all()


@pytest.mark.parametrize("cfg", ["bn2_relu", "bn2_aff_celu", "bn2_gelu_drop0"])
def test_ragged_bn2_scorer_matches_oracle_per_query(cfg):
    """Per-query BN2 (LTRBatchNorm2, base/utils.py:227-282) over a ragged batch: scores and every parameter gradient equal
    the oracle scoring each query alone (its statistics span that query's documents only) with gradients summed."""
    import ptranking_b200
    from tests.test_oracle_vs_golden import POINT_CFGS, point_cfg
    over = dict(POINT_CFGS[cfg]) if cfg in POINT_CFGS else dict(AF="GE", TL_AF="S", bn_type="BN2", bn_affine=True, num_layers=3)
    F = 136
    lens = [50, 7, 130, 33, 1, 64, 260]
    off = np.zeros(len(lens) + 1, dtype=np.int32); off[1:] = np.cumsum(lens)
    total = int(off[-1])
    sf = dict(sf_id="pointsf", opt="Adam", lr=1e-3, pointsf=point_cfg(F, **over))
    torch.manual_seed(2)
    r = ptranking_b200.ListNet(sf_para_dict=sf, gpu=True, device=DEV)
    r.init(); r.eval_mode()
    with torch.no_grad():                      # perturb the norm parameters off their init point
        for k, p in r.point_sf.named_parameters():
            if "bn" in k:
                p.add_(0.1 * torch.randn_like(p))
    net = rp.point_scorer(**sf["pointsf"])
    net.load_state_dict({k: v.cpu() for k, v in r.point_sf.state_dict().items()})
    net.eval()
    g = torch.Generator().manual_seed(5)
    X = torch.randn(total, F, generator=g); w = torch.randn(total, generator=g)
    offd = torch.from_numpy(off).to(DEV)
    s = r.forward_ragged(X.to(DEV), offd, max(lens))
    assert s.shape == (total,)
    r.grad_bucket.zero()
    (s * w.to(DEV)).sum().backward()
    want = []
    for b in range(len(lens)):
        sq = rp.point_forward(net, X[off[b]: off[b + 1]][None]).view(-1)
        (sq * w[off[b]: off[b + 1]]).sum().backward()          # parameter gradients accumulate over the queries
        want.append(sq.detach())
    want = torch.cat(want).numpy()
    # a one-document query has zero variance: the normalised value is 0/sqrt(eps) on both sides
    assert rel_err(s.detach().cpu().numpy(), want) <= 2e-5
    gscale = max(float(p.grad.abs().max()) for p in net.parameters())
    for (k, p), q in zip(r.point_sf.named_parameters(), net.parameters()):
        err = float((p.grad.cpu() - q.grad).abs().max())
        assert err <= 3e-5 * float(q.grad.abs().max()) + 2e-6 * gscale + 1e-9, (k, err, float(q.grad.abs().max()), gscale)


def test_ragged_bn2_equals_dense_bn2_on_uniform_lengths():
    import ptranking_b200
    from tests.test_oracle_vs_golden import point_cfg
    F, B, n = 136, 6, 96
    sf = dict(sf_id="pointsf", opt="Adam", lr=1e-3, pointsf=point_cfg(F, bn_type="BN2", bn_affine=True, num_layers=3, dropout=0.1))
    torch.manual_seed(2)
    r = ptranking_b200.ListNet(sf_para_dict=sf, gpu=True, device=DEV)
    r.init(); r.train_mode()                   # dropout ON: the ragged path must draw the same counter-based masks
    X = torch.randn(B, n, F, generator=torch.Generator().manual_seed(1)).to(DEV)
    off = torch.arange(0, B * n + 1, n, dtype=torch.int32, device=DEV)
    torch.manual_seed(9)
    from ptranking_b200 import ops
    o0 = ops._dropout_offset
    a = r.forward(X)
    ops._dropout_offset = o0                   # same dropout stream for the second call
    b = r.forward_ragged(X.reshape(B * n, F), off, n)
    assert rel_err(b.detach().cpu().numpy(), a.detach().cpu().numpy().reshape(-1)) <= 1e-5


@pytest.mark.parametrize("name,params", [("LambdaRank", dict(sigma=1.0)), ("RankNet", dict(sigma=1.0)), ("ListNet", {}), ("SoftRank", dict(delta=2.0)),
                                         ("LambdaLoss", dict(k=5)), ("ApproxNDCG", dict(alpha=10.0, batch_coupled=False)), ("ListMLE", {})])
def test_length_buckets_change_launch_geometry_not_results(name, params):
    """RaggedBatches orders a batch by length and cuts it into at most three length classes; each class is launched with CTAs sized
    for its own lists.  Same numbers as the single launch sized for the longest list (different kernels may serve the
    short and the long lists: fp32-rounding agreement, not bit equality), and the metric kernels agree exactly."""
    from ptranking_b200 import ops
    from ptranking_b200.data import length_buckets
    rng = np.random.default_rng(3)
    lens = np.sort(np.clip(rng.lognormal(4.45, 0.85, 300), 1, 1251).astype(int))[::-1].copy()
    lens[0] = 1251
    S, Y, off = _ragged(list(lens), seed=41, sigmoid=True)
    s = torch.from_numpy(np.concatenate(S)).to(DEV); y = torch.from_numpy(np.concatenate(Y)).to(DEV)
    offd = torch.from_numpy(off).to(DEV)
    buckets = length_buckets(lens)
    assert 2 <= len(buckets) <= 3
    kw = dict(params)
    if name == "ListMLE":
        kw["perm"] = ops.shuffle_ties_perm(y, seed=3, offset=1, offsets=offd, max_len=int(lens.max()), buckets=buckets)
        p2 = ops.shuffle_ties_perm(y, seed=3, offset=1, offsets=offd, max_len=int(lens.max()))
        assert torch.equal(kw["perm"], p2)              # the tie shuffle is keyed by flat document index: launch geometry is irrelevant
    l0, q0, g0 = ops.rank_loss_and_grad(name, s, y, offsets=offd, max_len=int(lens.max()), **kw)
    l1, q1, g1 = ops.rank_loss_and_grad(name, s, y, offsets=offd, max_len=int(lens.max()), buckets=buckets, **kw)
    assert rel_err(q1.cpu().numpy(), q0.cpu().numpy()) <= 2e-5 and abs(float(l1) - float(l0)) <= 2e-5 * abs(float(l0))
    g0, g1 = g0.cpu().numpy(), g1.cpu().numpy()
    for b in range(len(lens)):
        a, c = g0[off[b]: off[b + 1]], g1[off[b]: off[b + 1]]
        assert np.abs(a - c).max() <= 2e-5 * max(np.abs(a).max(), 1e-6) + 1e-8, (b, lens[b])
    nd0 = ops.ndcg_at_ks(s, y, [1, 5, 10], presort=True, offsets=offd, max_len=int(lens.max()))
    nd1 = ops.ndcg_at_ks(s, y, [1, 5, 10], presort=True, offsets=offd, max_len=int(lens.max()), buckets=buckets)
    m0 = ops.adhoc_metrics_at_ks(s, y, [1, 5, 10], presort=True, max_label=4.0, offsets=offd, max_len=int(lens.max()))
    m1 = ops.adhoc_metrics_at_ks(s, y, [1, 5, 10], presort=True, max_label=4.0, offsets=offd, max_len=int(lens.max()), buckets=buckets)
    assert torch.equal(nd0, nd1) and all(torch.equal(a, c) for a, c in zip(m0, m1))


@pytest.mark.parametrize("enc", ["DASALC", "AllRank", "AttnDIN"])
def test_list_scorer_ragged_batch_equals_query_by_query(enc):
    """Lists of different lengths through the attention scorer in ONE padded batch (pad -> masked softmax -> gather) give
    every query the scores, and every parameter the gradient, that processing the queries one by one gives (the dense path is
    pinned to the reference by the fixtures of tests/test_gpu_listsf.py; F = 24 is a multiple of four, so the aligned
    batched-GEMM kernel and the fused Q|K|V projection are on the path)."""
    import ptranking_b200
    from ptranking_b200 import ops
    F = 24
    sf = dict(sf_id="listsf", opt="Adagrad", lr=1e-3,
              listsf=dict(num_features=F, ff_dims=[16, 32, 24], AF="R", TL_AF="GE", apply_tl_af=False, BN=False, bn_type="BN2",
                          bn_affine=False, n_heads=2, encoder_layers=2, encoder_type=enc, dropout=0.0))
    torch.manual_seed(11)
    r = ptranking_b200.ListNet(sf_para_dict=sf, gpu=True, device=DEV)
    r.init()
    r.eval_mode()           # the tail net keeps the factory's dropout 0.1 whatever is configured (list_ranker.py:340-341): masks are
                            # keyed by position in the batch, so the comparison runs without dropout; autograd is still on
    lens = [40, 17, 33, 5, 64, 1, 28]
    rng = np.random.default_rng(5)
    X = torch.from_numpy(rng.standard_normal((sum(lens), F)).astype(np.float32)).to(DEV)
    y = torch.from_numpy(rng.integers(0, 5, sum(lens)).astype(np.float32)).to(DEV)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    offd = torch.from_numpy(off).to(DEV)
    params = r.get_parameters()

    def grads_of(loss):
        for p in params:
            p.grad = None
        loss.backward()
        return [p.grad.detach().clone() if p.grad is not None else torch.zeros_like(p) for p in params]

    s_rag = r.forward_ragged(X, offd, max(lens))
    assert s_rag.shape == (sum(lens),)
    g_rag = grads_of((s_rag * torch.cos(torch.arange(sum(lens), device=DEV, dtype=torch.float32))).sum())
    s_one, total = [], None
    for b, n in enumerate(lens):
        sq = r.forward(X[off[b]: off[b + 1]].unsqueeze(0))[0]
        s_one.append(sq)
    s_cat = torch.cat(s_one)
    g_one = grads_of((s_cat * torch.cos(torch.arange(sum(lens), device=DEV, dtype=torch.float32))).sum())
    assert rel_err(s_rag.detach().cpu().numpy(), s_cat.detach().cpu().numpy()) <= 1e-5
    scale = max(float(g.abs().max()) for g in g_one)
    for p, a, c in zip(params, g_rag, g_one):
        assert float((a - c).abs().max()) <= 2e-5 * scale, tuple(p.shape)
    # the same batch cut into two query ranges, each padded to its own longest list
    s_cls = r.forward_ragged(X, offd, max(lens), buckets=[(0, 3, 40), (3, 7, 64)])
    g_cls = grads_of((s_cls * torch.cos(torch.arange(sum(lens), device=DEV, dtype=torch.float32))).sum())
    assert rel_err(s_cls.detach().cpu().numpy(), s_cat.detach().cpu().numpy()) <= 1e-5
    for p, a, c in zip(params, g_cls, g_one):
        assert float((a - c).abs().max()) <= 2e-5 * scale, tuple(p.shape)
    # and one optimizer step on the ragged batch through the public training entry point
    loss, stop = r.train_op(X, y, offsets=offd, max_len=max(lens), buckets=[(0, 3, 40), (3, 7, 64)], presort=False,
                            label_type=ptranking_b200.LABEL_TYPE.MultiLabel)
    assert torch.isfinite(loss) and not stop
    # pad / unpad are inverse gathers
    P = ops.pad_lists(X, offd, max(lens))
    assert P.shape == (len(lens), max(lens), F) and torch.equal(ops.unpad_lists(P, offd, sum(lens)), X)
    assert float(P[1, lens[1]:].abs().max()) == 0.0


def test_unpad_lists_stops_at_the_padded_block():
    """A list longer than the padded length gives back only the n_max rows its block holds; its rows behind stay
    untouched."""
    from ptranking_b200 import _lib
    lib = _lib.load()
    lens, n_max, F = [9, 3, 5], 5, 4
    o = np.concatenate([[0], np.cumsum(lens)])
    offd = torch.tensor(o, dtype=torch.int32, device=DEV)
    padded = torch.arange(len(lens) * n_max * F, dtype=torch.float32, device=DEV).reshape(len(lens), n_max, F)
    flat = torch.full((sum(lens), F), -1.0, device=DEV)
    _lib.check(lib.ptrb200_unpad_lists(padded.data_ptr(), offd.data_ptr(), flat.data_ptr(), len(lens), n_max, F,
                                       torch.cuda.current_stream().cuda_stream), "unpad_lists")
    want = torch.full_like(flat, -1.0)
    for b, n in enumerate(lens):
        want[o[b]:o[b] + min(n, n_max)] = padded[b, :min(n, n_max)]
    assert torch.equal(flat, want)
