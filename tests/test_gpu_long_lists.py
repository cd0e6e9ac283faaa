"""The per-list kernels on lists of 1000 to 4096 documents (PTRB200_MAX_LIST_LEN), against the float64 closed forms with
the fp32 ATen port as referee.

The launchers change kernel, CTA width and pass structure with the list length, and a ragged launch sizes every CTA for
the longest list in it, so a short query can run under the long-list schedule:
 - LambdaRank: lambdarank_runs_kernel with one thread per document up to 512, 1024 threads up to 1420 (two passes above
   1024), 512 threads up to 2048 (the 1024-thread partner rows no longer fit in shared memory), then
   pairwise_bce_kernel<true>, one thread per row over all pairs;
 - RankNet: pairwise_bce_circ_kernel<false> up to 1024 documents, pairwise_bce_kernel<false> above;
 - every kernel that sorts in the CTA (LambdaRank, LambdaLoss, ApproxNDCG's iDCG on unsorted labels, the tie shuffle,
   both metric kernels) sorts 4096 keys for any list above 2048.
Bars (the rule of tests/test_gpu_losses.py): the kernel is within max(1e-5, 2 x the port's own distance from float64) of
the port, and within 5e-5 of float64.  Metric values are within 1e-6 of the port; orders are exact."""
import numpy as np
import pytest
import torch

from oracle import closed_form as cf
from oracle import ref_port as rp
from tests import wassrank_oracle as wo
from tests.helpers import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-5
TOL64 = 5e-5
MAX_LEN = 4096
MSLR_P = np.array([1940952, 1225770, 504958, 69010, 30435], dtype=np.float64)
MSLR_P /= MSLR_P.sum()

# where the launchers change schedule (module docstring), plus the 2048 / 2049 sort boundary and the limit
L_LAMBDARANK = [1000, 1025, 1420, 1421, 2047, 2048, 2049, 3000, 4095, 4096]
L_RANKNET = [1000, 1025, 2049, 4096]                  # circulant <= 1024 < thread per row
L_SORTED = [1000, 1025, 2048, 2049, 4096]             # 1024-thread CTA above 1024, 4096 sort keys above 2048
L_LINEAR = [1000, 1025, 2049, 4096]                   # no sort: only the CTA width changes
L_WASS = [1000, 1420, 2049, 4096]                     # fixed CTA; shared memory beyond the default above 1170

# id -> (loss, kernel parameters, lengths)
CFGS = {
    "RankNet": ("RankNet", dict(sigma=1.0), L_RANKNET),
    "LambdaRank": ("LambdaRank", dict(sigma=1.0), L_LAMBDARANK),
    "LambdaLoss2pp_k5": ("LambdaLoss", dict(k=5, sigma=1.0, mu=5.0, loss_type="NDCG_Loss2++", presort=True), L_SORTED),
    "LambdaLoss2_kn": ("LambdaLoss", dict(k=MAX_LEN, sigma=1.0, mu=5.0, loss_type="NDCG_Loss2", presort=True), L_SORTED),
    "LambdaLoss1_k10": ("LambdaLoss", dict(k=10, sigma=1.0, mu=5.0, loss_type="NDCG_Loss1", presort=True), L_SORTED),
    "ListNet": ("ListNet", {}, L_LINEAR),
    "ListMLE": ("ListMLE", {}, L_LINEAR),
    "ApproxNDCG_coupled": ("ApproxNDCG", dict(alpha=10.0, presort=True, batch_coupled=True), L_SORTED),
    "ApproxNDCG_per_query": ("ApproxNDCG", dict(alpha=10.0, presort=False, batch_coupled=False), L_SORTED),
    "RankMSE": ("RankMSE", {}, L_LINEAR),
    "RankCosine": ("RankCosine", {}, L_LINEAR),
    "STListNet": ("STListNet", dict(temperature=1.0), L_LINEAR),
    "SoftRank_kNone": ("SoftRank", dict(delta=2.0, top_k=None), L_LINEAR),
    "SoftRank_k10": ("SoftRank", dict(delta=2.0, top_k=10), L_LINEAR),
    "WassRank_eg": ("WassRank", dict(cost_type="eg", lam=0.1, sh_itr=20), L_WASS),
    "WassRank_p1": ("WassRank", dict(cost_type="p1", lam=0.1, sh_itr=20), L_WASS),
    "WassRank_ddg": ("WassRank", dict(cost_type="ddg", lam=0.1, sh_itr=20), L_WASS),
}
SWEEP = [(c, n) for c, (_, _, lens) in CFGS.items() for n in lens]


def _batch(cfg, n):
    """B = 1 above 2048 documents (each float64 [B,n,n] temporary is 134 MB per query at 4096), 2 below; NDCG_Loss1 is
    defined per query (the reference's form holds for B = 1 only)."""
    return 1 if n > 2048 or cfg == "LambdaLoss1_k10" else 2


def _inputs(cfg, B, n, seed):
    """MSLR-WEB30K label marginals, at least one relevant document per query, labels sorted descending (shuffled for the
    presort=False configuration); the scores' spread alternates with the seed.  -> (s, y, extra) with extra the
    tie-shuffled ListMLE ordering or STListNet's uniforms ([B,n] numpy arrays)."""
    rng = np.random.default_rng(seed)
    y = rng.choice(5, size=(B, n), p=MSLR_P).astype(np.float32)
    if n:
        y[:, 0] = np.maximum(y[:, 0], 1.0)
    y = -np.sort(-y, axis=1)
    s = (rng.standard_normal((B, n)) * (1.0 if seed % 2 else 0.25)).astype(np.float32)
    name, params, _ = CFGS[cfg]
    extra = {}
    if name == "ApproxNDCG" and not params["presort"]:
        y = rng.permuted(y, axis=1)
    if name == "ListMLE":
        g = torch.Generator().manual_seed(seed)
        extra["perm"] = rp.shuffle_ties_perm(torch.from_numpy(y), generator=g).numpy().astype(np.int32)
    if name == "STListNet":
        extra["unif"] = rng.random((B, n), dtype=np.float32)
    return s, y, extra


def _params(cfg, over):
    name, params, _ = CFGS[cfg]
    return name, dict(params, **(over or {}))


def _kernel(cfg, s, y, extra, offsets=None, buckets=None, over=None):
    """-> (batch loss, loss per query, gradient) from the kernel; ``s``/``y`` are [B,n], or flat with ``offsets``.
    ``over``: parameters that replace the configuration's."""
    from ptranking_b200 import ops
    name, params = _params(cfg, over)
    kw = dict(params)
    for k, v in extra.items():
        kw[k] = torch.from_numpy(np.ascontiguousarray(v)).to(DEV)
    if offsets is not None:
        lens = np.diff(offsets)
        kw.update(offsets=torch.from_numpy(offsets).to(DEV), max_len=int(lens.max()), buckets=buckets)
    st = torch.from_numpy(np.ascontiguousarray(s)).to(DEV)
    yt = torch.from_numpy(np.ascontiguousarray(y)).to(DEV)
    loss, lq, g = ops.rank_loss_and_grad(name, st, yt, **kw)
    torch.cuda.synchronize()
    return float(loss), lq.cpu().numpy(), g.cpu().numpy()


def _f64(cfg, s, y, extra, over=None):
    """float64 closed form of the batch -> (loss summed over queries, gradient)."""
    name, params = _params(cfg, over)
    p = {k: v for k, v in params.items() if k not in ("presort", "batch_coupled")}
    if name == "RankNet":
        return cf.ranknet(s, y, **p)
    if name == "LambdaRank":
        return cf.lambdarank(s, y, **p)
    if name == "LambdaLoss":
        return cf.lambdaloss(s, y, presort=params["presort"], **p)
    if name == "ListNet":
        return cf.listnet(s, y)
    if name == "ListMLE":
        return cf.listmle(s, extra["perm"])
    if name == "ApproxNDCG":
        return cf.approxndcg(s, y, presort=params["presort"], batch_coupled=params["batch_coupled"], **p)
    if name == "RankMSE":
        return cf.rankmse(s, y)
    if name == "RankCosine":
        return cf.rankcosine(s, y)
    if name == "STListNet":
        return cf.stlistnet(s, y, extra["unif"], **p)
    if name == "SoftRank":
        return cf.softrank(s, y, **p)
    return wo.closed_form(s, y, **p)


def _port(cfg, s, y, extra):
    """fp32 ATen port of the reference -> (loss, gradient) as float / numpy."""
    name, params, _ = CFGS[cfg]
    if name == "WassRank":
        l, g = wo.port_loss_and_grad(torch.from_numpy(s), torch.from_numpy(y), **params)
        return float(l), g.numpy()
    kw = {k: v for k, v in params.items() if k != "batch_coupled"}
    if name == "ApproxNDCG" and not params["batch_coupled"]:      # the port couples a batch: run it query by query
        parts = [rp.loss_and_grad(name, torch.from_numpy(s[b:b + 1]), torch.from_numpy(y[b:b + 1]), **kw)
                 for b in range(s.shape[0])]
        return float(sum(l for l, _ in parts)), np.concatenate([g.numpy() for _, g in parts])
    if name == "ListMLE":
        kw["perm"] = torch.from_numpy(extra["perm"].astype(np.int64))
    if name == "STListNet":
        kw["unif"] = torch.from_numpy(extra["unif"])
    l, g = rp.loss_and_grad(name, torch.from_numpy(s), torch.from_numpy(y), **kw)
    return float(l), g.numpy()


def _check(tag, loss, grad, port, f64):
    """The bar of tests/test_gpu_losses.py; the message carries the kernel's and the port's distances from float64."""
    (pl, pg), (fl, fg) = port, f64
    k_l, k_g = abs(loss - fl) / max(abs(fl), 1.0), rel_err(grad, fg)
    p_l, p_g = abs(pl - fl) / max(abs(fl), 1.0), rel_err(pg, fg)
    msg = f"{tag}: from float64 kernel loss {k_l:.2e} grad {k_g:.2e}, port loss {p_l:.2e} grad {p_g:.2e}"
    print(msg)
    tol_l, tol_g = max(TOL, 2.0 * p_l), max(TOL, 2.0 * p_g)
    assert abs(loss - pl) <= tol_l * max(abs(pl), 1.0), msg
    assert rel_err(grad, pg) <= tol_g, msg
    assert k_l <= 5 * TOL and k_g <= 5 * TOL, msg


def _check_wass(tag, loss, grad, port, f64):
    """WassRank's bar (tests/test_gpu_wassrank.py): float64 within 5e-5 relative to the loss and to the largest gradient
    entry; the fp32 port referees where it is finite (it returns NaN where exp(-C/lam) underflows)."""
    (pl, pg), (fl, fg) = port, f64
    k_l = abs(loss - fl) / max(abs(fl), 1e-30)
    k_g = np.abs(grad - fg).max() / max(np.abs(fg).max(), 1e-30)
    msg = f"{tag}: from float64 kernel loss {k_l:.2e} grad {k_g:.2e}"
    if np.isfinite(pl) and np.isfinite(pg).all():
        p_l, p_g = abs(pl - fl) / max(abs(fl), 1e-30), rel_err(pg, fg)
        msg += f", port loss {p_l:.2e} grad {p_g:.2e}"
        assert abs(loss - pl) <= max(TOL, 2.0 * p_l) * max(abs(pl), 1.0), msg
        assert rel_err(grad, pg) <= max(TOL, 2.0 * p_g), msg
    print(msg)
    assert np.isfinite(loss) and np.isfinite(grad).all(), msg
    assert k_l <= TOL64 and k_g <= TOL64, msg


# --------------------------------------------------------------------------- #
# 1. dense sweep over every schedule boundary
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("cfg,n", SWEEP, ids=[f"{c}-{n}" for c, n in SWEEP])
def test_dense_lists_match_float64(cfg, n):
    B = _batch(cfg, n)
    s, y, extra = _inputs(cfg, B, n, seed=n + 7 * B)
    loss, lq, grad = _kernel(cfg, s, y, extra)
    check = _check_wass if CFGS[cfg][0] == "WassRank" else _check
    check(f"{cfg} B={B} n={n}", loss, grad, _port(cfg, s, y, extra), _f64(cfg, s, y, extra))
    assert abs(float(lq.sum()) - loss) <= 1e-5 * max(abs(loss), 1e-30 if CFGS[cfg][0] == "WassRank" else 1.0)


# --------------------------------------------------------------------------- #
# 2. one query under every schedule its launch can choose
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("cfg,n,partners", [("LambdaRank", 997, [1000, 1420, 1421, 2048, 2049, 4096]),
                                            ("RankNet", 1001, [1024, 1025])], ids=["LambdaRank", "RankNet"])
def test_one_query_under_every_schedule(cfg, n, partners):
    """A ragged launch sizes its CTAs and picks its kernel from its longest list.  The same query next to partners of
    different lengths runs under 1024 threads (one or two passes), 512 threads, or one thread per row over all pairs
    (LambdaRank), circulant or thread per row (RankNet), and must give the float64 answer and one answer under all."""
    s, y, extra = _inputs(cfg, 1, n, seed=5)
    f64, port = _f64(cfg, s, y, extra), _port(cfg, s, y, extra)
    got = []
    for P in partners:
        sp, yp, _ = _inputs(cfg, 1, P, seed=P)
        off = np.array([0, n, n + P], dtype=np.int32)
        _, lq, g = _kernel(cfg, np.concatenate([s[0], sp[0]]), np.concatenate([y[0], yp[0]]), {}, offsets=off)
        _check(f"{cfg} n={n} next to {P}", float(lq[0]), g[None, :n], port, f64)
        got.append((float(lq[0]), g[:n]))
    l0, g0 = got[0]
    for P, (l, g) in zip(partners, got):
        assert abs(l - l0) <= 1e-5 * max(abs(l0), 1.0), (P, l, l0)
        assert rel_err(g, g0) <= 1e-5, (P, rel_err(g, g0))


# --------------------------------------------------------------------------- #
# 3. a mixed ragged batch: one launch, and length buckets
# --------------------------------------------------------------------------- #
# every schedule's lengths, empty and one-document lists, and enough long and mid-length queries (8 per class) that
# length_buckets cuts the batch into several launches
MIXED = [4096, 0, 1, 2049, 33, 1421, 1025, 512, 513, 3000, 2, 800, 600, 500, 450, 400, 300, 256, 200, 130]


def _f64_query(cfg, sq, yq, eq, B, inv_idcg_total, over):
    """float64 (loss, grad) of one query of a ragged batch of B queries, with the batch couplings of ApproxNDCG (every
    query scaled by sum_a 1/iDCG_a), RankMSE and WassRank (1/B)."""
    name, params, _ = CFGS[cfg]
    l, g = _f64(cfg, sq[None], yq[None], {k: v[None] for k, v in eq.items()}, over)
    if name == "ApproxNDCG" and params["batch_coupled"]:
        scale = inv_idcg_total * float(cf._idcg(-np.sort(-yq[None].astype(np.float64), axis=1))[0])
        return l * scale, g[0] * scale
    if name in ("RankMSE", "WassRank"):
        return l / B, g[0] / B
    return l, g[0]


@pytest.mark.parametrize("cfg", list(CFGS))
def test_mixed_ragged_batch_single_launch_and_buckets(cfg):
    from ptranking_b200.data import length_buckets
    queries = [_inputs(cfg, 1, n, seed=1000 + i) for i, n in enumerate(MIXED)]
    B = len(MIXED)

    def flat(order):
        s = np.concatenate([queries[i][0][0] for i in order])
        y = np.concatenate([queries[i][1][0] for i in order])
        extra = {k: np.concatenate([queries[i][2][k][0] for i in order]) for k in queries[0][2]}
        off = np.zeros(len(order) + 1, dtype=np.int32)
        off[1:] = np.cumsum([MIXED[i] for i in order])
        return s, y, extra, off

    # one launch in the given order; the same queries sorted longest first (the order RaggedBatches uses) and cut into
    # length buckets, one launch each
    single = flat(range(B))
    desc = sorted(range(B), key=lambda i: -MIXED[i])
    bucketed = flat(desc)
    buckets = length_buckets([MIXED[i] for i in desc])
    assert len(buckets) >= 2
    # WassRank: 5 Sinkhorn iterations instead of 20 (the same code paths) keep its float64 form, 40 [n,n] log-sum-exps
    # per query at 20 iterations, within a few seconds for the 9.7k documents of this batch
    over = dict(sh_itr=5) if CFGS[cfg][0] == "WassRank" else None
    _, lq1, g1 = _kernel(cfg, single[0], single[1], single[2], offsets=single[3], over=over)
    _, lq2, g2 = _kernel(cfg, bucketed[0], bucketed[1], bucketed[2], offsets=bucketed[3], buckets=buckets, over=over)
    inv = sum(1.0 / float(cf._idcg(-np.sort(-q[1].astype(np.float64), axis=1))[0]) for q in queries if q[1].size)
    wass = CFGS[cfg][0] == "WassRank"
    for i, n in enumerate(MIXED):
        j = desc.index(i)
        a = g1[single[3][i]: single[3][i + 1]]
        c = g2[bucketed[3][j]: bucketed[3][j + 1]]
        if n == 0:
            assert lq1[i] == 0.0 and lq2[j] == 0.0
            continue
        sq, yq, eq = queries[i][0][0], queries[i][1][0], {k: v[0] for k, v in queries[i][2].items()}
        fl, fg = _f64_query(cfg, sq, yq, eq, B, inv, over)
        for tag, l, g in (("single", lq1[i], a), ("buckets", lq2[j], c)):
            k_l = abs(float(l) - fl) / max(abs(fl), 1e-30 if wass else 1.0)
            k_g = np.abs(g - fg).max() / max(np.abs(fg).max(), 1e-30)
            assert np.isfinite(l) and np.isfinite(g).all(), (tag, n)
            assert k_l <= TOL64 and (k_g <= TOL64 or np.abs(g - fg).max() <= 1e-7), (tag, n, k_l, k_g)
        assert abs(float(lq1[i]) - float(lq2[j])) <= 1e-5 * max(abs(float(lq1[i])), 1e-30 if wass else 1.0), (n, lq1[i], lq2[j])
        assert np.abs(a - c).max() <= 1e-5 * max(np.abs(a).max(), 1e-6) + 1e-9, (n, rel_err(c, a))


def test_mixed_ragged_batch_metrics():
    from ptranking_b200 import ops
    from ptranking_b200.data import length_buckets
    rng = np.random.default_rng(12)
    desc = sorted(MIXED, reverse=True)
    S = [rng.standard_normal(n).astype(np.float32) for n in desc]
    Y = [rng.choice(5, size=n, p=MSLR_P).astype(np.float32) for n in desc]      # unsorted: the kernels sort the ideal list
    for yq in Y:
        if len(yq):
            yq[rng.integers(len(yq))] = 1.0 + rng.integers(4)        # one relevant document at least (iDCG > 0)
    off = np.zeros(len(desc) + 1, dtype=np.int32)
    off[1:] = np.cumsum(desc)
    s = torch.from_numpy(np.concatenate(S)).to(DEV)
    y = torch.from_numpy(np.concatenate(Y)).to(DEV)
    offd = torch.from_numpy(off).to(DEV)
    ks = [1, 3, 10, 100, 1025, 3000, 4096]
    buckets = length_buckets(desc)
    assert len(buckets) >= 2
    kw = dict(presort=False, offsets=offd, max_len=max(desc))
    nd, order = ops.ndcg_at_ks(s, y, ks, return_order=True, **kw)
    nd_b, order_b = ops.ndcg_at_ks(s, y, ks, return_order=True, buckets=buckets, **kw)
    m = ops.adhoc_metrics_at_ks(s, y, ks, max_label=4.0, **kw)
    m_b = ops.adhoc_metrics_at_ks(s, y, ks, max_label=4.0, buckets=buckets, **kw)
    assert torch.equal(nd, nd_b) and torch.equal(order, order_b) and all(torch.equal(a, c) for a, c in zip(m, m_b))
    nd, order = nd.cpu().numpy(), order.cpu().numpy()
    m = [t.cpu().numpy() for t in m]
    for b, (sq, yq) in enumerate(zip(S, Y)):
        if len(sq) == 0:
            assert not nd[b].any() and not any(t[b].any() for t in m)
            continue
        st, yt = torch.from_numpy(sq)[None], torch.from_numpy(yq)[None]
        assert np.array_equal(order[off[b]: off[b + 1]], torch.sort(st[0], descending=True, stable=True)[1].numpy())
        want = rp.evaluator_metrics_at_ks(st, yt, ks, presort=False, max_label=4.0)
        assert np.abs(nd[b] - want[0].numpy()[0]).max() <= 1e-6, (len(sq), nd[b], want[0])
        for got, w in zip(m, want):
            assert np.abs(got[b] - w.numpy()[0]).max() <= 1e-6, (len(sq), got[b], w)


# --------------------------------------------------------------------------- #
# 4. sort-dependent outputs at 4096 keys
# --------------------------------------------------------------------------- #
def test_ndcg_order_is_the_stable_sort_at_4096():
    """Scores rounded to one decimal: thousands of exact ties, so the index tie-break of the 4096-key sort decides the
    order, which must be torch.sort(stable=True)'s bit for bit."""
    from ptranking_b200 import ops
    rng = np.random.default_rng(21)
    B, n = 2, MAX_LEN
    s = np.round(rng.standard_normal((B, n)), 1).astype(np.float32)
    y = rng.choice(5, size=(B, n), p=MSLR_P).astype(np.float32)
    ks = [1, 10, 1000, 4095, 4096, 4097]
    out, order = ops.ndcg_at_ks(torch.from_numpy(s).to(DEV), torch.from_numpy(y).to(DEV), ks, presort=False, return_order=True)
    want_order = torch.sort(torch.from_numpy(s), dim=1, descending=True, stable=True)[1]
    assert np.array_equal(order.cpu().numpy(), want_order.numpy().astype(np.int32))
    sys_r = torch.gather(torch.from_numpy(y), 1, want_order)
    want = rp.ndcg_at_ks(sys_r, torch.sort(torch.from_numpy(y), dim=1, descending=True)[0], ks).numpy()
    assert np.abs(out.cpu().numpy() - want).max() <= 1e-6
    assert np.all(out.cpu().numpy()[:, -1] == 0.0)


@pytest.mark.parametrize("presort", [True, False])
def test_adhoc_metrics_at_4096(presort):
    """nDCG, nERR, AP and P at 32 cutoffs (the most one call takes), including n and n + 1, against the port."""
    from ptranking_b200 import ops
    rng = np.random.default_rng(22 + presort)
    B, n = 2, MAX_LEN
    s = rng.standard_normal((B, n)).astype(np.float32)
    y = rng.choice(5, size=(B, n), p=MSLR_P).astype(np.float32)
    y[:, 0] = 4.0
    if presort:
        y = -np.sort(-y, axis=1)
    ks = [1, 2, 3, 4, 5, 7, 10, 15, 20, 30, 50, 64, 100, 128, 200, 256, 300, 500, 512, 1000, 1024, 1025, 1500, 2000,
          2047, 2048, 2049, 3000, 4000, 4095, 4096, 4097]
    assert len(ks) == 32
    got = ops.adhoc_metrics_at_ks(torch.from_numpy(s).to(DEV), torch.from_numpy(y).to(DEV), ks, presort=presort)
    want = rp.evaluator_metrics_at_ks(torch.from_numpy(s), torch.from_numpy(y), ks, presort=presort)
    for name, g, w in zip(("nDCG", "nERR", "AP", "P"), got, want):
        g, w = g.cpu().numpy(), w.numpy()
        assert np.abs(g - w).max() <= 1e-6, (name, np.abs(g - w).max())
        assert np.all(g[:, -1] == 0.0), name


def test_shuffle_ties_perm_at_4096():
    from ptranking_b200 import ops
    rng = np.random.default_rng(23)
    B, n = 3, MAX_LEN
    y = rng.choice(5, size=(B, n), p=MSLR_P).astype(np.float32)
    y[1] = -np.sort(-y[1])
    y[2] = 0.0                                               # one tie group of 4096: the order is the noise alone
    yt = torch.from_numpy(y).to(DEV)
    p1 = ops.shuffle_ties_perm(yt, seed=4, offset=1).cpu().numpy()
    p1b = ops.shuffle_ties_perm(yt, seed=4, offset=1).cpu().numpy()
    p2 = ops.shuffle_ties_perm(yt, seed=4, offset=2).cpu().numpy()
    assert np.array_equal(p1, p1b)
    for p in (p1, p2):
        assert np.array_equal(np.sort(p, axis=1), np.tile(np.arange(n), (B, 1)))       # a permutation, up to index 4095
        assert np.all(np.diff(np.take_along_axis(y, p.astype(np.int64), 1), axis=1) <= 0)
    for b in range(B):
        assert not np.array_equal(p1[b], p2[b])
    assert not np.array_equal(p1[2], np.arange(n))
    # ragged: a list of 4096 behind a short one, positions within each list
    off = torch.tensor([0, 5, 5 + n], dtype=torch.int32, device=DEV)
    yr = torch.cat([torch.zeros(5, device=DEV), yt[0]])
    pr = ops.shuffle_ties_perm(yr, seed=4, offset=1, offsets=off, max_len=n).cpu().numpy()
    assert np.array_equal(np.sort(pr[5:]), np.arange(n)) and np.array_equal(np.sort(pr[:5]), np.arange(5))
    assert np.all(np.diff(y[0][pr[5:].astype(np.int64)]) <= 0)


# --------------------------------------------------------------------------- #
# 5. full-size properties on long lists
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("name,B,n", [("LambdaRank", 64, 4096), ("RankNet", 64, 4096), ("LambdaRank", 128, 1500)],
                         ids=["LambdaRank-64x4096", "RankNet-64x4096", "LambdaRank-128x1500"])
def test_full_size_properties_long_lists(name, B, n):
    cfg = name
    s, y, extra = _inputs(cfg, B, n, seed=B + n)
    _, lq, g = _kernel(cfg, s, y, extra)
    _, lq2, g2 = _kernel(cfg, s, y, extra)
    assert np.array_equal(g, g2) and np.array_equal(lq, lq2)                 # bit-identical reruns
    assert np.isfinite(g).all() and np.isfinite(lq).all()
    assert np.abs(g.sum(1)).max() <= 2e-4 * max(np.abs(g).max(), 1e-12) * np.sqrt(n)
    _, lqs, gs = _kernel(cfg, s[:3], y[:3], extra)
    assert np.array_equal(gs, g[:3]) and np.array_equal(lqs, lq[:3])       # queries are independent


# --------------------------------------------------------------------------- #
# 6. the list-length limit
# --------------------------------------------------------------------------- #
ENTRY = list({name: cfg for cfg, (name, _, _) in reversed(list(CFGS.items()))}.values())[::-1] + \
    ["shuffle_ties", "ndcg_at_ks", "adhoc_metrics_at_ks"]          # the first configuration of every loss


def _call_entry(entry, s, y, **layout):
    from ptranking_b200 import ops
    if entry == "shuffle_ties":
        return [ops.shuffle_ties_perm(y, seed=1, offset=1, **layout)]
    if entry == "ndcg_at_ks":
        return list(ops.ndcg_at_ks(s, y, [1, 10], return_order=True, **layout))
    if entry == "adhoc_metrics_at_ks":
        return list(ops.adhoc_metrics_at_ks(s, y, [1, 10], max_label=4.0, **layout))
    name, params, _ = CFGS[entry]
    kw = dict(params)
    if name == "ListMLE":
        kw["perm"] = torch.zeros(s.shape, dtype=torch.int32, device=DEV)
    if name == "STListNet":
        kw["unif"] = torch.full(s.shape, 0.5, device=DEV)
    return list(ops.rank_loss_and_grad(name, s, y, **kw, **layout))


@pytest.mark.parametrize("entry", ENTRY)
def test_list_length_limit(entry):
    """4096 documents are accepted, 4097 refused with the PTRB200_MAX_LIST_LEN message, as a dense [B,n] batch and as a
    ragged batch's max_len (the offsets describe one list of that length, so nothing is read out of bounds either way)."""
    from ptranking_b200 import _lib
    for n in (MAX_LEN, MAX_LEN + 1):
        rng = np.random.default_rng(n)
        y = torch.from_numpy(-np.sort(-rng.choice(5, size=(1, n), p=MSLR_P).astype(np.float32), axis=1)).to(DEV)
        y[0, 0] = 4.0
        s = torch.from_numpy(rng.standard_normal((1, n)).astype(np.float32)).to(DEV)
        off = torch.tensor([0, n], dtype=torch.int32, device=DEV)
        for layout, (sa, ya) in ((dict(), (s, y)), (dict(offsets=off, max_len=n), (s[0], y[0]))):
            if n <= MAX_LEN:
                out = _call_entry(entry, sa, ya, **layout)
                torch.cuda.synchronize()
                assert all(torch.isfinite(t.float()).all() for t in out), layout
            else:
                with pytest.raises(_lib.B200LibraryError, match="PTRB200_MAX_LIST_LEN"):
                    _call_entry(entry, sa, ya, **layout)


# --------------------------------------------------------------------------- #
# 7. a query without relevant documents (iDCG = 0)
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("partner", [1000, 3000])
def test_lambdarank_all_zero_query_does_not_depend_on_its_launch(partner):
    """Every normalised gain of an all-zero query is 0/0 and every pair ties.  Tie pairs are skipped on every schedule,
    so the query's loss and gradient are exactly zero whether its launch runs the runs kernel (longest list 1000) or the
    thread-per-row kernel (longest list 3000); the partner query is unaffected."""
    cfg, n = "LambdaRank", 700
    sp, yp, _ = _inputs(cfg, 1, partner, seed=partner)
    s0 = np.random.default_rng(3).standard_normal(n).astype(np.float32)
    off = np.array([0, n, n + partner], dtype=np.int32)
    _, lq, g = _kernel(cfg, np.concatenate([s0, sp[0]]), np.concatenate([np.zeros(n, np.float32), yp[0]]), {}, offsets=off)
    assert lq[0] == 0.0 and not g[:n].any(), (lq[0], np.abs(g[:n]).max())
    _check(f"partner n={partner}", float(lq[1]), g[None, n:], _port(cfg, sp, yp, {}), _f64(cfg, sp, yp, {}))
    # and all-zero lists alone in dense launches of both schedules
    for m in (n, 3000):
        s1 = np.random.default_rng(m).standard_normal((1, m)).astype(np.float32)
        _, lq1, g1 = _kernel(cfg, s1, np.zeros((1, m), np.float32), {})
        assert lq1[0] == 0.0 and not g1.any(), (m, lq1[0])
