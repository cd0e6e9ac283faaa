"""Per-op timings at BASELINE.json's config sizes (CUDA events, warm, 20 iterations) -> profiles/<tag>_op_table.md.
Not the headline bench: explains it (loss-only throughput, scorer forward/backward, metric kernel)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
import ptranking_b200
from ptranking_b200 import ops, LABEL_TYPE

args = [a for a in sys.argv[1:] if not a.startswith("--")]
tag = args[0] if args else "r02"
dev = "cuda:0"
rng = np.random.default_rng(137)
rows = []


def timeit(fn, iters=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def labels(B, n):
    y = rng.choice(5, size=(B, n), p=bench.MSLR_P).astype(np.float32)
    y[:, 0] = np.maximum(y[:, 0], 1)
    return torch.from_numpy(-np.sort(-y, axis=1)).to(dev)


HBM = bench.measured_peaks()["hbm_gbs"]

def divprob_rows():
    """DivProbRanker's fused loss kernel against an ATen restatement of the reference's loss (tests/divprob_oracle.py's
    fp32 port: head, [m, n, n] temporaries, autograd) on the same GPU: 64 queries of n documents, m = 8 subtopic rows,
    K = 1 and limit_delta = 0.01 (the reference's defaults).  The kernel takes the 64 queries in one launch; the
    restatement runs them one query at a time, as the reference's training loop does."""
    from tests import divprob_oracle as dpo
    out = []
    B, m = 64, 8
    for n in (50, 300, 1000):
        raws = [torch.from_numpy(dpo.draw_raw(rng, n, 1, 0.01, True)).to(dev) for _ in range(B)]
        mats = [torch.from_numpy((rng.random((m, n)) < 0.2).astype(np.float32)).to(dev) for _ in range(B)]
        u = torch.stack(raws)
        rele = ops.SubtopicRele.pack([R.cpu() for R in mats], dev)
        for loss in dpo.LOSSES:
            opt_id, metric = ("SuperSoft", loss) if loss in ("aNDCG", "nERR-IA") else (loss, None)
            kw = dict(K=1, limit_delta=0.01, top_k=None, norm=True)
            ms_k = timeit(lambda: ops.divprob_loss_and_grad(u, rele, opt_id=opt_id, metric=metric, **kw))

            def aten():
                for q in range(B):
                    leaf = raws[q].unsqueeze(0).clone().requires_grad_(True)
                    mus, vars = dpo.port_head(leaf, 1, 0.01)
                    dpo.port_loss(mus, vars, mats[q], loss, None, True).backward()
            ms_a = timeit(aten, iters=3, warm=1)
            out.append((f"DivProbRanker {loss} K=1 limit 0.01: fused kernel", f"B={B} n={n} m={m}", ms_k, B / ms_k * 1e3,
                        float('nan'), float('nan')))
            out.append((f"DivProbRanker {loss}: ATen restatement, one query per call (x{ms_a / ms_k:.0f})",
                        f"B={B} n={n} m={m}", ms_a, B / ms_a * 1e3, float('nan'), float('nan')))
    return out


if "--divprob" in sys.argv:
    print(f"{torch.cuda.get_device_name()}")
    print("| op | shape | ms | queries/s |\n|---|---|---|---|")
    for name, shape, ms, qps, _, _ in divprob_rows():
        print(f"| {name} | {shape} | {ms:.4f} | {qps:,.0f} |")
    sys.exit(0)

for name, params, shapes in [
    ("LambdaRank", dict(sigma=1.0), [(1024, 256), (256, 1024), (4096, 32)]),
    ("RankNet", dict(sigma=1.0), [(1024, 256)]),
    ("LambdaLoss", dict(k=5, sigma=1.0, mu=5.0, loss_type="NDCG_Loss2++"), [(1024, 256), (256, 1024)]),
    ("LambdaLoss", dict(k=1024, sigma=1.0, mu=5.0, loss_type="NDCG_Loss2++"), [(256, 1024)]),
    ("ListNet", {}, [(1024, 256), (256, 1024)]),
    ("ListMLE", {}, [(4096, 32), (1024, 256), (256, 1024)]),
    ("ApproxNDCG", dict(alpha=10.0), [(1024, 256), (512, 512)]),
    ("SoftRank", dict(delta=2.0, top_k=None), [(1024, 256), (256, 1024)]),
    ("STListNet", dict(temperature=1.0), [(1024, 256), (4096, 32)]),
    ("RankCosine", {}, [(1024, 256)]),
    ("RankMSE", {}, [(1024, 256)]),
    ("WassRank", dict(cost_type="eg"), [(1024, 256), (256, 1024)]),      # default settings: label-group schedule
    ("WassRank", dict(cost_type="ddg"), [(1024, 256)]),                  # O(n^2) walks
    ("WassRank", dict(cost_type="p1"), [(256, 1024)]),
    ("MDPRank", dict(distribution="PL", top_k=10), [(1024, 256), (256, 1024), (64, 4096)]),
    ("MDPRank", dict(distribution="PL", top_k=None), [(1024, 256), (256, 1024), (64, 4096)]),
    ("MDPRank", dict(distribution="STPL", top_k=10), [(1024, 256), (256, 1024), (64, 4096)]),
    ("MDPRank", dict(distribution="STPL", top_k=None), [(1024, 256), (256, 1024), (64, 4096)]),
]:
    for (B, n) in shapes:
        s = torch.sigmoid(torch.randn(B, n, device=dev))
        y = labels(B, n)
        kw = dict(params)
        if name == "ListMLE":
            kw["perm"] = ops.shuffle_ties_perm(y, seed=1, offset=1)
        if name in ("STListNet", "MDPRank"):
            kw.update(seed=1, offset=1)
        ms = timeit(lambda: ops.rank_loss_and_grad(name, s, y, **kw))
        algo = (16 if name == "ListMLE" else 12) * n * B
        tag = params.get('loss_type', params.get('cost_type', params.get('distribution', '')))
        if name == "MDPRank":
            tag += " k=%s" % (params['top_k'] or "n")
        rows.append((f"{name} {tag} {('k=%d' % params['k']) if 'k' in params else ''}".strip(), f"B={B} n={n}",
                     ms, B / ms * 1e3, algo / ms / 1e6, algo / ms / 1e6 / HBM))
# DALETOR (diversification): m = 8 subtopic rows of 0/1 relevance per query, rt 10, top_k 10 (the reference's defaults)
for (B, n) in [(1024, 256), (64, 4096)]:
    s = torch.randn(B, n, device=dev)
    rele = ops.SubtopicRele.pack([torch.from_numpy((rng.random((8, n)) < 0.2).astype(np.float32)) for _ in range(B)], dev)
    ms = timeit(lambda: ops.daletor_loss_and_grad(s, rele, rt=10.0, top_k=10))
    algo = (12 + 8 * 4) * n * B
    rows.append(("DALETOR m=8 k=10", f"B={B} n={n}", ms, B / ms * 1e3, algo / ms / 1e6, algo / ms / 1e6 / HBM))
    ms = timeit(lambda: ops.srd_metrics_at_ks(s, rele, [1, 3, 5, 10, 20], max_label=1.0))
    rows.append(("alpha-nDCG+ERR-IA+nERR-IA @5 cutoffs m=8", f"B={B} n={n}", ms, B / ms * 1e3, algo / ms / 1e6, algo / ms / 1e6 / HBM))
rows += divprob_rows()
# ndcg / all metrics
for (B, n) in [(1024, 256), (256, 1024)]:
    s = torch.randn(B, n, device=dev); y = labels(B, n)
    ms = timeit(lambda: ops.adhoc_metrics_at_ks(s, y, [1, 3, 5, 10, 20, 50], presort=True, max_label=4.0))
    rows.append(("nDCG+nERR+AP+P @6 cutoffs", f"B={B} n={n}", ms, B / ms * 1e3, 8 * n * B / ms / 1e6, 8 * n * B / ms / 1e6 / HBM))

# ragged batches: an MSLR-WEB30K-shaped length distribution (1..1251 documents, mean ~120) against uniform lists with
# the same number of documents, loss kernel alone and the whole training step (SURVEY 8f-2)
lens = np.clip(rng.lognormal(mean=4.45, sigma=0.85, size=4096), 1, 1251).astype(np.int64)
take = int(np.searchsorted(np.cumsum(lens), 1 << 18))
lens = np.sort(lens[:take])[::-1].copy()          # data.RaggedBatches orders a batch by length, longest first
from ptranking_b200.data import length_buckets
buckets = length_buckets(lens)
off = np.zeros(len(lens) + 1, dtype=np.int32); off[1:] = np.cumsum(lens)
total = int(off[-1])
yr = np.concatenate([-np.sort(-np.maximum(rng.choice(5, size=n_, p=bench.MSLR_P), (np.arange(n_) == 0).astype(np.int64)).astype(np.float32)) for n_ in lens])
s_r = torch.sigmoid(torch.randn(total, device=dev)); y_r = torch.from_numpy(yr).to(dev); off_d = torch.from_numpy(off).to(dev)
for name, params in [("LambdaRank", dict(sigma=1.0)), ("ListNet", {}), ("ApproxNDCG", dict(alpha=10.0))]:
    ms = timeit(lambda: ops.rank_loss_and_grad(name, s_r, y_r, offsets=off_d, max_len=int(lens.max()), **params))
    rows.append((f"{name} RAGGED one launch (lens 1..{int(lens.max())}, mean {lens.mean():.0f})", f"B={len(lens)} docs={total}", ms, len(lens) / ms * 1e3,
                 12 * total / ms / 1e6, 12 * total / ms / 1e6 / HBM))
    ms = timeit(lambda: ops.rank_loss_and_grad(name, s_r, y_r, offsets=off_d, max_len=int(lens.max()), buckets=buckets, **params))
    rows.append((f"{name} RAGGED {len(buckets)} length buckets", f"B={len(lens)} docs={total}", ms, len(lens) / ms * 1e3,
                 12 * total / ms / 1e6, 12 * total / ms / 1e6 / HBM))
Xs = torch.randn(total, 136, device=dev)
ms = timeit(lambda: ops.standard_scale(Xs, offsets=off_d, max_len=int(lens.max())))
rows.append(("per-query StandardScaler (ragged)", f"B={len(lens)} docs={total}", ms, len(lens) / ms * 1e3, 8 * 136 * total / ms / 1e6, 8 * 136 * total / ms / 1e6 / HBM))

# scorer forward / forward+backward (default pointsf) and full step
sf = bench.point_sf(136)
r = ptranking_b200.LambdaRank(sf_para_dict=sf, model_para_dict=dict(model_id="LambdaRank", sigma=1.0), gpu=True, device=dev)
r.init(); r.train_mode()
for (B, n) in [(1024, 256), (256, 1024), (4096, 32)]:
    X, y = bench.synth_batch(rng, B, n, 136, bench.MSLR_P)
    X, y = X.to(dev), y.to(dev)
    with torch.no_grad():
        ms_f = timeit(lambda: r.forward(X))
    ms_s = timeit(lambda: r.train_op(X, y, presort=True, label_type=LABEL_TYPE.MultiLabel, epoch_k=1))
    algo = n * B * (136 * 4 + 8)
    rows.append(("pointsf forward (5x100 GELU BN)", f"B={B} n={n}", ms_f, B / ms_f * 1e3, algo / ms_f / 1e6, algo / ms_f / 1e6 / HBM))
    rows.append(("LambdaRank train step (fwd+loss+bwd+Adam)", f"B={B} n={n}", ms_s, B / ms_s * 1e3, algo / ms_s / 1e6, algo / ms_s / 1e6 / HBM))
    if (B, n) == (1024, 256):       # the same step with WassRank's default settings (eg cost, lam 0.1, 20 iterations)
        rw = ptranking_b200.WassRank(sf_para_dict=sf, wass_para_dict=None, dict_cost_mats={}, dict_std_dists={}, gpu=True, device=dev)
        rw.init(); rw.train_mode()
        ms_w = timeit(lambda: rw.train_op(X, y, presort=True, label_type=LABEL_TYPE.MultiLabel, epoch_k=1))
        rows.append(("WassRank train step (fwd+loss+bwd+Adam)", f"B={B} n={n}", ms_w, B / ms_w * 1e3, algo / ms_w / 1e6, algo / ms_w / 1e6 / HBM))
        # and with MDPRank's default settings (PL, top_k 10, gamma 1, T 1)
        rm = ptranking_b200.MDPRank(sf_para_dict=sf, model_para_dict=dict(model_id="MDPRank", temperature=1.0, gamma=1.0, top_k=10,
                                                                          distribution="PL"), gpu=True, device=dev)
        rm.init(); rm.train_mode()
        ms_m = timeit(lambda: rm.train_op(X, y, presort=True, label_type=LABEL_TYPE.MultiLabel, epoch_k=1))
        rows.append(("MDPRank train step (fwd+loss+bwd+Adam)", f"B={B} n={n}", ms_m, B / ms_m * 1e3, algo / ms_m / 1e6, algo / ms_m / 1e6 / HBM))
# DALETOR with the default diversification pointsf (F = 100, so 300 inputs; 5 x 100 GELU, per-query BN; Adagrad): the
# reference's one query per step, and 1024 queries in one ragged step (queries_per_step = 1024)
sfd = dict(sf_id="pointsf", opt="Adagrad", lr=0.001, pointsf=dict(num_features=100, num_layers=5, AF="GE", TL_AF="GE",
                                                                  apply_tl_af=False, BN=True, bn_type="BN", bn_affine=True))
rd = ptranking_b200.DALETOR(sf_para_dict=sfd, model_para_dict=dict(model_id="DALETOR", rt=10.0, top_k=10), gpu=True, device=dev)
rd.init(); rd.train_mode()
for (B, n) in [(1, 256), (1024, 256)]:
    Xd = torch.randn(B * n, 300, device=dev)
    rele = ops.SubtopicRele.pack([torch.from_numpy((rng.random((8, n)) < 0.2).astype(np.float32)) for _ in range(B)], dev)
    offd = torch.arange(0, (B + 1) * n, n, dtype=torch.int32, device=dev)
    if B == 1:
        step = lambda: rd.div_custom_loss_function(rd.point_sf(Xd.view(1, n, 300)).view(1, -1), rele, presort=True)
    else:
        step = lambda: rd.div_custom_loss_function(rd.div_forward_ragged(Xd, offd, n), rele, presort=True, offsets=offd, max_len=n)
    ms_d = timeit(step)
    algo = B * n * (300 * 4 + 8)
    rows.append(("DALETOR train step (pointsf 300->5x100, per-query BN, Adagrad)", f"B={B} n={n}", ms_d, B / ms_d * 1e3,
                 algo / ms_d / 1e6, algo / ms_d / 1e6 / HBM))
# the same step on the ragged batch (batch-level BN: one long list to the scorer, per-query offsets to the loss)
Xr = torch.randn(total, 136, device=dev)
ms_s = timeit(lambda: r.train_op(Xr, y_r, presort=True, label_type=LABEL_TYPE.MultiLabel, epoch_k=1, offsets=off_d, max_len=int(lens.max()), buckets=buckets))
algo = total * (136 * 4 + 8)
rows.append((f"LambdaRank train step RAGGED (lens 1..{int(lens.max())})", f"B={len(lens)} docs={total}", ms_s, len(lens) / ms_s * 1e3, algo / ms_s / 1e6, algo / ms_s / 1e6 / HBM))
rows.append(("   -> documents/s ragged vs uniform 1024x256", "", float('nan'), total / ms_s * 1e3, float('nan'), float('nan')))

# list scorer (DASALC, 2 heads) forward + step, config (c) shape
for L in (3, 6):
    sfl = dict(sf_id="listsf", opt="Adagrad", lr=1e-3,
               listsf=dict(num_features=136, ff_dims=[128, 256, 512], AF="R", TL_AF="GE", apply_tl_af=False, BN=False, bn_type="BN2",
                           bn_affine=False, n_heads=2, encoder_layers=L, encoder_type="DASALC"))
    rl = ptranking_b200.ApproxNDCG(sf_para_dict=sfl, model_para_dict=dict(model_id="ApproxNDCG", alpha=10.0), gpu=True, device=dev)
    rl.init(); rl.train_mode()
    B, n = 64, 512
    X, y = bench.synth_batch(rng, B, n, 136, bench.MSLR_P)
    X, y = X.to(dev), y.to(dev)
    ms_s = timeit(lambda: rl.train_op(X, y, presort=True, label_type=LABEL_TYPE.MultiLabel, epoch_k=1), iters=5, warm=2)
    flops = 3 * n * (865280 + L * (147968 + 4 * n * 136)) * B
    rows.append((f"ApproxNDCG + listsf DASALC L={L} train step", f"B={B} n={n}", ms_s, B / ms_s * 1e3, flops / ms_s / 1e9, float('nan')))
    if L == 3:      # per-kernel breakdown of this step (CUDA events around every launch of the library; serialised)
        from ptranking_b200 import _lib
        _lib.kernel_timings(enable=True)
        for _ in range(2):
            rl.train_op(X, y, presort=True, label_type=LABEL_TYPE.MultiLabel, epoch_k=1)
        torch.cuda.synchronize()
        listsf_kernels = {k: (v[0] / 2, v[1] / 2) for k, v in _lib.kernel_timings().items()}
        _lib.kernel_timings(enable=False)
        # the same number of documents as lists of different lengths (MSLR-shaped, capped at 512): one padded batch, and
        # the batch cut into RaggedBatches' length classes, each padded to its own longest list
        ll = np.clip(rng.lognormal(mean=4.45, sigma=0.85, size=2048), 1, 512).astype(np.int64)
        ll = np.sort(ll[: int(np.searchsorted(np.cumsum(ll), B * n))])[::-1].copy()
        lo = np.zeros(len(ll) + 1, dtype=np.int32); lo[1:] = np.cumsum(ll)
        tot_l = int(lo[-1])
        Xl = torch.randn(tot_l, 136, device=dev)
        yl = torch.from_numpy(np.concatenate([-np.sort(-rng.choice(5, size=int(n_), p=bench.MSLR_P).astype(np.float32)) for n_ in ll])).to(dev)
        lo_d = torch.from_numpy(lo).to(dev)
        for label, bk in (("one padded batch", None), (f"{len(length_buckets(ll, edges=(64, 192)))} length classes", length_buckets(ll, edges=(64, 192)))):
            ms_r = timeit(lambda: rl.train_op(Xl, yl, presort=True, label_type=LABEL_TYPE.MultiLabel, epoch_k=1, offsets=lo_d,
                                              max_len=int(ll.max()), buckets=bk), iters=5, warm=2)
            rows.append((f"ApproxNDCG + listsf DASALC L={L} train step RAGGED, {label} (lens 1..{int(ll.max())}, mean {ll.mean():.0f})",
                         f"B={len(ll)} docs={tot_l}", ms_r, len(ll) / ms_r * 1e3, float('nan'), float('nan')))
        rows.append((f"   -> documents/s ragged (length classes); uniform 64x512: {B * n / ms_s * 1e3:,.0f}", "", float('nan'), tot_l / ms_r * 1e3, float('nan'), float('nan')))

os.makedirs("profiles", exist_ok=True)
with open(f"profiles/{tag}_op_table.md", "w") as f:
    f.write(f"# {tag}: per-op timings on one {torch.cuda.get_device_name()} (CUDA events, 20 warm iterations; `tools/op_bench.py`)\n\n")
    f.write("GB/s = ALGORITHMIC bytes (12n per query for a loss, n(4F+8) for the scorer) / time; frac = of the measured copy bandwidth "
            f"({HBM:.0f} GB/s).  For the list scorer the last-but-one column is GFLOP/s (algorithmic fwd+bwd FLOPs).\n\n")
    f.write("| op | shape | ms | queries/s | GB/s (GFLOP/s) | frac of HBM |\n|---|---|---|---|---|---|\n")
    for name, shape, ms, qps, gbs, frac in rows:
        f.write(f"| {name} | {shape} | {ms:.4f} | {qps:,.0f} | {gbs:,.1f} | {frac:.4f} |\n")
    f.write("\n## kernels of one ApproxNDCG + listsf DASALC L=3 step (B=64, n=512; launches and ms per step)\n\n| kernel | launches | ms |\n|---|---|---|\n")
    for k, (c, ms) in sorted(listsf_kernels.items(), key=lambda kv: -kv[1][1]):
        f.write(f"| `{k}` | {c:.0f} | {ms:.4f} |\n")
print(open(f"profiles/{tag}_op_table.md").read())
