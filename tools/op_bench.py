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

tag = sys.argv[1] if len(sys.argv) > 1 else "r02"
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
]:
    for (B, n) in shapes:
        s = torch.sigmoid(torch.randn(B, n, device=dev))
        y = labels(B, n)
        kw = dict(params)
        if name == "ListMLE":
            kw["perm"] = ops.shuffle_ties_perm(y, seed=1, offset=1)
        if name == "STListNet":
            kw.update(seed=1, offset=1)
        ms = timeit(lambda: ops.rank_loss_and_grad(name, s, y, **kw))
        algo = (16 if name == "ListMLE" else 12) * n * B
        rows.append((f"{name} {params.get('loss_type', '')} {('k=%d' % params['k']) if 'k' in params else ''}".strip(), f"B={B} n={n}",
                     ms, B / ms * 1e3, algo / ms / 1e6, algo / ms / 1e6 / HBM))
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
