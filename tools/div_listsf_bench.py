"""Time DALETOR with the diversification list scorer at the reference default (AttnDIN, 6 heads, 6 layers, F = 100, so
the encoder is 300 wide with 50-wide heads; uni_sf [600, 256, 128, 64, 1]):

* the train step (forward, DALETOR loss, backward, Adagrad) for one 256-document query, the reference's one query per
  step, and for 64 x 256 and 16 x 1024 documents in one ragged step;
* evaluation of a 200-query split (one scorer pass, one metric launch).

CUDA events after warm-up; the card's name and power limit are read in the same run.  ``--profile`` adds a separate
torch.profiler run of the 256-document step and the 64 x 256 step and prints the share of CUDA time per kernel group:
attention GEMMs, softmax, FF / linear kernels, LayerNorm, the new list-scorer kernels, the loss, the rest.

    python tools/div_listsf_bench.py [--heads 6] [--profile] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

DEV = "cuda:0"
F = 100
LISTSF = dict(encoder_type="AttnDIN", n_heads=6, encoder_layers=6, ff_dims=[256, 128, 64], AF="R", TL_AF="GE",
              apply_tl_af=False, BN=True, bn_type="BN", bn_affine=True)


def card():
    name = torch.cuda.get_device_name()
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def split(rng, lens, m=6):
    data = []
    for i, n in enumerate(lens):
        R = (rng.random((m, n)) < 0.2).astype(np.float32)
        R[0, 0] = 1.0
        data.append((f"q{i}", torch.from_numpy(rng.standard_normal((1, F)).astype(np.float32)), [""] * n,
                     torch.from_numpy(rng.standard_normal((n, F)).astype(np.float32)), None, None, torch.from_numpy(R)))
    return data


def ranker(heads):
    from ptranking_b200 import DALETOR
    sf = dict(sf_id="listsf", opt="Adagrad", lr=0.01, listsf=dict(num_features=F, **dict(LISTSF, n_heads=heads)))
    r = DALETOR(sf_para_dict=sf, model_para_dict=dict(model_id="DALETOR", rt=10.0, top_k=10), gpu=True, device=DEV)
    r.init()
    return r


def time_epoch(r, data, qps, reps):
    """ms per div_train step over ``reps`` epochs of ``data`` (every query counted), after one warm-up epoch."""
    r.queries_per_step = qps
    r.div_train(data, epoch_k=1)
    torch.cuda.synchronize()
    steps = len(r._split(data).steps(qps))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        r.div_train(data, epoch_k=1)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / (reps * steps)


def time_eval(r, data, reps):
    r.srd_performance_at_ks(test_data=data, ks=[1, 3, 5, 10, 20], max_label=1.0)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        r.srd_performance_at_ks(test_data=data, ks=[1, 3, 5, 10, 20], max_label=1.0)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


GROUPS = [("new list-scorer kernels", ("div_list", "pad_lists")),
          ("attention GEMMs", ("bgemm", "attn_gemm", "attention_tc", "attn_mma")),
          ("softmax", ("softmax",)),
          ("LayerNorm", ("layernorm",)),
          ("DALETOR loss", ("daletor",)),
          ("FF / linear kernels", ("rows_gemm", "wgrad", "ffnet", "bn", "gemm", "act", "dgrad", "colstat",
                                   "reduce_splits", "dy_finalize", "pack_b")),
          ("optimizer", ("adagrad",))]


def profile(r, data, qps):
    from torch.profiler import ProfilerActivity, profile as tprofile
    r.queries_per_step = qps
    r.div_train(data, epoch_k=1)
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        r.div_train(data, epoch_k=1)
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            per[ev.key] = per.get(ev.key, 0.0) + t
    total = sum(per.values())
    groups, top = {}, sorted(per.items(), key=lambda kv: -kv[1])[:15]
    for k, t in per.items():
        low = k.lower()
        g = next((name for name, pats in GROUPS if any(p in low for p in pats)), "other")
        groups[g] = groups.get(g, 0.0) + t
    return {g: round(100.0 * t / total, 1) for g, t in sorted(groups.items(), key=lambda kv: -kv[1])}, \
        [(k[:90], round(100.0 * t / total, 1)) for k, t in top]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--heads", type=int, default=6)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("div_listsf_bench needs a CUDA device")
    name, limit = card()
    torch.manual_seed(0)
    rng = np.random.default_rng(0)
    r = ranker(args.heads)
    res = dict(card=name, power_limit=limit, heads=args.heads, head_width=3 * F // args.heads)
    one = split(rng, [256] * 32)
    res["step_1x256_ms"] = round(time_epoch(r, one, 1, args.reps), 3)
    res["step_64x256_ms"] = round(time_epoch(r, split(rng, [256] * 64), 64, args.reps), 3)
    res["step_16x1024_ms"] = round(time_epoch(r, split(rng, [1024] * 16), 16, args.reps), 3)
    ev = split(rng, [int(n) for n in rng.integers(20, 400, 200)])
    res["eval_200q_ms"] = round(time_eval(r, ev, args.reps), 3)
    flop_doc = 6 * (720_000 + 1_200 * 256) + 389_248          # forward FLOP per document at n = 256 (from shapes)
    res["fwd_flop_per_doc_n256"] = flop_doc
    print(json.dumps(res))
    if args.profile:
        for tag, data, qps in (("1x256", one, 1), ("64x256", split(rng, [256] * 64), 64)):
            groups, top = profile(r, data, qps)
            res[f"profile_{tag}"] = groups
            res[f"top_kernels_{tag}"] = top
            print(json.dumps({f"profile_{tag}": groups}))
            for k, pct in top:
                print(f"  {pct:5.1f}%  {k}")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    t0 = time.time()
    main()
    print(f"done in {time.time() - t0:.1f} s")
