"""bf16 feature tensors against fp32 ones, step by step, in one process (arms alternated).

    python tools/bf16_features_bench.py [--shapes e:32,e:128,e:256,e:1024,b:256] [--rounds 2] [--json out.json]

Shapes: ``e:n`` = BASELINE config (e), ListMLE + the default pointwise scorer with math_mode="bf16", B = 2^18 / n;
``b:n`` = config (b), LambdaRank + the default scorer in 3xTF32, B = 2^18 / n.  136 features.  Per shape and arm:

  dev_ms      device-resident ms/step (features already on the GPU; CUDA events over a window of >= 1 s)
  e2e_ms      ms/step through data.RaggedBatches with pinned host batches and NeuralRanker.train's side-stream copies
              (host clock around whole epochs ending in a synchronise, >= 1 s)
  l0_*_ms     layer 0's kernels per step from the library's launch timing: the bf16 arm's own launch tags
              (rows_gemm_*_fwd_xbf16, wgrad_tc_xbf16); for the fp32 arm, its tag total minus the bf16 arm's
              total of the same tag (= the other layers, which both arms run identically)
  feat_MB     algorithmic feature bytes per step: HBM reads of X by layer 0 (forward + weight gradient) and the
              host-to-device copy, from shapes
  peak_MB     the arm's feature tensor plus the peak device memory one step allocates on top of what is resident
  equal       torch.equal of the scores and every parameter gradient of one forward/backward on the same weights

The card's name and power limit are read in the same run.  Needs a GPU; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np
import torch

F = 136
DOCS = 1 << 18
MSLR_P = np.array([1940952, 1225770, 504958, 69010, 30435], dtype=np.float64)
MSLR_P /= MSLR_P.sum()
ARMS = (("f32", torch.float32), ("bf16", torch.bfloat16))


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def make_ranker(key, seed=137):
    import ptranking_b200
    os.environ["PTRANKING_B200_MATH"] = "bf16" if key == "e" else "3xtf32"
    sf = dict(sf_id="pointsf", opt="Adam", lr=1e-4,
              pointsf=dict(num_features=F, num_layers=5, AF="GE", TL_AF="S", apply_tl_af=True, BN=True, bn_type="BN",
                           bn_affine=True, dropout=0.1))
    torch.manual_seed(seed)
    if key == "e":
        r = ptranking_b200.ListMLE(sf_para_dict=sf, gpu=True, device="cuda:0")
    else:
        r = ptranking_b200.LambdaRank(sf_para_dict=sf, model_para_dict=dict(model_id="LambdaRank", sigma=1.0), gpu=True,
                                      device="cuda:0")
    r.init()
    r.train_mode()
    return r


def synth(rng, B, n):
    X = rng.standard_normal((B, n, F), dtype=np.float32)
    y = rng.choice(len(MSLR_P), size=(B, n), p=MSLR_P).astype(np.float32)
    y[:, 0] = np.maximum(y[:, 0], 1.0)
    return X, -np.sort(-y, axis=1)


def step_fn(r, X, y):
    from ptranking_b200 import LABEL_TYPE
    return lambda: r.train_op(X, y, presort=True, label_type=LABEL_TYPE.MultiLabel)


def timed_ms(fn, min_s=1.0):
    """ms per call over a window of at least min_s seconds (CUDA events)."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); b.record(); b.synchronize()
    k = max(10, int(min_s * 1000.0 / max(a.elapsed_time(b), 1e-3)) + 1)
    a.record()
    for _ in range(k):
        fn()
    b.record(); b.synchronize()
    return a.elapsed_time(b) / k


def kernel_ms(fn, steps=10):
    from ptranking_b200 import _lib
    fn(); torch.cuda.synchronize()
    _lib.kernel_timings(True)
    try:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    finally:
        _lib.kernel_timings(False)
    return {k: ms / steps for k, (cnt, ms) in _lib.kernel_timings(None).items()}


def e2e_ms(r, queries, dt, min_s=1.0):
    from ptranking_b200 import LABEL_TYPE, data
    loader = data.RaggedBatches(queries, docs_per_batch=DOCS, feature_dtype=dt)
    nb = len(loader)
    r.train(loader, label_type=LABEL_TYPE.MultiLabel, presort=True)        # warm: pinned pages, kernels, allocator
    torch.cuda.synchronize()
    epochs, t0 = 0, time.perf_counter()
    while True:
        r.train(loader, label_type=LABEL_TYPE.MultiLabel, presort=True)
        epochs += 1
        if time.perf_counter() - t0 >= min_s:
            break
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1000.0 / (epochs * nb)


def equality(key, X32, y):
    """one forward/backward of the scorer on identical weights: bf16 features vs the same values in fp32"""
    from ptranking_b200 import ops
    res = {}
    for name, dt in ARMS:
        r = make_ranker(key, seed=5)
        ops._dropout_offset = 0
        s = r.point_sf(X32.to(dt))
        (s.squeeze(-1) * y).sum().backward()
        res[name] = (s.detach(), [p.grad.clone() for p in r.point_sf.ordered_parameters()])
    (sa, ga), (sb, gb) = res["f32"], res["bf16"]
    return bool(torch.equal(sa, sb) and all(torch.equal(a, b) for a, b in zip(ga, gb)))


def run_shape(key, n, rounds, rng):
    B = DOCS // n
    Xn, yn = synth(rng, B, n)
    Xb32 = torch.from_numpy(Xn).to(torch.bfloat16).float()             # the values both arms carry
    y = torch.from_numpy(yn).cuda()
    rows = B * n
    row = dict(shape=f"{key}:{n}", B=B, n=n)
    rankers = {name: make_ranker(key) for name, _ in ARMS}
    Xdev = {name: Xb32.to(dt).cuda() for name, dt in ARMS}
    dev = {name: [] for name, _ in ARMS}
    for _ in range(rounds):                                            # alternated arms
        for name, _ in ARMS:
            dev[name].append(timed_ms(step_fn(rankers[name], Xdev[name], y)))
    kt = {name: kernel_ms(step_fn(rankers[name], Xdev[name], y)) for name, _ in ARMS}
    for name, dt in ARMS:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        before = torch.cuda.memory_allocated()
        step_fn(rankers[name], Xdev[name], y)()
        torch.cuda.synchronize()
        e = 2 if dt == torch.bfloat16 else 4
        # this arm's features + what its step allocates on top of everything resident (both arms' features stay resident)
        peak = Xdev[name].nbytes + torch.cuda.max_memory_allocated() - before
        row[name] = dict(dev_ms=dev[name], peak_MB=peak / 1e6,
                         feat_hbm_MB=2 * rows * F * e / 1e6, feat_h2d_MB=rows * F * e / 1e6)
    for tag in ("rows_gemm_ws_fwd", "rows_gemm_tc_fwd", "wgrad_tc"):
        xb = kt["bf16"].get(tag + "_xbf16")
        if xb is not None:
            row["bf16"][f"l0_{tag}_ms"] = xb
            row["f32"][f"l0_{tag}_ms"] = kt["f32"].get(tag, 0.0) - kt["bf16"].get(tag, 0.0)
    del Xdev
    queries = [(f"q{i}", Xb32[i].numpy(), yn[i]) for i in range(B)]
    for _ in range(rounds):
        for name, dt in ARMS:
            row[name].setdefault("e2e_ms", []).append(e2e_ms(rankers[name], queries, dt))
    row["equal"] = equality(key, Xb32[: min(B, 256)].cuda(), y[: min(B, 256)])
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default="e:32,e:128,e:256,e:1024,b:256")
    ap.add_argument("--rounds", type=int, default=2, help="alternations of the two arms per timed figure")
    ap.add_argument("--json", default=None, help="also write the rows to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bf16_features_bench needs a CUDA device")
    info = gpu_info()
    print(f"# {info}")
    rng = np.random.default_rng(137)
    rows = []
    hdr = ("shape", "arm", "dev_ms", "e2e_ms", "l0_fwd_ms", "l0_wgrad_ms", "feat_hbm_MB", "feat_h2d_MB", "peak_MB", "equal")
    print(" | ".join(hdr))
    for s in args.shapes.split(","):
        key, n = s.split(":")
        row = run_shape(key, int(n), args.rounds, rng)
        rows.append(row)
        for name, _ in ARMS:
            a = row[name]
            fwd = a.get("l0_rows_gemm_ws_fwd_ms", a.get("l0_rows_gemm_tc_fwd_ms", float("nan")))
            print(" | ".join([row["shape"], name, "/".join(f"{v:.3f}" for v in a["dev_ms"]),
                              "/".join(f"{v:.3f}" for v in a["e2e_ms"]), f"{fwd:.4f}", f"{a.get('l0_wgrad_tc_ms', float('nan')):.4f}",
                              f"{a['feat_hbm_MB']:.1f}", f"{a['feat_h2d_MB']:.1f}", f"{a['peak_MB']:.0f}", str(row["equal"])]),
                  flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(gpu=info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
