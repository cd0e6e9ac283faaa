"""Train the list scorer at the reference's grid setting (BN2 head and tail nets) on variable-length data, one epoch at a
time, batched two ways:

* (a) ``LengthBucketedBatches``: equal-length buckets, one dense [B, n, F] step per bucket batch;
* (b) ``RaggedBatches`` with list-scorer bucket edges: one ragged step per batch, the encoder padded per length class.

Workload: seeded MSLR-WEB30K-shaped query lengths (lognormal, 1 to 1,251 documents, mean about 120), F = 136, labels
0-4; DASALC, 3 encoder layers, 2 heads, ff_dims 128/256/512, BN2, dropout 0.1, ApproxNDCG with Adagrad.  Each arm trains
its own ranker from the same initial weights.  After one warm-up epoch per arm the timed epochs alternate between the
arms; each is timed on the host clock between device synchronisations.  Prints one JSON line: queries/s per epoch and
the epoch losses of each arm, with the card's name and power limit read in the same run.

    python tools/listsf_ragged_bench.py [--queries 2000] [--docs-per-batch 16384] [--repeats 3]
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
F = 136
MSLR_P = np.array([1940952, 1225770, 504958, 69010, 30435], dtype=np.float64)     # MSLR-WEB30K's label frequencies
MSLR_P /= MSLR_P.sum()


def card():
    name = torch.cuda.get_device_name()
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def queries(num, seed):
    rng = np.random.default_rng(seed)
    lens = np.clip(rng.lognormal(4.45, 0.85, num), 1, 1251).astype(int)
    qs = []
    for i, n in enumerate(lens):
        y = rng.choice(5, size=n, p=MSLR_P).astype(np.float32)
        y[0] = max(y[0], 1.0)           # a query without a relevant document has no ideal DCG: ApproxNDCG is undefined
        qs.append((f"q{i}", rng.standard_normal((n, F)).astype(np.float32), y))
    return qs, lens


def ranker(seed):
    import ptranking_b200
    sf = dict(sf_id="listsf", opt="Adagrad", lr=1e-3,
              listsf=dict(num_features=F, ff_dims=[128, 256, 512], AF="R", TL_AF="GE", apply_tl_af=False, BN=True,
                          bn_type="BN2", bn_affine=False, n_heads=2, encoder_layers=3, encoder_type="DASALC", dropout=0.1))
    torch.manual_seed(seed)
    r = ptranking_b200.ApproxNDCG(sf_para_dict=sf, model_para_dict=dict(model_id="ApproxNDCG", alpha=10.0), gpu=True,
                                  device=DEV)
    r.init()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=2000)
    ap.add_argument("--docs-per-batch", type=int, default=16384)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--edges", default="32,64,128,256,512", help="RaggedBatches bucket edges")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("listsf_ragged_bench needs a CUDA device")
    from ptranking_b200 import LABEL_TYPE
    from ptranking_b200.data import LengthBucketedBatches, RaggedBatches
    qs, lens = queries(args.queries, seed=0)
    edges = tuple(int(e) for e in args.edges.split(","))
    loaders = {"bucketed": LengthBucketedBatches(qs, docs_per_batch=args.docs_per_batch),
               "ragged": RaggedBatches(qs, docs_per_batch=args.docs_per_batch, bucket_edges=edges)}
    rankers = {k: ranker(seed=1) for k in loaders}
    res = {k: dict(batches=len(loaders[k]), queries_per_s=[], epoch_losses=[]) for k in loaders}

    def epoch(k):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        loss, stop = rankers[k].train(loaders[k], epoch_k=1, presort=True, label_type=LABEL_TYPE.MultiLabel)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        assert not stop
        return len(qs) / dt, float(loss)

    for k in loaders:               # warm-up: module loads, allocator growth, every batch shape once
        res[k]["warmup_epoch_loss"] = epoch(k)[1]
    for _ in range(args.repeats):
        for k in loaders:
            qps, loss = epoch(k)
            res[k]["queries_per_s"].append(round(qps, 1))
            res[k]["epoch_losses"].append(loss)
    name, limit = card()
    ratio = [b / a for a, b in zip(res["bucketed"]["queries_per_s"], res["ragged"]["queries_per_s"])]
    print(json.dumps(dict(card=name, power_limit=limit,
                          workload=dict(queries=len(qs), docs=int(lens.sum()), mean_len=round(float(lens.mean()), 1),
                                        max_len=int(lens.max()), F=F, docs_per_batch=args.docs_per_batch,
                                        bucket_edges=list(edges), encoder="DASALC", encoder_layers=3, heads=2,
                                        norm="BN2", loss="ApproxNDCG"),
                          **res, ragged_over_bucketed=[round(x, 3) for x in ratio])))


if __name__ == "__main__":
    main()
