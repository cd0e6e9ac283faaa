"""Time one rerank-mode selection pass over a TREC-shaped split on the GPU, against the reference's per-query path.

    python tools/div_rerank_bench.py [--queries 198] [--k 50] [--repeats 5] [--out div_rerank_bench.json]

The split is generated from a seed: 198 queries (the TREC Web-track 2009-2012 diversification set's count), 100-wide
query and document representations, 100 to 300 documents per query, 1 to 6 subtopics.  The first stage is a
DivProbRanker with the reference driver's default pointsf scorer (5 layers, GELU, BN, dropout 0.1, ExpRele keys) in
training mode, as the driver leaves a loaded discriminator.

* device: RerankDIVDataset.select() -- one batched scorer forward, the select and the gather launches and the one
  relevance-mass read-back -- on the host clock after a synchronise; the pool is packed before the first, untimed, pass.
* reference (when the reference package is importable: baseline/_ref or PTRANKING_REFERENCE): the reference's
  RerankDIVDataset.__getitem__ over every query with a CPU DivProbRanker holding the same weights, as the driver runs it
  (gpu=False).

The card's name and power limit are read in the same run."""
import argparse
import copy
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
for cand in (os.path.join(ROOT, "baseline", "_ref"), os.environ.get("PTRANKING_REFERENCE", "")):
    if cand and os.path.isdir(os.path.join(cand, "ptranking")):
        sys.path.insert(0, cand)
        break

import ptranking_b200  # noqa: E402
from ptranking_b200.ltr_diversification.div_data import RerankDIVDataset  # noqa: E402

F = 100
SF = dict(sf_id="pointsf", opt="Adagrad", lr=0.001,
          pointsf=dict(num_features=F, num_layers=5, AF="GE", TL_AF="GE", apply_tl_af=False, BN=True, bn_type="BN",
                       bn_affine=True, dropout=0.1))
MP = dict(model_id="DivProbRanker", K=1, cluster=False, sort_id="ExpRele", top_k=None, opt_id="SuperSoft",
          limit_delta=0.01, metric="nERR-IA", opt_ideal=True, norm=True)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True)
    return r.stdout.strip()


def make_split(queries, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(queries):
        n, m = int(rng.integers(100, 301)), int(rng.integers(1, 7))
        q = torch.from_numpy(rng.standard_normal((1, F)).astype(np.float32))
        d = torch.from_numpy(rng.standard_normal((n, F)).astype(np.float32))
        R = torch.from_numpy((rng.random((m, n)) < 0.1).astype(np.float32))
        out.append((str(i), q, [f"{i}-{j}" for j in range(n)], d, 0.0, None, R))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=198)
    ap.add_argument("--k", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.manual_seed(0)
    data = make_split(args.queries)
    d = ptranking_b200.DivProbRanker(sf_para_dict=copy.deepcopy(SF), model_para_dict=dict(MP), gpu=True, device="cuda:0")
    d.init()
    d.train_mode()
    ds = RerankDIVDataset.from_queries(data, d, args.k)
    ds.pool()
    ds.select()
    torch.cuda.synchronize()
    dev_ms = []
    for _ in range(args.repeats):
        t0 = time.perf_counter()
        ds.select()
        torch.cuda.synchronize()
        dev_ms.append((time.perf_counter() - t0) * 1e3)
    res = dict(card=card(), queries=args.queries, docs=int(sum(x[3].shape[0] for x in data)), rerank_k=args.k,
               device_pass_ms=dev_ms)
    try:
        from ptranking.ltr_diversification.score_and_sort.div_prob_ranker import DivProbRanker as RefDivProbRanker
        from ptranking.ltr_diversification.util.div_data import RerankDIVDataset as RefRerank
    except ImportError:
        res["reference_pass_ms"] = "not measured: the reference package is not importable"
    else:
        ref = RefDivProbRanker(sf_para_dict=copy.deepcopy(SF), model_para_dict=dict(MP), gpu=False, device="cpu")
        ref.init()
        ref.point_sf.load_state_dict({k: v.cpu() for k, v in d.point_sf.state_dict().items()})
        ref_ds = RefRerank.__new__(RefRerank)
        ref_ds.list_torch_Qs, ref_ds.discriminator, ref_ds.rerank_k = data, ref, args.k
        ref_ds.gpu, ref_ds.device = False, None
        ref_ms = []
        for _ in range(max(1, min(args.repeats, 3))):
            t0 = time.perf_counter()
            for i in range(len(ref_ds)):
                ref_ds[i]
            ref_ms.append((time.perf_counter() - t0) * 1e3)
        res["reference_pass_ms"] = ref_ms
        res["reference_threads"] = torch.get_num_threads()
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
