"""Time building the diversification driver's plain splits (3 splits x 5 folds) with the reference's DIVDataset and
with the device one.

    python tools/div_data_bench.py [--queries 198] [--out div_data_bench.json]

The data is generated from a seed in the driver's layout: 198 queries (the TREC Web-track 2009-2012 diversification
set's count), 100-wide float64 representations ([1, 100] per document, as load_raw_data makes them), 100 to 300
documents per query, 1 to 6 subtopics as strings, a document covering each with probability 0.15.  Folds as the
driver cuts them: fold k tests on its fifth of the queries, validates on the next fifth and trains on the rest.

* device: ptranking_b200.ltr_diversification.div_data.DIVDataset for the 15 splits, on the host clock (each split
  reads its order back, so it ends synchronised).  The first split also indexes and uploads the document table; a
  first, untimed fold warms up CUDA and the library.
* reference (when the package is importable: baseline/_ref or PTRANKING_REFERENCE): its own DIVDataset, buffer=False,
  one CPU process.  The rows and matrices of fold 1 are checked against the device split's, gathered by document id.

The card's name and power limit are read in the same run."""
import argparse
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

from ptranking_b200.ltr_diversification.div_data import DIVDataset  # noqa: E402

F = 100
DATA_DICT = dict(data_id="WT_Div_0912_Implicit")
try:
    from ptranking.data.data_utils import SPLIT_TYPE
    SPLITS = (SPLIT_TYPE.Train, SPLIT_TYPE.Validation, SPLIT_TYPE.Test)
except ImportError:
    SPLITS = ("train", "vali", "test")        # the device DIVDataset only keeps the value


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True)
    return r.stdout.strip()


def make_dicts(queries, seed=0):
    rng = np.random.default_rng(seed)
    q_reprs, d_reprs, perms, q_docs = {}, {}, {}, {}
    for q in range(queries):
        n, m = int(rng.integers(100, 301)), int(rng.integers(1, 7))
        q_reprs[str(q)] = rng.standard_normal((1, F))
        pool = [f"q{q}-d{j}" for j in range(n)]
        subs = {}
        for doc in pool:
            d_reprs[doc] = rng.standard_normal((1, F))
            cover = [str(t + 1) for t in range(m) if rng.random() < 0.15]
            if cover:
                subs[doc] = cover
        perms[str(q)], q_docs[str(q)] = dict(alphaDCG=0.0, permutation=pool), subs
    return q_reprs, d_reprs, perms, q_docs


def folds(queries):
    parts = np.array_split(np.arange(queries), 5)
    for k in range(5):
        test, vali = parts[k], parts[(k + 1) % 5]
        train = np.concatenate([parts[j] for j in range(5) if j not in (k, (k + 1) % 5)])
        yield [[int(q) for q in s] for s in (train, vali, test)]


def build_all(cls, dicts, queries, **kw):
    q_reprs, d_reprs, perms, q_docs = dicts
    out, ms = [], []
    for split_qids in folds(queries):
        fold = []
        for split_type, qids in zip(SPLITS, split_qids):
            t0 = time.perf_counter()
            fold.append(cls(split_type=split_type, list_as_file=qids, data_dict=DATA_DICT, fold_dir="unused/folder1/",
                            presort=True, dictQueryRepresentation=q_reprs, dictDocumentRepresentation=d_reprs,
                            dictQueryPermutaion=perms, dictQueryDocumentSubtopics=q_docs, buffer=False, **kw))
            ms.append((time.perf_counter() - t0) * 1e3)
        out.append(fold)
    return out, ms


def check(dev_fold, ref_fold):
    """The device rows and matrices are the reference's, gathered by document id; returns the queries whose order is
    the reference's."""
    same = 0
    for dev, ref in zip(dev_fold, ref_fold):
        for b in range(len(ref)):
            _, q, perm, docs, _, _, R = dev[b]
            _, rq, rperm, rdocs, _, _, rR = ref[b]
            where = [rperm.index(d) for d in perm]
            assert np.array_equal(q.cpu().numpy(), rq.numpy())
            assert np.array_equal(docs.cpu().numpy(), rdocs.numpy()[where])
            assert np.array_equal(R.cpu().numpy(), rR.numpy()[:, where])
            same += perm == rperm
    return same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=198)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dicts = make_dicts(args.queries)
    torch.cuda.init()
    warm, _ = build_all(DIVDataset, make_dicts(args.queries, seed=1), args.queries)      # untimed
    del warm
    dev, dev_ms = build_all(DIVDataset, dicts, args.queries)
    res = dict(card=card(), queries=args.queries, docs=len(dicts[1]), splits=len(dev_ms),
               device_split_ms=[round(x, 2) for x in dev_ms], device_total_ms=round(sum(dev_ms), 1))
    try:
        from ptranking.ltr_diversification.util.div_data import DIVDataset as RefDIVDataset
    except ImportError:
        res["reference_total_ms"] = "not measured: the reference package is not importable"
    else:
        ref, ref_ms = build_all(RefDIVDataset, dicts, args.queries)
        res["reference_split_ms"] = [round(x, 1) for x in ref_ms]
        res["reference_total_ms"] = round(sum(ref_ms), 1)
        res["fold1_queries_checked"] = sum(len(s) for s in ref[0])
        res["fold1_same_order"] = check(dev[0], [s.list_torch_Qs for s in ref[0]])
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
