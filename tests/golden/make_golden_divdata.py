"""Golden fixture for the device DIVDataset, produced by the UNMODIFIED reference on CPU.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_divdata.py

Seeded TREC-shaped dicts (subtopic ids as strings, representations [1, F] float64) go through the reference's own
DIVDataset (buffer=False, presort=True, alpha=0.5): queries of 1 to 450 documents plus one of 4000, subtopic ids up to
20 with gaps, documents with empty subtopic lists, documents absent from q_doc_subtopics, a pool without any subtopic
and a pool with a repeated document.  Twelve small queries are redrawn until the greedy meets no tie (so the
reference's order does not depend on string hashing and must be met exactly).  Layout: tests/divdata_oracle.py.
"""
import os
import sys
import time
import warnings

import numpy as np

warnings.filterwarnings("ignore")
REF = os.environ.get("PTRANKING_REFERENCE", "/root/reference")
sys.path.insert(0, REF)
sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from ptranking.data.data_utils import SPLIT_TYPE  # noqa: E402
from ptranking.ltr_diversification.util.div_data import DIVDataset  # noqa: E402
from tests import divdata_oracle as oracle  # noqa: E402

F = 4
D = 4500


def draw_cover(rng, n, ids, p):
    """Per position: None (absent), [] (empty list) or a list of subtopic ids from ``ids``."""
    out = []
    for _ in range(n):
        u = rng.random()
        if u < 0.08:
            out.append(None)
        elif u < 0.14:
            out.append([])
        else:
            out.append([int(s) for s in ids if rng.random() < p])
    return out


def main():
    rng = np.random.default_rng(2026)
    table = rng.standard_normal((D, F))
    queries = []                                       # (pool rows, cover)
    lens = [1, 2, 3, 5, 8, 17, 33, 64, 120, 200, 300, 450] + [int(x) for x in rng.integers(1, 260, 16)]
    for n in lens:
        m = int(rng.integers(1, 21))
        ids = np.sort(rng.choice(np.arange(1, 21), size=m, replace=False))     # gaps in the ids
        queries.append((rng.choice(D, size=n, replace=False), draw_cover(rng, n, ids, float(rng.uniform(0.1, 0.5)))))
    queries.append((rng.choice(D, size=4000, replace=False), draw_cover(rng, 4000, np.arange(1, 21), 0.3)))
    queries.append((rng.choice(D, size=40, replace=False), [None if j % 3 else [] for j in range(40)]))   # no subtopic
    dup = rng.choice(D, size=30, replace=False)
    queries.append((np.concatenate([dup, dup[:5]]), draw_cover(rng, 35, np.arange(1, 9), 0.3)))  # repeated documents
    for _ in range(12):                                                           # tie-free
        n = int(rng.integers(2, 7))
        for _ in range(100000):
            cover = [[int(s) for s in np.arange(1, 21) if rng.random() < 0.25] for _ in range(n)]
            order = oracle.replay(cover)[0]
            if oracle.tie_free(cover, order):
                break
        else:
            raise RuntimeError("no tie-free draw")
        queries.append((rng.choice(D, size=n, replace=False), cover))

    out = {"num_queries": np.int64(len(queries)), "table": table}
    for i, (pool, cover) in enumerate(queries):
        out[f"pool_{i}"] = pool.astype(np.int32)
        out[f"q_{i}"] = rng.standard_normal((1, F))
        out[f"subs_{i}"] = np.asarray([-1 if c is None else len(c) for c in cover], dtype=np.int32)
        out[f"sids_{i}"] = np.asarray([s for c in cover if c for s in c], dtype=np.int32)
    z = out
    qids, q_reprs, doc_reprs, perms, q_docs = oracle.input_dicts(z)
    t0 = time.time()
    ds = DIVDataset(split_type=SPLIT_TYPE.Train, list_as_file=qids, data_dict=dict(data_id="WT_Div_0912_Implicit"),
                    fold_dir="unused/folder1/", presort=True, alpha=oracle.ALPHA, dictQueryRepresentation=q_reprs,
                    dictDocumentRepresentation=doc_reprs, dictQueryPermutaion=perms,
                    dictQueryDocumentSubtopics=q_docs, buffer=False)
    print(f"reference DIVDataset: {len(ds)} queries in {time.time() - t0:.1f} s")
    for i, (qid, q, perm_docs, docs, _, _, R) in enumerate(ds.list_torch_Qs):
        pos = {doc: j for j, doc in enumerate(dict.fromkeys(perms[str(qid)]["permutation"]))}   # set() drops repeats
        out[f"ref_order_{i}"] = np.asarray([pos[doc] for doc in perm_docs], dtype=np.int32)
        out[f"ref_docs_{i}"] = docs.numpy()
        out[f"ref_rele_{i}"] = R.numpy()
    np.savez_compressed(os.path.join(HERE, "divdata.npz"), **out)
    print(f"divdata.npz: {len(queries)} queries, lengths {min(len(t[2]) for t in ds.list_torch_Qs)}"
          f"..{max(len(t[2]) for t in ds.list_torch_Qs)}")


if __name__ == "__main__":
    main()
