"""Golden fixtures for rerank mode, produced by the UNMODIFIED reference on CPU.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_rerank.py

A pool of 30 synthetic queries with 1 to 300 documents goes through the reference's own DIVDataset (buffer=False, presort
with its ideal diversified ranking) and is wrapped in the reference's RerankDIVDataset with rerank_k in {1, 5, 50, 400}
for two first stages (tests.rerank_oracle.STAGES, starting weights from tests.daletor_oracle.seeded_state).  Stored:

* ``pool_<i>__{q,docs,rele}``: the DIVDataset tuple of query i (presorted doc rows and relevance matrix);
* ``<stage>__state__<key>``: the first stage's state dict;
* ``<stage>__keys_<i>``: its div_predict output for query i (the sort keys);
* ``<stage>_k<k>_<i>__{docs,rele}``: what RerankDIVDataset.__getitem__(i) returned -- [F] and [m] when one document is
  selected (the reference's squeeze).  At rerank_k = 400, above every list's length, the generator checks that the
  whole pool comes back in its order and stores nothing.

Documents are redrawn until every boundary a rerank_k cuts (between the k-th and the (k+1)-th key) is wider than
1e-3 of the query's key range for both stages, so fp32 rounding cannot change a selection.
"""
import os
import sys
import warnings

import numpy as np
import torch

warnings.filterwarnings("ignore")
REF = os.environ.get("PTRANKING_REFERENCE", "/root/reference")
sys.path.insert(0, REF)
sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from ptranking.data.data_utils import SPLIT_TYPE  # noqa: E402
from ptranking.ltr_diversification.score_and_sort.daletor import DALETOR  # noqa: E402
from ptranking.ltr_diversification.score_and_sort.div_prob_ranker import DivProbRanker  # noqa: E402
from ptranking.ltr_diversification.util.div_data import DIVDataset, RerankDIVDataset  # noqa: E402
from tests import daletor_oracle  # noqa: E402
from tests.rerank_oracle import F, KS, NUM_QUERIES, stage_config  # noqa: E402

MIN_GAP = 1e-3


def first_stage(name):
    mp, sf, mode = stage_config(name)
    cls = DivProbRanker if mp["model_id"] == "DivProbRanker" else DALETOR
    r = cls(sf_para_dict=sf, model_para_dict=mp, gpu=False, device="cpu")
    r.init()
    init = daletor_oracle.seeded_state({k: tuple(v.shape) for k, v in r.point_sf.state_dict().items()}, seed=31337)
    with torch.no_grad():
        for k, v in r.point_sf.state_dict().items():
            v.copy_(torch.from_numpy(init[k]))
    r.point_sf.train(mode == "train")
    return r


def well_separated(stages, q, d):
    with torch.no_grad():
        for r in stages.values():
            keys = np.sort(r.div_predict(torch.from_numpy(q), torch.from_numpy(d))[0].numpy().astype(np.float64))[::-1]
            span = max(keys[0] - keys[-1], 1e-6)
            for k in KS:
                if k < keys.size and keys[k - 1] - keys[k] <= MIN_GAP * span:
                    return False
    return True


def main():
    rng = np.random.default_rng(2025)
    torch.manual_seed(2025)
    stages = {name: first_stage(name) for name in ("divprob", "daletor")}
    lens = [1, 2, 5, 6, 49, 50, 51, 300, 299, 4] + [int(x) for x in rng.integers(1, 121, NUM_QUERIES - 10)]
    q_reprs, d_reprs, perms, q_docs = {}, {}, {}, {}
    for i, n in enumerate(lens):
        m = int(rng.integers(1, 7))
        q = rng.standard_normal((1, F))
        for _ in range(200):
            d = rng.standard_normal((n, F))
            if well_separated(stages, q.astype(np.float32), d.astype(np.float32)):
                break
        else:
            raise RuntimeError(f"query {i}: no tie-free draw")
        docs, subtopics = [], {}
        for j in range(n):
            doc = f"q{i}-d{j}"
            d_reprs[doc] = d[j:j + 1]
            docs.append(doc)
            cover = [str(t + 1) for t in range(m) if rng.random() < 0.3]
            if cover:
                subtopics[doc] = cover
        if not subtopics:
            subtopics[docs[0]] = ["1"]
        q_reprs[str(i)], perms[str(i)], q_docs[str(i)] = q, dict(alphaDCG=0.0, permutation=docs), subtopics
    kw = dict(split_type=SPLIT_TYPE.Train, list_as_file=list(range(len(lens))),
              data_dict=dict(data_id="WT_Div_0912_Implicit"), fold_dir="unused/folder1/", presort=True,
              dictQueryRepresentation=q_reprs, dictDocumentRepresentation=d_reprs, dictQueryPermutaion=perms,
              dictQueryDocumentSubtopics=q_docs, buffer=False)
    out = {"num_queries": np.int64(len(lens)), "ks": np.asarray(KS, dtype=np.int64)}
    for i, (_, q, _, d, _, _, R) in enumerate(DIVDataset(**kw).list_torch_Qs):
        out[f"pool_{i}__q"], out[f"pool_{i}__docs"], out[f"pool_{i}__rele"] = q.numpy(), d.numpy(), R.numpy()
    for name, r in stages.items():
        for k, v in r.point_sf.state_dict().items():
            out[f"{name}__state__{k}"] = v.numpy().copy()
        with torch.no_grad():
            for i in range(len(lens)):
                keys = r.div_predict(torch.from_numpy(out[f"pool_{i}__q"]), torch.from_numpy(out[f"pool_{i}__docs"]))
                out[f"{name}__keys_{i}"] = keys[0].numpy().copy()
        for k in KS:
            ds = RerankDIVDataset(discriminator=r, eval_dict=dict(rerank_k=k), **kw)
            for i in range(len(ds)):
                _, _, perm_docs, d, _, subtopics, R = ds[i]
                assert perm_docs is None and subtopics is None
                if k > max(lens):
                    assert torch.equal(d, torch.from_numpy(out[f"pool_{i}__docs"]).reshape(d.shape))
                    assert torch.equal(R, torch.from_numpy(out[f"pool_{i}__rele"]).reshape(R.shape))
                    continue
                out[f"{name}_k{k}_{i}__docs"], out[f"{name}_k{k}_{i}__rele"] = d.numpy().copy(), R.numpy().copy()
    np.savez_compressed(os.path.join(HERE, "div_rerank.npz"), **out)
    print(f"div_rerank.npz: {len(out)} arrays, {len(lens)} queries, lengths {min(lens)}..{max(lens)}")


if __name__ == "__main__":
    main()
