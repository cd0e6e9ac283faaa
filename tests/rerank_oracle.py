"""Rerank mode's fixture cases (tests/golden/make_golden_rerank.py) and a NumPy restatement of the selection.

Two first stages over one pool of synthetic queries: a DivProbRanker (pointsf, no BN, dropout 0, training mode, as
the driver leaves a loaded discriminator) and a DALETOR (pointsf with GELU hidden layers, evaluation mode).  Neither
uses BN: the reference's BN keeps no running statistics, so it refuses a one-document query in either mode.  Their
starting weights are daletor_oracle.seeded_state."""
import copy

import numpy as np

F = 8
KS = (1, 5, 50, 400)
NUM_QUERIES = 30
SF = dict(sf_id="pointsf", opt="Adagrad", lr=0.01,
          pointsf=dict(num_features=F, h_dim=16, num_layers=2, AF="R", TL_AF="S", apply_tl_af=False, BN=False,
                       bn_type=None, bn_affine=False, dropout=0.0))
STAGES = {
    "divprob": (dict(model_id="DivProbRanker", K=1, cluster=False, sort_id="ExpRele", limit_delta=0.01,
                     opt_id="SuperSoft", metric="aNDCG", top_k=10, opt_ideal=True, norm=True),
                SF, "train"),
    "daletor": (dict(model_id="DALETOR", rt=10.0, top_k=10),
                dict(SF, pointsf=dict(SF["pointsf"], AF="GE")), "eval"),
}


def stage_config(name):
    """-> (model dict, scorer dict, mode) of a first stage; fresh copies (the rankers write into them)."""
    mp, sf, mode = STAGES[name]
    return copy.deepcopy(mp), copy.deepcopy(sf), mode


def topk_ascending(keys, k):
    """The selection in NumPy: the indices of the top min(n, k) keys by (key descending, index ascending), ascending."""
    keys = np.asarray(keys, dtype=np.float32).reshape(-1)
    order = np.lexsort((np.arange(keys.size), -keys.astype(np.float64)))
    return np.sort(order[:k])


def pool_queries(z):
    """The fixture pool as DIVDataset tuples (qid, q_repr [1,F], perm_docs, doc_reprs [n,F], alphaDCG, None, R [m,n])."""
    import torch
    out = []
    for i in range(int(z["num_queries"])):
        d = z[f"pool_{i}__docs"]
        out.append((f"q{i}", torch.from_numpy(z[f"pool_{i}__q"]), [f"q{i}-d{j}" for j in range(d.shape[0])],
                    torch.from_numpy(d), 0.0, None, torch.from_numpy(z[f"pool_{i}__rele"])))
    return out
