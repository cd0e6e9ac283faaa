"""Golden fixtures for DivProbRanker, produced by the UNMODIFIED reference on CPU.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_divprob.py

The reference's Gaussian head is DivMDNRanker.div_forward (base/div_mdn_ranker.py:248-299); each case builds a
reference DivProbRanker and replaces its ``div_switch_forward`` by a function that returns a leaf raw output, so the
head, the losses of score_and_sort/div_prob_ranker.py and the sort keys are all the reference's own code.

* ``loss_*``: value and autograd gradient w.r.t. the raw output [n, D] of every supported loss -- SuperSoft aNDCG and
  nERR-IA at top_k in {None, 1, 10} (nERR-IA only where top_k <= n: the reference raises beyond), PairCLS, LambdaPairCLS with norm True / False -- over n in {1, 2, 7, 50, 300} and
  m in {1, 3, 8, 32}; every list takes one of the six (K, limit_delta) in {1, 5} x {None, 0.01, 0.1} in turn.  Inputs
  ``list_<i>__{raw_free,raw_pair,rele_bin,rele_flt}`` plus ``__meta`` = (n, m, K, limit_delta or 0).  ``raw_pair`` (the
  pair losses') is drawn by ``tests.divprob_oracle.draw_raw`` so that no pair is near fp32 saturation of
  1 - erfc(x)/2 while many are clearly saturated.  Every m >= 3 matrix has one relevance-free row.  Binary relevance
  for every loss, graded for three.  Results ``loss_<i>_<loss>_k<top_k>_<norm>_<bin|flt>__{loss,grad}``.
* ``key_*``: the three sort keys (div_predict) of a few lists.
* ``train_<sf>__*``: a pointsf and a listsf DivProbRanker trained by the reference's own ``div_train_op`` on three
  queries, one Adagrad step each, from seeded starting weights (tests.daletor_oracle.seeded_state for pointsf,
  tests.divlist_oracle.seeded_state for listsf); dropout off (pointsf) or eval mode (listsf).  Stored: the queries, the
  step losses, the first step's parameter gradients and the (mu, var) of each query after the three steps.
"""
import copy
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

from ptranking.ltr_diversification.score_and_sort.div_prob_ranker import DivProbRanker  # noqa: E402
from tests import daletor_oracle, divlist_oracle  # noqa: E402
from tests.divprob_oracle import TRAIN, draw_raw  # noqa: E402

HEADS = [(1, None), (5, None), (1, 0.01), (5, 0.1), (1, 0.1), (5, 0.01)]
CONFIGS = [("SuperSoft", "aNDCG", None, True), ("SuperSoft", "aNDCG", 1, True), ("SuperSoft", "aNDCG", 10, True),
           ("SuperSoft", "nERR-IA", None, True), ("SuperSoft", "nERR-IA", 1, True), ("SuperSoft", "nERR-IA", 10, True),
           ("PairCLS", None, None, True), ("LambdaPairCLS", None, None, True), ("LambdaPairCLS", None, None, False)]
GRADED = {("SuperSoft", "aNDCG", None, True), ("SuperSoft", "nERR-IA", 10, True), ("LambdaPairCLS", None, None, True)}


def case_name(opt_id, metric, top_k, norm):
    return f"{metric or opt_id}_k{top_k}_{'norm' if norm else 'raw'}"


def rele_mat(rng, m, n, graded):
    R = (rng.uniform(0.0, 2.0, (m, n)) * (rng.random((m, n)) < 0.4)) if graded else \
        (rng.random((m, n)) < 0.3).astype(np.float64)
    if m >= 3:
        R[rng.integers(m)] = 0.0
    return R.astype(np.float32)


def ranker(K, limit_delta, opt_id="SuperSoft", metric="aNDCG", top_k=None, norm=True, sf=None):
    sf = sf or dict(sf_id="pointsf", opt="Adagrad", lr=0.001,
                    pointsf=dict(num_features=4, h_dim=8, num_layers=2, AF="R", TL_AF="S", apply_tl_af=False, BN=False,
                                 bn_type=None, bn_affine=False, dropout=0.0))
    mp = dict(model_id="DivProbRanker", K=K, cluster=False, sort_id="ExpRele", top_k=top_k, opt_id=opt_id,
              limit_delta=limit_delta, metric=metric, opt_ideal=True, norm=norm)
    return DivProbRanker(sf_para_dict=sf, model_para_dict=mp, gpu=False, device="cpu")


def on_raw(r, raw):
    """The reference's head over a given raw output: (mus, vars) of DivMDNRanker.div_forward."""
    r.div_switch_forward = lambda q_repr, doc_reprs, sf=None: raw
    n = raw.shape[1]
    return r.div_forward(torch.zeros(1, 4), torch.zeros(n, 4))


def loss_cases(rng, out):
    i = 0
    for n in (1, 2, 7, 50, 300):
        for m in (1, 3, 8, 32):
            K, ld = HEADS[i % len(HEADS)]
            key = f"list_{i}"
            out[key + "__meta"] = np.asarray([n, m, K, ld or 0.0], dtype=np.float64)
            out[key + "__raw_free"] = draw_raw(rng, n, K, ld, False)
            out[key + "__raw_pair"] = draw_raw(rng, n, K, ld, True)
            out[key + "__rele_bin"], out[key + "__rele_flt"] = rele_mat(rng, m, n, False), rele_mat(rng, m, n, True)
            for cfg in CONFIGS:
                opt_id, metric, top_k, norm = cfg
                if metric == "nERR-IA" and top_k is not None and top_k > n:
                    continue            # the reference's cascade assignment raises when top_k exceeds the list
                for tag in ("bin", "flt") if cfg in GRADED else ("bin",):
                    r = ranker(K, ld, opt_id, metric, top_k, norm)
                    u = out[key + ("__raw_free" if opt_id == "SuperSoft" else "__raw_pair")]
                    leaf = torch.from_numpy(u).clone().unsqueeze(0).requires_grad_(True)
                    mus, vars = on_raw(r, leaf)
                    R = torch.from_numpy(out[f"{key}__rele_{tag}"])
                    kw = dict(presort=True)
                    if opt_id == "SuperSoft":
                        from ptranking.ltr_diversification.score_and_sort import div_prob_ranker as dp
                        if metric == "aNDCG":
                            loss = dp.alpha_dcg_as_a_loss(top_k=top_k, batch_mus=mus, batch_vars=vars, q_doc_rele_mat=R,
                                                          opt_ideal=True, presort=True, beta=0.5)
                        else:
                            loss = dp.err_ia_as_a_loss(top_k=top_k, batch_mus=mus, batch_vars=vars, q_doc_rele_mat=R,
                                                       opt_ideal=True, presort=True, max_label=1.0, device="cpu")
                    else:
                        from ptranking.ltr_diversification.score_and_sort import div_prob_ranker as dp
                        loss = dp.prob_lambda_loss(opt_id=opt_id, batch_mus=mus, batch_vars=vars, q_doc_rele_mat=R,
                                                   opt_ideal=True, presort=True, beta=0.5, device="cpu", norm=norm)
                    loss.backward()
                    name = f"loss_{i}_{case_name(*cfg)}_{tag}"
                    out[name + "__loss"] = np.float64(loss.detach())
                    out[name + "__grad"] = leaf.grad[0].numpy().copy()
            i += 1


def key_cases(rng, out):
    for i, (n, K, ld) in enumerate(((9, 1, None), (40, 5, 0.1), (120, 1, 0.01), (33, 5, None))):
        u = draw_raw(rng, n, K, ld, False)
        out[f"key_{i}__raw"] = u
        out[f"key_{i}__meta"] = np.asarray([n, 0, K, ld or 0.0], dtype=np.float64)
        for sort_id in ("ExpRele", "RERAR", "RiskAware"):
            r = ranker(K, ld)
            r.sort_id = sort_id
            r.div_switch_forward = lambda q_repr, doc_reprs, sf=None: torch.from_numpy(u).unsqueeze(0)
            with torch.no_grad():
                out[f"key_{i}__{sort_id}"] = r.div_predict(torch.zeros(1, 4), torch.zeros(n, 4))[0].numpy().copy()


def train_case(rng, name, out):
    mp, sf = TRAIN[name]
    F = sf[name]["num_features"]
    r = DivProbRanker(sf_para_dict=copy.deepcopy(sf), model_para_dict=dict(model_id="DivProbRanker", cluster=False,
                                                                          sort_id="ExpRele", opt_ideal=True, **mp),
                      gpu=False, device="cpu")
    r.init()
    if name == "pointsf":
        init = daletor_oracle.seeded_state({k: tuple(v.shape) for k, v in r.point_sf.state_dict().items()})
        with torch.no_grad():
            for k, v in r.point_sf.state_dict().items():
                v.copy_(torch.from_numpy(init[k]))
        named = lambda: [("point_sf", k, p) for k, p in r.point_sf.named_parameters()]
        r.train_mode()
    else:
        init = divlist_oracle.seeded_state(divlist_oracle.state_shapes(r.list_sf["encoder"], r.list_sf["uni_sf"]))
        with torch.no_grad():
            for part in ("encoder", "uni_sf"):
                for k, v in r.list_sf[part].state_dict().items():
                    v.copy_(torch.from_numpy(init[part][k]))
        named = lambda: [(part, k, p) for part in ("encoder", "uni_sf") for k, p in r.list_sf[part].named_parameters()]
        r.eval_mode()
    losses = []
    for i, (n, m) in enumerate(((40, 5), (23, 3), (64, 8))):
        q = rng.standard_normal((1, F)).astype(np.float32)
        d = rng.standard_normal((n, F)).astype(np.float32)
        R = rele_mat(rng, m, n, False)
        R[0, 0] = 1.0
        out[f"train_{name}__q{i}_q_repr"], out[f"train_{name}__q{i}_doc_reprs"], out[f"train_{name}__q{i}_rele"] = q, d, R
        loss, _ = r.div_train_op(torch.from_numpy(q), torch.from_numpy(d), torch.from_numpy(R), presort=True, epoch_k=1)
        losses.append(float(loss))
        if i == 0:
            for part, k, p in named():
                out[f"train_{name}__grad0__{part}__{k}"] = p.grad.numpy().copy()
    out[f"train_{name}__losses"] = np.asarray(losses, dtype=np.float64)
    with torch.no_grad():
        for i in range(3):
            q, d = (torch.from_numpy(out[f"train_{name}__q{i}_{f}"]) for f in ("q_repr", "doc_reprs"))
            mus, vars = r.div_forward(q, d)
            out[f"train_{name}__final_mu_q{i}"] = mus.numpy().copy()
            out[f"train_{name}__final_var_q{i}"] = vars.numpy().copy()


def main():
    rng = np.random.default_rng(2022)
    torch.manual_seed(2022)
    out = {}
    loss_cases(rng, out)
    key_cases(rng, out)
    for name in TRAIN:
        train_case(rng, name, out)
    np.savez_compressed(os.path.join(HERE, "divprob.npz"), **out)
    print(f"divprob.npz: {len(out)} arrays, {sum(1 for k in out if k.endswith('__loss'))} loss runs")


if __name__ == "__main__":
    main()
