"""Golden fixtures for the diversification path (DALETOR and the SRD metrics), produced by the UNMODIFIED reference.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_daletor.py

* ``loss_*``: ``alphaDCG_as_a_loss`` (ltr_diversification/score_and_sort/daletor.py:22-40) on a leaf score tensor, its
  value and autograd gradient, over n in {1, 2, 7, 50, 300}, m in {1, 3, 8, 20}, top_k in {None, 1, 2, 10} and
  rt in {1, 10, 50} with 0/1 subtopic relevance (one row of every m >= 3 matrix has none), plus graded (float)
  relevance at rt = 10.  Inputs ``list_n<n>_m<m>__{scores,rele_bin,rele_flt}``; results ``loss_<case>__{loss,grad}``,
  a case being ``n<n>_m<m>_k<top_k>_rt<rt>_<bin|flt>``.
* ``met_*``: the evaluator's sort (``torch.sort(descending=True)`` + gather, base/ranker.py:413-475) and the six metric
  functions of metric/srd/diversity_metric.py at ks = (1, 3, 5, 10, 20), including lists shorter than max(ks), a query
  with no relevance at all and one whose relevance lies beyond the first positions.  Keys
  ``met_<case>__{scores,rele,max_label,order,andcg_ks,err_ia_ks,nerr_ia_ks,andcg_k5,err_ia_k5,nerr_ia_k5}``.
* ``train__*``: a DALETOR pointsf (the reference's default diversification scorer, num_features = 100 so its input is
  300 wide, dropout off) trained by the reference's own ``div_train_op`` on three queries, one Adagrad step each:
  ``q<i>_{q_repr,doc_reprs,rele}``, the scores of query 0 before the first step ``pred0``, the parameter gradients of the
  first step ``grad0__<key>``, the losses ``losses`` and each query's scores after the three steps
  ``final_scores_q<i>``.  The starting weights are not stored: ``tests.daletor_oracle.seeded_state`` rebuilds them.
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
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))          # the repository: tests.daletor_oracle.seeded_state

from ptranking.ltr_diversification.score_and_sort.daletor import alphaDCG_as_a_loss, DALETOR  # noqa: E402
from ptranking.metric.srd import diversity_metric as dm  # noqa: E402
from tests.daletor_oracle import seeded_state  # noqa: E402

KS = (1, 3, 5, 10, 20)


def rele_mat(rng, m, n, graded):
    if graded:
        R = rng.uniform(0.0, 2.0, (m, n)) * (rng.random((m, n)) < 0.4)
    else:
        R = (rng.random((m, n)) < 0.3).astype(np.float64)
    if m >= 3:
        R[rng.integers(m)] = 0.0
    return R.astype(np.float32)


def loss_cases(rng, out):
    for n in (1, 2, 7, 50, 300):
        for m in (1, 3, 8, 20):
            s = rng.standard_normal((1, n)).astype(np.float32)
            Rb, Rf = rele_mat(rng, m, n, False), rele_mat(rng, m, n, True)
            lst = f"list_n{n}_m{m}"
            out[lst + "__scores"], out[lst + "__rele_bin"], out[lst + "__rele_flt"] = s, Rb, Rf
            for top_k in (None, 1, 2, 10):
                for rt in (1.0, 10.0, 50.0):
                    for tag, R in (("bin", Rb), ("flt", Rf)):
                        if tag == "flt" and rt != 10.0:
                            continue
                        leaf = torch.from_numpy(s).clone().requires_grad_(True)
                        loss = alphaDCG_as_a_loss(batch_preds=leaf, q_doc_rele_mat=torch.from_numpy(R), rt=rt,
                                                  top_k=top_k, device="cpu")
                        loss.backward()
                        key = f"loss_n{n}_m{m}_k{top_k}_rt{rt:g}_{tag}"
                        out[key + "__loss"] = np.float64(loss.detach())
                        out[key + "__grad"] = leaf.grad.numpy().copy()


def metric_cases(rng, out):
    specs = [("n30_m4", 30, 4, False), ("n12_m3", 12, 3, False), ("n3_m5", 3, 5, False), ("n25_m8_flt", 25, 8, True),
             ("n20_m1", 20, 1, False), ("n7_m2_none", 7, 2, False), ("n40_m6_late", 40, 6, False)]
    for name, n, m, graded in specs:
        R = rele_mat(rng, m, n, graded)
        if name.endswith("_none"):
            R[:] = 0.0
        if name.endswith("_late"):
            R[:, :15] = 0.0
        s = rng.standard_normal((1, n)).astype(np.float32)
        max_label = 2.0 if graded else 1.0
        Rt, st = torch.from_numpy(R), torch.from_numpy(s)
        _, order = torch.sort(st, dim=1, descending=True)
        sys_R = torch.gather(Rt, dim=1, index=order.expand(m, -1))
        key = f"met_{name}"
        out[key + "__scores"], out[key + "__rele"] = s, R
        out[key + "__max_label"] = np.float64(max_label)
        out[key + "__order"] = order[0].numpy().astype(np.int32)
        out[key + "__andcg_ks"] = dm.torch_alpha_ndcg_at_ks(sys_R, Rt, ks=list(KS), alpha=0.5).numpy()
        out[key + "__err_ia_ks"] = dm.torch_err_ia_at_ks(sys_R, max_label=max_label, ks=list(KS)).numpy()
        out[key + "__nerr_ia_ks"] = dm.torch_nerr_ia_at_ks(sys_R, Rt, max_label=max_label, ks=list(KS)).numpy()
        if n >= 5:
            out[key + "__andcg_k5"] = np.float64(dm.torch_alpha_ndcg_at_k(sys_R, Rt, k=5, alpha=0.5))
            out[key + "__err_ia_k5"] = np.float64(dm.torch_err_ia_at_k(sys_R, max_label=max_label, k=5))
            out[key + "__nerr_ia_k5"] = np.float64(dm.torch_nerr_ia_at_k(sys_R, Rt, max_label=max_label, k=5))


def train_case(rng, out):
    torch.manual_seed(2718)
    F = 100
    sf = dict(sf_id="pointsf", opt="Adagrad", lr=0.001,
              pointsf=dict(num_features=F, num_layers=5, AF="GE", TL_AF="GE", apply_tl_af=False,
                           BN=True, bn_type="BN", bn_affine=True, dropout=0.0))
    r = DALETOR(sf_para_dict=sf, model_para_dict=dict(model_id="DALETOR", rt=10.0, top_k=10), gpu=False, device="cpu")
    r.init()
    init = seeded_state({k: tuple(v.shape) for k, v in r.point_sf.state_dict().items()})
    with torch.no_grad():
        for k, v in r.point_sf.state_dict().items():
            v.copy_(torch.from_numpy(init[k]))
    losses = []
    for i, (n, m) in enumerate(((40, 5), (23, 3), (64, 8))):
        q = rng.standard_normal((1, F)).astype(np.float32)
        d = rng.standard_normal((n, F)).astype(np.float32)
        R = rele_mat(rng, m, n, False)
        R[0, 0] = 1.0
        out[f"train__q{i}_q_repr"], out[f"train__q{i}_doc_reprs"], out[f"train__q{i}_rele"] = q, d, R
        r.train_mode()
        if i == 0:
            with torch.no_grad():
                out["train__pred0"] = r.div_forward(torch.from_numpy(q), torch.from_numpy(d)).numpy().copy()
        loss, _ = r.div_train_op(torch.from_numpy(q), torch.from_numpy(d), torch.from_numpy(R), presort=True, epoch_k=1)
        losses.append(float(loss))
        if i == 0:
            for k, p in r.point_sf.named_parameters():
                out["train__grad0__" + k] = p.grad.numpy().copy()
    out["train__losses"] = np.asarray(losses, dtype=np.float64)
    r.train_mode()
    with torch.no_grad():
        for i in range(3):
            q, d = (torch.from_numpy(out[f"train__q{i}_{f}"]) for f in ("q_repr", "doc_reprs"))
            out[f"train__final_scores_q{i}"] = r.div_forward(q, d).numpy().copy()


def main():
    rng = np.random.default_rng(2021)
    torch.manual_seed(2021)
    out = {}
    loss_cases(rng, out)
    metric_cases(rng, out)
    train_case(rng, out)
    np.savez_compressed(os.path.join(HERE, "daletor.npz"), **out)
    print(f"daletor.npz: {len(out)} arrays, {sum(1 for k in out if k.endswith('__loss'))} loss runs, "
          f"{sum(1 for k in out if k.endswith('__andcg_ks'))} metric cases")


if __name__ == "__main__":
    main()
