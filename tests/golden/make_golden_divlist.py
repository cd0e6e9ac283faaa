"""Golden fixtures for the diversification list scorer (DALETOR with sf_id='listsf'), produced by the UNMODIFIED
reference.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_divlist.py

Every case builds the reference's DALETOR with a listsf dict, loads the seeded starting weights that
``tests.divlist_oracle.seeded_state`` rebuilds and runs in ``eval_mode()``: the MHSA dropout and the uni_sf's fixed 0.1
dropout are off, and the uni_sf BN keeps its per-call statistics.  The inputs are not stored either:
``tests.divlist_oracle.case_inputs`` rebuilds them.

* ``<enc>_h<heads>`` for the three encoder types and 6 / 2 heads, F = 12 (heads 6 and 18 wide), tests.divlist_oracle
  SMALL_LISTSF, three queries of 150, 2 and 37 documents: ``pred_q<i>`` (scores from the starting weights),
  ``loss_q<i>`` (one DALETOR step of that query from the starting weights), ``grad__<encoder|uni_sf>__<key>`` (the
  parameter gradients of that step for the query ``tests.divlist_oracle.grad_query`` names: the 150-document list at
  6 heads, the 37-document one at 2 heads), ``losses`` (three steps q0, q1, q2 in turn, Adagrad lr 0.01) and
  ``final_q<i>`` (each query's scores after those steps).
* ``default``: the reference default (div_parameter.py:98-104: AttnDIN, 6 heads, 6 layers) at F = 100 on 256, 2 and 37
  documents: ``pred_q<i>``, ``loss_q<i>``, ``losses`` and ``final_q<i>`` only.
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
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))          # the repository: tests.divlist_oracle

from ptranking.ltr_diversification.score_and_sort.daletor import DALETOR  # noqa: E402
from tests.divlist_oracle import SMALL, case_config, case_inputs, grad_query, seeded_state, state_shapes  # noqa: E402


def make_ranker(F, listsf):
    sf = dict(sf_id="listsf", opt="Adagrad", lr=0.01, listsf=dict(num_features=F, **copy.deepcopy(listsf)))
    r = DALETOR(sf_para_dict=sf, model_para_dict=dict(model_id="DALETOR", rt=10.0, top_k=10), gpu=False, device="cpu")
    r.init()
    init = seeded_state(state_shapes(r.list_sf["encoder"], r.list_sf["uni_sf"]))
    with torch.no_grad():
        for part in ("encoder", "uni_sf"):
            for k, v in r.list_sf[part].state_dict().items():
                v.copy_(torch.from_numpy(init[part][k]))
    r.eval_mode()
    return r


def run_case(name, out):
    F, listsf, _ = case_config(name)
    qs = case_inputs(name)
    r = make_ranker(F, listsf)
    with torch.no_grad():
        for i, (q, d, _) in enumerate(qs):
            out[f"{name}__pred_q{i}"] = r.div_forward(torch.from_numpy(q), torch.from_numpy(d)).numpy().copy()
    for i, (q, d, R) in enumerate(qs):          # one step of each query from the starting weights
        r = make_ranker(F, listsf)
        loss, _ = r.div_train_op(torch.from_numpy(q), torch.from_numpy(d), torch.from_numpy(R), presort=True, epoch_k=1)
        out[f"{name}__loss_q{i}"] = np.float64(loss.detach())
        if i == grad_query(name):
            for part in ("encoder", "uni_sf"):
                for k, p in r.list_sf[part].named_parameters():
                    out[f"{name}__grad__{part}__{k}"] = p.grad.numpy().copy()
    r = make_ranker(F, listsf)                  # three steps in turn
    losses = []
    for q, d, R in qs:
        loss, _ = r.div_train_op(torch.from_numpy(q), torch.from_numpy(d), torch.from_numpy(R), presort=True, epoch_k=1)
        losses.append(float(loss.detach()))
    out[f"{name}__losses"] = np.asarray(losses, dtype=np.float64)
    with torch.no_grad():
        for i, (q, d, _) in enumerate(qs):
            out[f"{name}__final_q{i}"] = r.div_forward(torch.from_numpy(q), torch.from_numpy(d)).numpy().copy()


def main():
    torch.manual_seed(2024)
    out = {}
    for name in SMALL + ["default"]:
        run_case(name, out)
    np.savez_compressed(os.path.join(HERE, "divlist.npz"), **out)
    print(f"divlist.npz: {len(out)} arrays")


if __name__ == "__main__":
    main()
