"""Golden fixtures for WassRank, produced by the UNMODIFIED reference.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_wassrank.py

The reference class's own custom_loss_function (mode 'SinkhornOT', wassrank/wassRank.py:43-86) runs on a leaf score
tensor; a throw-away SGD(lr=0) stands in for the optimizer it steps, and its per-call print goes to a discarded buffer.
The reference handles one query per call (OldSinkhornOT rejects the [B,n,n] cost of a larger batch), so every case is
one query.  eg / dg / ddg also run on float64 tensors (the reference accepts them there); p1 / p2 build their cost in a
FloatTensor whatever the input, so they have fp32 runs only.  NaN outputs are stored as they come.  Output:
wassrank.npz, keys "<cost>_lam<lam>_it<sh_itr>_<case>__<field>" with fields scores, labels, loss, grad, [loss64,
grad64], cost, lam, sh_itr.
"""
import contextlib
import io
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
sys.path.insert(0, HERE)

from make_golden import synth_labels, point_sf_dict, MSLR_P, MQ_P  # noqa: E402
from ptranking.ltr_adhoc.listwise.wassrank.wassRank import WassRank, WassRankParameter  # noqa: E402

COSTS = ["p1", "p2", "eg", "dg", "ddg"]


def run(para, s, y, dtype):
    r = WassRank(sf_para_dict=point_sf_dict(4), wass_para_dict=para, dict_cost_mats={}, dict_std_dists={},
                 gpu=False, device="cpu")
    leaf = torch.from_numpy(s).to(dtype).clone().requires_grad_(True)
    r.optimizer = torch.optim.SGD([leaf], lr=0.0)
    with contextlib.redirect_stdout(io.StringIO()):
        loss = r.custom_loss_function(leaf, torch.from_numpy(y).to(dtype), batch_ids=["q"])
    return np.float64(loss.detach().reshape(-1)[0]), leaf.grad.detach().numpy().copy()


def main():
    rng = np.random.default_rng(2019)
    torch.manual_seed(2019)
    default = WassRankParameter().default_para_dict()
    cases = []
    for n in (1, 2, 8, 50, 256, 1024):
        y = synth_labels(rng, 1, n, MQ_P if n == 50 else MSLR_P)
        for tag, s in (("sig", 1.0 / (1.0 + np.exp(-rng.standard_normal((1, n))))), ("wide", 2.5 * rng.standard_normal((1, n)))):
            cases.append((f"n{n}_{tag}", s.astype(np.float32), y, ((0.1, 20), (1.0, 5))))
    # labels in no particular order; real-valued labels (more distinct values than the kernel's label-group table)
    y = synth_labels(rng, 1, 50, MSLR_P, presort=False)
    cases.append(("n50_unsorted", (2.5 * rng.standard_normal((1, 50))).astype(np.float32), y, ((0.1, 20),)))
    y = np.round(4.0 * rng.random((1, 64)), 3).astype(np.float32)
    cases.append(("n64_real", (1.0 / (1.0 + np.exp(-rng.standard_normal((1, 64))))).astype(np.float32), y, ((0.1, 20), (1.0, 5))))
    out = {}
    for case, s, y, settings in cases:
        for cost in COSTS:
            for lam, it in settings:
                para = dict(default, cost_type=cost, lam=lam, sh_itr=it)
                key = f"{cost}_lam{lam}_it{it}_{case}"
                out[key + "__scores"], out[key + "__labels"] = s, y
                out[key + "__cost"], out[key + "__lam"], out[key + "__sh_itr"] = np.int64(COSTS.index(cost)), np.float64(lam), np.int64(it)
                out[key + "__loss"], out[key + "__grad"] = run(para, s, y, torch.float32)
                if cost in ("eg", "dg", "ddg"):
                    out[key + "__loss64"], out[key + "__grad64"] = run(para, s, y, torch.float64)
    np.savez_compressed(os.path.join(HERE, "wassrank.npz"), **out)
    nan = sum(1 for k in out if k.endswith("__loss") and not np.isfinite(out[k]))
    print(f"wassrank.npz: {len(out)} arrays, {sum(1 for k in out if k.endswith('__loss'))} cases, {nan} with a NaN fp32 loss")


if __name__ == "__main__":
    main()
