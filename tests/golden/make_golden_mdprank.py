"""Golden fixtures for MDPRank, produced by the UNMODIFIED reference.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_mdprank.py

The reference class's own custom_loss_function (ltr_adhoc/listwise/mdprank.py:24-79) runs on a leaf score tensor; a
throw-away SGD(lr=0) stands in for the optimizer it steps.  The reference asserts one query per call, so every case is
one query, and it raises when top_k exceeds the list's length, so the grid keeps top_k <= n.  Its random draw is
captured by wrapping torch.multinomial (PL: the sampled ordering) or torch.rand (STPL: the uniforms) while it runs; for
STPL the ordering is recomputed from the captured uniforms with the reference's own ops.  Output: mdprank.npz, keys
"n<n>_<tag>__scores" / "__labels" for each list and "<dist>_k<top_k>_g<gamma>_T<T>_n<n>_<tag>__<field>" for each run
of it, with fields loss, grad, perm (int16) and, for STPL, unif.
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
sys.path.insert(0, HERE)

from make_golden import synth_labels, point_sf_dict, MSLR_P, MQ_P  # noqa: E402
from ptranking.ltr_adhoc.listwise.mdprank import MDPRank  # noqa: E402

EPS = 1e-20


def run(dist, top_k, gamma, T, s, y):
    para = dict(model_id="MDPRank", gamma=gamma, top_k=top_k, temperature=T, distribution=dist)
    r = MDPRank(sf_para_dict=point_sf_dict(4), model_para_dict=para, gpu=False, device="cpu")
    leaf = torch.from_numpy(s).clone().requires_grad_(True)
    r.optimizer = torch.optim.SGD([leaf], lr=0.0)
    captured = {}
    name = "multinomial" if dist == "PL" else "rand"
    real = getattr(torch, name)

    def spy(*a, **k):
        out = real(*a, **k)
        captured["draw"] = out.detach().clone()
        return out
    setattr(torch, name, spy)
    try:
        loss = r.custom_loss_function(leaf, torch.from_numpy(y), presort=True)
    finally:
        setattr(torch, name, real)
    extra = {}
    if dist == "PL":
        perm = captured["draw"][0].numpy().astype(np.int32)
    else:
        u = captured["draw"]
        with torch.no_grad():
            logits = torch.from_numpy(s) + (-torch.log(-torch.log(u + EPS) + EPS))
            logits = logits if 1.0 == T else logits / T
            perm = torch.sort(logits, dim=1, descending=True)[1][0].numpy().astype(np.int32)
        extra["unif"] = u.numpy()
    return np.float64(loss.detach()), leaf.grad.detach().numpy().copy(), perm, extra


def main():
    rng = np.random.default_rng(3141)
    torch.manual_seed(3141)
    out = {}
    for n in (1, 2, 8, 50, 256, 1024):
        y = synth_labels(rng, 1, n, MQ_P if n == 50 else MSLR_P)
        for tag, s in (("sig", 1.0 / (1.0 + np.exp(-rng.standard_normal((1, n))))), ("wide", 2.5 * rng.standard_normal((1, n)))):
            s = s.astype(np.float32)
            out[f"n{n}_{tag}__scores"], out[f"n{n}_{tag}__labels"] = s, y
            for dist in ("PL", "STPL"):
                for top_k in (None, 1, 10):
                    if top_k is not None and top_k > n:
                        continue
                    for gamma in (1.0, 0.9):
                        for T in (1.0, 0.5, 0.1):
                            key = f"{dist}_k{top_k}_g{gamma}_T{T}_n{n}_{tag}"
                            loss, grad, perm, extra = run(dist, top_k, gamma, T, s, y)
                            out[key + "__loss"], out[key + "__grad"] = loss, grad
                            out[key + "__perm"] = perm[None].astype(np.int16)
                            for f, v in extra.items():
                                out[key + "__" + f] = v
    np.savez_compressed(os.path.join(HERE, "mdprank.npz"), **out)
    print(f"mdprank.npz: {len(out)} arrays, {sum(1 for k in out if k.endswith('__loss'))} runs")


if __name__ == "__main__":
    main()
