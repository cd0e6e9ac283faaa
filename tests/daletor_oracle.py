"""Two independent restatements of the diversification path, for the parity tests:

* ``port_loss``: DALETOR's alphaDCG_as_a_loss (ltr_diversification/score_and_sort/daletor.py:8-40) op for op in ATen
  (fp32, the reference's robust sigmoid and its saved gradient), differentiated by autograd; ``port_metrics``: the
  evaluator's sort + gather and the alpha-nDCG / ERR-IA / nERR-IA functions of metric/srd/diversity_metric.py, with the
  one intended change: a list shorter than a cutoff gives 0 there (the reference's alpha-nDCG@ks returns an [m, len(ks)]
  matrix for such a list).
* ``closed_form`` / ``closed_form_metrics``: the same quantities in float64 numpy from the formulas (DESIGN §4), with
  the gradient in closed form.
"""
import zlib

import numpy as np
import torch

from oracle.ref_port import _RobustSigmoid


def port_loss(scores, R, rt=10.0, top_k=10, alpha=0.5):
    """scores [1,n] (leaf or not), R [m,n] -> 0-dim loss; daletor.py:8-40 with the reference's operators."""
    diffs = scores.unsqueeze(2) - scores.unsqueeze(1)
    ind = _RobustSigmoid.apply(torch.transpose(diffs, 1, 2), rt)
    hat_pis = torch.sum(ind, dim=2) + 0.5
    Rx = R.unsqueeze(1).expand(-1, R.size(1), -1)
    prior = torch.sum(ind * Rx, dim=2) - R / 2.0
    gains = R * torch.pow((1.0 - alpha), prior) / torch.log2(1.0 + hat_pis)
    glob = torch.sum(gains, dim=1)
    return -(torch.sum(glob) if top_k is None else torch.sum(glob[0:top_k]))


def port_loss_and_grad(scores, R, rt=10.0, top_k=10, alpha=0.5):
    s = torch.as_tensor(scores, dtype=torch.float32).reshape(1, -1).clone().requires_grad_(True)
    loss = port_loss(s, torch.as_tensor(R, dtype=torch.float32), rt, top_k, alpha)
    loss.backward()
    return float(loss.detach()), s.grad[0].numpy().copy()


def _sig(x, rt):
    return np.where(x > 0, 1.0 / (1.0 + np.exp(-rt * np.abs(x))),
                    np.where(x < 0, np.exp(-rt * np.abs(x)) / (1.0 + np.exp(-rt * np.abs(x))), 0.5))


def closed_form(scores, R, rt=10.0, top_k=10, alpha=0.5):
    """float64 (loss, grad) from the closed form: sig_ij = sigma(rt (s_j - s_i)), pi_i = 1/2 + sum_j sig_ij,
    C_si = sum_j sig_ij R_sj - R_si/2, g_si = R_si (1-alpha)^C_si / log2(1+pi_i), L = -sum_{s<K} sum_i g_si;
    dL/ds_k = sum_i c_ik d_ik - sum_j c_kj d_kj with c_ij = a_i + sum_s b_si R_sj."""
    s = np.asarray(scores, dtype=np.float64).reshape(-1)
    R = np.asarray(R, dtype=np.float64)
    m = R.shape[0]
    rows = m if not top_k or top_k <= 0 else min(top_k, m)
    R = R[:rows]
    if rows == 0 or s.size == 0:
        return 0.0, np.zeros_like(s)
    sig = _sig(s[None, :] - s[:, None], rt)                  # [i, j]
    pi = 0.5 + sig.sum(axis=1)
    C = R @ sig.T - R / 2.0                                   # C[s, i] = sum_j sig_ij R_sj
    g = R * np.power(1.0 - alpha, C) / np.log2(1.0 + pi)[None, :]
    loss = -g.sum()
    d = rt * sig * (1.0 - sig)
    a = g.sum(axis=0) / ((1.0 + pi) * np.log(1.0 + pi))
    b = -np.log(1.0 - alpha) * g
    c = a[:, None] + b.T @ R                                  # c[i, j] = a_i + sum_s b_si R_sj
    grad = (c * d).sum(axis=0) - (c * d).sum(axis=1)
    return float(loss), grad


def _sys_rele(scores, R):
    s = torch.as_tensor(scores, dtype=torch.float32).reshape(1, -1)
    Rt = torch.as_tensor(R, dtype=torch.float32)
    _, order = torch.sort(s, dim=1, descending=True, stable=True)
    return torch.gather(Rt, dim=1, index=order.expand(Rt.size(0), -1)), Rt, order[0]


def port_metrics(scores, R, ks, max_label, alpha=0.5):
    """-> (andcg, err_ia, nerr_ia: float32 [len(ks)], order) with the reference's operators; 0 at cutoffs beyond n."""
    sys_R, ide_R, order = _sys_rele(scores, R)
    n, m = sys_R.size(1), sys_R.size(0)
    out = np.zeros((3, len(ks)), dtype=np.float32)
    t2 = torch.tensor([2.0])

    def dcgs(M, K):
        prior = torch.zeros_like(M[:, :K])
        prior[:, 1:K] = M[:, 0:K - 1]
        cnt = torch.cumsum(prior, dim=1)
        den = torch.log2(torch.arange(K, dtype=torch.float) + 2.0)
        return torch.cumsum(torch.sum(torch.pow(1.0 - alpha, cnt) * M[:, :K] / den, dim=0), dim=0)

    def errs(M, K):
        sat = (torch.pow(t2, M[:, :K]) - 1.0) / torch.pow(t2, max_label)
        cum = torch.cumprod(1.0 - sat, dim=1)
        casc = torch.ones_like(cum)
        casc[:, 1:K] = cum[:, 0:K - 1]
        rr = 1.0 / (torch.arange(K, dtype=torch.float).view(1, -1) + 1.0)
        return torch.sum(torch.cumsum(sat * casc * rr, dim=1), dim=0) / m

    used = [k for k in ks if k <= n]
    if used:
        K = max(used)
        ds, di, es, ei = dcgs(sys_R, K), dcgs(ide_R, K), errs(sys_R, K), errs(ide_R, K)
        for c, k in enumerate(ks):
            if k <= n:
                out[0, c] = float(ds[k - 1] / di[k - 1]) if di[k - 1] > 0 else 0.0
                out[1, c] = float(es[k - 1])
                out[2, c] = float(es[k - 1] / ei[k - 1]) if ei[k - 1] > 0 else 0.0
    return out[0], out[1], out[2], order.numpy()


def closed_form_metrics(scores, R, ks, max_label, alpha=0.5):
    """float64 alpha-nDCG / ERR-IA / nERR-IA at ks (0 beyond n) of the stable score-descending order."""
    s = np.asarray(scores, dtype=np.float64).reshape(-1)
    R = np.asarray(R, dtype=np.float64)
    m, n = R.shape
    order = np.argsort(-s, kind="stable")

    def run(M):
        cnt = np.zeros(m)
        casc = np.ones(m)
        dcg, err, d_out, e_out = 0.0, 0.0, [], []
        for p in range(n):
            r = M[:, p]
            dcg += float(np.sum(r * np.power(1.0 - alpha, cnt))) / np.log2(p + 2.0)
            cnt += r
            sat = (np.power(2.0, r) - 1.0) / 2.0 ** max_label
            err += float(np.sum(sat * casc)) / (p + 1.0)
            casc *= 1.0 - sat
            d_out.append(dcg)
            e_out.append(err / m if m else 0.0)
        return d_out, e_out

    ds, es = run(R[:, order])
    di, ei = run(R)
    out = np.zeros((3, len(ks)))
    for c, k in enumerate(ks):
        if k <= n:
            out[0, c] = ds[k - 1] / di[k - 1] if di[k - 1] > 0 else 0.0
            out[1, c] = es[k - 1]
            out[2, c] = es[k - 1] / ei[k - 1] if ei[k - 1] > 0 else 0.0
    return out[0], out[1], out[2], order


def seeded_state(shapes, seed=2718):
    """Starting weights of the train-step fixture, rebuilt from (seed, key) so the fixture does not have to store them:
    {key: float32 array} for a {key: shape} of a pointsf state dict -- xavier-normal Linear weights, small biases, BN
    weights near 1."""
    out = {}
    for key, shape in shapes.items():
        rng = np.random.default_rng([seed, zlib.crc32(key.encode())])
        if key.startswith("ff_") and key.endswith(".weight"):
            a = rng.standard_normal(shape) * np.sqrt(2.0 / (shape[0] + shape[1]))
        elif key.startswith("bn_") and key.endswith(".weight"):
            a = 1.0 + 0.1 * rng.standard_normal(shape)
        else:
            a = 0.1 * rng.standard_normal(shape)
        out[key] = a.astype(np.float32)
    return out
