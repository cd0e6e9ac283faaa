"""oracle/closed_form.py -- float64 numpy closed forms of the six ranking losses.

TEST INFRASTRUCTURE, NOT PRODUCT (same import rule as oracle/ref_port.py).

A second, independent statement of each loss value and its gradient with
respect to the scores, written from the math (SURVEY.md Appendix A) instead of
from autograd, in float64 so it can referee fp32 disagreements between the
CUDA kernels and the ATen restatement.  Formulas cite the reference lines whose
behaviour they encode.  ATen's BCE clamps (log >= -100,
max(p(1-p),1e-12)) act on the fp32-rounded sigmoid; ``_bce_terms`` reproduces that
rounding (p == 1.0f beyond x ~ 17.3) and keeps the rest in float64.  Pinned by
tests/test_oracle_vs_golden.py against outputs of the reference itself.
"""
from __future__ import annotations

import numpy as np

LN2 = np.log(2.0)


def _gain(y):
    return np.power(2.0, y) - 1.0


def _disc(n):
    return np.log2(np.arange(n, dtype=np.float64) + 2.0)


def _idcg(ideal):
    return (_gain(ideal) / _disc(ideal.shape[1])[None]).sum(1)


def _sigmoid(x):
    return 0.5 * (1.0 + np.tanh(0.5 * x))


def _stable_desc_order(s):
    """score descending, index ascending among equals (the total order the kernels use)."""
    return np.argsort(-s, axis=1, kind="stable")


def _bce_terms(x, pbar, w, fp32_sigmoid=True):
    """weighted BCE over logits x: loss cell and d(cell)/dx with ATen's clamps.

    ATen evaluates p = sigmoid(x) in fp32 and then takes log(p), log(1-p) and p(1-p)
    of that rounded p (binary_cross_entropy: log >= -100, backward max(p(1-p),1e-12)).
    With fp32_sigmoid=True the rounding of p is reproduced (p == 1.0f for x > ~17.3,
    so log(1-p) hits the -100 clamp); everything downstream stays float64."""
    if fp32_sigmoid:
        x32 = x.astype(np.float32)
        with np.errstate(over="ignore"):
            p32 = (np.float32(1.0) / (np.float32(1.0) + np.exp(-x32))).astype(np.float32)
        p = p32.astype(np.float64)
        one_m_p = (np.float32(1.0) - p32).astype(np.float64)
        with np.errstate(divide="ignore"):
            logp = np.maximum(np.log(p), -100.0)
            log1mp = np.maximum(np.log(one_m_p), -100.0)
    else:
        p = _sigmoid(x)
        one_m_p = 1.0 - p
        logp = np.maximum(-np.logaddexp(0.0, -x), -100.0)
        log1mp = np.maximum(-np.logaddexp(0.0, x), -100.0)
    cell = -w * (pbar * logp + (1.0 - pbar) * log1mp)
    pq = p * one_m_p
    dcell = w * (p - pbar) * pq / np.maximum(pq, 1e-12)
    return cell, dcell


def ranknet(s, y, sigma=1.0):
    """pairwise/ranknet.py:32-36: all i<j in input order, ties count with target 1/2."""
    s = s.astype(np.float64); y = y.astype(np.float64)
    B, n = s.shape
    x = sigma * (s[:, :, None] - s[:, None, :])
    pbar = 0.5 * (1.0 + np.clip(y[:, :, None] - y[:, None, :], -1.0, 1.0))
    upper = np.triu(np.ones((n, n)), 1)[None]
    cell, dcell = _bce_terms(x, pbar, upper)
    g = sigma * dcell
    return cell.sum(), g.sum(2) - g.sum(1)


def lambdarank(s, y, sigma=1.0):
    """listwise/lambdarank.py:39-56 + metric_utils.py:19-45; y presorted descending."""
    s = s.astype(np.float64); y = y.astype(np.float64)
    B, n = s.shape
    order = _stable_desc_order(s)
    ss = np.take_along_axis(s, order, 1)
    ys = np.take_along_axis(y, order, 1)
    ng = _gain(ys) / _idcg(y)[:, None]
    inv_d = 1.0 / _disc(n)
    delta = np.abs(ng[:, :, None] - ng[:, None, :]) * np.abs(inv_d[None, :, None] - inv_d[None, None, :])
    x = sigma * (ss[:, :, None] - ss[:, None, :])
    pbar = 0.5 * (1.0 + np.clip(ys[:, :, None] - ys[:, None, :], -1.0, 1.0))
    w = delta * np.triu(np.ones((n, n)), 1)[None]
    cell, dcell = _bce_terms(x, pbar, w)
    g = sigma * dcell
    gs = g.sum(2) - g.sum(1)
    grad = np.zeros_like(s)
    np.put_along_axis(grad, order, gs, 1)
    return cell.sum(), grad


def lambdaloss(s, y, k=5, sigma=1.0, loss_type="NDCG_Loss2++", mu=5.0, presort=True, eps=1e-8):
    """listwise/lambdaloss.py:73-132."""
    s = s.astype(np.float64); y = y.astype(np.float64)
    B, n = s.shape
    ideal = y if presort else -np.sort(-y, axis=1)
    if presort:
        target, back = s, None
    else:
        back = np.argsort(-y, axis=1, kind="stable")
        target = np.take_along_axis(s, back, 1)
    order = _stable_desc_order(target)
    ss = np.take_along_axis(target, order, 1)
    ys = np.take_along_axis(ideal, order, 1)
    ng = _gain(ys) / _idcg(ideal)[:, None]
    D = _disc(n)                       # D(r) = log2(r+2) ; reference's dists_1D = 1/D
    idx = np.arange(n)
    gap = np.abs(idx[:, None] - idx[None, :])
    dgap = np.abs(np.log2(gap + 1.0) - np.log2(gap + 2.0)) * (gap > 0)      # |D(d-1) - D(d)|, diag zeroed
    ngd = np.abs(ng[:, :, None] - ng[:, None, :])
    if loss_type == "NDCG_Loss1":
        w = np.broadcast_to((ng * D[None])[:, None, :], (B, n, n))          # w_j, broadcast over rows
    elif loss_type == "NDCG_Loss2":
        w = dgap[None] * ngd
    elif loss_type == "NDCG_Loss2++":
        w = (np.abs(D[:, None] - D[None, :]) + mu * dgap)[None] * ngd
    else:
        raise NotImplementedError(loss_type)
    dx = np.clip(ss[:, :, None] - ss[:, None, :], -1e8, 1e8)
    p = _sigmoid(sigma * dx)
    pc = np.maximum(p, eps)
    u = np.power(pc, w)
    uc = np.maximum(u, eps)
    K = min(k, n)
    mask = np.zeros((n, n), bool); mask[:K, :K] = True
    mask = np.broadcast_to(mask[None], (B, n, n)).copy()
    if loss_type != "NDCG_Loss1":
        mask &= (ys[:, :, None] - ys[:, None, :]) > 0
    loss = -(np.log2(uc) * mask).sum()
    live = mask & (p >= eps) & (u >= eps)
    g = np.where(live, -w * sigma * (1.0 - p) / LN2, 0.0)                   # d/d(s_i - s_j)
    gs = g.sum(2) - g.sum(1)
    gt = np.zeros_like(s)
    np.put_along_axis(gt, order, gs, 1)
    if back is not None:
        grad = np.zeros_like(s)
        np.put_along_axis(grad, back, gt, 1)
    else:
        grad = gt
    return loss, grad


def _softmax(v):
    e = np.exp(v - v.max(1, keepdims=True))
    return e / e.sum(1, keepdims=True)


def listnet(s, y):
    """listwise/listnet.py:39."""
    s = s.astype(np.float64); y = y.astype(np.float64)
    logsm = s - s.max(1, keepdims=True)
    logsm = logsm - np.log(np.exp(logsm).sum(1, keepdims=True))
    return -(_softmax(y) * logsm).sum(), _softmax(s) - _softmax(y)


def listmle(s, perm):
    """listwise/listmle.py:83-97 with the tie-shuffled ordering given."""
    s = s.astype(np.float64)
    z = np.take_along_axis(s, perm.astype(np.int64), 1)
    m = z.max(1, keepdims=True)
    e = np.exp(z - m)
    C = np.cumsum(e[:, ::-1], 1)[:, ::-1]
    loss = (np.log(C) + m - z).sum()
    gz = e * np.cumsum(1.0 / C, 1) - 1.0
    grad = np.zeros_like(s)
    np.put_along_axis(grad, perm.astype(np.int64), gz, 1)
    return loss, grad


def approxndcg(s, y, alpha=10.0, presort=True, batch_coupled=True):
    """listwise/approxNDCG.py:19-28,45-62.  batch_coupled=True keeps the [B]/[B,1]
    broadcast (every query scaled by sum_a 1/iDCG_a, :58-61)."""
    s = s.astype(np.float64); y = y.astype(np.float64)
    B, n = s.shape
    if presort:
        target, ideal, back = s, y, None
    else:
        back = np.argsort(-y, axis=1, kind="stable")
        ideal = np.take_along_axis(y, back, 1)
        target = np.take_along_axis(s, back, 1)
    sg = _sigmoid(alpha * (target[:, None, :] - target[:, :, None]))        # [b,i,j] = sig(a(s_j - s_i))
    pi = sg.sum(2) + 0.5
    G = _gain(ideal)
    lg = np.log2(pi + 1.0)
    dcg = (G / lg).sum(1)
    inv = 1.0 / _idcg(ideal)
    scale = np.full(B, inv.sum()) if batch_coupled else inv
    loss = -(scale * dcg).sum()
    c = scale[:, None] * G / (lg ** 2 * (pi + 1.0) * LN2)
    d = alpha * sg * (1.0 - sg)                                              # symmetric in (i,j)
    gt = (d * (c[:, :, None] - c[:, None, :])).sum(1)                        # grad_j = sum_i d_ij (c_i - c_j)
    if back is not None:
        grad = np.zeros_like(s)
        np.put_along_axis(grad, back, gt, 1)
    else:
        grad = gt
    return loss, grad


def rankmse(s, y):
    """pointwise/rank_mse.py:13-22: mean over queries of the summed squared error."""
    s = s.astype(np.float64); y = y.astype(np.float64)
    B = s.shape[0]
    return ((s - y) ** 2).sum() / B, 2.0 * (s - y) / B


def rankcosine(s, y, eps=1e-8):
    """listwise/rank_cosine.py:33 with ATen's cosine_similarity (each vector divided by max(norm, eps))."""
    s = s.astype(np.float64); y = y.astype(np.float64)
    ns = np.sqrt((s * s).sum(1, keepdims=True)); ny = np.sqrt((y * y).sum(1, keepdims=True))
    S = np.maximum(ns, eps); Y = np.maximum(ny, eps)
    sy = (s * y).sum(1, keepdims=True)
    cos = sy / (S * Y)
    dcos = y / (S * Y) - np.where(ns > eps, sy * s / (S * S * np.maximum(ns, 1e-300) * Y), 0.0)
    return (2.0 * (1.0 - cos)).sum(), -2.0 * dcos


def stlistnet(s, y, unif, temperature=1.0):
    """listwise/st_listnet.py:41-49 with the uniform draw given.  The Gumbel transform is evaluated in fp32 like the
    reference (its 1e-20 guards are below float64's resolution of u but not of fp32's)."""
    u = unif.astype(np.float32)
    g = -np.log(-np.log(u + np.float32(1e-20)) + np.float32(1e-20))
    z = (s.astype(np.float64) + g.astype(np.float64)) / temperature
    y = y.astype(np.float64)
    logsm = z - z.max(1, keepdims=True)
    logsm = logsm - np.log(np.exp(logsm).sum(1, keepdims=True))
    return -(_softmax(y) * logsm).sum(), (_softmax(z) - _softmax(y)) / temperature


def softrank(s, y, delta=2.0, top_k=None):
    """listwise/softrank.py:46-72 (nDCG, labels presorted)."""
    from math import pi, sqrt
    from scipy.special import erfc
    s = s.astype(np.float64); y = y.astype(np.float64)
    B, n = s.shape
    den = sqrt(2.0 * 2.0 * delta * delta)
    x = (s[:, :, None] - s[:, None, :]) / den                       # [b,i,j]
    phi = 0.5 * erfc(x)
    off = 1.0 - np.eye(n)[None]
    r = (phi * off).sum(2) + 1.0
    G = _gain(y)
    K = n if top_k is None else min(top_k, n)
    mask = (np.arange(n) < K)[None, :]
    lg = np.log2(r + 1.0)
    idcg = _idcg(y)[:, None]
    loss = -((G / lg) * mask / idcg).sum()
    c = mask * G / (idcg * lg ** 2 * (r + 1.0) * LN2)
    e = -np.exp(-x * x) / (sqrt(pi) * den) * off
    grad = (e * (c[:, :, None] - c[:, None, :])).sum(2)
    return loss, grad


def ndcg_at_ks(scores, labels, ks, presort=True):
    """metric/adhoc/adhoc_metric.py:219-260 over the ranking base/ranker.py:50-56 builds."""
    s = scores.astype(np.float64); y = labels.astype(np.float64)
    B, n = s.shape
    order = _stable_desc_order(s)
    sys_r = np.take_along_axis(y, order, 1)
    ideal = y if presort else -np.sort(-y, axis=1)
    D = _disc(n)[None]
    sys_c = np.cumsum(_gain(sys_r) / D, 1)
    ide_c = np.cumsum(_gain(ideal) / D, 1)
    out = np.zeros((B, len(ks)))
    for c, k in enumerate(ks):
        if k <= n:
            with np.errstate(divide="ignore", invalid="ignore"):
                out[:, c] = sys_c[:, k - 1] / ide_c[:, k - 1]
    return out, order
