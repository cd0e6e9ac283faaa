"""Test-side restatements of WassRank (mode 'SinkhornOT', 'ST' / 'BothST' histograms) that referee the CUDA kernel.

TEST INFRASTRUCTURE, NOT PRODUCT: the shipped package never imports it.  Two independent statements, both pinned to
outputs of the unmodified reference (tests/golden/wassrank.npz, made by tests/golden/make_golden_wassrank.py) by
tests/test_oracle_wassrank.py:

* ``port_loss`` / ``port_loss_and_grad`` -- an op-for-op ATen restatement of the reference's K-matrix formulation
  (wassrank/wassRank.py:43-86, OldSinkhornOT at pytorch_wasserstein.py:323-394), applied query by query.  It
  reproduces the reference's NaNs where exp(-C/lam) underflows in fp32.
* ``closed_form`` -- the same maths in float64, in the log domain (finite everywhere).

Both extend the reference to B > 1 the way the kernel does: every query gets its own cost matrix, the loss is the mean
over the queries and the gradient carries 1/B (at B = 1 this is the reference exactly).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------- #
# ATen port of the reference's K-matrix computation
# --------------------------------------------------------------------------- #
def wass_cost_mat(labels_row, cost_type, non_rele_gap=100.0, var_penalty=math.e, gain_base=4.0):
    """get_explicit_cost_mat for one query, wassrank/wasserstein_cost_mat.py:47-139 -> [n,n].  Positions, ddg's
    discounts and eg's gap / penalty scalars live in FloatTensors there (:52, :73, :97, :103, :106), whatever the
    labels' dtype."""
    y = labels_row.reshape(1, -1)
    n = y.size(1)
    if cost_type in ("p1", "p2"):                                         # :47-60
        pos = (torch.arange(n) + 1.0).type(torch.FloatTensor)
        C = torch.abs(pos.view(-1, 1) - pos.view(1, -1))
        return torch.pow(C, 2.0) if cost_type == "p2" else C
    if cost_type == "eg":                                                 # :84-111
        gains = torch.pow(gain_base, y) - 1.0
        with_gap = torch.where(gains < 1.0, -torch.FloatTensor([non_rele_gap]), gains)
        D = torch.abs(with_gap.view(1, n, 1) - with_gap.view(1, 1, n))
        C = torch.where(D < 1.0, torch.FloatTensor([var_penalty]), D)
        return (C - (torch.eye(n).type(torch.FloatTensor) * var_penalty).expand(1, -1, -1))[0]
    if cost_type not in ("dg", "ddg"):
        raise NotImplementedError(cost_type)
    gains = torch.pow(2.0, y) - 1.0                                       # :63-81
    D = torch.abs(torch.unsqueeze(gains, dim=2) - torch.unsqueeze(gains, dim=1))
    if cost_type == "ddg":
        disc = torch.unsqueeze(1.0 / torch.log2(torch.arange(n).type(torch.FloatTensor) + 2.0), dim=0)
        D = D * torch.abs(torch.unsqueeze(disc, dim=2) - torch.unsqueeze(disc, dim=1))
    return D[0]


class _OldSinkhornOT(torch.autograd.Function):
    """OldSinkhornOT, wassrank/pytorch_wasserstein.py:323-394, for one query of a batch of ``batch_queries``: the
    K-matrix iteration with max-stabilised products (NaN where exp(-C/lam) underflows, as there).  The loss and the
    saved gradient carry 1/batch_queries (at one query this is the reference exactly)."""

    @staticmethod
    def forward(ctx, pred, target, cost, lam, sh_num_iter, batch_queries):
        na, nb = cost.size(0), cost.size(1)
        K = torch.exp(-cost / lam)
        KM = cost * K
        log_a, log_b = torch.log(pred), torch.log(target)
        log_u = cost.new(1, na).fill_(-math.log(na))
        log_v = cost.new(1, nb).fill_(-math.log(nb))
        for _ in range(sh_num_iter):
            u_max = torch.max(log_u, dim=1, keepdim=True)[0]
            log_v = log_b - torch.log(torch.mm(K.t(), torch.exp(log_u - u_max).t()).t()) - u_max
            v_max = torch.max(log_v, dim=1, keepdim=True)[0]
            log_u = log_a - torch.log(torch.mm(K, torch.exp(log_v - v_max).t()).t()) - v_max
        v_max = torch.max(log_v, dim=1, keepdim=True)[0]
        part1 = torch.log(torch.mm(KM, torch.exp(log_v - v_max).t()).t()) + v_max
        wnorm = torch.exp(log_u + part1).mean(0).sum()
        grad = log_u * lam
        grad = grad - torch.mean(grad, dim=1, keepdim=True)
        grad = grad - torch.mean(grad, dim=1, keepdim=True)
        grad = grad / 1                                                   # the reference's batch size
        ctx.save_for_backward(grad / batch_queries)
        return (wnorm / batch_queries).reshape(1)

    @staticmethod
    def backward(ctx, grad_output):
        res = ctx.saved_tensors[0].clone()
        if grad_output[0] != 1:
            res.mul_(grad_output[0])
        return res, None, None, None, None, None


def port_loss(preds, labels, cost_type="eg", lam=0.1, sh_itr=20, non_rele_gap=100.0, var_penalty=math.e, gain_base=4.0):
    """WassRank.custom_loss_function, mode 'SinkhornOT', 'ST' / 'BothST' histograms (wassrank/wassRank.py:43-86,
    wasserstein_cost_mat.py:181-203), applied query by query: the mean over the batch of each query's loss."""
    B = preds.size(0)
    total = None
    for b in range(B):
        C = wass_cost_mat(labels[b], cost_type, non_rele_gap, var_penalty, gain_base)
        std_hist = F.softmax(labels[b:b + 1], dim=1)
        pred_hist = F.softmax(preds[b:b + 1], dim=1)
        q = _OldSinkhornOT.apply(pred_hist, std_hist, C, lam, sh_itr, B)
        total = q if total is None else total + q
    return total[0]


def port_loss_and_grad(scores, labels, **params):
    """(loss, d loss / d scores as the reference's backward defines it) on a leaf fp32 copy of ``scores``."""
    s = scores.detach().clone().float().requires_grad_(True)
    loss = port_loss(s, labels.float(), **params)
    loss.backward()
    return loss.detach(), s.grad.detach()


# --------------------------------------------------------------------------- #
# float64 log-domain closed form
# --------------------------------------------------------------------------- #
def _lse(x, axis):
    """log-sum-exp along ``axis``; -inf where every entry is -inf."""
    m = np.max(x, axis=axis, keepdims=True)
    m = np.where(np.isfinite(m), m, 0.0)
    with np.errstate(divide="ignore"):
        return np.squeeze(np.log(np.exp(x - m).sum(axis=axis, keepdims=True)) + m, axis)


def wass_cost(y, cost_type, non_rele_gap=100.0, var_penalty=np.e, gain_base=4.0):
    """get_explicit_cost_mat of one query (wassrank/wasserstein_cost_mat.py:47-139) in float64.  The quantities the
    reference keeps in FloatTensors whatever the labels' dtype -- positions, ddg's discounts (:52, :73-74) and eg's gap
    and penalty (:97, :103, :106) -- are fp32-rounded as there."""
    y = np.asarray(y, dtype=np.float64)
    n = y.shape[0]
    if cost_type in ("p1", "p2"):
        C = np.abs(np.subtract.outer(np.arange(n), np.arange(n))).astype(np.float64)
        return C * C if cost_type == "p2" else C
    if cost_type == "eg":
        gap, vp = float(np.float32(non_rele_gap)), float(np.float32(var_penalty))
        g = np.power(float(gain_base), y) - 1.0
        g = np.where(g < 1.0, -gap, g)
        D = np.abs(np.subtract.outer(g, g))
        C = np.where(D < 1.0, vp, D)
        np.fill_diagonal(C, 0.0)
        return C
    g = np.power(2.0, y) - 1.0
    C = np.abs(np.subtract.outer(g, g))
    if cost_type == "ddg":
        # fp32 1 / log2(i + 2) with the logarithm correctly rounded to fp32 (numpy's own fp32 log2 is not, ATen's is),
        # and their differences taken in fp32 as well
        disc = np.float32(1.0) / np.log2(np.arange(n, dtype=np.float64) + 2.0).astype(np.float32)
        C = C * np.abs(np.subtract.outer(disc, disc)).astype(np.float64)
    elif cost_type != "dg":
        raise NotImplementedError(cost_type)
    return C


def closed_form(s, y, cost_type="eg", lam=0.1, sh_itr=20, non_rele_gap=100.0, var_penalty=np.e, gain_base=4.0):
    """WassRank, mode 'SinkhornOT' (wassrank/wassRank.py:43-86, OldSinkhornOT pytorch_wasserstein.py:323-394), in the
    log domain, query by query: the mean over the batch of
        sum_i exp(log_u_i + LSE_{j: C_ij > 0}(log C_ij - C_ij/lam + log_v_j))
    after sh_itr Sinkhorn iterations from log_u = log_v = -log n, and the reference's gradient: g = lam log_u centred
    twice, / B, through the softmax of the scores."""
    s = np.asarray(s, dtype=np.float64); y = np.asarray(y, dtype=np.float64)
    B, n = s.shape
    loss, grad = 0.0, np.zeros_like(s)
    for b in range(B):
        C = wass_cost(y[b], cost_type, non_rele_gap, var_penalty, gain_base)
        nK = -C / lam
        la = s[b] - _lse(s[b], 0)
        lb = y[b] - _lse(y[b], 0)
        lu = np.full(n, -np.log(n))
        lv = np.full(n, -np.log(n))
        for _ in range(sh_itr):
            lv = lb - _lse(nK + lu[:, None], 0)
            lu = la - _lse(nK + lv[None, :], 1)
        with np.errstate(divide="ignore"):
            lc = np.where(C > 0.0, np.log(np.where(C > 0.0, C, 1.0)) + nK, -np.inf)
        loss += np.exp(lu + _lse(lc + lv[None, :], 1)).sum() / B
        g = lam * lu
        g = g - g.mean()
        g = g - g.mean()
        g = g / B
        a = np.exp(la)
        grad[b] = a * (g - (a * g).sum())
    return loss, grad
