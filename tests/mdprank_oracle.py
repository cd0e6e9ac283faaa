"""Test-side restatements of MDPRank that referee the CUDA kernel.

TEST INFRASTRUCTURE, NOT PRODUCT: the shipped package never imports it.  Two independent statements, both pinned to
outputs of the unmodified reference (tests/golden/mdprank.npz, made by tests/golden/make_golden_mdprank.py) by
tests/test_oracle_mdprank.py:

* ``port_loss_and_grad`` -- an op-for-op ATen restatement of MDPRank.custom_loss_function (ltr_adhoc/listwise/mdprank.py:
  24-79 with sample_ranking_PL / sample_ranking_PL_gumbel_softmax, ltr_adhoc/util/sampling_utils.py:31-79), applied
  query by query, with the draws injectable: ``perm`` replaces PL's torch.multinomial, ``unif`` STPL's torch.rand.
* ``closed_form`` -- the loss and its gradient in float64 numpy, from the formulas rather than from autograd.

Both extend the reference the way the kernel does: any number of queries (the batch loss is the sum over queries) and
top_k clamped to the list's length (the reference raises when top_k exceeds it).
"""
import numpy as np
import torch

EPS = 1e-20


def _k_eff(top_k, n):
    return n if (top_k is None or top_k <= 0 or top_k > n) else int(top_k)


def port_query_loss(preds, labels, distribution="PL", top_k=None, gamma=1.0, temperature=1.0, perm=None, unif=None):
    """Loss of one query ([1,n] tensors), as mdprank.py:33-71 computes it."""
    if distribution == "PL":                                              # sampling_utils.py:31-56
        if perm is None:
            target = torch.div(preds, temperature) if 1.0 != temperature else preds
            m, _ = torch.max(target, dim=1, keepdim=True)
            perm = torch.multinomial(torch.exp(target - m), replacement=False, num_samples=preds.size(1))
        inds = perm.reshape(1, -1).long()
        action_preds = torch.gather(preds, dim=1, index=inds)
    elif distribution == "STPL":                                          # sampling_utils.py:59-79
        if unif is None:
            unif = torch.rand(preds.size())
        gumbel = -torch.log(-torch.log(unif.reshape(preds.shape) + EPS) + EPS)
        logits = preds + gumbel if 1.0 == temperature else (preds + gumbel) / temperature
        action_preds, inds = torch.sort(logits, dim=1, descending=True)
    else:
        raise NotImplementedError(distribution)
    k = _k_eff(top_k, labels.size(1))
    action_stds = torch.gather(labels, dim=1, index=inds)
    gains = torch.pow(2.0, action_stds) - 1.0
    ranks = torch.arange(k, dtype=torch.float).view(1, -1)
    rewards = gains[:, 0:k] / torch.log2(2.0 + ranks)
    G = torch.flip(torch.cumsum(torch.flip(rewards, dims=[1]), dim=1), dims=[1])
    if gamma != 1.0:
        G = G * torch.cumprod(torch.ones(k).view(1, -1) * gamma, dim=1)
    m, _ = torch.max(action_preds, dim=1, keepdim=True)
    y = torch.exp(action_preds - m)
    lcse = torch.log(torch.flip(torch.cumsum(torch.flip(y, dims=[1]), dim=1), dims=[1])) + m
    neg_log_probs = lcse[:, 0:k] - action_preds[:, 0:k]
    return torch.sum(torch.sum(neg_log_probs * G[:, 0:k], dim=1)), inds[0]


def port_loss_and_grad(scores, labels, distribution="PL", top_k=None, gamma=1.0, temperature=1.0, perm=None, unif=None):
    """(batch loss, d loss / d scores, sampled orderings [B,n]) on a leaf fp32 copy of ``scores`` ([B,n])."""
    s = scores.detach().clone().float().requires_grad_(True)
    y = labels.float()
    total, orders = None, []
    for b in range(s.size(0)):
        q, order = port_query_loss(s[b:b + 1], y[b:b + 1], distribution, top_k, gamma, temperature,
                                   None if perm is None else perm[b], None if unif is None else unif[b:b + 1])
        total = q if total is None else total + q
        orders.append(order)
    total.backward()
    return total.detach(), s.grad.detach(), torch.stack(orders)


def stpl_order(s, unif, temperature):
    """STPL's ordering of one or more [n] rows: the fp32 perturbed logits sorted descending (ties by position)."""
    s = np.asarray(s, dtype=np.float32); u = np.asarray(unif, dtype=np.float32)
    z = gumbel_logits(s, u, temperature)
    return np.argsort(-z, axis=-1, kind="stable"), z


def gumbel_logits(s, u, temperature):
    """(s + g) / T in fp32, g = -log(-log(u + 1e-20) + 1e-20) (sampling_utils.py:66-76)."""
    eps = np.float32(EPS)
    g = -np.log(-np.log(u + eps) + eps)
    z = s + g
    return z if temperature == 1.0 else (z / np.float32(temperature)).astype(np.float32)


def closed_form(s, y, order, distribution="PL", top_k=None, gamma=1.0, temperature=1.0, unif=None, with_scales=False):
    """float64 loss and gradient for [B,n] scores / labels and the sampled orderings ``order`` [B,n] (positions within
    each list).  The action values are s[order] (PL) or the perturbed logits (s + g) / T at ``order`` (STPL, the
    uniforms in ``unif``).  With e_j = exp(a_j - max a), C_t = sum_{j>=t} e_j and G_t = gamma^{t+1} sum_{t<=t'<k} r_t':
        loss = sum_{t<k} (log C_t + max a - a_t) G_t,   d loss / d a_j = e_j sum_{t<=min(j,k-1)} G_t / C_t - [j<k] G_j.
    ``with_scales``: also return the sizes fp32 rounding is relative to -- sum_b (1 + max |a|) sum_t |G_t| for the loss
    (each term differences log C_t and a_t) and max_t |G_t| / T for the gradient (each entry differences two terms of
    that size)."""
    s = np.asarray(s, dtype=np.float64); y = np.asarray(y, dtype=np.float64)
    B, n = s.shape
    loss, grad = 0.0, np.zeros_like(s)
    k = _k_eff(top_k, n)
    loss_scale, grad_scale = 0.0, 0.0
    for b in range(B):
        o = np.asarray(order[b], dtype=np.int64)
        if distribution == "PL":
            a, scale = s[b][o], 1.0
        else:
            eps = EPS
            g = -np.log(-np.log(np.asarray(unif[b], dtype=np.float64) + eps) + eps)
            a, scale = ((s[b] + g) / temperature)[o], 1.0 / temperature
        r = (np.power(2.0, y[b][o][:k]) - 1.0) / np.log2(np.arange(k) + 2.0)
        G = np.cumsum(r[::-1])[::-1] * (np.power(gamma, np.arange(1, k + 1)) if gamma != 1.0 else 1.0)
        m = a.max()
        e = np.exp(a - m)
        C = np.cumsum(e[::-1])[::-1]
        loss += float(np.sum((np.log(C[:k]) + m - a[:k]) * G))
        Q = np.cumsum(G / C[:k])
        q = np.concatenate([Q, np.full(n - k, Q[-1])])
        ga = e * q
        ga[:k] -= G
        grad[b][o] = ga * scale
        loss_scale += (1.0 + np.abs(a).max()) * np.abs(G).sum()
        grad_scale = max(grad_scale, np.abs(G).max() * scale)
    if with_scales:
        return loss, grad, loss_scale, grad_scale
    return loss, grad
