"""Two independent restatements of DivProbRanker's losses, for the parity tests:

* ``port_head`` / ``port_loss`` / ``port_sort_key``: the Gaussian head (base/div_mdn_ranker.py:276-326), the expected
  ranks (util/prob_utils.py:62-80), SuperSoft aNDCG / nERR-IA, PairCLS and LambdaPairCLS
  (score_and_sort/div_prob_ranker.py:29-231, util/div_lambda_utils.py:26-43, metric/srd/diversity_metric.py:13-30,
  143-183) with opt_ideal, op for op in fp32 ATen, differentiated by autograd.
* ``closed_form``: the same losses in float64 numpy with the gradient w.r.t. (mu, v) in closed form (DESIGN §4):
  dL/dmu_k = -sum_j w_kj A_kj, dL/dv_k = sum_j w_kj z_kj / (2 sigma_kj) A_kj, with A_kj = c_kj - c_jk,
  w_kj = phi(z_kj) / sigma_kj, and ``head_grad`` chains it to the raw output.
"""
import numpy as np
import torch
import torch.nn.functional as F

from tests import divlist_oracle

LOSSES = ("aNDCG", "nERR-IA", "PairCLS", "LambdaPairCLS")

# The training fixtures' rankers: (model dict without model_id / cluster / sort_id / opt_ideal, sf_para_dict)
TRAIN = {
    # the reference's default model dict (SuperSoft nERR-IA, K 1, limit_delta 0.01) on a small pointsf
    "pointsf": (dict(K=1, limit_delta=0.01, opt_id="SuperSoft", metric="nERR-IA", top_k=None, norm=True),
                dict(sf_id="pointsf", opt="Adagrad", lr=0.01,
                     pointsf=dict(num_features=20, h_dim=16, num_layers=3, AF="GE", TL_AF="GE", apply_tl_af=False,
                                  BN=True, bn_type="BN", bn_affine=True, dropout=0.0))),
    # the grid's K = 5 SuperSoft aNDCG at top_k 10 on the small list scorer of tests.divlist_oracle
    "listsf": (dict(K=5, limit_delta=None, opt_id="SuperSoft", metric="aNDCG", top_k=10, norm=True),
               dict(sf_id="listsf", opt="Adagrad", lr=0.01,
                    listsf=dict(num_features=divlist_oracle.SMALL_F,
                                **dict(divlist_oracle.SMALL_LISTSF, encoder_type="AttnDIN", n_heads=2)))),
}


def port_head(raw, K, limit_delta):
    """raw [1, n, D] (D = 2 or 3K) -> (mus, vars) [1, n]."""
    if 1 == K:
        mus, std_vars = torch.split(raw, 1, dim=2)
        var = torch.exp(std_vars) if limit_delta is None else torch.sigmoid(std_vars) * limit_delta
        return torch.squeeze(mus, dim=2), torch.squeeze(var, dim=2)
    w, mu_i, std_var_i = torch.split(raw, K, dim=2)
    var_i = torch.exp(std_var_i) if limit_delta is None else torch.sigmoid(std_var_i) * limit_delta
    coef = torch.softmax(w, dim=2)
    return torch.sum(coef * mu_i, dim=2), torch.sum(coef * var_i, dim=2)


def _pairs(mus, vars):
    return mus.unsqueeze(2) - mus.unsqueeze(1), vars.unsqueeze(2) + vars.unsqueeze(1)


def port_expected_rank(mus, vars):
    d, v = _pairs(mus, vars)
    phi0 = 0.5 * torch.erfc(d / torch.sqrt(2 * v))
    sub = torch.triu(phi0, diagonal=1) + torch.tril(phi0, diagonal=-1)
    return torch.sum(sub, dim=2) + 1.0, sub


def _alpha_dcg(R, alpha=0.5):
    n = R.size(1)
    prior = torch.zeros_like(R)
    prior[:, 1:n] = R[:, 0:n - 1]
    cnt = torch.cumsum(prior, dim=1)
    den = torch.log2(torch.arange(n, dtype=torch.float, device=R.device) + 2.0).view(1, -1)
    return torch.sum(torch.sum(torch.pow((1.0 - alpha), cnt) * R / den, dim=0))


def _delta_alpha_dcg(R, alpha=0.5, norm=True):
    m, n = R.size()
    prior = torch.zeros_like(R)
    prior[:, 1:n] = R[:, 0:n - 1]
    focus = torch.pow((1.0 - alpha), torch.cumsum(prior, dim=1))
    gains = torch.pow(2.0, R) - 1.0
    gdiff = gains.unsqueeze(2) - gains.unsqueeze(1)
    disc = 1.0 / torch.log2(torch.arange(n, dtype=torch.float, device=R.device) + 2.0)
    c1 = disc.view(1, -1, 1) * focus.unsqueeze(2).expand(-1, -1, n)
    c2 = disc.view(1, 1, -1) * focus.unsqueeze(1).expand(-1, n, -1)
    delta = torch.abs(torch.sum(gdiff * c1, dim=0) - torch.sum(gdiff * c2, dim=0))
    return delta / _alpha_dcg(R, alpha) if norm else delta


def port_loss(mus, vars, R, loss, top_k=None, norm=True, beta=0.5):
    """mus, vars [1, n] (differentiable), R [m, n] -> 0-dim loss."""
    if "aNDCG" == loss:
        E, sub = port_expected_rank(mus, vars)
        cover = torch.sum(sub * R.unsqueeze(1).expand(-1, R.size(1), -1), dim=2)
        g = torch.sum(R * torch.pow((1.0 - beta), cover) / torch.log2(1.0 + E), dim=1)
        return -(torch.sum(g) if top_k is None else torch.sum(g[0:top_k]))
    if "nERR-IA" == loss:
        E, _ = port_expected_rank(mus, vars)
        n = R.size(1)
        k = n if top_k is None else top_k
        t2 = torch.tensor([2.0], device=R.device)
        lab = R[:, 0:k]
        sat = (torch.pow(t2, lab) - 1.0) / torch.pow(t2, 1.0)
        cum = torch.cumprod(torch.ones_like(lab) - sat, dim=1)
        casc = torch.ones_like(cum)
        casc[:, 1:k] = cum[:, 0:k - 1]
        return -torch.sum(torch.sum(sat * casc * (1.0 / E[:, 0:k]), dim=1))
    d, v = _pairs(mus, vars)
    p = 1.0 - 0.5 * torch.erfc(d / torch.sqrt(2 * v))
    S = torch.clamp(R.unsqueeze(2) - R.unsqueeze(1), min=-1.0, max=1.0)
    t = torch.mean(0.5 * (1.0 + S), dim=0, keepdim=True)
    W = None if "PairCLS" == loss else torch.triu(_delta_alpha_dcg(R, beta, norm).unsqueeze(0), diagonal=1)
    bce = F.binary_cross_entropy(input=torch.triu(p, diagonal=1), target=torch.triu(t, diagonal=1), weight=W,
                                 reduction='none')
    return torch.sum(torch.sum(bce, dim=(2, 1)))


def port_loss_and_grad(raw, R, loss, K=1, limit_delta=None, top_k=None, norm=True):
    """raw [n, D] -> (loss, d loss / d raw [n, D]) in fp32 through the head."""
    u = torch.as_tensor(np.asarray(raw, dtype=np.float32)).reshape(1, -1, 2 if K == 1 else 3 * K).clone()
    u.requires_grad_(True)
    mus, vars = port_head(u, K, limit_delta)
    L = port_loss(mus, vars, torch.as_tensor(np.asarray(R, dtype=np.float32)), loss, top_k, norm)
    L.backward()
    return float(L.detach()), u.grad[0].numpy().copy()


def port_sort_key(raw, sort_id, K=1, limit_delta=None):
    u = torch.as_tensor(np.asarray(raw, dtype=np.float32)).reshape(1, -1, 2 if K == 1 else 3 * K)
    mus, vars = port_head(u, K, limit_delta)
    if 'RERAR' == sort_id:
        return (1.0 / port_expected_rank(mus, vars)[0])[0].numpy()
    if 'RiskAware' == sort_id:
        return (mus - 0.1 * vars)[0].numpy()
    return mus[0].numpy()


# ---------------------------------------------------------------------------------------------------------------- #
# float64 closed form
# ---------------------------------------------------------------------------------------------------------------- #
def head64(raw, K, limit_delta):
    u = np.asarray(raw, dtype=np.float64).reshape(-1, 2 if K == 1 else 3 * K)
    T = (lambda x: np.exp(x)) if limit_delta is None else (lambda x: limit_delta / (1.0 + np.exp(-x)))
    if K == 1:
        return u[:, 0].copy(), T(u[:, 1])
    lg = u[:, :K] - u[:, :K].max(axis=1, keepdims=True)
    w = np.exp(lg) / np.exp(lg).sum(axis=1, keepdims=True)
    return (w * u[:, K:2 * K]).sum(axis=1), (w * T(u[:, 2 * K:])).sum(axis=1)


def head_grad(raw, K, limit_delta, gmu, gv):
    """Chain (dL/dmu, dL/dv) through the head -> dL/draw [n, D], float64."""
    u = np.asarray(raw, dtype=np.float64).reshape(-1, 2 if K == 1 else 3 * K)
    if limit_delta is None:
        T = np.exp
        dT = np.exp
    else:
        T = lambda x: limit_delta / (1.0 + np.exp(-x))
        dT = lambda x: limit_delta * np.exp(-x) / (1.0 + np.exp(-x)) ** 2
    g = np.zeros_like(u)
    if K == 1:
        g[:, 0], g[:, 1] = gmu, gv * dT(u[:, 1])
        return g
    lg = u[:, :K] - u[:, :K].max(axis=1, keepdims=True)
    w = np.exp(lg) / np.exp(lg).sum(axis=1, keepdims=True)
    dw = gmu[:, None] * u[:, K:2 * K] + gv[:, None] * T(u[:, 2 * K:])
    g[:, :K] = w * (dw - (w * dw).sum(axis=1, keepdims=True))
    g[:, K:2 * K] = gmu[:, None] * w
    g[:, 2 * K:] = gv[:, None] * w * dT(u[:, 2 * K:])
    return g


def _erfc(x):
    from scipy.special import erfc
    return erfc(x)


def closed_form_mv(mu, v, R, loss, top_k=None, norm=True, beta=0.5):
    """float64 (loss, dL/dmu, dL/dv) from the closed form."""
    from scipy.special import erfc
    mu, v = np.asarray(mu, np.float64), np.asarray(v, np.float64)
    R = np.asarray(R, np.float64)
    m, n = R.shape
    sig = np.sqrt(v[:, None] + v[None, :])
    z = (mu[:, None] - mu[None, :]) / sig
    P = 0.5 * erfc(z / np.sqrt(2.0))
    np.fill_diagonal(P, 0.0)
    E = 1.0 + P.sum(axis=1)
    c = np.zeros((n, n))
    if loss == "aNDCG":
        rows = m if top_k is None else min(top_k, m)
        Rr = R[:rows]
        C = Rr @ P.T                                        # C[s, i] = sum_j P_ij R_sj
        g = Rr * np.power(1.0 - beta, C) / np.log2(1.0 + E)[None, :]
        L = -g.sum()
        a = g.sum(axis=0) / ((1.0 + E) * np.log(1.0 + E))
        b = -np.log(1.0 - beta) * g
        c = a[:, None] + b.T @ Rr
    elif loss == "nERR-IA":
        k = n if top_k is None else min(top_k, n)
        sat = (np.power(2.0, R) - 1.0) / 2.0
        casc = np.ones_like(sat)
        casc[:, 1:] = np.cumprod(1.0 - sat, axis=1)[:, :-1]
        ws = (sat * casc).sum(axis=0)
        L = -(ws[:k] / E[:k]).sum()
        a = np.zeros(n)
        a[:k] = ws[:k] / E[:k] ** 2
        c = np.repeat(a[:, None], n, axis=1)
    else:
        p = 1.0 - P
        t = (0.5 * (1.0 + np.clip(R[:, :, None] - R[:, None, :], -1.0, 1.0))).mean(axis=0)
        if loss == "LambdaPairCLS":
            prior = np.zeros_like(R)
            prior[:, 1:] = np.cumsum(R, axis=1)[:, :-1]
            h = np.power(1.0 - beta, prior) / np.log2(np.arange(n) + 2.0)[None, :]
            G = np.power(2.0, R) - 1.0
            gd = G[:, :, None] - G[:, None, :]
            W = np.abs((gd * h[:, :, None]).sum(axis=0) - (gd * h[:, None, :]).sum(axis=0))
            if norm:
                with np.errstate(invalid='ignore'):     # 0 / 0 without relevance, as the reference
                    W = W / (R * h).sum()
        else:
            W = np.ones((n, n))
        iu = np.triu(np.ones((n, n), dtype=bool), k=1)
        with np.errstate(divide='ignore'):
            lp, l1p = np.maximum(np.log(p), -100.0), np.maximum(np.log1p(-p), -100.0)
        bce = -(t * lp + (1.0 - t) * l1p) * W
        L = bce[iu].sum()
        dbce = W * (p - t) / np.maximum((1.0 - p) * p, 1e-12)
        c = np.where(iu, -dbce, 0.0)
    A = c - c.T
    wgt = np.exp(-0.5 * z * z) / np.sqrt(2.0 * np.pi) / sig
    np.fill_diagonal(A, 0.0)
    gmu = -(wgt * A).sum(axis=1)
    gv = (wgt * z / (2.0 * sig) * A).sum(axis=1)
    return float(L), gmu, gv


def closed_form(raw, R, loss, K=1, limit_delta=None, top_k=None, norm=True):
    """float64 (loss, dL/draw [n, D])."""
    mu, v = head64(raw, K, limit_delta)
    L, gmu, gv = closed_form_mv(mu, v, R, loss, top_k, norm)
    return L, head_grad(raw, K, limit_delta, gmu, gv)


def autograd64(raw, R, loss, K=1, limit_delta=None, top_k=None, norm=True):
    """float64 autograd of the port's formulas (for checking the closed form)."""
    u = torch.as_tensor(np.asarray(raw, dtype=np.float64)).reshape(1, -1, 2 if K == 1 else 3 * K).clone()
    u.requires_grad_(True)
    with _default_dtype(torch.float64):
        mus, vars = port_head(u, K, limit_delta)
        L = port_loss(mus, vars, torch.as_tensor(np.asarray(R, dtype=np.float64)), loss, top_k, norm)
    L.backward()
    return float(L.detach()), u.grad[0].numpy().copy()


class _default_dtype:
    def __init__(self, dt):
        self.dt = dt

    def __enter__(self):
        self.old = torch.get_default_dtype()
        torch.set_default_dtype(self.dt)

    def __exit__(self, *a):
        torch.set_default_dtype(self.old)


def draw_raw(rng, n, K, limit_delta, pair_safe):
    """Raw scorer output [n, D] (float32).  ``pair_safe``: means in clusters, so that every pair's
    |x| = |mu_i - mu_j| / sqrt(2 (v_i + v_j)) is either below 1.5 or above 6 (clearly saturated in fp32) -- never in the
    band where 1 - erfc(x)/2 is within a few ulp of 0 or 1 and the reference's 1e-12 BCE clamp turns an ulp of erfc into
    a large gradient difference."""
    D = 2 if K == 1 else 3 * K
    for _ in range(1000):
        u = rng.standard_normal((n, D)).astype(np.float32)
        if K > 1:
            u[:, :K] *= 0.5
        if not pair_safe:
            return u
        mu, v = head64(u, K, limit_delta)
        vmax = float(v.max())
        cl = rng.integers(0, max(1, min(4, n)), size=n)
        jit = rng.uniform(-0.4, 0.4, size=n) * np.sqrt(float(v.min()))
        target = cl * 9.0 * np.sqrt(2.0 * 2.0 * vmax) + jit
        if K == 1:
            u[:, 0] = target
        else:
            u[:, K:2 * K] = (target - mu)[:, None] + u[:, K:2 * K]
        mu32 = torch.as_tensor(u)[None]
        m_, v_ = port_head(mu32.float(), K, limit_delta)
        m_, v_ = m_[0].double().numpy(), v_[0].double().numpy()
        x = np.abs(m_[:, None] - m_[None, :]) / np.sqrt(2.0 * (v_[:, None] + v_[None, :]))
        if not np.any((x > 1.5) & (x < 6.0)):
            return u
    raise RuntimeError("no pair-safe draw")
