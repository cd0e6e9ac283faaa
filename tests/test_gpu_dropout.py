"""Every dropout site of the library against the mask specification (tests/dropout_ref.py), not against another kernel.

(a) Layer-0 masks, bit for bit, in every math mode: a training-mode call on X equals an eval-mode call on the replica's
    X' = mask * X * scale (the kernels' product is the same fp32 multiply), and dX = mask * scale * dX'.
(b) Whole training passes against float64: the reference stacked FF net with each nn.Dropout replaced by the replica's
    fixed mask, over norms, BN2 tile packings, widths, activations, rates and the bench shapes.
(c) Key domains: an FF call's masks and a one-mask call's (elementwise dropout, attention) never share a key, also
    through the list scorer's shared offset counter.
(d) The elementwise and attention masks against the replica directly.
"""
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import ref_port as rp
from tests import dropout_ref as dref
from tests.helpers import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED = 0x5EED_2024_0BAD_F00D
OFFSET = 9
RAGGED_LENS = [37, 100, 64, 9]          # 210 rows: the last 128-row tile is a partial one


def _ragged(lens):
    offsets = torch.zeros(len(lens) + 1, dtype=torch.int32)
    offsets[1:] = torch.cumsum(torch.tensor(lens), 0)
    return offsets


def _params(spec, dims, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    out = []
    for l, names in enumerate(spec.slots):
        for nm in names:
            if nm == "weight":
                t = torch.randn(dims[l + 1], dims[l], device=DEV, generator=g) / np.sqrt(dims[l])
            elif nm in ("gamma", "aff_w"):
                t = 1.0 + 0.1 * torch.randn(dims[l + 1], device=DEV, generator=g)
            else:
                t = 0.1 * torch.randn(dims[l + 1], device=DEV, generator=g)
            out.append(t)
    return out


def _f32(v):
    return torch.tensor(float(v), dtype=torch.float32, device=DEV)


# --------------------------------------------------------------------------------------------------------------------
# (a) layer-0 masks, bit for bit
# --------------------------------------------------------------------------------------------------------------------
def _run(spec, params, X, dO, ragged, training, seed=SEED, offset=OFFSET):
    from ptranking_b200 import ops
    Xl = X.detach().clone().requires_grad_(True)
    pm = [q.detach().clone().requires_grad_(True) for q in params]
    kw = dict(offsets=ragged[0], max_len=ragged[1]) if ragged else {}
    out = ops.ffnet_apply(Xl, spec, pm, training=training, seed=seed, offset=offset, **kw)
    (out * dO).sum().backward()
    return out.detach(), [q.grad for q in pm], Xl.grad


@pytest.mark.parametrize("F", [136, 64, 46, 220, 4])
@pytest.mark.parametrize("xdtype", ["fp32", "bf16"])
@pytest.mark.parametrize("layout", ["dense", "ragged"])
@pytest.mark.parametrize("mode", ["simt", "3xtf32", "tf32", "bf16"])
def test_layer0_mask_is_the_specified_stream(mode, layout, xdtype, F):
    """Net [F, 100, 1]: layer 0's input is its only dropout site.  Training on X must equal eval on the replica's
    mask(X) * scale in the output and every parameter gradient, and dX must be mask * scale * dX(eval), all torch.equal."""
    from ptranking_b200 import ops
    if mode == "simt" and layout == "ragged":
        pytest.skip("ragged per-query BN2 needs the tensor-core path")
    p = 0.25
    dims = [F, 100, 1]
    norm = "BN" if layout == "dense" else "BN2"
    spec = ops.FFNetSpec(dims, "GE", "S", norm, True, p, math_mode=mode)
    spec0 = ops.FFNetSpec(dims, "GE", "S", norm, True, 0.0, math_mode=mode)
    params = _params(spec, dims, F)
    g = torch.Generator(device=DEV).manual_seed(F + 1)
    if layout == "ragged":
        offsets = _ragged(RAGGED_LENS)
        rows, shape, ragged = int(offsets[-1]), (int(offsets[-1]), F), (offsets.to(DEV), max(RAGGED_LENS))
    else:
        rows, shape, ragged = 3 * 50, (3, 50, F), None
    X = torch.randn(*shape, device=DEV, generator=g)
    if xdtype == "bf16":
        X = X.to(torch.bfloat16)
    dO = torch.randn(*shape[:-1], 1, device=DEV, generator=g)
    keep = torch.from_numpy(dref.ff_mask(SEED, OFFSET, 0, p, rows, F)).to(DEV).view(shape)
    sc = _f32(dref.scale(p))
    zero = torch.zeros((), device=DEV)
    Xm = torch.where(keep, X.float() * sc, zero)
    o_t, g_t, dx_t = _run(spec, params, X, dO, ragged, True)
    o_e, g_e, dx_e = _run(spec0, params, Xm, dO, ragged, False)
    assert torch.equal(o_t, o_e), (o_t - o_e).abs().max().item()
    for i, (a, b) in enumerate(zip(g_t, g_e)):
        assert torch.equal(a, b), (i, (a - b).abs().max().item())
    want = torch.where(keep, dx_e * sc, zero).to(dx_t.dtype)
    assert torch.equal(dx_t, want), ((dx_t != want).sum().item(), ((dx_t == 0) != ~keep).sum().item())


# --------------------------------------------------------------------------------------------------------------------
# (b) whole training passes against float64
# --------------------------------------------------------------------------------------------------------------------
class FixedMask(nn.Module):
    """nn.Dropout with the replica's mask: x * keep * scale over the rows ``sl`` of the batch's flattened rows."""

    def __init__(self, keep, scale):
        super().__init__()
        self.m = keep.double() * float(scale)
        self.sl = slice(None)

    def forward(self, x):
        return x * self.m[self.sl].view(x.shape)


# B, n (0 = ragged RAGGED_LENS), dims, AF, TL_AF (None: no tail activation), norm ("BNq": BN per query), affine, p
FLOAT64_CASES = {
    "nonorm": (4, 50, [136, 100, 100, 1], "GE", "S", None, False, 0.1),
    "bn_affine": (4, 64, [136, 100, 100, 1], "GE", "S", "BN", True, 0.1),
    "bn_plain_p05": (4, 64, [136, 100, 100, 1], "R", "S", "BN", False, 0.5),
    "bn_deep_p09": (4, 64, [136, 100, 100, 100, 1], "GE", "S", "BN", True, 0.9),
    "bn_hidden4": (4, 64, [136, 4, 4, 1], "R", "S", "BN", True, 0.1),
    "bn_F220": (4, 50, [220, 100, 100, 1], "GE", "S", "BN", True, 0.25),
    "bnq_affine": (3, 60, [136, 100, 100, 1], "GE", "S", "BNq", True, 0.1),
    "bn2_n1_F46": (5, 1, [46, 100, 100, 1], "R", "S", "BN2", False, 0.1),
    "bn2_n33_hidden4_p09": (3, 33, [64, 100, 4, 1], "CE", None, "BN2", False, 0.9),
    "bn2_n50_affine": (3, 50, [136, 100, 100, 1], "GE", "S", "BN2", True, 0.1),
    "bn2_n128_F46_p05": (2, 128, [46, 100, 100, 1], "GE", "S", "BN2", True, 0.5),
    "bn2_n129": (2, 129, [136, 100, 100, 1], "S", "S", "BN2", False, 0.1),
    "bn2_n200": (3, 200, [136, 100, 100, 1], "R", "S", "BN2", False, 0.1),
    "bn2_n512_wide": (2, 512, [136, 128, 256, 512, 136], "R", "R", "BN2", False, 0.1),
    "wide_out8": (2, 96, [136, 128, 256, 512, 8], "R", None, None, False, 0.1),
    "wide320_bn": (3, 40, [64, 320, 8], "GE", "S", "BN", True, 0.5),
    "out3_rows600": (2, 300, [136, 100, 3], "S", "R", "BN", False, 0.1),
    "nonorm_F46_p09": (7, 33, [46, 100, 100, 1], "CE", None, None, False, 0.9),
    "ragged_bn2": (0, 0, [136, 100, 100, 1], "GE", "S", "BN2", True, 0.1),
    "ragged_bn2_F46_p05": (0, 0, [46, 100, 100, 1], "R", "S", "BN2", False, 0.5),
}
FULL_CASES = {
    # the bench's default scorer (5 x 100 GELU) at 1024 x 256 x 136 with batch BN and 256 x 1024 x 136 with BN2
    "full_bn": (1024, 256, [136] + [100] * 5 + [1], "GE", "S", "BN", True, 0.1),
    "full_bn2": (256, 1024, [136] + [100] * 5 + [1], "GE", "S", "BN2", False, 0.1),
}
# (out, gradients, floor): out relative to the float64 output's max; a gradient to its float64 max plus floor * the net's
# largest gradient.  3xTF32 and SIMT are fp32-grade (the bound of test_point_scorer_forward_backward).  Single-pass TF32
# (10-bit mantissa operands) was measured on an H100 SXM (700 W) over the cases it runs: at most 2.1e-3 on the output
# (no norm, p = 0.9), and on a gradient at most 0.73 of 5e-3 * its max + 1e-4 * the largest gradient; the bounds leave
# 2x.  TF32 runs only the nets without a ReLU: rounded operands flip the sign of pre-activations near 0, and at a ReLU
# kink that moves single gradient elements by up to 20 % of the gradient's max, which no elementwise bound can tell from
# a wrong mask.  Those nets run in SIMT and 3xTF32.
TOLS = {"simt": (1e-5, 2e-5, 1e-6), "3xtf32": (1e-5, 2e-5, 1e-6), "tf32": (4e-3, 1e-2, 1e-4)}


def _float64_pass(case, mode, seed=SEED, offset=OFFSET):
    """-> dict of (got, want) pairs: out, dX and every parameter gradient by state_dict name."""
    from ptranking_b200 import ops
    from ptranking_b200.base.utils import StackedFFNet
    B, n, dims, AF, TL, norm, affine, p = case
    per_query = norm == "BNq"
    torch.manual_seed(sum(dims) + B + n)
    net = StackedFFNet(dims, AF=AF, TL_AF=TL or "S", apply_tl_af=TL is not None, dropout=p, BN=norm is not None,
                       bn_type="BN" if per_query else norm, bn_affine=affine, math_mode=mode, bn_per_query=per_query).to(DEV)
    with torch.no_grad():
        for name, q in net.named_parameters():
            if "weight" in name and name.startswith("ff_"):
                continue
            q.add_(0.1 * torch.randn_like(q))
    ref = rp.stacked_ffnet(dims, AF, TL or "S", TL is not None, 0.0, norm is not None, "BN" if per_query else norm, affine)
    ref.load_state_dict({k: v.detach().cpu() for k, v in net.state_dict().items()})
    ref = ref.double().to(DEV)

    if n == 0:
        offsets = _ragged(RAGGED_LENS)
        rows = int(offsets[-1])
        groups = [(int(offsets[i]), int(offsets[i + 1])) for i in range(len(RAGGED_LENS))]
        X = torch.randn(rows, dims[0], device=DEV)
        dO = torch.randn(rows, dims[-1], device=DEV)
        kw = dict(offsets=offsets.to(DEV), max_len=max(RAGGED_LENS))
    else:
        rows = B * n
        groups = [(b * n, (b + 1) * n) for b in range(B)] if per_query else None
        X = torch.randn(B, n, dims[0], device=DEV)
        dO = torch.randn(B, n, dims[-1], device=DEV)
        kw = {}
    masks = []
    for l in range(len(dims) - 2):       # every Linear but the last has a dropout on its input
        keep = torch.from_numpy(dref.ff_mask(seed, offset, l, p, rows, dims[l])).to(DEV)
        masks.append(FixedMask(keep, dref.scale(p)))
        ref._modules[f"dr_{l + 1}"] = masks[-1]

    Xg = X.clone().requires_grad_(True)
    out = ops.ffnet_apply(Xg, net.spec, net.ordered_parameters(), training=True, seed=seed, offset=offset, **kw)
    (out * dO).sum().backward()

    Xd = X.double().requires_grad_(True)
    if groups is None:
        out_ref = ref(Xd)
    else:       # per-query statistics: the reference net on one query at a time, masks by global row
        parts, Xrows = [], Xd.reshape(rows, dims[0])
        for r0, r1 in groups:
            for m in masks:
                m.sl = slice(r0, r1)
            parts.append(ref(Xrows[r0:r1].unsqueeze(0)).squeeze(0))
        out_ref = torch.cat(parts).view(out.shape)
    (out_ref * dO.double()).sum().backward()
    res = {"out": (out.detach(), out_ref.detach()), "dX": (Xg.grad, Xd.grad)}
    lib_params = dict(net.named_parameters())
    for name, q in ref.named_parameters():
        res[name] = (lib_params[name].grad.view(q.shape), q.grad)
    return res


def _errors(res):
    """-> {name: (max abs error, max abs reference)} and the largest parameter gradient."""
    errs = {k: (float((a.double() - b).abs().max()), float(b.abs().max())) for k, (a, b) in res.items()}
    gscale = max(v[1] for k, v in errs.items() if k not in ("out", "dX"))
    return errs, gscale


def _check(res, mode):
    tol_out, tol_g, floor = TOLS[mode]
    errs, gscale = _errors(res)
    e, m = errs.pop("out")
    assert e <= tol_out * m, ("out", e / m)
    for k, (e, m) in errs.items():
        assert e <= tol_g * m + floor * gscale + 1e-9, (k, e, m, gscale)


@pytest.mark.parametrize("mode", ["simt", "3xtf32", "tf32"])
@pytest.mark.parametrize("case", list(FLOAT64_CASES))
def test_training_pass_matches_float64(case, mode):
    c = FLOAT64_CASES[case]
    if mode == "simt" and c[1] == 0:
        pytest.skip("ragged per-query BN2 needs the tensor-core path")
    if mode == "tf32" and "R" in (c[3], c[4]):
        pytest.skip("TF32 against float64 is bounded on nets without a ReLU (see TOLS)")
    _check(_float64_pass(c, mode), mode)


@pytest.mark.parametrize("case", list(FULL_CASES))
def test_full_size_training_pass_matches_float64(case):
    _check(_float64_pass(FULL_CASES[case], "3xtf32"), "3xtf32")


# --------------------------------------------------------------------------------------------------------------------
# (c) key domains
# --------------------------------------------------------------------------------------------------------------------
def _ew_keep(shape, p, seed, offset):
    from ptranking_b200 import ops
    out = ops._ew(ops.EW_DROPOUT, torch.ones(shape, device=DEV), None, p, seed, offset)
    return out != 0, out


@pytest.mark.parametrize("o", [1, 3])
def test_ff_and_one_mask_calls_never_share_a_mask(o):
    """The layer-0 mask of an FF call at offset o (read off dX, as in (a)) and the elementwise-dropout mask at offset
    64*o, over the same number of elements: different streams, and each one is the replica's."""
    from ptranking_b200 import ops
    rows, F, p = 256, 136, 0.5
    dims = [F, 100, 1]
    spec = ops.FFNetSpec(dims, "R", None, None, False, p, math_mode="3xtf32")
    params = _params(spec, dims, 3)
    X = torch.randn(1, rows, F, device=DEV)
    _, _, dx = _run(spec, params, X, torch.randn(1, rows, 1, device=DEV), None, True, offset=o)
    ff_keep = (dx != 0).view(rows, F)
    ew_keep, _ = _ew_keep((rows, F), p, SEED, 64 * o)
    agree = float((ew_keep == ff_keep).float().mean())
    assert agree < 0.6, agree                       # independent streams agree on half the elements at p = 0.5
    assert np.array_equal(ff_keep.cpu().numpy(), dref.ff_mask(SEED, o, 0, p, rows, F))
    assert np.array_equal(ew_keep.cpu().numpy(), dref.call_mask(SEED, 64 * o, p, (rows, F)))


def test_list_scorer_step_keys_are_distinct(monkeypatch):
    """One training step of the list scorer (AllRank encoder: attention and elementwise dropout; head and tail FF nets):
    log every offset the library takes from ops.next_dropout_offset, map it through the key rules, and require the key
    indices to be pairwise distinct, with no one-mask key inside any FF call's block of layer slots."""
    import ptranking_b200
    from ptranking_b200 import LABEL_TYPE, ops
    log = []
    counter = ops.next_dropout_offset

    def logged():
        o = counter()
        caller = sys._getframe(1)
        log.append((caller.f_code.co_name, o, dict(caller.f_locals)))
        return o

    monkeypatch.setattr(ops, "next_dropout_offset", logged)
    F, p = 20, 0.2
    sf = dict(sf_id="listsf", opt="Adagrad", lr=1e-3,
              listsf=dict(num_features=F, ff_dims=[16, 32, 24], AF="R", TL_AF="GE", apply_tl_af=False, BN=True,
                          bn_type="BN2", bn_affine=False, n_heads=2, encoder_layers=2, encoder_type="AllRank", dropout=p))
    torch.manual_seed(0)
    r = ptranking_b200.ListNet(sf_para_dict=sf, gpu=True, device=DEV)
    r.init()
    r.train_mode()
    X = torch.randn(3, 40, F, device=DEV)
    y = torch.sort(torch.randint(0, 5, (3, 40), device=DEV).float(), dim=1, descending=True)[0]
    for _ in range(2):
        r.train_op(X, y, presort=True, label_type=LABEL_TYPE.MultiLabel)
    ff_keys, call_keys, kinds = [], [], set()
    for fn, o, loc in log:
        if fn == "ffnet_apply":
            spec = loc["spec"]
            if loc["training"] and spec.dropout_p > 0:
                ff_keys += [dref.ff_index(o, l) for l in range(spec.L - 1)]
                kinds.add(fn)
        elif fn in ("attention_packed", "dropout"):
            if loc.get("dropout_p", loc.get("p", 0.0)) > 0:
                call_keys.append(dref.call_index(o))
                kinds.add(fn)
        else:
            raise AssertionError(f"unexpected consumer of the dropout offset counter: {fn}")
    assert kinds == {"ffnet_apply", "attention_packed", "dropout"}, kinds
    keys = ff_keys + call_keys
    assert len(set(keys)) == len(keys)
    assert all(k % dref.FF_KEYS_PER_OFFSET < dref.MAX_FF_LAYERS - 1 for k in ff_keys)
    assert all(k % dref.FF_KEYS_PER_OFFSET >= dref.MAX_FF_LAYERS - 1 for k in call_keys)


# --------------------------------------------------------------------------------------------------------------------
# (d) elementwise and attention masks against the replica
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,p,seed,offset", [
    ((1001,), 0.1, SEED, 1),
    ((3, 77, 5), 0.5, 0, 2 ** 40 + 5),
    ((64, 136), 0.9, 2 ** 64 - 1, 12),
    ((262144, 136), 0.1, 1234, 5),
])
def test_elementwise_dropout_is_the_specified_stream(shape, p, seed, offset):
    keep, out = _ew_keep(shape, p, seed, offset)
    want = torch.from_numpy(dref.call_mask(seed, offset, p, shape)).to(DEV)
    assert torch.equal(keep, want), (keep != want).sum().item()
    assert torch.equal(out[keep], torch.full_like(out[keep], float(dref.scale(p))))


def test_attention_dropout_with_the_specified_mask_matches_float64():
    """test_attention_dropout_matches_float64 with the mask taken from the replica's key rule ((z*n + row)*n + col under
    the one-mask key of the offset) instead of the elementwise kernel.  (2, 152, 2, 68) takes the alignment-specialised
    GEMM kernel, n = 150 and D = 46 the general one."""
    from tests.test_gpu_listsf import _attention, _attention_float64
    p, seed, offset = 0.25, 11, 4
    for B, n, H, D in ((2, 152, 2, 68), (2, 150, 2, 68), (2, 130, 1, 46)):
        g = torch.Generator().manual_seed(B * 1000 + n + D)
        Q, K, V, dO = (torch.randn(B, n, H * D, generator=g) for _ in range(4))
        keep = torch.from_numpy(dref.call_mask(seed, offset, p, (B * H, n, n)))
        mask = keep.double() * float(dref.scale(p))
        refs = _attention_float64(Q, K, V, H, dO, mask)
        Qc, Kc, Vc = (t.to(DEV).requires_grad_(True) for t in (Q, K, V))
        o = _attention(Qc, Kc, Vc, H, p, seed=seed, offset=offset)
        (o * dO.to(DEV)).sum().backward()
        for name, a, b, tol in zip(("O", "dQ", "dK", "dV"), (o.detach(), Qc.grad, Kc.grad, Vc.grad), refs, (3e-6, 5e-6, 5e-6, 5e-6)):
            assert rel_err(a.cpu().numpy(), b.numpy()) <= tol, ((B, n, H, D), name)
