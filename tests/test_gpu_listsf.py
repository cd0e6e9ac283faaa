"""GPU parity of the list (MHSA) scorer: attention core, reference LayerNorm, and the whole
ListNeuralRanker for the three encoder types against tensors produced by the unmodified reference."""
import numpy as np
import pytest
import torch

from oracle import ref_port as rp
from tests.helpers import load, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _attention(Q, K, V, H, p, seed=None, offset=None):
    """The attention core over separate Q, K, V: the packed entry point on their concatenation (autograd splits the
    [B,n,3F] gradient back into dQ, dK, dV).  F % 4 == 0 exactly when 3F % 4 == 0 and the K and V blocks start 16-byte
    aligned, so each contraction takes the same kernel as it would with Q, K, V in three tensors."""
    from ptranking_b200 import ops
    return ops.attention_packed(torch.cat((Q, K, V), -1), H, p, seed=seed, offset=offset)


def _attention_float64(Q, K, V, H, dO, mask=None):
    """float64 reference of list_ranker.py:226-248 with the dropout mask (kept elements already scaled) as a tensor:
    returns O and dQ, dK, dV for the incoming gradient dO."""
    B, n, F = Q.shape
    D = F // H
    q, k, v = (t.double().requires_grad_(True) for t in (Q, K, V))
    split = lambda t: t.view(B, n, H, D).permute(0, 2, 1, 3)
    att = torch.softmax(split(q) @ split(k).transpose(-1, -2) / np.sqrt(D), dim=-1)
    if mask is not None:
        att = att * mask.double().view(B, H, n, n)
    o_ref = (att @ split(v)).permute(0, 2, 1, 3).reshape(B, n, H * D)
    (o_ref * dO.double()).sum().backward()
    return o_ref.detach(), q.grad, k.grad, v.grad


@pytest.mark.parametrize("shape", [(2, 24, 2, 10), (3, 200, 2, 68), (1, 512, 2, 68), (2, 37, 4, 17), (1, 1, 2, 23), (2, 130, 1, 46)])
def test_attention_matches_float64(shape):
    B, n, H, D = shape
    g = torch.Generator().manual_seed(B * 1000 + n)
    Q, K, V = (torch.randn(B, n, H * D, generator=g) for _ in range(3))
    dO = torch.randn(B, n, H * D, generator=g)
    refs = _attention_float64(Q, K, V, H, dO)
    Qc, Kc, Vc = (t.to(DEV).requires_grad_(True) for t in (Q, K, V))
    o = _attention(Qc, Kc, Vc, H, 0.0)
    (o * dO.to(DEV)).sum().backward()
    # 3xTF32 tensor-core path: split accumulators keep it at fp32 grade (north-star bound: 1e-5)
    for name, a, b, tol in zip(("O", "dQ", "dK", "dV"), (o.detach(), Qc.grad, Kc.grad, Vc.grad), refs, (3e-6, 5e-6, 5e-6, 5e-6)):
        assert rel_err(a.cpu().numpy(), b.numpy()) <= tol, name


def test_attention_dropout_matches_float64():
    """Dropout in the forward contraction, the softmax backward and the transposed dV contraction against float64 autograd
    on softmax(QK^T/sqrt(d)) * M with the mask M drawn by the elementwise dropout kernel over ones [B*H, n, n]: that kernel
    keys element i by its flat index, which is the attention's element id (z*n + row)*n + col.  (2, 152, 2, 68) takes the
    alignment-specialised GEMM kernel; n = 150 and D = 46 take the general one."""
    from ptranking_b200 import ops
    p, seed, offset = 0.25, 11, 4
    for B, n, H, D in ((2, 152, 2, 68), (2, 150, 2, 68), (2, 130, 1, 46)):
        g = torch.Generator().manual_seed(B * 1000 + n + D)
        Q, K, V, dO = (torch.randn(B, n, H * D, generator=g) for _ in range(4))
        mask = ops._ew(ops.EW_DROPOUT, torch.ones(B * H, n, n, device=DEV), None, p, seed, offset).cpu()
        assert 0.2 < float((mask == 0).double().mean()) < 0.3
        refs = _attention_float64(Q, K, V, H, dO, mask)
        Qc, Kc, Vc = (t.to(DEV).requires_grad_(True) for t in (Q, K, V))
        o = _attention(Qc, Kc, Vc, H, p, seed=seed, offset=offset)
        (o * dO.to(DEV)).sum().backward()
        for name, a, b, tol in zip(("O", "dQ", "dK", "dV"), (o.detach(), Qc.grad, Kc.grad, Vc.grad), refs, (3e-6, 5e-6, 5e-6, 5e-6)):
            assert rel_err(a.cpu().numpy(), b.numpy()) <= tol, ((B, n, H, D), name)


@pytest.mark.parametrize("shape", [(2, 152, 2, 68), (1, 512, 2, 68), (3, 24, 2, 12), (2, 260, 1, 136), (2, 640, 2, 68), (2, 200, 4, 32)])
@pytest.mark.parametrize("p", [0.0, 0.25])
def test_attention_tc_aligned_kernel_equals_general_kernel(shape, p, monkeypatch):
    """The alignment-specialised batched-GEMM kernel stages the same operand images and issues the same MMAs as the
    general one (which remains the path of shapes that are not multiples of four): identical bits, dropout included."""
    B, n, H, D = shape
    torch.manual_seed(n)
    Q0, K0, V0, G = (torch.randn(B, n, H * D, device=DEV) for _ in range(4))
    outs = []
    for general in ("0", "1"):
        monkeypatch.setenv("PTRB200_BGEMM_GENERAL", general)
        Q, K, V = (t.clone().requires_grad_(True) for t in (Q0, K0, V0))
        o = _attention(Q, K, V, H, p, seed=21, offset=2)
        (o * G).sum().backward()
        outs.append([t.detach().clone() for t in (o, Q.grad, K.grad, V.grad)])
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_attention_dropout_consistent_between_forward_and_backward():
    B, n, H, D = 2, 96, 2, 16
    torch.manual_seed(0)
    Q, K = torch.randn(B, n, H * D, device=DEV), torch.randn(B, n, H * D, device=DEV)
    V = torch.randn(B, n, H * D, device=DEV, requires_grad=True)
    o1 = _attention(Q, K, V, H, 0.3, seed=5, offset=9)
    o2 = _attention(Q, K, V, H, 0.3, seed=5, offset=9)
    o3 = _attention(Q, K, V, H, 0.3, seed=5, offset=10)
    assert torch.equal(o1, o2) and not torch.equal(o1, o3)
    # O is linear in V for a fixed mask: finite-difference-free check  dL/dV . V == L  for L = sum(O*G)
    G = torch.randn_like(o1)
    (o1 * G).sum().backward()
    lhs = float((V.grad * V).sum()), float((o1 * G).sum())
    assert abs(lhs[0] - lhs[1]) <= 1e-3 * max(abs(lhs[1]), 1.0)
    # expectation over masks ~ no-dropout output
    o0 = _attention(Q, K, V, H, 0.0)
    mean = torch.stack([_attention(Q, K, V, H, 0.3, seed=7, offset=100 + i) for i in range(64)]).mean(0)
    assert float((mean - o0).abs().mean()) < 0.15 * float(o0.abs().mean())


@pytest.mark.parametrize("shape", [(48, 20), (600, 136), (5, 512), (1000, 33)])
def test_layernorm_ref_matches_oracle(shape):
    from ptranking_b200 import ops
    rows, F = shape
    g = torch.Generator().manual_seed(rows + F)
    x = torch.randn(2, rows // 2 if rows % 2 == 0 else rows, F, generator=g)[:1] if rows % 2 else torch.randn(2, rows // 2, F, generator=g)
    ln = rp.RefLayerNorm(F)
    with torch.no_grad():
        ln.a_2.add_(0.1 * torch.randn(F, generator=g)); ln.b_2.add_(0.1 * torch.randn(F, generator=g))
    dy = torch.randn(x.shape, generator=g)
    xr = x.clone().requires_grad_(True)
    y_ref = ln(xr)
    (y_ref * dy).sum().backward()
    xc = x.to(DEV).requires_grad_(True)
    a2, b2 = ln.a_2.detach().to(DEV).requires_grad_(True), ln.b_2.detach().to(DEV).requires_grad_(True)
    y = ops.layernorm_ref(xc, a2, b2, 1e-6)
    (y * dy.to(DEV)).sum().backward()
    assert rel_err(y.detach().cpu().numpy(), y_ref.detach().numpy()) <= 2e-6
    assert rel_err(xc.grad.cpu().numpy(), xr.grad.numpy()) <= 2e-5
    assert rel_err(a2.grad.cpu().numpy(), ln.a_2.grad.numpy()) <= 2e-5
    assert rel_err(b2.grad.cpu().numpy(), ln.b_2.grad.numpy()) <= 2e-5


def _list_ranker(cls_name, F, enc, bn, model_para=None):
    import ptranking_b200
    sf = dict(sf_id="listsf", opt="Adagrad", lr=1e-3,
              listsf=dict(num_features=F, ff_dims=[16, 32, 24], AF="R", TL_AF="GE", apply_tl_af=False, BN=bn, bn_type="BN2",
                          bn_affine=False, n_heads=2, encoder_layers=2, encoder_type=enc, dropout=0.0))
    C = getattr(ptranking_b200, cls_name)
    r = C(sf_para_dict=sf, gpu=True, device=DEV) if model_para is None else C(sf_para_dict=sf, model_para_dict=model_para, gpu=True, device=DEV)
    r.init()
    return r


def _load_parts(r, z, prefix):
    for part in ("head_ffnns", "encoder", "tail_ffnns"):
        sd = {k.split("::")[2]: torch.from_numpy(z[k]) for k in z.files if k.startswith(f"{prefix}::{part}::")}
        r.list_sf[part].load_state_dict(sd)          # the reference's own key names


@pytest.mark.parametrize("enc", ["DASALC", "AllRank", "AttnDIN"])
@pytest.mark.parametrize("bn", [0, 1])
def test_list_scorer_forward_backward(enc, bn):
    z = load("scorers.npz")
    key = f"list_{enc}_bn{bn}"
    r = _list_ranker("ListNet", 20, enc, bool(bn))
    _load_parts(r, z, key + "__param")
    r.eval_mode()
    X = torch.from_numpy(z[key + "__X"]).to(DEV)
    s = r.forward(X)
    assert rel_err(s.detach().cpu().numpy(), z[key + "__scores"]) <= 1e-5
    (s * torch.from_numpy(z[key + "__dscores"]).to(DEV)).sum().backward()
    refs = {k: z[k] for k in z.files if k.startswith(key + "__grad::")}
    gscale = max(np.abs(v).max() for v in refs.values())
    checked = 0
    for part in ("head_ffnns", "encoder", "tail_ffnns"):
        for name, p in r.list_sf[part].named_parameters():
            ref = refs[f"{key}__grad::{part}::{name}"]
            got = p.grad.cpu().numpy() if p.grad is not None else np.zeros_like(ref)
            assert np.abs(got - ref).max() <= 3e-5 * np.abs(ref).max() + 2e-6 * gscale + 1e-9, (part, name)
            checked += 1
    assert checked == len(refs)


def test_list_train_steps_match_reference():
    from ptranking_b200 import LABEL_TYPE
    z = load("train_steps.npz")
    run = "ApproxNDCG_list"
    r = _list_ranker("ApproxNDCG", 20, "DASALC", False, dict(model_id="ApproxNDCG", alpha=10.0))
    _load_parts(r, z, run + "__init")
    r.eval_mode()
    X, y = z[run + "__X"], z[run + "__labels"]
    for t in range(3):
        loss, stop = r.train_op(torch.from_numpy(X[t]).to(DEV), torch.from_numpy(y[t]).to(DEV), presort=True, label_type=LABEL_TYPE.MultiLabel)
        ref = z[run + "__losses"][t]
        assert not stop and abs(float(loss.detach()) - ref) <= 3e-5 * max(abs(ref), 1.0), (t, float(loss.detach()), ref)
    s = r.predict(torch.from_numpy(X[0]).to(DEV)).detach().cpu().numpy()
    assert rel_err(s, z[run + "__final_scores"]) <= 5e-5
