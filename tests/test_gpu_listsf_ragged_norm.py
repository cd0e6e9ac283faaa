"""Ragged batches through the list scorer with BN / BN2 in its head and tail nets: the head and tail run once on the flat
rows (per-query or whole-batch statistics over real documents only), the encoder on each length class padded with masked
keys.  Checked against the dense scorer run query by query (BN2), the dense scorer on equal lengths (BN) and a float64
CPU restatement (BN on mixed lengths), and through a training step, the evaluator and bf16 features."""
import copy

import numpy as np
import pytest
import torch

from oracle import ref_port as rp
from tests.helpers import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ENCS = ["DASALC", "AllRank", "AttnDIN"]
NORMS = {"BN2": ("BN2", False), "BN2_affine": ("BN2", True), "BN": ("BN", False), "BN_affine": ("BN", True)}
FS = [24, 46, 136]          # 46 (MQ2007/2008): the head's F-wide normalised output layer is padded on the ragged BN2 call
FF_DIMS = [32, 64]
# longest first, as data.RaggedBatches orders a batch: a list longer than 512, lists longer than one 128-row tile, a 1
LENS = [600, 200, 130, 64, 40, 7, 3, 1]
CLASSES = [(0, 1, 600), (1, 3, 200), (3, 5, 64), (5, 8, 7)]
SPLITS = {"one_class": None, "classes": CLASSES}
GRAD64_TOL = 1.5e-4         # see test_bn2_ragged_equals_query_by_query
TRAIN_GRAD_TOL = 5e-4       # see test_bn2_ragged_train_step


def _ranker(enc, norm, F, cls="ListNet", dropout=0.0, seed=11):
    import ptranking_b200
    bn_type, affine = NORMS[norm]
    sf = dict(sf_id="listsf", opt="Adagrad", lr=1e-3,
              listsf=dict(num_features=F, ff_dims=list(FF_DIMS), AF="R", TL_AF="GE", apply_tl_af=False, BN=True,
                          bn_type=bn_type, bn_affine=affine, n_heads=2, encoder_layers=2, encoder_type=enc, dropout=dropout))
    torch.manual_seed(seed)
    C = getattr(ptranking_b200, cls)
    r = C(sf_para_dict=sf, gpu=True, device=DEV) if cls != "ApproxNDCG" else \
        C(sf_para_dict=sf, model_para_dict=dict(model_id="ApproxNDCG", alpha=10.0), gpu=True, device=DEV)
    r.init()
    with torch.no_grad():                      # norm parameters off their init point, so that scale and shift matter
        for part in ("head_ffnns", "tail_ffnns"):
            for k, p in r.list_sf[part].named_parameters():
                if "bn" in k:
                    p.add_(0.1 * torch.randn_like(p))
    return r


def _batch(lens, F, seed):
    rng = np.random.default_rng(seed)
    X = torch.from_numpy(rng.standard_normal((sum(lens), F)).astype(np.float32))
    y = torch.from_numpy(rng.integers(0, 5, sum(lens)).astype(np.float32))
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    return X, y, off


def _grads(params, loss):
    for p in params:
        p.grad = None
    loss.backward()
    return [p.grad.detach().clone() if p.grad is not None else torch.zeros_like(p) for p in params]


def _weights(total):
    return torch.cos(torch.arange(total, device=DEV, dtype=torch.float32))


def _names(r):
    """Parameter names of r.get_parameters(), in its order."""
    by_id = {id(p): f"{part}.{k}" for part in ("head_ffnns", "encoder", "tail_ffnns") for k, p in r.list_sf[part].named_parameters()}
    return [by_id[id(p)] for p in r.get_parameters()]


def _check_against(r, s, g, s_want, g_want, tag):
    """The bars of the BN=False ragged test (test_gpu_ragged.py): scores 1e-5 relative, gradients 2e-5 x the largest."""
    assert rel_err(s.detach().cpu().numpy(), s_want.detach().cpu().numpy()) <= 1e-5, tag
    scale = max(float(c.abs().max()) for c in g_want)
    for name, a, c in zip(_names(r), g, g_want):
        assert float((a - c).abs().max()) <= 2e-5 * scale, (tag, name, float((a - c).abs().max()), scale)


@pytest.mark.parametrize("split", list(SPLITS))
@pytest.mark.parametrize("F", FS)
@pytest.mark.parametrize("norm", ["BN2", "BN2_affine"])
@pytest.mark.parametrize("enc", ENCS)
def test_bn2_ragged_equals_query_by_query(enc, norm, F, split):
    """Per-query BN2: the ragged batch gives every query the scores, and every parameter the gradient, that the dense
    forward gives the queries one at a time (the dense path is pinned to the reference by test_gpu_listsf.py and
    test_gpu_r2_parity.py).  A one-document query has zero variance: its normalised value is 0/sqrt(eps) on both sides.

    Bars: scores 1e-5 relative; every gradient within 2e-5 x the largest gradient of the query-by-query run, or, where
    the two fp32 runs differ by more, within GRAD64_TOL x that scale of float64 truth (the oracle's modules, each query
    alone).  The wider bar is needed by the head's first layers: they sit behind four per-query BN2 layers, and the
    lists of 3 and 7 documents have near-constant channels whose 1/sqrt(var + 1e-5) amplifies rounding.  Measured on
    an H100: the ragged gradients of head_ffnns.ff_2..ff_4 lie up to 9e-5 of scale from float64, the query-by-query
    ones up to 2.5e-5; every other gradient agrees within 2e-5."""
    r = _ranker(enc, norm, F)
    r.eval_mode()              # no dropout (the tail keeps the factory's 0.1); autograd stays on
    X, _, off = _batch(LENS, F, seed=F)
    X, offd = X.to(DEV), torch.from_numpy(off).to(DEV)
    params = r.get_parameters()
    w = _weights(X.shape[0])
    s = r.forward_ragged(X, offd, max(LENS), buckets=SPLITS[split])
    assert s.shape == (X.shape[0],)
    g = _grads(params, (s * w).sum())
    s_one = torch.cat([r.forward(X[off[b]: off[b + 1]].unsqueeze(0))[0] for b in range(len(LENS))])
    g_one = _grads(params, (s_one * w).sum())
    assert rel_err(s.detach().cpu().numpy(), s_one.detach().cpu().numpy()) <= 1e-5
    # float64 truth: the oracle's modules, each query alone
    net64 = _oracle(r, enc, norm, F).double()
    Xc, w64 = X.cpu().double(), w.cpu().double()
    s64 = torch.cat([net64(Xc[off[b]: off[b + 1]][None])[0] for b in range(len(LENS))])
    (s64 * w64).sum().backward()
    p64 = dict(net64.named_parameters())
    scale = max(float(c.abs().max()) for c in g_one)
    report = []
    for name, a, c in zip(_names(r), g, g_one):
        e = float((a - c).abs().max())
        g64 = p64[_port_name(*name.split(".", 1))].grad.reshape(a.shape)
        e_rag, e_one = float((a.cpu().double() - g64).abs().max()), float((c.cpu().double() - g64).abs().max())
        report.append((name, e / scale, e_rag / scale, e_one / scale))
    for name, e, e_rag, e_one in report:
        assert e <= 2e-5 or e_rag <= GRAD64_TOL, (name, e, e_rag, e_one)


@pytest.mark.parametrize("split", ["one_class", "classes"])
@pytest.mark.parametrize("F", FS)
@pytest.mark.parametrize("norm", ["BN", "BN_affine"])
@pytest.mark.parametrize("enc", ENCS)
def test_bn_ragged_on_equal_lengths_equals_dense(enc, norm, F, split):
    """Batch-level BN over a ragged batch normalises over every real document of the batch: on lists of one length that
    is the dense [B, n, F] path's BN, so scores and gradients agree."""
    r = _ranker(enc, norm, F)
    r.eval_mode()
    params = r.get_parameters()
    B = 4
    for n in (1, 130, 520):
        X, _, off = _batch([n] * B, F, seed=n + F)
        X, offd = X.to(DEV), torch.from_numpy(off).to(DEV)
        w = _weights(B * n)
        buckets = [(0, 1, n), (1, 3, n), (3, 4, n)] if split == "classes" else None
        s = r.forward_ragged(X, offd, n, buckets=buckets)
        g = _grads(params, (s * w).sum())
        s_dense = r.forward(X.view(B, n, F)).reshape(-1)
        g_dense = _grads(params, (s_dense * w).sum())
        _check_against(r, s, g, s_dense, g_dense, (enc, norm, F, split, n))


def _port_name(part, name):
    """ListNeuralRanker parameter (part, name) -> oracle.ref_port.RefListScorer parameter name."""
    if part != "encoder":
        return ("head." if part == "head_ffnns" else "tail.") + name
    if not name.startswith("layers."):
        return "final_" + name                                   # AllRank's closing LayerNorm
    for a, b in (("sublayer_cont.norm.", "norm."), ("sublayer_cont.0.norm.", "norm0."), ("sublayer_cont.1.norm.", "norm1."),
                 ("fc.w1.", "w1."), ("fc.w2.", "w2.")):
        name = name.replace(a, b)
    return name


def _oracle(r, enc, norm, F):
    """oracle.ref_port.RefListScorer with r's weights, in eval mode (dropout off; batch statistics all the same)."""
    bn_type, affine = NORMS[norm]
    net = rp.RefListScorer(F, ff_dims=FF_DIMS, AF="R", TL_AF="GE", apply_tl_af=False, BN=True, bn_type=bn_type,
                           bn_affine=affine, n_heads=2, encoder_layers=2, dropout=0.0, encoder_type=enc)
    state = {_port_name(part, k): v.detach().cpu().clone() for part in ("head_ffnns", "encoder", "tail_ffnns")
             for k, v in r.list_sf[part].named_parameters()}
    net.load_state_dict(state, strict=True)
    return net.eval()


def _restated_forward(net, X, off, enc):
    """The scorer over a ragged batch, written out with the oracle's modules: head and tail over all real rows with
    batch statistics (LTRBatchNorm: biased variance, eps 1e-5), the encoder query by query."""
    H = net.head(X[None])[0]
    src = X if enc == "DASALC" else H
    E = torch.cat([net.encode(src[off[b]: off[b + 1]][None])[0] for b in range(len(off) - 1)])
    z = {"AllRank": lambda: E, "DASALC": lambda: (E + 1.0) * H, "AttnDIN": lambda: E + X}[enc]()
    return net.tail(z[None])[0, :, 0]


@pytest.mark.parametrize("split", list(SPLITS))
@pytest.mark.parametrize("F", FS)
@pytest.mark.parametrize("norm", ["BN", "BN_affine"])
@pytest.mark.parametrize("enc", ENCS)
def test_bn_ragged_on_mixed_lengths_equals_float64(enc, norm, F, split):
    """Batch-level BN over lists of different lengths against a float64 restatement on the CPU.  Bars: scores within
    2e-5 relative of float64 (or 5x the fp32 restatement's own distance from it), every parameter gradient within
    3e-5 of its largest element + 2e-6 of the largest gradient (or 8x the fp32 restatement's distance)."""
    r = _ranker(enc, norm, F)
    r.eval_mode()
    X, _, off = _batch(LENS, F, seed=3 * F)
    w = torch.cos(torch.arange(X.shape[0], dtype=torch.float64))
    net = _oracle(r, enc, norm, F)
    net64 = copy.deepcopy(net).double()
    s32 = _restated_forward(net, X, off, enc); (s32 * w.float()).sum().backward()
    s64 = _restated_forward(net64, X.double(), off, enc); (s64 * w).sum().backward()
    s64n = s64.detach().numpy()
    s = r.forward_ragged(X.to(DEV), torch.from_numpy(off).to(DEV), max(LENS), buckets=SPLITS[split])
    e_fwd, e_ref = rel_err(s.detach().cpu().numpy(), s64n), rel_err(s32.detach().numpy(), s64n)
    assert e_fwd <= max(2e-5, 5.0 * e_ref), (e_fwd, e_ref)
    (s * w.float().to(DEV)).sum().backward()
    p32, p64 = dict(net.named_parameters()), dict(net64.named_parameters())
    gscale = max(float(p.grad.abs().max()) for p in net64.parameters())
    bad, checked = [], 0
    for part in ("head_ffnns", "encoder", "tail_ffnns"):
        for name, p in r.list_sf[part].named_parameters():
            pn = _port_name(part, name)
            g = p.grad.cpu().double().reshape(p64[pn].shape) if p.grad is not None else torch.zeros_like(p64[pn])
            g64, g32 = p64[pn].grad, p32[pn].grad.double()
            e_ours, e_32 = float((g - g64).abs().max()), float((g32 - g64).abs().max())
            if e_ours > max(3e-5 * float(g64.abs().max()) + 2e-6 * gscale + 1e-12, 8.0 * e_32):
                bad.append((part, name, e_ours, e_32, float(g64.abs().max())))
            checked += 1
    assert not bad, bad
    assert checked == len(p64)


def _flat(r):
    return r.grad_bucket.flat_param.detach().clone(), r.grad_bucket.flat.detach().clone()


@pytest.mark.parametrize("F", [46, 136])
@pytest.mark.parametrize("enc", ENCS)
def test_bn2_ragged_train_step(enc, F):
    """train_op (ListNet, Adagrad) on a ragged BN2 batch cut into length classes: finite loss, one optimizer step, and the
    parameters that one step on the query-by-query gradient sum gives.  The gradients agree within TRAIN_GRAD_TOL x the
    largest gradient, wider than the forward test's bars: ListNet's softmax weights the few top documents of each list
    heavily, and the head's first layers sit behind four per-query BN2 layers whose 1/sqrt(var + 1e-5) amplifies rounding
    on the short lists.  Measured on an H100: up to 3.4e-4 of scale, on head_ffnns.ff_2.weight (AllRank, F = 46); the
    encoder's gradients up to 4.2e-5.
    Adagrad's first step is lr * sign(g + wd p): where the two gradients are too close to zero to agree on that sign an
    element may move by 2 lr; fewer than 1 % of the elements may differ at all.  With dropout p = 0.1, two runs from
    one seed are bit-identical."""
    from ptranking_b200 import LABEL_TYPE, ops
    X, y, off = _batch(LENS, F, seed=7 + F)
    X, y, offd = X.to(DEV), y.to(DEV), torch.from_numpy(off).to(DEV)
    kw = dict(offsets=offd, max_len=max(LENS), buckets=CLASSES, presort=False, label_type=LABEL_TYPE.MultiLabel)
    a = _ranker(enc, "BN2", F)
    b = _ranker(enc, "BN2", F)
    p0, _ = _flat(a)
    assert torch.equal(p0, _flat(b)[0])
    a.eval_mode(); b.eval_mode()
    loss, stop = a.train_op(X, y, **kw)
    assert torch.isfinite(loss) and not stop
    assert a.optimizer.num_steps == 1
    s_one = torch.cat([b.forward(X[off[q]: off[q + 1]].unsqueeze(0))[0] for q in range(len(LENS))])
    loss_one = b.custom_loss_function(s_one, y, **kw)
    assert abs(float(loss) - float(loss_one)) <= 1e-5 * max(abs(float(loss_one)), 1.0)
    (pa, ga), (pb, gb) = _flat(a), _flat(b)
    scale = float(gb.abs().max())
    for name, u, v in zip(_names(a), a.get_parameters(), b.get_parameters()):
        e = float((u.grad - v.grad).abs().max())
        assert e <= TRAIN_GRAD_TOL * scale, (name, e / scale)
    lr, wd = a.lr, a.weight_decay

    def adagrad_first_step(g):          # torch.optim.Adagrad from zero state: p - lr * g' / (|g'| + eps), g' = g + wd p
        gd = g.double() + wd * p0.double()
        return p0.double() - lr * gd / (gd.abs() + 1e-10)
    step_a, step_b = adagrad_first_step(ga), adagrad_first_step(gb)
    assert float((pa.double() - step_a).abs().max()) <= 1e-7 and float((pb.double() - step_b).abs().max()) <= 1e-7
    # so the parameters differ only where the two gradients, within the bars above, disagree on the step
    assert float((pa.double() - step_b).abs().max()) <= float((step_a - step_b).abs().max()) + 1e-7
    assert float((pa - pb).abs().max()) <= 2.0 * lr * 1.001
    assert float(((pa - pb).abs() > 1e-6).float().mean()) < 0.01
    # dropout on: the same seed and dropout counter give the same masks, hence the same bits
    outs = []
    for _ in range(2):
        r = _ranker(enc, "BN2", F, dropout=0.1, seed=5)
        r.train_mode()
        ops._dropout_offset = 1000
        loss, _ = r.train_op(X, y, **kw)
        outs.append((loss.detach().clone(), *_flat(r)))
    assert all(torch.equal(u, v) for u, v in zip(*outs))


def _queries(lens, F, seed):
    rng = np.random.default_rng(seed)
    qs = []
    for i, n in enumerate(lens):
        y = rng.integers(0, 5, n).astype(np.float32)
        y[0] = max(y[0], 1.0)                    # nDCG of a query without a relevant document is 0/0
        qs.append((f"q{i}", rng.standard_normal((n, F)).astype(np.float32), y))
    return qs


@pytest.mark.parametrize("enc", ENCS)
def test_bn2_evaluator_ragged_equals_length_buckets(enc):
    """nDCG and the four ad-hoc metrics over one split, batched ragged and batched by equal length, agree."""
    from ptranking_b200 import LABEL_TYPE
    from ptranking_b200.data import LengthBucketedBatches, RaggedBatches
    F = 46
    rng = np.random.default_rng(1)
    lens = list(np.clip(rng.lognormal(3.8, 0.8, 60), 1, 200).astype(int)) + [1, 1, 150, 150]
    qs = _queries(lens, F, seed=2)
    r = _ranker(enc, "BN2", F)
    rag = RaggedBatches(qs, docs_per_batch=2048, presort=False, pin_memory=False, bucket_edges=(32, 64, 128))
    buck = LengthBucketedBatches(qs, docs_per_batch=2048, presort=False, pin_memory=False)
    ks = [1, 5, 10]
    nd_r = r.ndcg_at_ks(test_data=rag, ks=ks, label_type=LABEL_TYPE.MultiLabel, presort=False)
    nd_b = r.ndcg_at_ks(test_data=buck, ks=ks, label_type=LABEL_TYPE.MultiLabel, presort=False)
    assert float((nd_r - nd_b).abs().max()) <= 1e-6, (nd_r, nd_b)
    m_r = r.adhoc_performance_at_ks(test_data=rag, ks=ks, label_type=LABEL_TYPE.MultiLabel, max_label=4.0, presort=False)
    m_b = r.adhoc_performance_at_ks(test_data=buck, ks=ks, label_type=LABEL_TYPE.MultiLabel, max_label=4.0, presort=False)
    for u, v in zip(m_r, m_b):
        assert float((u - v).abs().max()) <= 1e-6, (m_r, m_b)


@pytest.mark.parametrize("norm", ["BN2", "BN"])
@pytest.mark.parametrize("F", [46, 136])
@pytest.mark.parametrize("enc", ["DASALC", "AttnDIN"])
def test_bf16_ragged_features_equal_fp32(enc, F, norm):
    """RaggedBatches(feature_dtype=torch.bfloat16) batches give the scores and gradients of the same values in fp32."""
    from ptranking_b200.data import RaggedBatches
    lens = [520] * 8 + [200] * 8 + [60] * 8 + [1, 3, 7, 20, 5, 9, 2, 1]      # >= 8 queries per length class
    qs = _queries(lens, F, seed=F)
    qs32 = [(q, torch.from_numpy(x).bfloat16().float().numpy(), y) for q, x, y in qs]
    r = _ranker(enc, norm, F)
    r.eval_mode()
    params = r.get_parameters()
    res = []
    for data, dtype in ((qs, torch.bfloat16), (qs32, torch.float32)):
        batch = next(iter(RaggedBatches(data, docs_per_batch=10 ** 6, presort=False, pin_memory=False,
                                        bucket_edges=(32, 128, 256), feature_dtype=dtype)))
        _, X, _, off, max_len, buckets = batch
        assert X.dtype == dtype and len(buckets) >= 3
        s = r.forward_ragged(X.to(DEV), off.to(DEV), max_len, buckets=buckets)
        res.append((s.detach().clone(), _grads(params, (s * _weights(s.numel())).sum())))
    assert torch.equal(res[0][0], res[1][0])
    assert all(torch.equal(u, v) for u, v in zip(res[0][1], res[1][1]))
