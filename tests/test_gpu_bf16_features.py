"""bf16 feature tensors read natively by the stacked-FF scorer.

A bf16 feature matrix must give bit for bit what the same values give as fp32 (bf16 values are exact in fp32 and tf32;
dropout masks are keyed by element index): forward output, every parameter gradient and dX, in every math mode, norm,
dropout setting, for dense and ragged batches.  Every comparison below is torch.equal against the fp32 entry fed
``X_bf16.float()``.  Two further checks make sure the bf16 path is really the native one (launch tags, peak memory).
"""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.test_oracle_vs_golden import point_cfg

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

MODES = ["3xtf32", "tf32", "bf16", "simt"]
NORMS = [None, "BN", "BN2"]
RAGGED_LENS = [37, 100, 64, 9]          # 210 rows: the last 128-row tile is a partial one


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


def _run(spec, params, X, dO, ragged, need_dx=True, training=True):
    from ptranking_b200 import ops
    Xl = X.detach().clone().requires_grad_(need_dx)
    pm = [q.detach().clone().requires_grad_(True) for q in params]
    kw = dict(offsets=ragged[0], max_len=ragged[1]) if ragged else {}
    out = ops.ffnet_apply(Xl, spec, pm, training=training, seed=1234, offset=7, **kw)
    (out * dO).sum().backward()
    return out.detach(), [q.grad for q in pm], (Xl.grad if need_dx else None)


def _compare(dims, AF, TL, norm, p, mode, ragged_batch, seed=0, B=3, n=50):
    """Runs the net once on bf16 features and once on the same values as fp32; asserts bit equality."""
    from ptranking_b200 import ops
    spec = ops.FFNetSpec(dims, AF if len(dims) > 2 else None, TL, norm, True, p, math_mode=mode)
    params = _params(spec, dims, seed)
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    if ragged_batch:
        lens = torch.tensor(RAGGED_LENS)
        offsets = torch.zeros(len(RAGGED_LENS) + 1, dtype=torch.int32)
        offsets[1:] = torch.cumsum(lens, 0)
        shape, ragged = (int(lens.sum()), dims[0]), (offsets.to(DEV), int(lens.max()))
    else:
        shape, ragged = (B, n, dims[0]), None
    Xb = torch.randn(*shape, device=DEV, generator=g).to(torch.bfloat16)
    dO = torch.randn(*shape[:-1], dims[-1], device=DEV, generator=g)
    ob, gb, dxb = _run(spec, params, Xb, dO, ragged)
    of, gf, dxf = _run(spec, params, Xb.float(), dO, ragged)
    assert dxb.dtype == torch.bfloat16
    assert torch.equal(ob, of)
    for i, (a, b) in enumerate(zip(gb, gf)):
        assert torch.equal(a, b), (i, (a - b).abs().max().item())
    assert torch.equal(dxb, dxf.to(torch.bfloat16))


@pytest.mark.parametrize("F", [136, 46, 220, 4])
@pytest.mark.parametrize("ragged", [False, True], ids=["dense", "ragged"])
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("norm", NORMS, ids=["nonorm", "BN", "BN2"])
@pytest.mark.parametrize("mode", MODES)
def test_bf16_features_equal_fp32_values(mode, norm, p, ragged, F):
    if mode == "simt" and ragged and norm == "BN2":
        pytest.skip("ragged per-query BN2 needs the tensor-core path (refused for fp32 features as well)")
    _compare([F, 100, 100, 1], "GE", "S", norm, p, mode, ragged, seed=F)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("norm", NORMS, ids=["nonorm", "BN", "BN2"])
def test_bf16_features_wide_stack_rows_gemm_tc(mode, norm):
    """136 -> 256 -> 512: layer 0 runs the one-tile-per-CTA kernel (N > 128), with output-column tiles."""
    _compare([136, 256, 512, 1], "R", None, norm, 0.1, mode, False, seed=5, B=4, n=96)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("ragged", [False, True], ids=["dense", "ragged"])
def test_bf16_features_column_blocked_wgrad(mode, ragged):
    """F = 700 (Yahoo): layer 0's weight gradient runs column-blocked (three input blocks, the last 188 wide); the row
    pitch of 1400 bytes is not 16-byte aligned, so the bf16 rows are staged by hand."""
    _compare([700, 100, 1], "GE", "S", "BN", 0.1, mode, ragged, seed=7, B=2, n=100)


def test_bf16_features_full_size_default_scorer():
    _compare([136] + [100] * 5 + [1], "GE", "S", "BN", 0.1, "3xtf32", False, seed=9, B=1024, n=256)


def _lambdarank(F):
    import ptranking_b200
    sf = dict(sf_id="pointsf", opt="Adam", lr=1e-3, pointsf=point_cfg(F))
    torch.manual_seed(11)
    r = ptranking_b200.LambdaRank(sf_para_dict=sf, model_para_dict=dict(model_id="LambdaRank", sigma=1.0), gpu=True, device=DEV)
    r.init()
    return r


def test_three_adam_steps_on_bf16_batches_equal_fp32_steps():
    """The LambdaRank drop-in at 1024 x 256 x 136: three Adam steps on bf16 batches leave the weights bit-equal to three
    steps on the same values in fp32."""
    from ptranking_b200 import LABEL_TYPE
    g = torch.Generator().manual_seed(3)
    Xs = [torch.randn(1024, 256, 136, generator=g).to(torch.bfloat16).to(DEV) for _ in range(3)]
    ys = [torch.sort(torch.randint(0, 5, (1024, 256), generator=g).float(), dim=1, descending=True)[0].to(DEV) for _ in range(3)]
    a, b = _lambdarank(136), _lambdarank(136)
    b.point_sf.load_state_dict({k: v.clone() for k, v in a.point_sf.state_dict().items()})
    for X, y in zip(Xs, ys):
        la, _ = a.train_op(X, y, presort=True, label_type=LABEL_TYPE.MultiLabel)
        lb, _ = b.train_op(X.float(), y, presort=True, label_type=LABEL_TYPE.MultiLabel)
        assert torch.equal(la, lb)
    for (k, va), (_, vb) in zip(a.point_sf.state_dict().items(), b.point_sf.state_dict().items()):
        assert torch.equal(va, vb), k


@pytest.mark.parametrize("mode", ["3xtf32", "tf32", "bf16"])
def test_native_bf16_kernels_run_and_nothing_widens(mode):
    """The timing report lists the bf16-input launch tags and no widening kernel (F = 136 on the tensor cores)."""
    from ptranking_b200 import _lib, ops
    dims = [136, 100, 100, 1]
    spec = ops.FFNetSpec(dims, "GE", "S", "BN", True, 0.1, math_mode=mode)
    params = _params(spec, dims, 0)
    Xb = torch.randn(8, 64, 136, device=DEV).to(torch.bfloat16)
    dO = torch.randn(8, 64, 1, device=DEV)
    torch.cuda.synchronize()
    _lib.kernel_timings(None)                     # drain earlier records
    _lib.kernel_timings(True)
    try:
        _run(spec, params, Xb, dO, None)
        wide = ops.FFNetSpec([136, 256, 512, 1], "R", None, None, False, 0.0, math_mode=mode)
        _run(wide, _params(wide, [136, 256, 512, 1], 1), Xb, torch.randn(8, 64, 1, device=DEV), None)
        torch.cuda.synchronize()
    finally:
        _lib.kernel_timings(False)
    tags = _lib.kernel_timings(None)
    for t in ("rows_gemm_ws_fwd_xbf16", "rows_gemm_tc_fwd_xbf16", "wgrad_tc_xbf16"):
        assert t in tags, (t, sorted(tags))
    assert "copy_cols_bf16_kernel" not in tags and "copy_cols_kernel" not in tags, sorted(tags)


def test_bf16_features_lower_peak_memory():
    """Forward + backward of the default scorer at 1024 x 256 x 136: bf16 features peak lower than fp32 features, and
    no hidden fp32 copy of them is made (peak minus the feature tensor itself is not higher)."""
    from ptranking_b200 import ops
    dims = [136] + [100] * 5 + [1]
    spec = ops.FFNetSpec(dims, "GE", "S", "BN", True, 0.1, math_mode="3xtf32")
    params = [q.requires_grad_(True) for q in _params(spec, dims, 0)]
    host = {torch.float32: torch.randn(1024, 256, 136)}
    host[torch.bfloat16] = host[torch.float32].to(torch.bfloat16)
    peaks, nbytes = {}, {}
    for dt in (torch.float32, torch.bfloat16, torch.float32, torch.bfloat16):       # second round: allocator warm
        for q in params:
            q.grad = None
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        X = host[dt].to(DEV)                       # the features are part of what is measured
        out = ops.ffnet_apply(X, spec, params, training=True, seed=1, offset=1)
        out.sum().backward()
        torch.cuda.synchronize()
        peaks[dt], nbytes[dt] = torch.cuda.max_memory_allocated() - base, X.nbytes
        del out, X
    assert peaks[torch.bfloat16] < peaks[torch.float32], peaks
    # an fp32 copy of the bf16 features made on the way in would put the bf16 run above this
    assert peaks[torch.bfloat16] - nbytes[torch.bfloat16] <= peaks[torch.float32] - nbytes[torch.float32], peaks


def _ffnet_desc(spec, params):
    return spec.describe([q.detach().contiguous() for q in params])


def test_ffnet_entry_points_refuse_misaligned_bf16_and_unknown_dtype():
    from ptranking_b200 import _lib, ops
    lib = _lib.load()
    dims = [136, 100, 1]
    spec = ops.FFNetSpec(dims, "GE", None, None, False, 0.0, math_mode="3xtf32")
    params = _params(spec, dims, 0)
    desc = _ffnet_desc(spec, params)
    B, n = 2, 64
    Xb = torch.randn(B * n * 136 + 4, device=DEV).to(torch.bfloat16)
    out = torch.empty(B, n, 1, device=DEV)
    nbytes = lib.ptrb200_ffnet_workspace_bytes(C.byref(desc), _lib.DTYPE_BF16, B, n, 0)
    assert nbytes > 0
    ws = torch.empty(int(nbytes), dtype=torch.uint8, device=DEV)
    stream = torch.cuda.current_stream().cuda_stream
    ok = lib.ptrb200_ffnet_forward(C.byref(desc), Xb.data_ptr(), _lib.DTYPE_BF16, out.data_ptr(), ws.data_ptr(), int(nbytes),
                                   B, n, None, 0, 0, 1, 1, stream)
    assert ok == 0
    rc = lib.ptrb200_ffnet_forward(C.byref(desc), Xb.data_ptr() + 2, _lib.DTYPE_BF16, out.data_ptr(), ws.data_ptr(), int(nbytes),
                                   B, n, None, 0, 0, 1, 1, stream)
    assert rc == -1 and b"aligned" in lib.ptrb200_last_error()
    rc = lib.ptrb200_ffnet_forward(C.byref(desc), Xb.data_ptr(), 7, out.data_ptr(), ws.data_ptr(), int(nbytes),
                                   B, n, None, 0, 0, 1, 1, stream)
    assert rc == -1 and b"dtype" in lib.ptrb200_last_error()
    assert lib.ptrb200_ffnet_workspace_bytes(C.byref(desc), 7, B, n, 0) == -1
    gdesc, _ = spec.grads([q.detach() for q in params])
    dO = torch.randn(B, n, 1, device=DEV)
    rc = lib.ptrb200_ffnet_backward(C.byref(desc), C.byref(gdesc), Xb.data_ptr() + 2, _lib.DTYPE_BF16, dO.data_ptr(), None,
                                    ws.data_ptr(), int(nbytes), B, n, None, 0, 0, 1, 1, stream)
    assert rc == -1 and b"aligned" in lib.ptrb200_last_error()
    torch.cuda.synchronize()


@pytest.mark.parametrize("ragged", [False, True], ids=["dense", "ragged"])
@pytest.mark.parametrize("clip", [None, 3.0], ids=["noclip", "istella_clip"])
def test_standard_scale_bf16_output(ragged, clip):
    from ptranking_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(2)
    if ragged:
        offsets = torch.tensor([0, 37, 137, 201, 210], dtype=torch.int32, device=DEV)
        X = 5.0 * torch.randn(210, 46, device=DEV, generator=g)
        kw = dict(offsets=offsets, max_len=100)
    else:
        X = 5.0 * torch.randn(4, 60, 136, device=DEV, generator=g)
        kw = {}
    X[..., 3] = 2.5                                # a constant column
    ref = ops.standard_scale(X, clip_max=clip, **kw).to(torch.bfloat16)
    got = ops.standard_scale(X, clip_max=clip, out_dtype=torch.bfloat16, **kw)
    assert got.dtype == torch.bfloat16 and torch.equal(got, ref)


def _queries(nq, F, seed):
    rng = np.random.default_rng(seed)
    out = []
    for q in range(nq):
        n = int(rng.integers(2, 200))
        out.append((f"q{q}", rng.standard_normal((n, F)).astype(np.float32), rng.integers(0, 5, n).astype(np.float32)))
    return out


def test_two_listmle_epochs_through_bf16_loader_equal_fp32_loader():
    """Two ListMLE epochs through RaggedBatches(feature_dtype=bf16) against two through an fp32 loader fed the pre-rounded
    values: epoch losses, weights and the evaluation metrics are equal."""
    import ptranking_b200
    from ptranking_b200 import LABEL_TYPE, data, ops
    qs = _queries(300, 136, 0)
    rounded = [(q, torch.from_numpy(X).to(torch.bfloat16).float().numpy(), y) for q, X, y in qs]
    res = {}
    for name, src, dt in (("bf16", qs, torch.bfloat16), ("f32", rounded, torch.float32)):
        loader = data.RaggedBatches(src, docs_per_batch=8192, shuffle_seed=1, feature_dtype=dt)
        sf = dict(sf_id="pointsf", opt="Adam", lr=1e-3, pointsf=point_cfg(136, dropout=0.1))
        torch.manual_seed(5)
        ops._tie_offset, ops._dropout_offset = 0, 0
        r = ptranking_b200.ListMLE(sf_para_dict=sf, gpu=True, device=DEV)
        r.init()
        losses = [r.train(loader, label_type=LABEL_TYPE.MultiLabel, presort=True)[0] for _ in range(2)]
        perf = r.adhoc_performance_at_ks(test_data=loader, ks=[1, 5, 10], label_type=LABEL_TYPE.MultiLabel, presort=True)
        res[name] = (losses, {k: v.clone() for k, v in r.point_sf.state_dict().items()}, perf)
    (lb, wb, pb), (lf, wf, pf) = res["bf16"], res["f32"]
    for a, b in zip(lb, lf):
        assert torch.equal(a, b)
    for k in wb:
        assert torch.equal(wb[k], wf[k]), k
    for a, b in zip(pb, pf):
        assert torch.equal(torch.as_tensor(a), torch.as_tensor(b))
