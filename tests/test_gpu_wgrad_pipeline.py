"""The weight-gradient kernel (wgrad_tc) against float64, called on its own (ptrb200_tc_wgrad) and inside the scorer.
It keeps one row tile's MMAs in flight while it stages the next tile into the other operand buffer.  A race on the
operand buffers shows up as wrong or run-to-run different gradients, so the pipeline cases are also run twice for bit
equality, at row counts that give the persistent CTAs 0, 1, 2, ...
tiles up to one more than the raw-ring depth, with a short last tile."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _tile_rows_and_stages(N, K, passes):
    """The tile height and raw-ring depth launch_wgrad picks for the un-fused operands (wgrad_smem in ffnet.cu)."""
    KP = (K + 15) // 16 * 16
    op = (128 + KP) * 128 * (2 if passes == 3 else 1)
    fixed = 1024 + 2 * op + 128 + 3 * 128 * 4
    for h in (32, 24, 16, 8):
        rawz, rawp = (h * N * 4 + 127) // 128 * 128, (h * K * 4 + 127) // 128 * 128
        for st in (4, 3, 2):
            if fixed + st * (rawz + rawp) <= 227 * 1024:
                return h, st
    raise AssertionError("no tile height fits")


GRID = 296          # ptrb200_tc_wgrad's persistent CTAs, one partial each


def _tc_wgrad(dZ, P, passes):
    from ptranking_b200 import _lib
    lib = _lib.load()
    rows, N = dZ.shape
    K = P.shape[1]
    out = torch.full((N, K), float("nan"), dtype=torch.float32, device=DEV)
    part = torch.empty(GRID * N * K, dtype=torch.float32, device=DEV)
    _lib.check(lib.ptrb200_tc_wgrad(dZ.data_ptr(), P.data_ptr(), out.data_ptr(), part.data_ptr(), rows, N, K, passes,
                                    torch.cuda.current_stream().cuda_stream), "tc_wgrad")
    return out


@pytest.mark.parametrize("shape", [(32, 100, 136), (64, 8, 32), (1000, 100, 100), (4096, 1, 100), (37, 128, 256), (5000, 100, 136)])
def test_tc_wgrad_matches_float64(shape):
    """dW = dZ^T P through operands transposed into K-major wgmma tiles while they are staged."""
    rows, N, K = shape
    g = torch.Generator(device="cpu").manual_seed(rows + N + K)
    dZ = torch.randn(rows, N, generator=g).to(DEV)
    P = torch.randn(rows, K, generator=g).to(DEV)
    ref = dZ.double().t() @ P.double()
    for passes, tol in ((3, 5e-6), (1, 5e-3)):
        out = _tc_wgrad(dZ, P, passes)
        torch.cuda.synchronize()
        err = float((out.double() - ref).abs().max()) / float(ref.abs().max())
        assert err <= tol, (shape, passes, err)


@pytest.mark.parametrize("N", [1, 100, 128])
@pytest.mark.parametrize("K", [100, 136, 256])
def test_tc_wgrad_tile_counts_match_float64(N, K):
    for passes, tol in ((3, 5e-6), (1, 5e-3)):
        R, stages = _tile_rows_and_stages(N, K, passes)
        # CTA b runs tiles b, b + GRID, ...: GRID * k + j tiles give the CTAs k + 1 or k tiles; the last tile is 3 rows short
        for k in range(stages + 1):
            rows = R * (GRID * k + GRID // 3) - 3
            g = torch.Generator(device="cpu").manual_seed(rows * 7 + N + K)
            dZ = torch.randn(rows, N, generator=g).to(DEV)
            P = torch.randn(rows, K, generator=g).to(DEV)
            ref = dZ.double().t() @ P.double()
            a = _tc_wgrad(dZ, P, passes)
            b = _tc_wgrad(dZ, P, passes)
            torch.cuda.synchronize()
            err = float((a.double() - ref).abs().max()) / float(ref.abs().max())
            assert err <= tol, (passes, rows, R, err)
            assert torch.equal(a, b), (passes, rows)


_ACTS = {"GE": lambda t: torch.nn.functional.gelu(t), "S": torch.sigmoid, "R": torch.relu, None: lambda t: t}


def _ffnet64(X, spec, params):
    """float64 restatement of the stacked net ops.ffnet_apply runs: Linear, batch-level BN (biased variance, eps 1e-5,
    optional affine), activation; no dropout."""
    h = X.double().reshape(-1, spec.dims[0])
    i = 0
    for l, names in enumerate(spec.slots):
        W, b = params[i].double(), params[i + 1].double()
        h = h @ W.t() + b
        has_act = l < spec.L - 1 or spec.act_tail is not None
        if has_act and spec.norm == "BN":
            h = (h - h.mean(0)) / torch.sqrt(h.var(0, unbiased=False) + 1e-5)
            if "gamma" in names:
                h = h * params[i + 2].double() + params[i + 3].double()
        if has_act:
            h = _ACTS[spec.act_hidden if l < spec.L - 1 else spec.act_tail](h)
        i += len(names)
    return h


def _params(spec, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    out = []
    for l, names in enumerate(spec.slots):
        for nm in names:
            if nm == "weight":
                t = torch.randn(spec.dims[l + 1], spec.dims[l], generator=g) / np.sqrt(spec.dims[l])
            elif nm == "gamma":
                t = 1.0 + 0.1 * torch.randn(spec.dims[l + 1], generator=g)
            else:
                t = 0.1 * torch.randn(spec.dims[l + 1], generator=g)
            out.append(t.to(DEV))
    return out


SCORER_CASES = {
    # the default pointwise scorer: normalisation backward folded into the staging (fused dZ), 305 tiles of 32 rows
    # over 132 CTAs on an H100 (2 or 3 each, the ring is 2 deep), the last tile 31 rows
    "fused_dz": (3, 3253, [136, 100, 100, 100, 100, 100, 1], "GE", "S", "BN", True, torch.float32),
    # the same with bf16 features: layer 0's raw ring carries 2-byte elements
    "bf16_x": (3, 3253, [136, 100, 100, 100, 100, 100, 1], "GE", "S", "BN", True, torch.bfloat16),
    # the list scorer's tail net: 128 -> 256, 256 -> 512 and 512 -> 1 run column-blocked (several dZ / input blocks)
    "column_blocked": (2, 1531, [136, 128, 256, 512, 1], "R", None, None, False, torch.float32),
}


@pytest.mark.parametrize("case", list(SCORER_CASES))
def test_scorer_weight_gradients_match_float64(case):
    from ptranking_b200 import ops
    B, n, dims, AF, TL, norm, affine, xdtype = SCORER_CASES[case]
    spec = ops.FFNetSpec(dims, AF, TL, norm, affine, 0.0)
    params = _params(spec, seed=len(case))
    g = torch.Generator(device="cpu").manual_seed(11)
    X = torch.randn(B, n, dims[0], generator=g).to(DEV).to(xdtype)
    dO = torch.randn(B, n, dims[-1], generator=g).to(DEV)
    runs = []
    for _ in range(2):
        pm = [q.clone().requires_grad_(True) for q in params]
        out = ops.ffnet_apply(X, spec, pm, training=True, seed=5, offset=0)
        (out * dO).sum().backward()
        runs.append([q.grad.clone() for q in pm])
    pr = [q.double().requires_grad_(True) for q in params]
    (_ffnet64(X, spec, pr) * dO.double().reshape(-1, dims[-1])).sum().backward()
    gscale = max(float(q.grad.abs().max()) for q in pr)
    i = 0
    for l, names in enumerate(spec.slots):
        ref, got = pr[i].grad, runs[0][i]                 # the weight gradient of layer l
        err = float((got.double() - ref).abs().max())
        assert err <= 2e-5 * float(ref.abs().max()) + 2e-6 * gscale, (case, l, err, float(ref.abs().max()))
        i += len(names)
    for a, b in zip(*runs):
        assert torch.equal(a, b), case
