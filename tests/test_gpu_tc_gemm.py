"""wgmma GEMM building block vs a float64 matmul: 3xTF32 restores fp32-level accuracy, 1xTF32 does not."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _gemm(A, B, passes):
    from ptranking_b200 import _lib
    lib = _lib.load()
    M, K = A.shape
    N = B.shape[0]
    out = torch.empty((M, N), dtype=torch.float32, device="cuda")
    _lib.check(lib.ptrb200_tc_gemm_nt(A.data_ptr(), B.data_ptr(), out.data_ptr(), M, N, K, passes,
                                      torch.cuda.current_stream().cuda_stream), "tc_gemm_nt")
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("shape", [(128, 112, 32), (300, 100, 136), (1000, 100, 100), (257, 256, 64),
                                   (128, 16, 8), (64, 1, 100), (4096, 100, 136), (129, 100, 7), (5, 3, 33)])
def test_tc_gemm_matches_float64(shape):
    M, N, K = shape
    g = torch.Generator(device="cpu").manual_seed(M * 31 + N * 7 + K)
    A = torch.randn(M, K, generator=g).cuda()
    B = (torch.randn(N, K, generator=g) * 0.3).cuda()
    ref = (A.double() @ B.double().t())
    scale = float(ref.abs().max())
    c3 = _gemm(A, B, 3)
    c1 = _gemm(A, B, 1)
    e3 = float((c3.double() - ref).abs().max()) / scale
    e1 = float((c1.double() - ref).abs().max()) / scale
    ef = float(((A @ B.t()).double() - ref).abs().max()) / scale      # cuBLAS fp32 for scale
    print(f"{shape}: 3xTF32 {e3:.2e}  1xTF32 {e1:.2e}  cublas-fp32 {ef:.2e}")
    assert e3 <= 3e-6, e3
    assert e1 <= 3e-3, e1
    assert e1 > e3 or K <= 8


@pytest.mark.parametrize("shape", [(32, 100, 136), (64, 8, 32), (1000, 100, 100), (4096, 1, 100), (37, 128, 256), (5000, 100, 136)])
def test_tc_wgrad_matches_float64(shape):
    """dW = dZ^T P through operands transposed into K-major wgmma tiles while they are staged."""
    from ptranking_b200 import _lib
    lib = _lib.load()
    rows, N, K = shape
    g = torch.Generator(device="cpu").manual_seed(rows + N + K)
    dZ = torch.randn(rows, N, generator=g).cuda()
    P = torch.randn(rows, K, generator=g).cuda()
    ref = dZ.double().t() @ P.double()
    out = torch.empty((N, K), dtype=torch.float32, device="cuda")
    part = torch.empty(296 * N * K, dtype=torch.float32, device="cuda")
    for passes, tol in ((3, 5e-6), (1, 5e-3)):
        _lib.check(lib.ptrb200_tc_wgrad(dZ.data_ptr(), P.data_ptr(), out.data_ptr(), part.data_ptr(), rows, N, K, passes,
                                        torch.cuda.current_stream().cuda_stream), "tc_wgrad")
        torch.cuda.synchronize()
        err = float((out.double() - ref).abs().max()) / float(ref.abs().max())
        nz = float((out == 0).float().mean())
        print(f"{shape} passes={passes}: err {err:.2e}  zero-frac {nz:.3f}  |out| {float(out.abs().max()):.3f} |ref| {float(ref.abs().max()):.3f}")
        if err > tol:   # diagnostics: is the result a permutation / transpose of the truth?
            o, r = out.double().cpu(), ref.cpu()
            print("   corr(out, ref) =", float(torch.corrcoef(torch.stack([o.flatten(), r.flatten()]))[0, 1]))
            print("   sorted-value err =", float((o.flatten().sort()[0] - r.flatten().sort()[0]).abs().max()))
        assert err <= tol, err
