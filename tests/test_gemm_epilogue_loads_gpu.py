"""GPU tests of the shared-memory (TMA) GEMM epilogues at shapes where a tile's last column groups lie past N and its
last rows past M: the epilogue loads the bias and gate values of several column groups before using them, reading a
clamped column for the groups past N.  Every output is checked against the fp64 product, and bitwise against the same
GEMM written from registers (an output row stride the TMA store cannot take), which does the same per-element
arithmetic."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def gemm(A, W, bias, gate, gate_stride, rows_per_sample, out, ldc, epi):
    from dgs_b200 import _lib
    M, K = A.shape
    N = W.shape[0]
    _lib.check(_lib.lib().dgs_gemm_bf16(A.data_ptr(), W.data_ptr(), None if bias is None else bias.data_ptr(),
                                        None if gate is None else gate.data_ptr(), out.data_ptr(), M, N, K, epi, ldc,
                                        gate_stride, rows_per_sample, stream()))


@pytest.mark.parametrize("M", [2, 130, 4098])
@pytest.mark.parametrize("N", [1056, 3072, 4128])
@pytest.mark.parametrize("epi", [0, 1, 2])
def test_tma_epilogue_partial_tiles(epi, N, M):
    """epi 0: bias -> bf16, 1: bias + GELU -> bf16, 2: x += gate[sample] * (acc + b) in place (two samples)."""
    K = 256
    g = torch.Generator(DEV).manual_seed(1000 * epi + N + M)
    A = torch.randn(M, K, device=DEV, generator=g).to(torch.bfloat16)
    W = (torch.randn(N, K, device=DEV, generator=g) * 0.06).to(torch.bfloat16)
    bias = torch.randn(N, device=DEV, generator=g) * 0.1
    y = A.double() @ W.double().t() + bias.double()
    pad = 8 if epi < 2 else 4  # a padded row the TMA store takes (16-byte multiple); + 2 elements it does not
    if epi < 2:
        ref = torch.nn.functional.gelu(y, approximate="tanh") if epi == 1 else y
        tma = torch.full((M, N + pad), 7.0, dtype=torch.bfloat16, device=DEV)
        reg = torch.full((M, N + 2), 7.0, dtype=torch.bfloat16, device=DEV)
        gemm(A, W, bias, None, 0, 1, tma, N + pad, epi)
        gemm(A, W, bias, None, 0, 1, reg, N + 2, epi)
        torch.cuda.synchronize()
        assert rel(tma[:, :N].float(), ref) < 2.5e-3
        assert bool((tma[:, N:] == 7.0).all())
        assert torch.equal(tma[:, :N], reg[:, :N])
    else:
        rps = (M + 1) // 2
        gate = torch.randn(2, 3 * N, device=DEV, generator=g)  # rows of an adaLN table, the gate at column offset N
        x = torch.randn(M, N, device=DEV, generator=g)
        sample = torch.arange(M, device=DEV) // rps
        ref = x.double() + gate[sample, N:2 * N].double() * y
        tma = torch.full((M, N + pad), 7.0, device=DEV)
        reg = torch.full((M, N + 2), 7.0, device=DEV)
        tma[:, :N] = x
        reg[:, :N] = x
        gemm(A, W, bias, gate[:, N:], gate.stride(0), rps, tma, N + pad, epi)
        gemm(A, W, bias, gate[:, N:], gate.stride(0), rps, reg, N + 2, epi)
        torch.cuda.synchronize()
        assert rel(tma[:, :N], ref) < 2e-5
        assert bool((tma[:, N:] == 7.0).all())
        assert torch.equal(tma[:, :N], reg[:, :N])
