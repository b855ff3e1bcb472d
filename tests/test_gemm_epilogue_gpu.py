"""GPU tests of the GEMM epilogue paths: the in-place gate/residual update that the DiT's attn.proj and mlp.fc2 run
(staged in shared memory and added into the residual stream by a TMA reduce-add), and output row strides that the
TMA store can (16-byte multiples) or cannot take (those are written from registers)."""
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


@pytest.mark.parametrize("K", [1024, 4096])
def test_gate_residual_in_place_block_shapes(K):
    """x += gate * (A W^T + b) at M = 4098 tokens, N = 1024: attn.proj (K = 1024) and mlp.fc2 (K = 4096) of one block,
    with the gate read from a row of the adaLN table.  The reduce-add rounds g * v before adding it to x: one fp32
    rounding more than fmaf, far below the tolerance."""
    from dgs_b200 import _lib
    M, N, L = 4098, 1024, 24
    g = torch.Generator(DEV).manual_seed(K)
    A = torch.randn(M, K, device=DEV, generator=g).to(torch.bfloat16)
    W = (torch.randn(N, K, device=DEV, generator=g) * 0.03).to(torch.bfloat16)
    bias = torch.randn(N, device=DEV, generator=g) * 0.1
    x = torch.randn(M, N, device=DEV, generator=g)
    mod = torch.randn(1, L * 6 * N + 4 * N, device=DEV, generator=g)  # the adaLN table of one sample
    gate = mod[:, 2 * N:]
    ref = x.double() + gate[:, :N].double() * (A.double() @ W.double().t() + bias.double())
    out = x.clone()
    _lib.check(_lib.lib().dgs_gemm_bf16(A.data_ptr(), W.data_ptr(), bias.data_ptr(), gate.data_ptr(), out.data_ptr(), M, N,
                                        K, 2, N, mod.stride(0), M, stream()))
    torch.cuda.synchronize()
    e = rel(out, ref)
    print(f"in-place gate/residual {M}x{N}x{K}: rel={e:.2e}")
    assert e < 2e-5
    # the last rows (the 2-row tail of the 33rd 128-row tile) are updated like every other row
    assert rel(out[-2:], ref[-2:]) < 2e-5


@pytest.mark.parametrize("pad", [0, 2, 4, 64])
@pytest.mark.parametrize("epi", [0, 3])
def test_output_row_stride(epi, pad):
    """ldc = N + pad elements: bf16 rows of 16-byte multiples (pad 0, 64) and fp32 rows (pad 0, 4, 64) are stored by
    the TMA unit, the others from registers.  The padding columns are left untouched."""
    from dgs_b200 import _lib
    M, N, K = 4098, 1024, 512
    g = torch.Generator(DEV).manual_seed(pad)
    A = torch.randn(M, K, device=DEV, generator=g).to(torch.bfloat16)
    W = (torch.randn(N, K, device=DEV, generator=g) * 0.05).to(torch.bfloat16)
    bias = torch.randn(N, device=DEV, generator=g)
    dt = torch.bfloat16 if epi == 0 else torch.float32
    out = torch.full((M, N + pad), 7.0, dtype=dt, device=DEV)
    _lib.check(_lib.lib().dgs_gemm_bf16(A.data_ptr(), W.data_ptr(), bias.data_ptr(), None, out.data_ptr(), M, N, K, epi,
                                        N + pad, 0, 1, stream()))
    torch.cuda.synchronize()
    ref = A.float() @ W.float().t() + bias
    assert rel(out[:, :N].float(), ref) < (2.5e-3 if epi == 0 else 2e-5)
    assert bool((out[:, N:] == 7.0).all())
