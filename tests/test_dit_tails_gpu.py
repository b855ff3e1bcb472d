"""GPU tests of the DiT kernels at token counts with ragged tails: the in-place gate/residual GEMM epilogue on
128 x 256 tiles (staged two column blocks at a time, the rows past M clipped by the TMA reduce-add), and the attention
forward with last key blocks of 1 to 98 valid keys and last query blocks that leave warpgroup 1 without a valid row."""
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


# 4098 / 8196: 1 and 2 samples of obj-256 (one or two 128 x 256 tiles per CTA); 1, 130, 257: rows tails of 1, 2, 1
@pytest.mark.parametrize("M", [4098, 8196, 1, 130, 257])
@pytest.mark.parametrize("K", [1024, 4096])
def test_gate_residual_tails(M, K):
    from dgs_b200 import _lib
    N = 1024
    g = torch.Generator(DEV).manual_seed(M + K)
    A = torch.randn(M, K, device=DEV, generator=g).to(torch.bfloat16)
    W = (torch.randn(N, K, device=DEV, generator=g) * 0.03).to(torch.bfloat16)
    bias = torch.randn(N, device=DEV, generator=g) * 0.1
    rows = 4098 if M > 4098 else M  # 8196: two samples, each with its own gate row
    x = torch.randn(M, N, device=DEV, generator=g)
    mod = torch.randn((M + rows - 1) // rows, 6 * N, device=DEV, generator=g)
    gate = mod[:, 2 * N:]
    ref = x.double() + gate[:, :N].double().repeat_interleave(rows, 0)[:M] * (A.double() @ W.double().t() + bias.double())
    # guard rows after the output: the clipped tile rows past M must not be written
    buf = torch.cat([x, torch.full((130, N), 7.0, device=DEV)])
    _lib.check(_lib.lib().dgs_gemm_bf16(A.data_ptr(), W.data_ptr(), bias.data_ptr(), gate.data_ptr(), buf.data_ptr(), M, N,
                                        K, 2, N, mod.stride(0), rows, stream()))
    torch.cuda.synchronize()
    out = buf[:M]
    e = rel(out, ref)
    print(f"gate/residual M={M} K={K}: rel={e:.2e}")
    assert e < 2e-5
    assert rel(out[-(M % 128 or 128):], ref[-(M % 128 or 128):]) < 2e-5
    assert bool((buf[M:] == 7.0).all())


# the last key block holds 2, 1, 15, 64, 1, 2 and 98 valid keys; the last query block has as many rows, so its
# warpgroup 1 (rows 64..127) has no valid row in all but the last case
@pytest.mark.parametrize("N", [4098, 4097, 4111, 4160, 4225, 130, 4194])
def test_attention_tails(N):
    from dgs_b200 import _lib
    L = _lib.lib()
    B, H = 1, 2
    g = torch.Generator(DEV).manual_seed(N)
    qkv = (torch.randn(B, N, 3, H, 64, device=DEV, generator=g) * 1.5).to(torch.bfloat16)
    out = torch.zeros(B, N, H * 64, dtype=torch.bfloat16, device=DEV)
    out_t = torch.zeros_like(out)
    Np = (N + 127) // 128 * 128
    lse = torch.full((B, H, Np), float("nan"), device=DEV)
    _lib.check(L.dgs_attention_fwd(qkv.data_ptr(), out.data_ptr(), B, N, H, stream()))
    _lib.check(L.dgs_attention_fwd_train(qkv.data_ptr(), out_t.data_ptr(), lse.data_ptr(), B, N, H, stream()))
    torch.cuda.synchronize()
    q, k, v = [t.float().permute(0, 2, 1, 3) for t in qkv.unbind(2)]
    s = (q @ k.transpose(-1, -2)) * 0.125
    ref = (torch.softmax(s, dim=-1) @ v).permute(0, 2, 1, 3).reshape(B, N, H * 64)
    e = rel(out.float(), ref)
    print(f"attention N={N}: rel={e:.2e}")
    assert e < 3e-3
    assert rel(out.float(), ref.to(torch.bfloat16).float()) < 2.5e-3
    # the last rows (the query tail) like every other row, and the training variant computes the same output
    assert rel(out[:, -(N % 128 or 128):].float(), ref[:, -(N % 128 or 128):]) < 3e-3
    assert torch.equal(out, out_t)
    lse_ref = torch.logsumexp(s, dim=-1) * 1.4426950408889634
    assert float((lse[:, :, :N] - lse_ref).abs().max()) < 2e-3
