"""GPU tests of the DiT kernels at token counts with ragged tails (the GEMM's are in test_gemm_gpu.py): the attention
forward with last key blocks of 1 to 98 valid keys and last query blocks that leave warpgroup 1 without a valid row."""
import pytest
import torch

from util import rel_l2 as rel

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


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
    _lib.check(L.dgs_attention_fwd(qkv.data_ptr(), out.data_ptr(), B, N, H, _lib.stream(None)))
    _lib.check(L.dgs_attention_fwd_train(qkv.data_ptr(), out_t.data_ptr(), lse.data_ptr(), B, N, H, _lib.stream(None)))
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
