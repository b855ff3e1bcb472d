"""CPU tests of the "fp8_attention" inference precision's oracle (oracle/fp8_attention.py), of its planted defects against
the GPU bounds of tests/test_fp8_attention_gpu.py, and of the argument checks of the new entry points."""
import ctypes as C
import os

import pytest
import torch

from oracle.fp8 import quantize_e4m3
from oracle.fp8_attention import (FP8_ATTENTION_DEFECTS, attention_fp8_matched, key_of_slot,
                                  quantize_attention_operands)
from test_fp8_attention_gpu import ATT_VS_MATCHED
from util import rel_l2 as _rel


def _qkv(B, N, H, seed, std=1.5):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, N, 3 * H * 64, generator=g) * std).to(torch.bfloat16)


def _plain(qkv, H):
    B, N, _ = qkv.shape
    q, k, v = qkv.double().reshape(B, N, 3, H, 64).permute(2, 0, 3, 1, 4)
    return (torch.softmax(q @ k.transpose(-1, -2) / 8, -1) @ v).permute(0, 2, 1, 3).reshape(B, N, H * 64)


def test_key_order_is_a_permutation_matching_the_fragments():
    assert sorted(key_of_slot(a) for a in range(16)) == list(range(16))
    for u in range(4):  # the quad thread u holds score columns {2u, 2u+1, 8+2u, 9+2u} and supplies A's k = 4u..4u+3
        assert [key_of_slot(4 * u + i) for i in range(4)] == [2 * u, 2 * u + 1, 8 + 2 * u, 9 + 2 * u]


@pytest.mark.parametrize("N", [1, 77, 128, 130, 300])
def test_quantizer_scales_order_and_padding(N):
    B, H = 2, 3
    qkv = _qkv(B, N, H, N)
    qkv[0, :, 2 * H * 64:] = 0  # sample 0: all of V zero -> scale 1
    ops = quantize_attention_operands(qkv, H)
    nkb = (N + 127) // 128
    assert ops["vt8"].shape == (B, H, 64, nkb * 128) and ops["sk"].shape == (B, H, nkb)
    t = qkv.float().reshape(B, N, 3, H, 64)
    # scales: 2^ceil(log2(amax / 448)) per (token, head) and per (128-key block, head) over the valid keys
    for s, amax in ((ops["sq"], t[:, :, 0].abs().amax(-1).permute(0, 2, 1)),
                    (ops["sk"][:, :, -1], t[:, 128 * (nkb - 1):, 1].abs().amax(-1).amax(1)),
                    (ops["sv"][1, :, -1], t[1, 128 * (nkb - 1):, 2].abs().amax(-1).amax(0))):
        assert torch.equal(torch.log2(s), torch.ceil(torch.log2(amax / 448)))
    assert torch.all(ops["sv"][0] == 1)
    # q8 is the per-(token, head) e4m3 quantization
    q_ref, _ = quantize_e4m3(t[:, :, 0], 64)
    assert torch.equal(ops["q8"], q_ref.view(torch.uint8))
    # vt8: slot a of every 16 keys holds key key_of_slot(a); the pad keys are zero bytes
    v = ops["vt8"].view(torch.float8_e4m3fn).float() * ops["sv"].repeat_interleave(128, -1)[:, :, None, :]
    for a in range(min(nkb * 128, 256)):
        key = 16 * (a // 16) + key_of_slot(a % 16)
        if key < N:
            # one e4m3 rounding: 2^-4 relative, or half a subnormal step (2^-10 of the scale)
            assert torch.allclose(v[..., a], t[:, key, 2], rtol=2 ** -4, atol=float(ops["sv"].max()) * 2 ** -10)
    pad = torch.tensor([16 * (a // 16) + key_of_slot(a % 16) >= N for a in range(nkb * 128)])
    assert torch.all(ops["vt8"][..., pad] == 0)


def _dequantized_qkv(ops, N):
    from oracle.fp8_attention import _slot_keys
    e = lambda t: t.view(torch.float8_e4m3fn).double()  # noqa: E731
    nk = ops["sk"].shape[-1]
    q = e(ops["q8"]) * ops["sq"].permute(0, 2, 1)[..., None].double()
    k = e(ops["k8"]) * ops["sk"].repeat_interleave(128, -1)[:, :, :N].permute(0, 2, 1)[..., None].double()
    inv = torch.empty(nk * 128, dtype=torch.long)
    inv[_slot_keys(nk * 128, "cpu")] = torch.arange(nk * 128)
    v = (e(ops["vt8"]) * ops["sv"].repeat_interleave(128, -1)[:, :, None, :].double())[..., inv][..., :N]
    return torch.stack([q, k, v.permute(0, 3, 1, 2)], 2).reshape(1, N, -1)


@pytest.mark.parametrize("N", [1, 130, 515])
def test_matched_attention_is_close_to_plain(N):
    B, H = 1, 2
    qkv = _qkv(B, N, H, 7 + N)
    ops = quantize_attention_operands(qkv, H)
    got = attention_fp8_matched(ops, N)
    e_p = _rel(got, _plain(_dequantized_qkv(ops, N), H))
    e_all = _rel(got, _plain(qkv, H))
    print(f"N={N}: matched fp8 attention vs fp64 softmax of the dequantized operands {e_p:.2e}, of the bf16 ones {e_all:.2e}")
    assert e_p < 0.03     # the e4m3 rounding of P alone (measured 1.3e-2)
    assert e_all < 0.12   # plus that of q, k and v at N(0, 1.5^2) inputs (measured 7.6e-2)


@pytest.mark.parametrize("defect", FP8_ATTENTION_DEFECTS)
def test_defects_move_the_output_far_beyond_the_gpu_bound(defect):
    B, H, N = 1, 2, 300
    qkv = _qkv(B, N, H, 3)
    qkv[:, 128:256, 2 * H * 64:] *= 40  # V scales that differ from block to block
    ops = quantize_attention_operands(qkv, H)
    good = attention_fp8_matched(ops, N)
    bad = attention_fp8_matched(ops, N, defects=(defect,))
    e = _rel(bad, good)
    print(f"{defect}: {e:.2e}")
    assert e > 10 * ATT_VS_MATCHED


def test_new_entry_points_validate_arguments():
    from dgs_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    p = C.c_void_p(16)
    assert L.dgs_attention_quantize_e4m3(None, p, p, p, p, p, p, 1, 4, 1, None) == 1
    assert L.dgs_attention_quantize_e4m3(p, p, p, p, p, p, p, 1, 0, 1, None) == 1
    assert b"bad shape" in L.dgs_last_error()
    assert L.dgs_attention_fwd_fp8(p, p, p, p, p, None, p, 1, 4, 1, None) == 1
    assert L.dgs_attention_fwd_fp8(p, p, p, p, p, p, p, 1, 4, 0, None) == 1
    w = _lib.DitWeights(width=1024, heads=16, layers=1, patch=8, n_gaussians=2, mlp_hidden=4096)
    n0 = L.dgs_dit_workspace_bytes_fp8(C.byref(w), 1, 4, 256, 256)
    assert L.dgs_dit_workspace_bytes_fp8_ex(C.byref(w), 1, 4, 256, 256, 0) == n0 > 0
    n1 = L.dgs_dit_workspace_bytes_fp8_ex(C.byref(w), 1, 4, 256, 256, _lib.FP8_ATTENTION)
    N, Nk = 4098, 4224
    assert n1 >= n0 + 2 * N * 1024 + 16 * 64 * Nk + 4 * 16 * N
    assert L.dgs_dit_workspace_bytes_fp8_ex(C.byref(w), 1, 4, 256, 256, 2) == 0
    w8 = _lib.DitWeightsFp8(*([16] * 6))
    io = _lib.DitIO(B=1, V=4, H=256, W=256)
    assert L.dgs_dit_forward_fp8_ex(C.byref(w), C.byref(w8), C.byref(io), 2, p, n1, None) == 1
    assert b"flags" in L.dgs_last_error()


def test_set_inference_precision_modes():
    from dgs_b200.denoiser import DGSDenoiser
    model = DGSDenoiser(dict(patch_size=8, num_layers=1))
    for mode in ("fp8_attention", "fp8", "bf16"):
        assert model.set_inference_precision(mode).inference_precision == mode
    with pytest.raises(ValueError, match="'bf16', 'fp8' or 'fp8_attention'"):
        model.set_inference_precision("fp8-attention")
    assert model.inference_precision == "bf16"
