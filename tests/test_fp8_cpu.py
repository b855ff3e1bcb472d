"""CPU checks of the FP8 path's format and of its GPU tests' machinery (no GPU):

* oracle/fp8.py's quantizer: power-of-two scales, an all-zero group, saturation, the 1 x 128 group layout, and
  round-to-nearest-even on every e4m3 code and every midpoint between neighbouring codes;
* the argument checks of the new C-ABI entries, which reject bad calls before touching the device;
* power: with the FP8-matched block standing in for the kernels, two planted defects (a k-block's group scale taken
  from the wrong group, one output channel's weight scale dropped) move the block increment by more than twice the
  bound tests/test_fp8_gpu.py applies on the H100.
"""
import ctypes

import pytest
import torch

from test_dit_gpu import rel
from test_fp8_gpu import BLOCK_FP8

D = 1024


def _codes():
    """every finite e4m3 value, ascending, with its byte"""
    b = torch.arange(256, dtype=torch.uint8)
    v = b.view(torch.float8_e4m3fn).float()
    keep = torch.isfinite(v)
    v, b = v[keep], b[keep]
    order = torch.argsort(v)
    return v[order], b[order]


def test_scales_are_powers_of_two_and_bound_the_group():
    from oracle.fp8 import quantize_e4m3
    g = torch.Generator().manual_seed(0)
    x = torch.randn(64, 512, generator=g) * torch.exp2(torch.randint(-30, 30, (64, 1), generator=g).float())
    q, s = quantize_e4m3(x, 128)
    assert s.shape == (64, 4)
    m, _ = torch.frexp(s)
    assert bool((m == 0.5).all())  # powers of two
    amax = x.reshape(64, 4, 128).abs().amax(-1)
    assert bool((amax <= 448 * s).all()) and bool((amax > 224 * s).all())  # the smallest such power
    assert bool((q.float().abs().reshape(64, 4, 128).amax(-1) <= 448).all())


def test_zero_group_and_saturation():
    from oracle.fp8 import quantize_e4m3
    x = torch.zeros(3, 256)
    x[1, :128] = 448.0
    x[1, 5] = -448.0
    x[2, 128:] = 1e-3
    q, s = quantize_e4m3(x, 128)
    assert s[0].tolist() == [1.0, 1.0] and bool((q[0].float() == 0).all())
    assert s[1, 0] == 1.0 and q[1, 0].float() == 448.0 and q[1, 5].float() == -448.0
    assert s[1, 1] == 1.0 and s[2, 0] == 1.0  # zero groups
    # amax just above a boundary takes the next power, and nothing saturates beyond +-448
    y = torch.full((1, 128), 448.0 * (1 + 2 ** -20))
    qy, sy = quantize_e4m3(y, 128)
    assert sy.item() == 2.0 and qy.float().max().item() == 224.0


def test_group_layout():
    from oracle.fp8 import dequantize_e4m3, quantize_e4m3
    x = torch.ones(2, 384)
    x[0, 128:256] *= 1000
    x[1, 256:] *= 1e-3
    q, s = quantize_e4m3(x, 128)
    assert s[0, 1] > s[0, 0] and s[0, 0] == s[0, 2]
    assert s[1, 2] < s[1, 0]
    assert torch.allclose(dequantize_e4m3(q, s, 128), x, rtol=2 ** -4)


def test_round_to_nearest_even_on_every_code_and_midpoint():
    from oracle.fp8 import quantize_e4m3
    v, b = _codes()
    pos = v[v >= 0]
    # group scale 1: a group whose amax is 448 (the last column) holds the values to quantize
    def q1(vals):
        x = torch.cat([vals, torch.tensor([448.0])])[None]
        q, s = quantize_e4m3(x, x.shape[1])
        assert s.item() == 1.0
        return q[0, :-1]
    # every code quantizes to itself, byte for byte
    assert torch.equal(q1(v).view(torch.uint8), b)
    # every midpoint between neighbouring non-negative codes rounds to the neighbour with the even (0) last bit
    lo, hi = pos[:-1], pos[1:]
    mid = (lo.double() + hi.double()) / 2
    assert bool((mid.float().double() == mid).all())  # midpoints are exact in fp32
    got = q1(mid.float()).float()
    lo_b = q1(lo).view(torch.uint8)
    want = torch.where((lo_b & 1) == 0, lo, hi)
    assert torch.equal(got, want)
    # and the negative side mirrors it
    assert torch.equal(q1(-mid.float()).float(), -want)


def test_argument_validation_without_gpu():
    """The FP8 entries reject bad arguments with a status and a message, without touching the device."""
    from test_abi import _ensure_built
    from dgs_b200 import _lib
    _ensure_built()
    L = _lib.lib()
    fake = ctypes.c_void_p(256)

    def gemm(M=256, N=1024, K=1024, sa=fake, sw=fake, epi=0, out_scale=None, gate=None):
        return L.dgs_gemm_fp8(fake, sa, fake, sw, None, gate, fake, out_scale, M, N, K, epi, N, 0, 1, None)
    assert gemm(K=1000) == 1 and b"K % 128" in L.dgs_last_error()
    assert gemm(N=1000) == 1 and b"N % 128" in L.dgs_last_error()
    assert gemm(sa=None) == 1 and b"NULL scales" in L.dgs_last_error()
    assert gemm(sw=None) == 1 and b"NULL scales" in L.dgs_last_error()
    assert gemm(epi=6) == 1 and b"out_scale" in L.dgs_last_error()
    assert gemm(epi=2) == 1 and b"gate" in L.dgs_last_error()
    assert gemm(epi=1, out_scale=fake) == 1 and b"epilogue" in L.dgs_last_error()
    assert L.dgs_ln_modulate_fp8(fake, fake, fake, 6 * D, fake, fake, 1, 10, 512, 1e-6, None) == 1
    assert b"width" in L.dgs_last_error()
    assert L.dgs_ln_modulate_fp8(fake, fake, fake, 6 * D, fake, None, 1, 10, D, 1e-6, None) == 1
    assert b"NULL" in L.dgs_last_error()
    assert L.dgs_quantize_rows_e4m3(fake, 4, 16, fake, None, None) == 1 and b"NULL" in L.dgs_last_error()
    # the forward: inference only, width 1024 only, FP8 weights required, workspace size
    w = _lib.DitWeights(width=1024, heads=16, layers=2, patch=8, n_gaussians=2, mlp_hidden=4096)
    w8 = _lib.DitWeightsFp8(*([256] * 6))
    io = _lib.DitIO(B=1, V=4, H=32, W=32, images=256, ray_o=256, ray_d=256, t=256, xyz=256, features=256, scaling=256,
                    rotation=256, opacity=256, train_state=256)
    bf = L.dgs_dit_workspace_bytes(ctypes.byref(w), 1, 4, 32, 32)
    b8 = L.dgs_dit_workspace_bytes_fp8(ctypes.byref(w), 1, 4, 32, 32)
    assert b8 > bf > 0
    fwd = lambda nbytes=b8, ww=w, w8_=w8: L.dgs_dit_forward_fp8(ctypes.byref(ww), None if w8_ is None else ctypes.byref(w8_),  # noqa: E731
                                                                  ctypes.byref(io), fake, nbytes, None)
    assert fwd() == 1 and b"inference only" in L.dgs_last_error()
    io.train_state = None
    assert fwd(nbytes=bf) == 1 and b"workspace too small" in L.dgs_last_error()
    assert fwd(w8_=None) == 1 and b"NULL FP8" in L.dgs_last_error()
    w8.fc2_s = None
    assert fwd(w8_=w8) == 1 and b"NULL FP8" in L.dgs_last_error()
    w8.fc2_s = 256
    w.width = 512
    assert fwd() == 1 and b"width" in L.dgs_last_error()
    assert L.dgs_dit_workspace_bytes_fp8(ctypes.byref(w), 1, 4, 32, 32) == 0


@pytest.fixture(scope="module")
def block_case():
    from dit_regime import apply_trained_scale
    from oracle.dit import DenoiserOracle, block_modulation64, conditioning64
    torch.manual_seed(0)
    o = apply_trained_scale(DenoiserOracle(layers=2), seed=0)
    blk = o.transformer[1]
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1, 130, D, generator=g, dtype=torch.float64) * 1.5
    mod = block_modulation64(blk, conditioning64(o, torch.tensor([400])))
    return blk, x, mod


@pytest.mark.parametrize("defect", ["group_scale_from_wrong_group", "weight_scale_dropped"])
def test_block_bound_rejects_planted_defects(block_case, defect):
    from oracle.fp8 import dit_block_fp8_matched
    blk, x, mod = block_case
    good = dit_block_fp8_matched(blk, x, mod)["x_out"] - x
    bad = dit_block_fp8_matched(blk, x, mod, defects=(defect,))["x_out"] - x
    e = rel(bad, good)
    print(f"{defect}: block increment moves by {e:.2e} (GPU bound {BLOCK_FP8:.1e})")
    assert e > 2 * BLOCK_FP8


def test_fp8_matched_block_is_close_to_the_plain_block(block_case):
    """Sanity: the FP8 block differs from the fp64 block by the e4m3 rounding of three GEMM inputs, a few percent."""
    from oracle.dit import dit_block_matched
    from oracle.fp8 import dit_block_fp8_matched
    blk, x, mod = block_case
    plain = dit_block_matched(blk, x, mod, rounding=False)["x_out"] - x
    e = rel(dit_block_fp8_matched(blk, x, mod)["x_out"] - x, plain)
    print(f"fp8-matched vs plain fp64 block increment: {e:.2e}")
    assert 1e-3 < e < 0.1
