"""CPU checks of the bf16 attention model (oracle/attention.py) that tests/test_attention_gpu.py holds the kernels to:

* with rounding off it is the plain fp64 softmax and its gradient; with rounding on it differs from them by bf16
  noise only; at N <= 128 (one key block) it is the one-shot rounded softmax, bit for bit; its lse2 is the log-sum-exp
  of the scores of the rounded inputs;
* power: with the model standing in for the kernels, each planted defect (ATTENTION_DEFECTS) moves what it corrupts
  by at least twice the bound the GPU test applies, at a shape and in a logit regime the GPU test runs.
"""
import math

import pytest
import torch

from oracle.attention import (ATTENTION_DEFECTS, C, attention_bwd_matched, attention_fwd_matched)
from test_attention_gpu import (BWD_DK_REL, BWD_DQ_REL, BWD_DV_REL, FWD_DIFF_FRAC, FWD_LSE, FWD_OUT_REL, REGIMES,
                                SHAPES, bits_stats, make_qkv)
from util import rel_l2 as rel

CPU_SHAPES = [s for s in SHAPES if s[0] * s[1] * s[2] <= 2000]  # the GPU test's shapes small enough for the CPU


def _plain(qkv):
    """fp64 softmax(q k^T / 8) v of the bf16 inputs -> (out [B, N, H * 64], lse2 [B, H, N])."""
    q, k, v = qkv.double().permute(2, 0, 3, 1, 4).unbind(0)
    s = q @ k.transpose(-1, -2) / 8
    B, H, N, _ = q.shape
    out = (torch.softmax(s, -1) @ v).permute(0, 2, 1, 3).reshape(B, N, H * 64)
    return out, torch.logsumexp(s, -1) / math.log(2.0)


def _lse_err(a, b):
    return float(((a - b).abs() / b.abs().clamp(min=1)).max())


def _case(B, N, H, regime, seed=0):
    qkv = make_qkv(B, N, H, regime, seed, device="cpu")
    g = torch.Generator().manual_seed(N + H)
    dout = torch.randn(B, N, H * 64, generator=g).to(torch.bfloat16)
    return qkv, dout


@pytest.mark.parametrize("N", [1, 77, 130, 300])
def test_unrounded_model_is_the_fp64_softmax_and_its_gradient(N):
    qkv, dout = _case(2, N, 2, "scale1.5")
    out, lse2 = attention_fwd_matched(qkv, rounding=False)
    ref, ref_lse = _plain(qkv)
    assert rel(out, ref) < 1e-12
    assert float((lse2 - ref_lse).abs().max()) < 1e-12
    x = qkv.double().requires_grad_(True)
    q, k, v = x.permute(2, 0, 3, 1, 4).unbind(0)
    o = (torch.softmax(q @ k.transpose(-1, -2) / 8, -1) @ v).permute(0, 2, 1, 3).reshape(2, N, 128)
    o.backward(dout.double())
    dqkv, dsum = attention_bwd_matched(qkv, out, dout, lse2, rounding=False)
    for i in range(3 if N > 1 else 1):  # N = 1: dq = dk = 0
        assert rel(dqkv[:, :, i], x.grad[:, :, i]) < 1e-12, i
    if N == 1:
        assert float(dqkv[:, :, :2].abs().max()) < 1e-12
    assert rel(dsum, (out * dout.double()).reshape(2, N, 2, 64).sum(-1).transpose(1, 2)) < 1e-14


@pytest.mark.parametrize("regime", list(REGIMES))
def test_rounded_model_differs_by_bf16_noise_only(regime):
    B, N, H = 3, 271, 3
    qkv, dout = _case(B, N, H, regime)
    out, lse2 = attention_fwd_matched(qkv)
    ref, ref_lse = _plain(qkv)
    e_out = rel(out, ref)
    e_lse = _lse_err(lse2, ref_lse)
    plain_out, plain_lse = attention_fwd_matched(qkv, rounding=False)
    dq = attention_bwd_matched(qkv, out, dout, lse2)[0]
    dq_plain = attention_bwd_matched(qkv, plain_out, dout, plain_lse, rounding=False)[0]
    e_bwd = [rel(dq[:, :, i], dq_plain[:, :, i]) for i in range(3)]
    print(f"{regime}: rounded model vs fp64 softmax: out {e_out:.2e}  lse2 {e_lse:.2e}  dq/dk/dv "
          + " ".join(f"{e:.2e}" for e in e_bwd))
    assert 1e-4 < e_out < 4e-3   # the bf16 roundings of P and of out: 2^-9 relative each, uncorrelated
    assert e_lse < 2e-7          # fp32 scores and fp32 lse2
    assert all(1e-4 < e < 1e-2 for e in e_bwd), e_bwd


@pytest.mark.parametrize("N", [1, 64, 77, 128])
@pytest.mark.parametrize("regime", list(REGIMES))
def test_one_key_block_is_the_one_shot_rounded_softmax(N, regime):
    """With a single key block the online softmax has nothing to rescale: the model is the rounded softmax written
    in one piece, bit for bit."""
    B, H = 2, 3
    qkv, _ = _case(B, N, H, regime)
    out, lse2 = attention_fwd_matched(qkv)
    f32 = lambda t: t.float().double()  # noqa: E731
    q, k, v = qkv.double().permute(2, 0, 3, 1, 4).unbind(0)
    s = f32(q @ k.transpose(-1, -2))
    m = s.amax(-1, keepdim=True)
    p = f32(torch.exp2(f32(s * C - f32(m * C))))
    p = torch.where(p < 2.0 ** -126, torch.zeros_like(p), p)
    l = p.sum(-1, keepdim=True)
    o = f32((p.to(torch.bfloat16).double() @ v) * f32(1.0 / f32(l)))
    ref = o.permute(0, 2, 1, 3).reshape(B, N, H * 64).to(torch.bfloat16)
    assert torch.equal(out, ref)
    assert torch.equal(lse2, f32(m[..., 0] * C + f32(torch.log2(f32(l[..., 0])))))


@pytest.mark.parametrize("regime", list(REGIMES))
def test_lse2_is_the_log_sum_exp_of_the_rounded_inputs(regime):
    qkv, _ = _case(2, 383, 5, regime)
    _, lse2 = attention_fwd_matched(qkv)
    _, ref = _plain(qkv)
    e = _lse_err(lse2, ref)
    print(f"{regime}: lse2 vs fp64 logsumexp {e:.2e}")
    assert e < 2e-7


def test_ulp_distance_of_bf16_bits():
    a = torch.tensor([1.0, -1.0, 0.0, 3.0, -2.0 ** -130, 2.0 ** -130], dtype=torch.bfloat16)
    b = torch.tensor([1.0078125, -0.99609375, -0.0, 3.0, 2.0 ** -130, 2.0 ** -130], dtype=torch.bfloat16)
    frac, small, ulp = bits_stats(a.repeat(64 // 6 + 1)[:64], b.repeat(64 // 6 + 1)[:64])
    assert ulp > 1 and 0 < frac < 1  # the sign change of a tiny value is many ulps, but small against the row
    assert small < 2.0 ** -120
    assert bits_stats(a[:4].repeat(16), b[:4].repeat(16))[2] == 1  # one ulp up, one ulp down, -0 = +0


def _fwd_power(qkv, defect):
    out, lse2 = attention_fwd_matched(qkv)
    bad, bad_lse = attention_fwd_matched(qkv, defects=(defect,))
    return max(rel(bad, out) / FWD_OUT_REL, _lse_err(bad_lse, lse2) / FWD_LSE, bits_stats(bad, out)[0] / FWD_DIFF_FRAC)


def _bwd_power(qkv, dout, defect):
    out, lse2 = attention_fwd_matched(qkv)
    good = attention_bwd_matched(qkv, out, dout, lse2)[0]
    bad = attention_bwd_matched(qkv, out, dout, lse2, defects=(defect,))[0]
    return max(rel(bad[:, :, i], good[:, :, i]) / b for i, b in enumerate((BWD_DQ_REL, BWD_DK_REL, BWD_DV_REL)))


def test_planted_defects_exceed_the_gpu_bounds():
    """Each defect's effect, as a multiple of the GPU bound on the check that sees it best (out norm-wise, lse2, the
    share of differing out bits; dq / dk / dv), at B = 3, N = 271, H = 3 (three key blocks, a ragged key and query tail,
    two 64-query blocks of the backward past the first 192 rows) in each logit regime of the GPU test."""
    B, N, H = 3, 271, 3
    assert (B, N, H) in SHAPES
    power = {}
    for defect in ATTENTION_DEFECTS:
        for regime in REGIMES:
            qkv, dout = _case(B, N, H, regime)
            if defect in ("dkv_query_tail_dropped", "ds_scale_dropped_in_dq"):
                power[defect, regime] = _bwd_power(qkv, dout, defect)
            else:
                power[defect, regime] = _fwd_power(qkv, defect)
    for defect in ATTENTION_DEFECTS:
        print(f"{defect:24s} " + "  ".join(f"{r} {power[defect, r]:9.1f}" for r in REGIMES) + "  x the GPU bound")
    for defect in ATTENTION_DEFECTS:
        assert max(power[defect, r] for r in REGIMES) >= 2, defect


def test_defects_that_fade_with_n_still_exceed_the_gpu_bounds_at_4098():
    """The pad key's weight is ~1/N and the exp2 bias and the bf16(P) row sum average out over the keys: at the obj-256
    token count, in the flat regime where they are weakest, they still pass 2x the bound (one head: heads are
    independent, so H = 16 only repeats the case)."""
    qkv, _ = _case(1, 4098, 1, "flat")
    power = {d: _fwd_power(qkv, d) for d in ("pad_key_unmasked", "exp2_bias", "l_from_rounded_p")}
    print("N = 4098, flat: " + "  ".join(f"{d} {v:.1f}" for d, v in power.items()) + "  x the GPU bound; "
          "below resolution: none")
    for d, v in power.items():
        assert v >= 2, d


def test_backward_rejects_more_than_64_heads():
    import ctypes as C
    import os
    from dgs_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    p = C.c_void_p(16)
    assert L.dgs_attention_bwd(p, p, p, p, p, p, 1, 4, 65, None) == 1
    assert b"bad shape" in L.dgs_last_error()
