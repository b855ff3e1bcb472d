"""GPU tests of the "fp8_attention" inference precision (DGS_FP8_ATTENTION): the quantize pass bitwise against
oracle/fp8_attention.py, the FP8 attention kernel against the matched fp64 oracle and the fp32 softmax, one block against
the FP8-attention-matched oracle block, and the whole denoiser against the fp32 oracle with the emulated model's own
error as the yardstick.

Every bound below was set from the errors measured on an H100 80GB HBM3 over seeds 0, 1, 2; the measured worst case is
written next to it.
"""
import math

import pytest
import torch

from dit_regime import dit_inputs
from fp8_ops import _attr, _err, _models, _views, attention_fwd_fp8, block_product, quantize_attention
from util import rel_l2 as rel

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
D = 1024

# ---- bounds, with the worst case measured on the H100 over seeds 0-2 ----
# kernel vs attention_fp8_matched on the same e4m3 operands: worst 5.06e-3 (N = 16386).  The kernel's fp32 arguments of
# the exponentials (and ex2.approx) differ from the oracle's fp64 ones in the last bits, which now and then puts P on the
# other side of an e4m3 rounding midpoint (one 2^-4 step), plus the bf16 output rounding.  The planted defects of
# tests/test_fp8_attention_cpu.py move the output by more than ten times this bound.
ATT_VS_MATCHED = 8e-3
# kernel vs the fp32 softmax of the bf16 q, k, v: worst 9.71e-2 (N = 16386).  This is the e4m3 rounding of q, k, v and P
# at N(0, 1.5^2) inputs (logit std 2.25, peaky rows): the oracle on the same operands is as far from the fp32 softmax.
ATT_VS_FP32 = 0.12
# block increment vs dit_block_fp8_matched(attention_fp8=True): worst 2.83e-2 (N = 16386; 1.90e-2 at N = 4098); the
# x_mid increment fed the product's h1q: worst 3.02e-2 (N = 16386).  The FP8 qkv GEMM's accumulation error moves q, k, v
# by a bf16 rounding here and there, and that moves their e4m3 roundings; the FP8 GEMM block's own bound is 2e-2.
BLOCK_FP8_ATT = 4.5e-2
E2E_SLACK = 1e-3  # the bf16 path's own end-to-end bound, added to 1.5 x the emulation's error


# the shapes of tests/test_dit_gpu.py::test_attention_vs_fp32_softmax
SHAPES = [(1, 4098, 16), (2, 1026, 16), (1, 128, 2), (1, 130, 1), (2, 77, 4), (1, 1, 1), (1, 16386, 2), (1, 2050, 20),
          (1, 1500, 16), (3, 4098, 16)]


@pytest.mark.parametrize("B,N,H", SHAPES)
def test_quantize_pass_bitwise(B, N, H):
    from oracle.fp8_attention import quantize_attention_operands
    g = torch.Generator(DEV).manual_seed(N)
    qkv = (torch.randn(B, N, 3 * H * 64, device=DEV, generator=g) * 1.5).to(torch.bfloat16)
    qkv[:, :, 2 * H * 64:2 * H * 64 + 64] = 0  # head 0's V all zero: scale 1
    got = quantize_attention(qkv, B, N, H)
    ref = quantize_attention_operands(qkv, H)
    torch.cuda.synchronize()
    for k in ref:
        assert torch.equal(got[k], ref[k]), k


@pytest.mark.parametrize("B,N,H", SHAPES)
def test_attention_fp8_vs_matched_and_fp32(B, N, H):
    from oracle.fp8_attention import attention_fp8_matched
    g = torch.Generator(DEV).manual_seed(N)
    qkv = (torch.randn(B, N, 3 * H * 64, device=DEV, generator=g) * 1.5).to(torch.bfloat16)
    ops = quantize_attention(qkv, B, N, H)
    out = attention_fwd_fp8(ops, B, N, H)
    e_m = rel(out.float(), attention_fp8_matched(ops, N).float())
    q, k, v = [t.float().permute(0, 2, 1, 3) for t in qkv.reshape(B, N, 3, H, 64).unbind(2)]
    ref = (torch.softmax((q @ k.transpose(-1, -2)) * 0.125, dim=-1) @ v).permute(0, 2, 1, 3).reshape(B, N, H * 64)
    e_f = rel(out.float(), ref)
    print(f"fp8 attention B={B} N={N} H={H}: vs matched {e_m:.2e}  vs fp32 softmax {e_f:.2e}")
    assert e_m < ATT_VS_MATCHED
    assert e_f < ATT_VS_FP32


# N = 4098: obj-256; N = 16386: obj-512 / scene-512 / the pipline_obj.py demo (one seed: the fp64 oracle is slow there)
@pytest.mark.parametrize("seed,N", [(0, 4098), (1, 4098), (2, 4098), (0, 16386)])
def test_block_fp8_attention_trained_scale(seed, N):
    from dgs_b200.denoiser import DGSDenoiser
    from dit_regime import apply_trained_scale
    from oracle.dit import block_modulation64, conditioning64
    from oracle.fp8_attention import dit_block_fp8_matched
    torch.manual_seed(seed)
    model = apply_trained_scale(DGSDenoiser(dict(patch_size=8, num_layers=2)), seed).to(DEV)
    blk = model.transformer[seed % 2]
    g = torch.Generator(DEV).manual_seed(seed)
    x = (torch.randn(1, N, D, device=DEV, generator=g) * 1.5).contiguous()
    mod = block_modulation64(blk, conditioning64(model, torch.tensor([100 + 300 * seed], device=DEV)))
    prod = block_product(blk, x, mod.float().contiguous(), N, attention_fp8=True)
    xd = x.double()
    ref = dit_block_fp8_matched(blk, xd, mod, attention_fp8=True)
    e_blk = rel(prod["x_out"] - x, ref["x_out"] - xd)
    fed = dit_block_fp8_matched(blk, xd, mod, feed={"h1q": prod["h1q"]}, attention_fp8=True)
    e_att = rel(prod["x_mid"] - x, fed["x_mid"] - xd)
    print(f"fp8-attention block N={N} seed {seed}: increment {e_blk:.2e}  x_mid increment (fed h1q) {e_att:.2e}")
    assert e_blk < BLOCK_FP8_ATT
    assert e_att < BLOCK_FP8_ATT


E2E_CASES = [(24, False, False), (24, False, True), (2, True, True)]


def _psnr(a, b):
    mse = float((a - b).double().pow(2).mean())
    return 10 * math.log10(float(b.double().abs().max()) ** 2 / max(mse, 1e-30))


@pytest.mark.parametrize("layers,scene,trained", E2E_CASES)
def test_end_to_end_fp8_attention(layers, scene, trained):
    from oracle.fp8_attention import emulate_fp8
    worst = []
    for seed in (0, 1, 2):
        model, oracle = _models(layers, scene, trained, seed)
        inputs = dit_inputs(1, 4, 256, 256, seed=seed)
        with torch.no_grad():
            r_out, r_ia = oracle.image_to_gaussians(*inputs)
            ref = (r_out, r_ia, _views(model, _attr(r_out), 4, 256, 256))
            e_out, e_ia = emulate_fp8(oracle, attention=True).image_to_gaussians(*inputs)
            e_em = _err(e_out, e_ia, _views(model, _attr(e_out), 4, 256, 256), ref)
            b_out, _ = model.image_to_gaussians(*inputs)
            b_views = _views(model, b_out, 4, 256, 256)
            model.set_inference_precision("fp8_attention")
            f_out, f_ia = model.image_to_gaussians(*inputs)
            f_views = _views(model, f_out, 4, 256, 256)
            e_f8 = _err(f_out, f_ia, f_views, ref)
        print(f"e2e fp8_attention layers={layers} scene={scene} trained={trained} seed={seed}: vs fp32 {e_f8:.2e}  "
              f"emulated {e_em:.2e}  gate {1.5 * e_em + E2E_SLACK:.2e}  PSNR(renders vs bf16) {_psnr(f_views, b_views):.1f} dB")
        worst.append((e_f8, e_em))
        del model, oracle
    for e_f8, e_em in worst:
        assert e_f8 <= 1.5 * e_em + E2E_SLACK, worst


def test_bf16_and_fp8_untouched_by_an_fp8_attention_call():
    from dgs_b200.train import DitTrainer
    model, _ = _models(2, False, True, 0)
    inputs = dit_inputs(1, 4, 64, 64, seed=0)
    outs = {}
    with torch.no_grad():
        for mode in ("bf16", "fp8", "fp8_attention", "fp8", "bf16"):
            model.set_inference_precision(mode)
            out, ia = model.image_to_gaussians(*inputs)
            outs.setdefault(mode, []).append((out, ia))
    torch.cuda.synchronize()
    for mode in ("bf16", "fp8"):
        (a, a_ia), (b, b_ia) = outs[mode]
        assert all(torch.equal(a[k], b[k]) for k in a) and torch.equal(a_ia, b_ia), mode
    f, _ = outs["fp8_attention"][0]
    a, _ = outs["fp8"][0]
    assert not all(torch.equal(a[k], f[k]) for k in a)  # the FP8 attention did run
    DitTrainer(model)
    model.train()
    model.set_inference_precision("fp8_attention")
    with pytest.raises(RuntimeError, match="FP8"):
        with torch.enable_grad():
            model.image_to_gaussians(*inputs)


def test_sampler_fp8_attention_three_steps():
    import torch.nn.functional as F
    from dgs_b200 import synth
    from dgs_b200.diffusion import create_diffusion
    model, _ = _models(2, False, True, 0)
    B, V, H, W = 1, 4, 64, 64
    g = torch.Generator(DEV).manual_seed(5)
    images = torch.rand(B, V, 3, H, W, device=DEV, generator=g) * 2 - 1
    c2w, fx = synth.orbit_cameras(V, W, H)
    c2w, fx = torch.tensor(c2w[None], device=DEV), torch.tensor(fx[None], device=DEV)
    ray_o = torch.randn(B, V, 3, 1, 1, device=DEV, generator=g).expand(B, V, 3, H, W).contiguous()
    ray_d = F.normalize(torch.randn(B, V, 3, H, W, device=DEV, generator=g), dim=2)
    x_T = torch.randn(B, V - 1, 3, H, W, device=DEV, generator=g)
    noise = torch.randn(3, B, V - 1, 3, H, W, device=DEV, generator=g)
    d = create_diffusion(timestep_respacing="3")
    batch = dict(image=images, image_noisy=x_T, ray_o=ray_o, ray_d=ray_d, c2w=c2w, fxfycxcy=fx)
    model.set_inference_precision("fp8_attention")
    got = [o["sample"] for o in d.p_sample_loop_progressive(model, x_T.shape, batch, noise_fn=lambda i, like: noise[i])]
    assert len(got) == 3 and all(torch.isfinite(s).all() for s in got)
