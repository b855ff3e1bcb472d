"""SSIM and PSNR on the H100 (dgs_b200.ssim over dgs_ssim_forward / dgs_ssim_backward, and dgs_b200.metrics) against the
fp64 reference (oracle/ssim.py) and against pytorch_msssim's own fp32 arithmetic on F.conv2d (TF32 off).

Inputs are renderings of a synthetic Gaussian scene on a white background (the targets), paired with
  * "independent": a rendering of another scene from the same cameras,
  * "noise": the target plus structured noise on the object only,
  * "flat": both renderings of "independent" made piecewise constant over 16 x 16 blocks, so sigma = 0 over whole
    windows,
  * "smooth": a low-contrast, blurred version of the target and a smooth perturbation of it of amplitude ~0.02, so that
    sigma^2 ~ C2 and skimage's sample covariance (k = 121/120) moves SSIM by ~3e-4,
  * "overshoot": the target plus a smooth perturbation and a horizontal ramp from -1.05 to 1.05, not clamped, so every
    rendering leaves [0, 1] on both sides (as an unclamped network output does) and PSNR's clamp to [0, 1] changes every
    image's value.

Bounds: worst of seeds 0-2 over every shape and kind, measured on an H100 80GB HBM3 (see the constants).  SSIM and PSNR
are compared as absolute errors per image; d x as relative L2 over the batch.  The floor is fp32 cancellation in
E[x^2] - mx^2, which the reference's fp32 arithmetic shares."""
import functools
import json
import math
import types

import pytest
import torch
import torch.nn.functional as F

from oracle.ssim import SAMPLE_COV, psnr64, ssim64, ssim_scipy32, ssim_torch32

pytestmark = pytest.mark.gpu
DEV = "cuda"

# Worst of seeds 0-2 over every shape, n (1, 3, 40) and kind on an H100 80GB HBM3 (400 W power limit), with margin.
# At 11 x 11 each channel has one valid pixel, so nothing averages the per-pixel fp32 floor; it has bounds of its own.
SSIM_F64 = 3e-5             # |ssim - fp64|, both variants: measured 1.60e-5 (37x61 "smooth"); "overshoot" 1.1e-6
SSIM_F64_ONE_PIXEL = 3e-4   # the same at 11 x 11: measured 1.47e-4 ("flat", sigma = 0 at a white pixel)
SSIM_T32 = 3e-5             # |ssim - pytorch_msssim's fp32 arithmetic|, both variants: measured 1.60e-5
SSIM_T32_ONE_PIXEL = 2e-4   # the same at 11 x 11: measured 9.0e-5
PSNR_F64 = 1e-5             # dB, |psnr - fp64|: measured 2.35e-6; "overshoot" (the clamp at work) 7.3e-7
GRAD_F64 = 6e-4             # relative L2 of d x over the batch against fp64 autograd: measured 2.69e-4 (11x11 "flat");
                            # 5.1e-5 at 37x61 and up
SCIPY_F32 = 5e-6            # |MetricComputer ssim - skimage's float32 scipy path|: measured 1.48e-6 (512x512 "flat")
GRAD_E2E = 2e-5             # Gaussian-parameter gradients of the training loss, native SsimLoss against the fp32 torch
                            # module: measured 3.5e-6

SIZES = [(11, 11), (37, 61), (64, 96), (256, 256), (512, 512)]
KINDS = ["independent", "noise", "flat", "smooth", "overshoot"]
N_MAX = 40


def _render(seed, n, H, W):
    from dgs_b200 import synth
    from dgs_b200.renderer import Renderer

    class Cfg:
        gaussians_sh_degree = 0
        use_gssplat = False
    g = synth.make_gaussians(4000, seed, "trained")
    c2w, fx = synth.orbit_cameras(n, W, H)
    t = [torch.tensor(g[k][None], device=DEV) for k in ("xyz", "features", "scaling", "rotation", "opacity")]
    with torch.no_grad():
        img = Renderer(Cfg())(*t, H, W, torch.tensor(c2w[None], device=DEV), torch.tensor(fx[None], device=DEV))
    return img[0].clamp(0, 1)


def _blocks(x, b=16):
    """piecewise constant over b x b blocks (the block's top-left value)"""
    H, W = x.shape[-2:]
    return x[..., ::b, ::b].repeat_interleave(b, -2).repeat_interleave(b, -1)[..., :H, :W].contiguous()


def _low(n, H, W, gen, div=8):
    return F.interpolate(torch.randn(n, 3, max(2, H // div), max(2, W // div), device=DEV, generator=gen), size=(H, W),
                         mode="bilinear")


@functools.lru_cache(maxsize=6)
def make_pair(kind, H, W, seed):
    """-> (x = the rendering, y = the target), both [N_MAX, 3, H, W] fp32; in [0, 1] except the "overshoot" rendering."""
    n = N_MAX
    target = _render(seed, n, H, W)
    gen = torch.Generator(DEV).manual_seed(seed)
    if kind in ("independent", "flat"):
        other = _render(seed + 100, n, H, W)
        if kind == "flat":
            target, other = _blocks(target), _blocks(other)
    elif kind == "noise":
        yy, xx = torch.meshgrid(torch.arange(H, device=DEV), torch.arange(W, device=DEV), indexing="ij")
        stripes = torch.sin(0.7 * xx + 0.3 * yy)[None, None]
        obj = (target < 0.995).any(dim=1, keepdim=True)
        other = (target + (0.05 * _low(n, H, W, gen) + 0.02 * stripes) * obj).clamp(0, 1)
    elif kind == "overshoot":  # the ramp takes every image's first column below 0 and its last column above 1
        ramp = 1.05 * (2 * torch.arange(W, device=DEV, dtype=torch.float32) / (W - 1) - 1)
        other = target + 0.2 * _low(n, H, W, gen, div=4) * (ramp.abs() < 1) + ramp
    else:  # smooth
        blur = lambda t: F.avg_pool2d(F.avg_pool2d(t, 5, 1, 2, count_include_pad=False), 5, 1, 2,  # noqa: E731
                                      count_include_pad=False)
        target = 0.5 + 0.1 * (blur(target) - 0.5)
        other = target + 0.02 * _low(n, H, W, gen, div=6)
    return other.contiguous(), target.contiguous()


def _rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def _native_train(x, y, dout, data_range=1.0):
    from dgs_b200.ssim import SSIM
    xg = x.clone().requires_grad_(True)
    out = SSIM(data_range=data_range)(xg, y)
    out.backward(dout)
    torch.cuda.synchronize()
    return out.detach(), xg.grad


def _fp64(x, y, dout):
    xg = x.double().clone().requires_grad_(True)
    v = ssim64(xg, y.double(), k=1.0)
    (v * dout.double()).sum().backward()
    return v.detach(), xg.grad


@pytest.fixture(autouse=True)
def _no_tf32():
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = prev


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", [1, 3, 40])
@pytest.mark.parametrize("HW", SIZES, ids=lambda s: "x".join(map(str, s)))
def test_against_references(HW, n, kind, seed):
    from dgs_b200.ssim import ssim_psnr
    H, W = HW
    x, y = (t[:n] for t in make_pair(kind, H, W, seed))
    dout = torch.rand(n, device=DEV, generator=torch.Generator(DEV).manual_seed(seed)) + 0.5
    loss_v, grad = _native_train(x, y, dout)
    met_v, psnr = ssim_psnr(x, y, sample_covariance=True, psnr=True)
    ref_v, ref_g = _fp64(x, y, dout)
    with torch.no_grad():
        ref_met = ssim64(x, y, k=SAMPLE_COV)
        ref_psnr = psnr64(x, y)
        t32 = ssim_torch32(x, y)
        t32_met = ssim_torch32(x, y, k=SAMPLE_COV)
    e = dict(loss=float((loss_v.double() - ref_v).abs().max()), metric=float((met_v.double() - ref_met).abs().max()),
             loss_t32=float((loss_v - t32).abs().max()), metric_t32=float((met_v - t32_met).abs().max()),
             psnr=float((psnr.double() - ref_psnr).abs().max()), grad=_rel_l2(grad, ref_g))
    print(f"\n[ssim-err] {kind} n={n} {H}x{W} seed={seed}: ssim={[round(float(v), 5) for v in loss_v[:3]]} "
          f"k-shift={float((ref_met - ref_v).abs().max()):.2e} psnr={[round(float(v), 3) for v in psnr[:3]]} "
          + " ".join(f"{k}={v:.2e}" for k, v in e.items()))
    one_pixel = (H, W) == (11, 11)
    bound_f64, bound_t32 = (SSIM_F64_ONE_PIXEL, SSIM_T32_ONE_PIXEL) if one_pixel else (SSIM_F64, SSIM_T32)
    assert e["loss"] < bound_f64 and e["metric"] < bound_f64
    assert e["loss_t32"] < bound_t32 and e["metric_t32"] < bound_t32
    assert e["psnr"] < PSNR_F64
    assert e["grad"] < GRAD_F64
    if kind == "smooth" and not one_pixel:  # the sample covariance is visible (~3e-4) well above the bound
        assert float((ref_met - ref_v).abs().min()) > 5 * SSIM_F64
    if kind == "overshoot":  # every image leaves [0, 1], and the clamp moves every PSNR far above the bound
        assert bool(((x < 0).flatten(1).any(1) & (x > 1).flatten(1).any(1)).all())
        assert float((psnr64(x, y, ("psnr_unclamped",)) - ref_psnr).abs().min()) > 100 * PSNR_F64


@pytest.mark.parametrize("HW", SIZES, ids=lambda s: "x".join(map(str, s)))
def test_batch_size_and_training_state_do_not_change_bits(HW):
    """n = 40, n = 3 and n = 1 give the same bits per image; so do inference and training forwards."""
    from dgs_b200.ssim import SSIM, ssim_psnr
    H, W = HW
    x, y = make_pair("noise", H, W, 1)
    dout = torch.rand(N_MAX, device=DEV, generator=torch.Generator(DEV).manual_seed(5)) + 0.5
    big_v, big_g = _native_train(x, y, dout)
    for sl in (slice(0, 3), slice(7, 8)):
        v, g = _native_train(x[sl], y[sl], dout[sl])
        assert torch.equal(v, big_v[sl]) and torch.equal(g, big_g[sl])
    with torch.no_grad():
        inf = SSIM()(x, y)
    assert torch.equal(inf, big_v)
    s_all, p_all = ssim_psnr(x, y)
    s1, p1 = ssim_psnr(x[7:8], y[7:8])
    assert torch.equal(s1, s_all[7:8]) and torch.equal(p1, p_all[7:8])
    s_np, none = ssim_psnr(x, y, psnr=False)
    assert none is None and torch.equal(s_np, s_all)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float64])
def test_other_input_dtypes_are_read_as_fp32(dtype):
    x, y = make_pair("independent", 64, 96, 0)
    x, y = x[:3].to(dtype), y[:3].to(dtype)
    dout = torch.ones(3, device=DEV)
    v, g = _native_train(x, y, dout)
    v32, g32 = _native_train(x.float(), y.float(), dout)
    assert v.dtype == torch.float32 and g.dtype == dtype
    assert torch.equal(v, v32) and torch.equal(g, g32.to(dtype))


@pytest.mark.parametrize("HW", [(11, 11), (64, 96), (256, 256)], ids=lambda s: "x".join(map(str, s)))
def test_identical_inputs(HW):
    from dgs_b200.ssim import ssim_psnr
    _, y = make_pair("independent", *HW, 0)
    y = y[:3]
    v, _ = _native_train(y.clone(), y, torch.ones(3, device=DEV))
    s, p = ssim_psnr(y.clone(), y)
    assert bool(torch.isinf(p).all()) and bool((p > 0).all())
    assert float((v - 1).abs().max()) < 1e-6 and float((s - 1).abs().max()) < 1e-6


def test_data_range():
    """data_range R only sets C1 = (0.01 R)^2 and C2 = (0.03 R)^2: images scaled by R give the value at R = 1."""
    x, y = (t[:3] for t in make_pair("smooth", 64, 96, 0))
    dout = torch.ones(3, device=DEV)
    v255, _ = _native_train(x * 255, y * 255, dout, data_range=255.0)
    ref = ssim64(x * 255, y * 255, data_range=255.0)
    assert float((v255.double() - ref).abs().max()) < SSIM_F64


class _TorchSsimLoss(torch.nn.Module):
    """1 - pytorch_msssim's fp32 arithmetic: the reference's SsimLoss on torch ops."""

    def forward(self, x, y):
        return 1 - ssim_torch32(x, y)


def test_training_loss_end_to_end():
    """fused_render_and_loss with lambda_ssim = 0.5: Gaussian-parameter gradients with the native SsimLoss match the same
    call with the fp32 torch module in its place."""
    from dgs_b200 import losses, synth
    from dgs_b200.renderer import Renderer
    from dgs_b200.ssim import SsimLoss

    class Cfg:
        gaussians_sh_degree = 0
        use_gssplat = False
    B, V, H, W = 2, 3, 64, 64
    target = torch.stack([_render(7, V, H, W), _render(8, V, H, W)])
    g = synth.make_gaussians(3000, 3, "trained")
    c2w, fx = synth.orbit_cameras(V, W, H)
    c2w = torch.tensor(c2w[None], device=DEV).expand(B, -1, -1, -1).contiguous()
    fx = torch.tensor(fx[None], device=DEV).expand(B, -1, -1).contiguous()
    model = types.SimpleNamespace(gs_renderer=Renderer(Cfg()))
    lambdas = dict(lambda_diffusion=1.0, lambda_ssim=0.5)
    grads, values = [], []
    for module in (SsimLoss(), _TorchSsimLoss()):
        leaves = [torch.tensor(g[k][None], device=DEV).expand(B, *g[k].shape).contiguous().requires_grad_(True)
                  for k in ("xyz", "features", "scaling", "rotation", "opacity")]
        gs = types.SimpleNamespace(**dict(zip(("xyz", "features", "scaling", "rotation", "opacity"), leaves)))
        lc = losses.LossComputer(ssim_module=module)
        res, _ = losses.fused_render_and_loss(model, gs, c2w, fx, H, W, target, loss_computer=lc, lambdas=lambdas)
        res["loss"].backward()
        values.append((float(res["loss"]), float(res["loss_ssim"])))
        grads.append([p.grad.clone() for p in leaves])
    e = max(_rel_l2(a, b) for a, b in zip(*grads))
    print(f"\n[ssim-err] e2e loss (native, torch) = {values}; worst Gaussian-gradient rel L2 = {e:.2e}")
    assert values[0][1] > 0.05
    assert abs(values[0][1] - values[1][1]) < SSIM_T32
    assert e < GRAD_E2E


def _lpips_module(seed=0):
    from lpips_regime import random_lpips_state_dict
    from dgs_b200.lpips import LPIPS
    sd = random_lpips_state_dict(seed)
    return LPIPS.from_state_dict(sd).to(DEV), sd


def test_metric_computer_against_references():
    """psnr / ssim / lpips of MetricComputer against psnr64, the fp64 skimage variant, skimage's float32 scipy path and
    the fp32 LPIPS reference module (after the same bilinear resize to 256 x 256)."""
    from oracle.lpips import LPIPSOracle
    from test_lpips_gpu import VALUE_F64 as LPIPS_VALUE_F64
    from dgs_b200.metrics import MetricComputer
    lp, sd = _lpips_module(0)
    mc = MetricComputer(lp)
    ref_lp = LPIPSOracle(sd, dtype=torch.float32)
    for kind, (H, W) in (("independent", (256, 256)), ("noise", (64, 96)), ("flat", (512, 512)),
                         ("overshoot", (37, 61))):
        x, y = make_pair(kind, H, W, 0)
        r, t = x[:6].view(2, 3, 3, H, W), y[:6].view(2, 3, 3, H, W)   # [scenes, views, 3, H, W]
        psnr, ssim, lpips = mc(t, r)
        assert psnr.shape == ssim.shape == lpips.shape == (6,)
        rf, tf = r.reshape(6, 3, H, W), t.reshape(6, 3, H, W)
        e_psnr = float((psnr.double() - psnr64(tf, rf)).abs().max())
        e_ssim = float((ssim.double() - ssim64(tf, rf, k=SAMPLE_COV)).abs().max())
        e_sc = float((ssim.double().cpu() - torch.tensor(ssim_scipy32(tf.cpu(), rf.cpu()))).abs().max())
        with torch.no_grad():
            up = lambda v: F.interpolate(v, size=[256, 256], mode="bilinear") * 2.0 - 1.0  # noqa: E731
            ref_l = ref_lp(up(rf), up(tf)).reshape(-1)
        e_lp = float(((lpips - ref_l) / ref_l).abs().max())
        print(f"\n[ssim-err] metrics {kind} {H}x{W}: psnr {e_psnr:.2e} ssim {e_ssim:.2e} scipy32 {e_sc:.2e} "
              f"lpips {e_lp:.2e}")
        assert e_psnr < PSNR_F64 and e_ssim < SSIM_F64 and e_sc < SCIPY_F32 and e_lp < LPIPS_VALUE_F64
        one = mc.compute_lpips(tf[:1], rf[:1])
        assert one.shape == (1,) and torch.equal(one, lpips[:1])
        assert torch.equal(mc.compute_ssim(tf, rf), ssim) and torch.equal(mc.compute_psnr(tf, rf), psnr)


def test_compute_metrics_on_a_results_directory(tmp_path):
    """5 scenes x 4 views written as the reference's evaluation writes them: chunk 2 and chunk 8 give the same JSON, and
    the values are MetricComputer's over all 20 images."""
    from dgs_b200.metrics import MetricComputer, compute_metrics
    H, W = 64, 96
    x, y = make_pair("noise", H, W, 2)
    for i in range(5):
        torch.save({"render_images": x[4 * i:4 * i + 4].cpu(), "image": y[4 * i:4 * i + 4].cpu()},
                   tmp_path / f"{i:04d}.pt")
    lp, _ = _lpips_module(1)
    mc = MetricComputer(lp)
    texts = []
    for chunk in (2, 8):
        compute_metrics(str(tmp_path), chunk=chunk, metric_computer=mc)
        texts.append((tmp_path / "eval_result.json").read_text())
    assert texts[0] == texts[1]
    res = json.loads(texts[0])
    psnr, ssim, lpips = mc(x[:20], y[:20])
    assert math.isclose(res["psnr"], float(psnr.mean()), rel_tol=1e-6)
    assert math.isclose(res["ssim"], float(ssim.mean()), rel_tol=1e-6)
    assert math.isclose(res["lpips"], float(lpips.mean()), rel_tol=1e-6)
