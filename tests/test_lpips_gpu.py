"""LPIPS-VGG on the H100 (dgs_b200.lpips.LPIPS over dgs_lpips_forward / dgs_lpips_backward) against the fp64 reference
(oracle/lpips.py), with He-scaled random VGG weights, non-zero biases and non-negative lin weights (tests/lpips_regime.py).

Inputs are renderings of a synthetic Gaussian scene on a white background (the targets), paired with
  * "independent": a rendering of another scene from the same cameras (LPIPS ~0.3-0.6), or
  * "noise": the target plus smooth structured noise on the object only (LPIPS ~0.02-0.1, the late-training regime),
  * "flat": both renderings of "independent" averaged over 16 x 16 blocks (piecewise constant; LPIPS ~0.08-0.3), so that
    inside each block every max-pool window holds four exactly equal activations and the tie rule decides where the
    gradient goes,
so every kind contains white regions where the two inputs are identical.

Bounds (seeds 0-2, every shape, measured on an H100 80GB HBM3; see the constants below): per-image relative error of the
value; relative L2 of d in0 over the batch, in full and after averaging over 8 x 8 pixel blocks.  The full gradient is
dominated by bf16 rounding flips: where two activations of a max-pool window lie within one bf16 step, or a
pre-activation near 0 rounds to the other side, the gradient takes another path.  The rounding-matched reference itself
differs from plain fp64 by ~25 % in full; the block means, which a systematic error (a wrong kernel flip, tap or
normalisation) moves but scattered routing flips do not, agree far more closely."""
import types

import pytest
import torch
import torch.nn.functional as F

from lpips_regime import random_lpips_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"

# Worst of seeds 0-2 over every shape and both kinds of pair on an H100 80GB HBM3 (700 W power limit), with margin.
# against the rounding-matched fp64 reference
VALUE_MATCHED = 2e-3        # measured 1.4e-3 (a "noise" pair, LPIPS ~0.02, among 40); 3.8e-4 flat, 2.1e-4 independent
GRAD_MATCHED = 0.15         # measured 0.104
GRAD_BLOCK_MATCHED = 0.05   # measured 3.2e-2
# against plain fp64
VALUE_F64 = 5e-3            # measured 3.5e-3
GRAD_F64 = 0.4              # measured 0.27
GRAD_BLOCK_F64 = 0.1        # measured 6.0e-2
# Gaussian-parameter gradients of the training loss, native module against the fp32 reference module
GRAD_E2E = 0.08             # measured 4.2e-2


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


def make_pair(kind, n, H, W, seed):
    """-> (in0 = the rendering, in1 = the target), both [n, 3, H, W] in [-1, 1]."""
    target = _render(seed, n, H, W)
    if kind in ("independent", "flat"):
        other = _render(seed + 100, n, H, W)
        if kind == "flat":
            flat = lambda x: F.interpolate(F.avg_pool2d(x, 16), scale_factor=16, mode="nearest")  # noqa: E731
            target, other = flat(target), flat(other)
    else:
        gen = torch.Generator(DEV).manual_seed(seed)
        low = F.interpolate(torch.randn(n, 3, H // 8, W // 8, device=DEV, generator=gen), size=(H, W), mode="bilinear")
        yy, xx = torch.meshgrid(torch.arange(H, device=DEV), torch.arange(W, device=DEV), indexing="ij")
        stripes = torch.sin(0.7 * xx + 0.3 * yy)[None, None]
        obj = (target < 0.995).any(dim=1, keepdim=True)
        other = (target + (0.05 * low + 0.02 * stripes) * obj).clamp(0, 1)
    return other * 2 - 1, target * 2 - 1


def _module(seed, sd=None):
    from dgs_b200.lpips import LPIPS
    return LPIPS.from_state_dict(sd or random_lpips_state_dict(seed)).to(DEV)


def _run(m, in0, in1, dout):
    x = in0.clone().requires_grad_(True)
    out = m(x, in1)
    out.backward(dout.view(-1, 1, 1, 1))
    torch.cuda.synchronize()
    return out.detach().reshape(-1), x.grad


def _oracle(sd, in0, in1, dout, matched):
    from oracle.lpips import lpips64, weights_from_state_dict
    w = weights_from_state_dict(sd)
    w = {k: ([t.to(DEV) for t in v] if isinstance(v, list) else v.to(DEV)) for k, v in w.items()}
    x = in0.double().clone().requires_grad_(True)
    out = lpips64(w, x, in1.double(), matched=matched)
    (out * dout.double()).sum().backward()
    return out.detach(), x.grad


def _rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def block_mean(g, k=8):
    return F.avg_pool2d(g.double(), k)


def grad_errors(g, ref):
    """-> (relative L2 in full, relative L2 of the 8 x 8 block means)"""
    return _rel_l2(g, ref), _rel_l2(block_mean(g), block_mean(ref))


SHAPES = [(1, 256, 256), (3, 256, 256), (1, 64, 96), (3, 64, 96), (40, 64, 96)]


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("kind", ["independent", "noise", "flat"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_against_fp64_reference(shape, kind, seed):
    n, H, W = shape
    sd = random_lpips_state_dict(seed)
    m = _module(seed, sd)
    if n > 3:  # processed in chunks of 3 images
        from dgs_b200 import _lib
        m.max_workspace_bytes = 3 * _lib.lib().dgs_lpips_workspace_bytes(1, H, W) + 4096
    in0, in1 = make_pair(kind, n, H, W, seed)
    dout = torch.rand(n, device=DEV, generator=torch.Generator(DEV).manual_seed(seed)) + 0.5
    val, grad = _run(m, in0, in1, dout)
    res = {}
    for matched in (True, False):
        rv, rg = _oracle(sd, in0, in1, dout, matched)
        res[matched] = (float(((val.double() - rv) / rv).abs().max()),) + grad_errors(grad, rg)
    print(f"\n{kind} n={n} {H}x{W} seed={seed}: lpips={[round(float(v), 4) for v in val[:3]]}  "
          f"matched: value {res[True][0]:.2e} grad {res[True][1]:.2e} block {res[True][2]:.2e}  "
          f"fp64: value {res[False][0]:.2e} grad {res[False][1]:.2e} block {res[False][2]:.2e}")
    lo, hi = dict(independent=(0.3, 0.6), noise=(0.02, 0.1), flat=(0.08, 0.3))[kind]
    assert lo / 2 < float(val.mean()) < hi * 2  # the regime the bounds were measured in
    assert res[True][0] < VALUE_MATCHED and res[True][1] < GRAD_MATCHED and res[True][2] < GRAD_BLOCK_MATCHED
    assert res[False][0] < VALUE_F64 and res[False][1] < GRAD_F64 and res[False][2] < GRAD_BLOCK_F64


@pytest.mark.parametrize("shape", [(3, 256, 256), (2, 64, 96)], ids=lambda s: "x".join(map(str, s)))
def test_identical_inputs_give_exact_zero(shape):
    n, H, W = shape
    m = _module(0)
    _, target = make_pair("noise", n, H, W, 0)
    val, grad = _run(m, target.clone(), target, torch.ones(n, device=DEV))
    assert torch.equal(val, torch.zeros_like(val))
    assert torch.equal(grad, torch.zeros_like(grad))


@pytest.mark.parametrize("shape", [(3, 256, 256), (3, 64, 96)], ids=lambda s: "x".join(map(str, s)))
def test_inference_and_training_forward_agree_bitwise(shape):
    n, H, W = shape
    m = _module(1)
    in0, in1 = make_pair("independent", n, H, W, 1)
    with torch.no_grad():
        inf = m(in0, in1).reshape(-1)
    train, _ = _run(m, in0, in1, torch.ones(n, device=DEV))
    assert torch.equal(inf, train)


@pytest.mark.parametrize("HW", [(256, 256), (64, 96)], ids=lambda s: "x".join(map(str, s)))
def test_results_do_not_depend_on_batch_or_chunk(HW):
    """n = 40 in chunks of 3 (a workspace for 3 images) and in one chunk, n = 3 and n = 1: the same bits."""
    from dgs_b200 import _lib
    H, W = HW
    n = 40
    m = _module(2)
    in0, in1 = make_pair("noise", n, H, W, 2)
    dout = torch.rand(n, device=DEV, generator=torch.Generator(DEV).manual_seed(5)) + 0.5
    m.max_workspace_bytes = 1 << 40
    big_v, big_g = _run(m, in0, in1, dout)
    m.max_workspace_bytes = 3 * _lib.lib().dgs_lpips_workspace_bytes(1, H, W) + 4096
    assert m.workspace(n, H, W, DEV).numel() < _lib.lib().dgs_lpips_workspace_bytes(4, H, W)
    small_v, small_g = _run(m, in0, in1, dout)
    assert torch.equal(big_v, small_v) and torch.equal(big_g, small_g)
    m.max_workspace_bytes = 1 << 40
    v3, g3 = _run(m, in0[:3], in1[:3], dout[:3])
    v1, g1 = _run(m, in0[7:8], in1[7:8], dout[7:8])
    assert torch.equal(v3, big_v[:3]) and torch.equal(g3, big_g[:3])
    assert torch.equal(v1, big_v[7:8]) and torch.equal(g1, big_g[7:8])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float64])
def test_other_input_dtypes_are_read_as_fp32(dtype):
    """fp16 / bf16 / fp64 images give the value of their fp32 conversion, and the gradient comes back in their dtype;
    a module converted with .to(bf16) gives what a module built from the bf16-rounded weights gives."""
    n, H, W = 2, 64, 96
    sd = random_lpips_state_dict(0)
    m = _module(0, sd)
    in0, in1 = make_pair("independent", n, H, W, 0)
    in0, in1 = in0.to(dtype), in1.to(dtype)
    dout = torch.ones(n, device=DEV)
    v, g = _run(m, in0, in1, dout)
    v32, g32 = _run(m, in0.float(), in1.float(), dout)
    assert g.dtype == dtype
    assert torch.equal(v, v32) and torch.equal(g, g32.to(dtype))
    sd16 = {k: t.to(torch.bfloat16).float() for k, t in sd.items()}
    vb, gb = _run(_module(0, sd).to(torch.bfloat16), in0.float(), in1.float(), dout)
    vr, gr = _run(_module(0, sd16), in0.float(), in1.float(), dout)
    assert torch.equal(vb, vr) and torch.equal(gb, gr)


def test_training_loss_end_to_end():
    """fused_render_and_loss with lambda_lpips = 0.5: Gaussian-parameter gradients with the native module match the same
    call with the fp32 reference module in its place."""
    from dgs_b200 import losses, synth
    from dgs_b200.renderer import Renderer
    from oracle.lpips import LPIPSOracle

    class Cfg:
        gaussians_sh_degree = 0
        use_gssplat = False
    B, V, H, W = 1, 3, 64, 64
    sd = random_lpips_state_dict(0)
    target = _render(7, V, H, W)[None]
    g = synth.make_gaussians(3000, 3, "trained")
    c2w, fx = synth.orbit_cameras(V, W, H)
    c2w, fx = torch.tensor(c2w[None], device=DEV), torch.tensor(fx[None], device=DEV)
    model = types.SimpleNamespace(gs_renderer=Renderer(Cfg()))
    lambdas = dict(lambda_diffusion=1.0, lambda_lpips=[150, 0.0, 0.5, 151])
    grads, values = [], []
    for module in (_module(0, sd), LPIPSOracle(sd, dtype=torch.float32)):
        leaves = [torch.tensor(g[k][None], device=DEV, requires_grad=True)
                  for k in ("xyz", "features", "scaling", "rotation", "opacity")]
        gs = types.SimpleNamespace(**dict(zip(("xyz", "features", "scaling", "rotation", "opacity"), leaves)))
        lc = losses.LossComputer(lpips_module=module)
        prev = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = False
        try:
            res, _ = losses.fused_render_and_loss(model, gs, c2w, fx, H, W, target, loss_computer=lc, lambdas=lambdas,
                                                  global_step=200)
            res["loss"].backward()
        finally:
            torch.backends.cudnn.allow_tf32 = prev
        values.append((float(res["loss"]), float(res["loss_lpips"])))
        grads.append([p.grad.clone() for p in leaves])
    e = max(_rel_l2(a, b) for a, b in zip(*grads))
    print(f"\nloss (native, reference) = {values}; worst Gaussian-gradient rel L2 = {e:.2e}")
    assert values[0][1] > 0.05
    assert abs(values[0][1] - values[1][1]) < VALUE_F64 * values[1][1]
    assert e < GRAD_E2E
