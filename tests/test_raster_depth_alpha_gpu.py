"""Depth and alpha maps of the batched sm_90a rasterizer (Renderer.forward_buffers, render_batch_forward(aux=True),
render_batch_backward(grad_depth=, grad_alpha=)):
  * the colour, final_T, n_contrib, loss_sum and colour-only gradients do not change,
  * depth, alpha and the gradients of every map against the CPU oracle (render_buffers_oracle.render_batch_buffers),
  * alpha == 1 - final_T bit for bit, the binning paths agree bit for bit, the view-chunked fallback matches one batch,
  * obj-256 full-size properties.
Tolerances: against the oracle's fp64 build, 1e-4 relative (norm-wise), or if larger twice its fp32 build's own distance from
fp64 or (map gradients) twice the colour-only gradient's distance on the same scene (_oracle_case); 2e-5 for atomics-order
differences between two runs."""
import numpy as np
import pytest
import torch

from test_raster_gpu import DEV, TOL, T, _batch_inputs
from util import rel_l2 as _rel

pytestmark = pytest.mark.gpu
NAMES = ("xyz", "features", "scaling", "rotation", "opacity")


class Cfg:
    gaussians_sh_degree = 0
    use_gssplat = False


def _upstream(B, V, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, V, 3, H, W, generator=g), torch.randn(B, V, 1, H, W, generator=g),
            torch.randn(B, V, 1, H, W, generator=g))


def _grads(outs, leaves, ups):
    """Gradients of sum <output, upstream>; an input the outputs do not depend on (features, for depth and alpha) -> 0."""
    loss = sum((o * u.to(o.device)).sum() for o, u in zip(outs, ups) if u is not None)
    g = torch.autograd.grad(loss, leaves, retain_graph=True, allow_unused=True)
    return [torch.zeros_like(x) if d is None else d for d, x in zip(g, leaves)]


def test_colour_final_T_n_contrib_loss_unchanged():
    from dgs_b200 import raster
    from dgs_b200.renderer import Renderer
    B, V, P, W, H = 2, 3, 1500, 64, 48
    raw, c2w, fx = _batch_inputs(B, V, P, W, H)
    gr, gd, ga = _upstream(B, V, H, W, 11)
    lv1 = [T(raw[k]).requires_grad_() for k in NAMES]
    lv2 = [T(raw[k]).requires_grad_() for k in NAMES]
    r = Renderer(Cfg())
    img = r(*lv1, H, W, T(c2w), T(fx))
    buf = r.forward_buffers(*lv2, H, W, T(c2w), T(fx))
    assert set(buf) == {"render", "depth", "alpha"} and buf["depth"].shape == buf["alpha"].shape == (B, V, 1, H, W)
    assert torch.equal(img, buf["render"])
    img.backward(gr.to(DEV))
    buf["render"].backward(gr.to(DEV))  # no gradient reaches depth / alpha: the plain backward
    for k, a, b in zip(NAMES, lv1, lv2):
        assert _rel(b.grad, a.grad) < 2e-5, k
    t = [T(raw[k]) for k in NAMES]
    i1, s1 = raster.render_batch_forward(*t, H, W, T(c2w), T(fx))
    i2, d2, a2, s2 = raster.render_batch_forward(*t, H, W, T(c2w), T(fx), aux=True)
    assert torch.equal(i1, i2) and s1["R"] == s2["R"] and s1["chunks"] == s2["chunks"]
    e1 = raster.export_state(B * V, P, W, H, 0, s1["geom"], s1["binning"], s1["img"])
    e2 = raster.export_state(B * V, P, W, H, 0, s2["geom"], s2["binning"], s2["img"])
    assert torch.equal(e1["final_T"], e2["final_T"]) and torch.equal(e1["n_contrib"], e2["n_contrib"])
    assert torch.equal(a2.reshape(-1), 1.0 - e2["final_T"])
    # fused MSE together with the maps: loss_sum bitwise equal to the MSE alone
    target = torch.rand(B, V, 3, H, W, device=DEV, generator=torch.Generator(DEV).manual_seed(2))
    l1, l2 = (torch.zeros(B, dtype=torch.float64, device=DEV) for _ in range(2))
    i3, _ = raster.render_batch_forward(*t, H, W, T(c2w), T(fx), mse_target=target, mse_loss_sum=l1)
    i4, d4, a4, s4 = raster.render_batch_forward(*t, H, W, T(c2w), T(fx), mse_target=target, mse_loss_sum=l2, aux=True)
    assert torch.equal(l1, l2) and torch.equal(i3, i4) and torch.equal(d4, d2) and torch.equal(a4, a2)
    coef = torch.full((B,), 1e-3, device=DEV)
    g_m = raster.render_batch_backward(s4, None, mse_coef=coef, grad_depth=gd.to(DEV), grad_alpha=ga.to(DEV))
    g_a = raster.render_batch_backward(s4, None, grad_depth=gd.to(DEV), grad_alpha=ga.to(DEV))
    g_c = raster.render_batch_backward(s4, None, mse_coef=coef)
    for a, b, c in zip(g_m, g_a, g_c):  # linear in the upstream gradient: MSE + aux = MSE alone + aux alone
        assert _rel(b + c, a) < 2e-5


def _oracle(raw, c2w, fx, H, W, upstreams, f64):
    """render_batch_buffers' maps and, per upstream set, its five gradients, from the oracle's fp32 or fp64 build."""
    from oracle import raster as orc
    from render_buffers_oracle import render_batch_buffers
    orc.set_f64(f64)
    try:
        cpu = [torch.tensor(raw[k], requires_grad=True) for k in NAMES]
        maps = render_batch_buffers(*cpu, H, W, torch.tensor(c2w), torch.tensor(fx))
        return [m.detach() for m in maps], {tag: _grads(maps, cpu, ups) for tag, ups in upstreams}
    finally:
        orc.set_f64(False)


def _oracle_case(B, V, P, W, H, dist):
    """Maps and gradients against the oracle's fp64 build, within max(1e-4, 2 x the oracle's own fp32 noise) -- the
    noise-floor rule of test_raster_gpu.check_grads: on the 10,000-Gaussian C1 scenes the fp32 oracle is itself up to ~5e-4
    (norm-wise) from fp64 in some gradients (cancellation in the blend's accumulators when a pixel's opacity nears 1).
    Every quantity is reported before the failures are raised."""
    from dgs_b200.renderer import Renderer
    raw, c2w, fx = _batch_inputs(B, V, P, W, H, dist=dist)
    gr, gd, ga = _upstream(B, V, H, W, 7)
    upstreams = (("render", (gr, None, None)), ("all", (gr, gd, ga)), ("depth", (None, gd, None)),
                 ("alpha", (None, None, ga)))
    ref64, g64 = _oracle(raw, c2w, fx, H, W, upstreams, True)
    ref32, g32 = _oracle(raw, c2w, fx, H, W, upstreams, False)
    gpu = [T(raw[k]).requires_grad_() for k in NAMES]

    def render():  # the forward's arenas serve one backward: a fresh forward per upstream gradient
        buf = Renderer(Cfg()).forward_buffers(*gpu, H, W, T(c2w), T(fx))
        return buf["render"], buf["depth"], buf["alpha"]
    assert float(ref64[2].max()) > 0.1  # something was blended
    bad = []

    def check(tag, ours, exact, fp32, colour_err=0.0):
        floor = _rel(fp32, exact)
        e, tol = _rel(ours, exact), max(TOL, 2.0 * floor, 2.0 * colour_err)
        print(f"  [{dist}] {tag}: rel_l2={e:.3e} (fp32 oracle {floor:.3e}, colour-only {colour_err:.3e}, tol {tol:.1e})")
        if not e < tol:
            bad.append((tag, e, tol))
    for name, a, b, c in zip(("render", "depth", "alpha"), render(), ref64, ref32):
        check(name, a, b, c)
    # The colour-only gradients come from the plain kernels (test_colour_final_T_n_contrib_loss_unchanged: equal to the
    # plain render's).  Their distance from fp64 is this renderer's fp32 noise on the scene -- on the 10,000-Gaussian
    # "fine" scene up to ~3e-4 in dL/dscaling -- and the map gradients may be as far, no farther than twice that.
    colour = [_rel(a, b) for a, b in zip(_grads(render(), gpu, upstreams[0][1]), g64["render"])]
    print(f"  [{dist}] render/d*: rel_l2 {' '.join(f'{e:.3e}' for e in colour)} (the plain colour path; not asserted here)")
    for tag, ups in upstreams[1:]:
        for k, a, b, c, ce in zip(NAMES, _grads(render(), gpu, ups), g64[tag], g32[tag], colour):
            check(f"{tag}/d{k}", a, b, c, ce)
    assert not bad, (dist, bad)


def test_batched_depth_alpha_vs_oracle():
    _oracle_case(2, 3, 1500, 64, 48, "trained")


@pytest.mark.parametrize("dist", ["trained", "init", "fine"])
def test_c1_distributions_depth_alpha_vs_oracle(dist):
    _oracle_case(1, 2, 10000, 256, 256, dist)  # the scene size of the single-view C1 tests


def test_crowded_depth_alpha_vs_oracle():
    """Tile lists longer than the small-scene sort takes: the small path counts, then falls back to the global one."""
    from dgs_b200 import _lib, raster
    L = _lib.lib()
    raw, c2w, fx = _batch_inputs(1, 2, 10000, 48, 48, dist="init")
    L.dgs_profile_enable(1)
    _lib.profile_read()
    raster.render_batch_forward(*[T(raw[k]) for k in NAMES], 48, 48, T(c2w), T(fx), aux=True)
    spans = _lib.profile_read()
    L.dgs_profile_enable(0)
    assert spans["raster.scan"][1] >= 2 and spans["raster.tile_ranges"][1] >= 1, spans
    _oracle_case(1, 2, 10000, 48, 48, "init")


def _aux_run(t, c2w, fx, H, W, near_log2, ups):
    from dgs_b200 import raster
    img, depth, alpha, st = raster.render_batch_forward(*t, H, W, c2w, fx, near_log2=near_log2, aux=True)
    g = raster.render_batch_backward(st, ups[0], grad_depth=ups[1], grad_alpha=ups[2])
    return img, depth, alpha, st, g


@pytest.mark.parametrize("dist,P", [("init", 2 + 4 * 256 * 256), ("fine", 400000)])
def test_binning_paths_agree(dist, P):
    """Single pass, two-phase (phase A's partial depth continued by phase B) and adaptive binning: the same maps bit for
    bit, the aux gradients equal up to atomics order."""
    B, V, W, H = 1, 4, 256, 256
    raw, c2w, fx = _batch_inputs(B, V, P, W, H, dist=dist)
    t = [T(raw[k]) for k in NAMES]
    ups = [u.to(DEV) for u in _upstream(B, V, H, W, 3)]
    base = _aux_run(t, T(c2w), T(fx), H, W, 0, (None, ups[1], ups[2]))
    for near in (3, -1):
        other = _aux_run(t, T(c2w), T(fx), H, W, near, (None, ups[1], ups[2]))
        print(f"[{dist}] near_log2={near} chunks={other[3]['chunks']}")
        if near == 3:
            assert other[3]["chunks"][0] < base[3]["R"] // 2
            assert (other[3]["chunks"][1] > 0) == (dist == "fine")
        assert torch.equal(base[0], other[0]) and torch.equal(base[1], other[1]) and torch.equal(base[2], other[2])
        for a, b in zip(base[4], other[4]):
            assert _rel(b, a) < 2e-5


def test_view_chunked_depth_alpha_equal_single_batch(monkeypatch):
    from dgs_b200 import raster
    from dgs_b200._lib import DgsError
    from dgs_b200.renderer import Renderer
    B, V, P, W, H = 2, 5, 1200, 64, 48
    raw, c2w, fx = _batch_inputs(B, V, P, W, H)
    ups = _upstream(B, V, H, W, 5)

    def run():
        g = [T(raw[k]).requires_grad_() for k in NAMES]
        buf = Renderer(Cfg()).forward_buffers(*g, H, W, T(c2w), T(fx))
        outs = (buf["render"], buf["depth"], buf["alpha"])
        return [o.detach() for o in outs], _grads(outs, g, ups)
    maps1, grads1 = run()
    real = raster._render_batch_forward_one
    calls = []

    def overflowing(xyz, features, scaling, rotation, opacity, Hh, Ww, C2W, fxf, *a, **k):
        calls.append(C2W.shape[1])
        if C2W.shape[1] > 2:
            raise DgsError("libdgs_b200 status 4: instance count 3000000000 exceeds 2^31-1 (render the views in smaller batches)")
        return real(xyz, features, scaling, rotation, opacity, Hh, Ww, C2W, fxf, *a, **k)
    monkeypatch.setattr(raster, "_render_batch_forward_one", overflowing)
    maps2, grads2 = run()
    assert calls == [5, 2, 3, 1, 2]
    for a, b in zip(maps1, maps2):
        assert torch.equal(a, b)
    for k, a, b in zip(NAMES, grads1, grads2):
        assert _rel(b, a) < 1e-5, k


def test_full_size_properties_obj256():
    """B=1, V=4, 256^2, 262,146 init-like Gaussians: finite maps, 0 <= alpha < 1, 0.2 alpha <= depth <= max_z alpha
    (every blended Gaussian lies beyond the 0.2 near plane), gradients linear in the upstream gradient."""
    from dgs_b200 import raster
    B, V, P, W, H = 1, 4, 2 + 4 * 256 * 256, 256, 256
    raw, c2w, fx = _batch_inputs(B, V, P, W, H, dist="init")
    t = [T(raw[k]) for k in NAMES]
    img, depth, alpha, st = raster.render_batch_forward(*t, H, W, T(c2w), T(fx), aux=True)
    assert bool(torch.isfinite(depth).all() and torch.isfinite(alpha).all())
    assert float(alpha.min()) >= 0.0 and float(alpha.max()) < 1.0
    ex = raster.export_state(B * V, P, W, H, 0, st["geom"], st["binning"], st["img"])
    max_z = float(ex["depth"].max())
    eps = 1e-5 * max_z
    assert bool((depth >= 0.2 * alpha - eps).all()) and bool((depth <= max_z * alpha + eps).all())
    ups = [u.to(DEV) for u in _upstream(B, V, H, W, 9)]
    d1 = raster.render_batch_backward(st, ups[0], grad_depth=ups[1], grad_alpha=ups[2])
    d2 = raster.render_batch_backward(st, 2.0 * ups[0], grad_depth=2.0 * ups[1], grad_alpha=2.0 * ups[2])
    for a, b in zip(d1, d2):
        assert bool(torch.isfinite(a).all())
        assert _rel(b, 2.0 * a) < 1e-5
    print(f"obj-256: R={st['R']} alpha mean={float(alpha.mean()):.3f} depth/alpha max={float((depth / alpha.clamp_min(1e-6)).max()):.3f}")
