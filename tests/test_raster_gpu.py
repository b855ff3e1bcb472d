"""GPU parity tests of the sm_90a rasterizer, all through the C ABI (libdgs_b200.so):
  * vs the CPU oracle (oracle/raster_oracle.c) on seeded C1 scenes,
  * vs stored outputs of the UNMODIFIED reference kernels (tests/golden/c1_ref_*.npz),
  * drop-in package autograd contract, batched renderer, edge cases, full-size properties.
Tolerance: 1e-4 relative (norm-wise) on colour and on every gradient; integer
outputs (radii, num_rendered, sorted lists, n_contrib) bit-exact up to the rare fp32 threshold flips
that FMA contraction differences between compilers can cause (bounded explicitly below)."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from util import max_abs, oracle_forward, rel_l2, scene_c1

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_golden as mg  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = 1e-4
DEV = "cuda:0"


def T(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype, device=DEV)


def ours_forward(sc, sh=None, degree=0, colors=None, cov3d=None):
    from dgs_b200 import raster
    a = sc["act"]
    e = torch.empty(0, device=DEV)
    out = raster.rasterize_gaussians(
        T(np.ones(3)), T(a["means3D"]), e if colors is None else T(colors), T(a["opacities"]),
        e if cov3d is not None else T(a["scales"]), e if cov3d is not None else T(a["rotations"]), 1.0,
        e if cov3d is None else T(cov3d), T(sc["view"]), T(sc["proj"]), sc["tanx"], sc["tany"], sc["H"], sc["W"],
        e if colors is not None else T(a["shs"] if sh is None else sh), degree, T(sc["campos"]), False, False)
    return out


def ours_backward(sc, fwd, dpix, sh=None, degree=0, colors=None, cov3d=None):
    from dgs_b200 import raster
    a = sc["act"]
    e = torch.empty(0, device=DEV)
    R, color, radii, geom, binning, img = fwd
    return raster.rasterize_gaussians_backward(
        T(np.ones(3)), T(a["means3D"]), radii, e if colors is None else T(colors),
        e if cov3d is not None else T(a["scales"]), e if cov3d is not None else T(a["rotations"]), 1.0,
        e if cov3d is None else T(cov3d), T(sc["view"]), T(sc["proj"]), sc["tanx"], sc["tany"], T(dpix),
        e if colors is not None else T(a["shs"] if sh is None else sh), degree, T(sc["campos"]), geom, R, binning,
        img, False)


GRAD_NAMES = ["dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales",
              "dL_drotations"]


def check_grads(ours, ref, tag, skip=(), noise_floor=None):
    """`noise_floor`: optional {name: rel_l2 of the REFERENCE kernels vs the fp64-accumulating oracle} on the same
    inputs -- the fp32 atomics-order / cancellation noise of the specification itself (dL/drotation and dL/dscale are
    differences of nearly equal terms).  We must be within max(1e-4, 2x that floor)."""
    for name, g in zip(GRAD_NAMES, ours):
        if name in skip or ref[name].size == 0:
            continue
        err = rel_l2(g.cpu().numpy(), ref[name])
        tol = TOL if not noise_floor else max(TOL, 2.0 * noise_floor.get(name, 0.0))
        print(f"  [{tag}] {name}: rel_l2={err:.3e} max_abs={max_abs(g.cpu().numpy(), ref[name]):.3e} (tol {tol:.1e})")
        assert err < tol, (tag, name, err)


NOISE_FLOOR_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sh_noise_floor.json")


def reference_noise_floor(key, sc, st, dpix, sh, degree, colors=None, cov3d=None):
    """rel_l2 of the reference kernels' own fp32 gradients vs the oracle: computed live where oracle/_ref is built, else
    the values tests/golden/make_golden.py stored in tests/golden/sh_noise_floor.json."""
    from oracle import build_ref
    ref = build_ref.load_module()
    if ref is None:
        return json.load(open(NOISE_FLOOR_PATH))[key]
    return mg.noise_floor(ref, sc, st, dpix, sh, degree, colors, cov3d, DEV)


@pytest.mark.parametrize("dist", ["trained", "init", "fine", "crowded"])
def test_c1_forward_backward_vs_oracle(dist):
    from oracle import raster as orc
    from dgs_b200 import raster
    # crowded: tile lists longer than the small-scene binning's shared-memory sort takes, so the forward falls back to
    # the global binning after the small path's counting pass
    sc = scene_c1(P=10000, dist="init", W=48, H=48) if dist == "crowded" else scene_c1(P=10000, dist=dist)
    st = oracle_forward(sc)
    fwd = ours_forward(sc)
    R, color, radii, geom, binning, img = fwd
    ex = raster.export_state(1, sc["P"], sc["W"], sc["H"], R, geom, binning, img)
    if dist == "crowded":
        assert int((st["ranges"][:, 1].astype(np.int64) - st["ranges"][:, 0]).max()) > 4096
    n_rad = int((radii.cpu().numpy() != st["radii"]).sum())
    print(f"[{dist}] R ours={R} oracle={st['num_rendered']} radii mismatches={n_rad}")
    assert n_rad <= 2 and abs(R - st["num_rendered"]) <= 64
    assert rel_l2(ex["xy"].cpu().numpy(), st["xy"]) < 1e-6
    assert rel_l2(ex["conic_opacity"].cpu().numpy(), st["conic_opacity"]) < 1e-5
    assert rel_l2(ex["rgb"].cpu().numpy(), st["rgb"]) < 1e-6
    if n_rad == 0:
        assert R == st["num_rendered"]
        assert np.array_equal(ex["point_list"].cpu().numpy().astype(np.uint32), st["point_list"])  # stable order
        assert np.array_equal(ex["ranges"].cpu().numpy().astype(np.uint32), st["ranges"])
        nc = (ex["n_contrib"].cpu().numpy().astype(np.int64) != st["n_contrib"].astype(np.int64)).mean()
        print(f"[{dist}] n_contrib mismatch fraction {nc:.2e}")
        assert nc < 1e-3
    err = rel_l2(color.cpu().numpy(), st["color"])
    print(f"[{dist}] colour rel_l2={err:.3e} max_abs={max_abs(color.cpu().numpy(), st['color']):.3e}")
    assert err < TOL
    dpix = np.random.default_rng(1).normal(0, 1, (3, sc["H"], sc["W"])).astype(np.float32)
    g_ref = orc.rasterize_backward(st, dpix)
    g = ours_backward(sc, fwd, dpix)
    check_grads(g, g_ref, dist)


@pytest.mark.parametrize("dist", ["trained", "init"])
def test_c1_vs_reference_kernels(dist):
    """Three-way agreement: our kernels vs the reference's own kernels, whose outputs on these seeded scenes are stored in
    tests/golden/c1_ref_<dist>.npz (tests/golden/make_golden.py: every radius, a fixed sample of colours and gradients)."""
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"c1_ref_{dist}.npz"))
    sc = scene_c1(P=10000, dist=dist)
    Rr, radii_r, pix, gi = int(z["num_rendered"]), torch.as_tensor(z["radii"], device=DEV), z["pix"], z["gauss"]
    fwd = ours_forward(sc)
    R, color, radii = fwd[0], fwd[1], fwd[2]
    color_s = color.cpu().numpy().reshape(-1)[pix]
    print(f"[{dist}] R ours={R} ref={Rr}; colour rel_l2={rel_l2(color_s, z['color']):.3e}")
    # radius = ceil(3 sqrt(lambda)) may flip by one on an exact-integer boundary (FMA contraction differs between
    # the two compilations); bound it instead of demanding bit equality
    n_bad = int((radii.to(radii_r.dtype) != radii_r).sum())
    assert n_bad <= 2 and int((radii.to(radii_r.dtype) - radii_r).abs().max()) <= 1 and abs(R - Rr) <= 64, (n_bad, R, Rr)
    assert rel_l2(color_s, z["color"]) < TOL
    dpix = np.random.default_rng(1).normal(0, 1, (3, sc["H"], sc["W"])).astype(np.float32)
    g = [t[torch.as_tensor(gi, device=t.device)] if t.numel() else t for t in ours_backward(sc, fwd, dpix)]
    ref_d = {n: (z[n] if n in z.files else np.zeros(0, np.float32)) for n in GRAD_NAMES}
    check_grads(g, ref_d, "ref-" + dist)


def test_sh_degree3_colors_precomp_cov_precomp():
    from oracle import raster as orc
    sc = scene_c1(P=3000, dist="trained", W=160, H=96)
    rng = np.random.default_rng(7)
    dpix = rng.normal(0, 1, (3, sc["H"], sc["W"])).astype(np.float32)
    sh = rng.normal(0, 0.4, (sc["P"], 16, 3)).astype(np.float32)
    for deg in (1, 2, 3):
        st = oracle_forward(sc, sh=sh, degree=deg)
        fwd = ours_forward(sc, sh=sh, degree=deg)
        assert rel_l2(fwd[1].cpu().numpy(), st["color"]) < TOL
        floor = reference_noise_floor(f"sh{deg}", sc, st, dpix, sh, deg)
        print(f"  [sh{deg}] reference-kernel noise floor vs oracle: {floor}")
        check_grads(ours_backward(sc, fwd, dpix, sh=sh, degree=deg), orc.rasterize_backward(st, dpix), f"sh{deg}",
                    noise_floor=floor)
    cols = rng.uniform(0, 1, (sc["P"], 3)).astype(np.float32)
    st = oracle_forward(sc, colors=cols)
    fwd = ours_forward(sc, colors=cols)
    assert rel_l2(fwd[1].cpu().numpy(), st["color"]) < TOL
    check_grads(ours_backward(sc, fwd, dpix, colors=cols), orc.rasterize_backward(st, dpix), "colors_precomp",
                noise_floor=reference_noise_floor("colors_precomp", sc, st, dpix, None, 0, colors=cols))
    cov = oracle_forward(sc)["cov3D"]
    st = oracle_forward(sc, cov3d=cov)
    fwd = ours_forward(sc, cov3d=cov)
    assert rel_l2(fwd[1].cpu().numpy(), st["color"]) < TOL
    check_grads(ours_backward(sc, fwd, dpix, cov3d=cov), orc.rasterize_backward(st, dpix), "cov_precomp",
                skip=("dL_dscales", "dL_drotations"),
                noise_floor=reference_noise_floor("cov_precomp", sc, st, dpix, sc["act"]["shs"], 0, cov3d=cov))


def test_edge_cases_empty_culled_ragged():
    from dgs_b200 import raster
    sc = scene_c1(P=64, W=100, H=70)
    a = sc["act"]
    e = torch.empty(0, device=DEV)
    # P == 0 is legal (rasterize_points.cu:81)
    out = raster.rasterize_gaussians(T(np.ones(3)), torch.zeros(0, 3, device=DEV), e, torch.zeros(0, 1, device=DEV),
                                     torch.zeros(0, 3, device=DEV), torch.zeros(0, 4, device=DEV), 1.0, e,
                                     T(sc["view"]), T(sc["proj"]), sc["tanx"], sc["tany"], 70, 100,
                                     torch.zeros(0, 1, 3, device=DEV), 0, T(sc["campos"]), False, False)
    assert out[0] == 0 and out[1].shape == (3, 70, 100)
    # wrong shape -> same error text as the reference
    with pytest.raises(RuntimeError, match="means3D must have dimensions"):
        raster.rasterize_gaussians(T(np.ones(3)), torch.zeros(5, 4, device=DEV), e, e, e, e, 1.0, e, T(sc["view"]),
                                   T(sc["proj"]), 1.0, 1.0, 8, 8, e, 0, T(sc["campos"]), False, False)
    # everything behind the camera -> background only, zero gradients
    behind = dict(sc)
    behind["act"] = dict(a)
    behind["act"]["means3D"] = np.tile(sc["campos"][None] * 2.0, (64, 1)).astype(np.float32)
    fwd = ours_forward(behind)
    assert fwd[0] == 0 and torch.all(fwd[1] == 1.0) and torch.all(fwd[2] == 0)
    g = ours_backward(behind, fwd, np.ones((3, 70, 100), np.float32))
    assert all(float(t.abs().sum()) == 0.0 for t in g)
    # ragged image size (not a multiple of 16) vs oracle
    st = oracle_forward(sc)
    fwd = ours_forward(sc)
    assert fwd[0] == st["num_rendered"] and rel_l2(fwd[1].cpu().numpy(), st["color"]) < TOL


def test_mark_visible_matches_oracle():
    from oracle import raster as orc
    from dgs_b200 import raster
    sc = scene_c1(P=4000, radius=0.8)  # camera inside the cloud: both outcomes occur
    vis = raster.mark_visible(T(sc["act"]["means3D"]), T(sc["view"]), T(sc["proj"])).cpu().numpy()
    ref = orc.mark_visible(sc["act"]["means3D"], sc["view"])
    assert vis.dtype == bool and 0 < vis.sum() < vis.size and np.array_equal(vis, ref)


def test_dropin_package_autograd_contract():
    """`from diff_gaussian_rasterization import ...` exactly as gs_core.py:10-13 / 874-945 uses it."""
    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    from oracle import raster as orc
    sc = scene_c1(P=5000, dist="trained", W=128, H=128)
    a = sc["act"]
    leaves = {k: T(a[k]).requires_grad_() for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    means2D = torch.zeros_like(leaves["means3D"], requires_grad=True)
    settings = GaussianRasterizationSettings(
        image_height=sc["H"], image_width=sc["W"], tanfovx=sc["tanx"], tanfovy=sc["tany"], bg=T(np.ones(3)),
        scale_modifier=1.0, viewmatrix=T(sc["view"]), projmatrix=T(sc["proj"]), sh_degree=0, campos=T(sc["campos"]),
        prefiltered=False, debug=False)
    rast = GaussianRasterizer(raster_settings=settings)
    color, radii = rast(means3D=leaves["means3D"], means2D=means2D, shs=leaves["shs"], colors_precomp=None,
                        opacities=leaves["opacities"], scales=leaves["scales"], rotations=leaves["rotations"],
                        cov3D_precomp=None)
    dpix = np.random.default_rng(2).normal(0, 1, (3, sc["H"], sc["W"])).astype(np.float32)
    color.backward(T(dpix))
    st = oracle_forward(sc)
    g = orc.rasterize_backward(st, dpix)
    assert rel_l2(color.detach().cpu().numpy(), st["color"]) < TOL
    pairs = dict(means3D="dL_dmeans3D", shs="dL_dsh", opacities="dL_dopacity", scales="dL_dscales",
                 rotations="dL_drotations")
    for k, gk in pairs.items():
        assert rel_l2(leaves[k].grad.cpu().numpy(), g[gk]) < TOL, k
    assert rel_l2(means2D.grad.cpu().numpy(), g["dL_dmeans2D"]) < TOL
    assert radii.dtype == torch.int32 and np.array_equal(radii.cpu().numpy(), st["radii"])
    with pytest.raises(Exception, match="SHs or precomputed colors"):
        rast(means3D=leaves["means3D"], means2D=means2D, opacities=leaves["opacities"], scales=leaves["scales"],
             rotations=leaves["rotations"])
    with pytest.raises(Exception, match="scale/rotation pair or precomputed 3D covariance"):
        rast(means3D=leaves["means3D"], means2D=means2D, opacities=leaves["opacities"], shs=leaves["shs"])


def _batch_inputs(B, V, P, W, H, dist="trained"):
    from dgs_b200 import synth
    gs = [synth.make_gaussians(P, 10 + i, dist) for i in range(B)]
    raw = {k: np.stack([g[k] for g in gs]) for k in gs[0]}
    rng = np.random.default_rng(3)
    raw["rotation"] = raw["rotation"] * rng.uniform(0.5, 2.0, (B, P, 1)).astype(np.float32)  # un-normalised
    c2w, fx = zip(*[synth.orbit_cameras(V, W, H, az0=15.0 * i) for i in range(B)])
    return raw, np.stack(c2w), np.stack(fx)


def test_batched_renderer_vs_oracle_renderer():
    """Renderer.forward/backward (renderer.py:34-92 + gs_core.py:949-1060 semantics) in ONE launch set."""
    from dgs_b200.renderer import Renderer
    from oracle import renderer as orr
    B, V, P, W, H = 2, 3, 1500, 64, 48
    raw, c2w, fx = _batch_inputs(B, V, P, W, H)
    names = ("xyz", "features", "scaling", "rotation", "opacity")
    cpu = [torch.tensor(raw[k], requires_grad=True) for k in names]
    ref = orr.render_batch(*cpu, H, W, torch.tensor(c2w), torch.tensor(fx))
    dimg = torch.tensor(np.random.default_rng(4).normal(0, 1, ref.shape).astype(np.float32))
    ref.backward(dimg)

    class Cfg:
        gaussians_sh_degree = 0
        use_gssplat = False
    gpu = [T(raw[k]).requires_grad_() for k in names]
    img = Renderer(Cfg())(*gpu, H, W, T(c2w), T(fx))
    assert img.shape == (B, V, 3, H, W) and img.dtype == torch.float32
    err = rel_l2(img.detach().cpu().numpy(), ref.detach().numpy())
    print(f"batched colour rel_l2={err:.3e}")
    assert err < TOL
    img.backward(dimg.to(DEV))
    for k, c, g in zip(names, cpu, gpu):
        e = rel_l2(g.grad.cpu().numpy(), c.grad.numpy())
        print(f"  batched d{k}: rel_l2={e:.3e}")
        assert e < TOL, k


def test_view_chunked_render_equals_single_batch(monkeypatch):
    """The > 2^31-1 instances fallback (dgs_b200/raster.py: views rendered in halves, gradients summed over the chunks)
    on the real kernels: the overflow status is injected for every call with more than 2 views, so a 5-view batch runs as
    chunks of (1, 1) and (1, 2) views; images must be bit-identical to the one-batch render (each view's blend is
    independent) and the per-Gaussian gradients equal up to the order of the cross-view sums."""
    from dgs_b200 import raster
    from dgs_b200._lib import DgsError
    from dgs_b200.renderer import Renderer
    B, V, P, W, H = 2, 5, 1200, 64, 48
    raw, c2w, fx = _batch_inputs(B, V, P, W, H)
    names = ("xyz", "features", "scaling", "rotation", "opacity")
    dimg = T(np.random.default_rng(5).normal(0, 1, (B, V, 3, H, W)).astype(np.float32))

    class Cfg:
        gaussians_sh_degree = 0
        use_gssplat = False

    def run():
        g = [T(raw[k]).requires_grad_() for k in names]
        img = Renderer(Cfg())(*g, H, W, T(c2w), T(fx))
        img.backward(dimg)
        return img.detach(), [t.grad for t in g]
    img1, grads1 = run()
    real = raster._render_batch_forward_one
    calls = []

    def overflowing(xyz, features, scaling, rotation, opacity, Hh, Ww, C2W, fxf, *a, **k):
        calls.append(C2W.shape[1])
        if C2W.shape[1] > 2:
            raise DgsError("libdgs_b200 status 4: instance count 3000000000 exceeds 2^31-1 (render the views in smaller batches)")
        return real(xyz, features, scaling, rotation, opacity, Hh, Ww, C2W, fxf, *a, **k)
    monkeypatch.setattr(raster, "_render_batch_forward_one", overflowing)
    img2, grads2 = run()
    assert calls == [5, 2, 3, 1, 2]
    assert torch.equal(img1, img2)
    for k, a, b in zip(names, grads1, grads2):
        e = rel_l2(b.cpu().numpy(), a.cpu().numpy())
        print(f"  chunked d{k}: rel_l2={e:.3e}")
        assert e < 1e-5, k


def test_full_size_properties_obj256():
    """The obj-256 denoise-step shape: P = 2 + 4*256*256 init-like Gaussians, 4 views at 256x256.
    Size-independent properties: partition of unity, (tile, depth) sortedness with stable ties,
    range lengths sum to R, linearity of the backward in dL/dpix."""
    from dgs_b200 import raster
    B, V, P, W, H = 1, 4, 2 + 4 * 256 * 256, 256, 256
    raw, c2w, fx = _batch_inputs(B, V, P, W, H, dist="init")
    raw["features"] = np.full_like(raw["features"], (1.0 - 0.5) / 0.28209479177387814)  # rgb == 1 exactly
    t = [T(raw[k]) for k in ("xyz", "features", "scaling", "rotation", "opacity")]
    img, state = raster.render_batch_forward(*t, H, W, T(c2w), T(fx), near_log2=0)  # single pass: lists exportable
    assert float((img - 1.0).abs().max()) < 5e-5  # sum_i w_i + T_final == 1
    R = state["R"]
    ex = raster.export_state(B * V, P, W, H, R, state["geom"], state["binning"], state["img"])
    assert int(ex["tiles_touched"].to(torch.int64).sum()) == R
    rng = ex["ranges"].to(torch.int64)
    assert int((rng[:, 1] - rng[:, 0]).sum()) == R
    pl = ex["point_list"].to(torch.int64)
    # depth along the sorted list must be non-decreasing inside every (view, tile) range
    tile_of = torch.repeat_interleave(torch.arange(rng.shape[0], device=DEV), rng[:, 1] - rng[:, 0])
    view_of = tile_of // 256
    depth = ex["depth"][view_of * P + pl]
    same_tile = tile_of[1:] == tile_of[:-1]
    assert bool(torch.all(depth[1:][same_tile] >= depth[:-1][same_tile]))
    ties = same_tile & (depth[1:] == depth[:-1])
    assert bool(torch.all(pl[1:][ties] > pl[:-1][ties]))
    # backward linearity: grad(2*g) == 2*grad(g) up to atomics-order noise
    g1 = torch.randn(img.shape, device=DEV, generator=torch.Generator(DEV).manual_seed(0))
    d1 = raster.render_batch_backward(state, g1)
    d2 = raster.render_batch_backward(state, 2.0 * g1)
    for a_, b_ in zip(d1, d2):
        assert rel_l2((2.0 * a_).cpu().numpy(), b_.cpu().numpy()) < 1e-5
    print(f"obj-256 init-like: R={R} ({R / (B * V):.0f} instances/view)")


@pytest.mark.parametrize("dist,P,expect_phase_b", [("init", 2 + 4 * 256 * 256, False), ("fine", 400000, True)])
def test_two_phase_binning_is_exact(dist, P, expect_phase_b):
    """near_log2 = 3: phase A bins/blends only the nearest 1/8 of each view's Gaussians; dense scenes stop there, sparse
    ones continue with phase B from the saved per-pixel state.  Images, final_T and n_contrib must be BIT-identical to
    the single-pass result (same blend order), gradients equal up to atomics-order noise."""
    from dgs_b200 import raster
    B, V, W, H = 1, 4, 256, 256
    raw, c2w, fx = _batch_inputs(B, V, P, W, H, dist=dist)
    t = [T(raw[k]) for k in ("xyz", "features", "scaling", "rotation", "opacity")]
    img1, st1 = raster.render_batch_forward(*t, H, W, T(c2w), T(fx), near_log2=0)
    img2, st2 = raster.render_batch_forward(*t, H, W, T(c2w), T(fx), near_log2=3)
    print(f"[{dist}] R={st1['R']} single-pass chunks={st1['chunks']} two-phase chunks={st2['chunks']}")
    assert st1["R"] == st2["R"] and st1["chunks"] == (st1["R"], 0)
    assert st2["chunks"][0] < st1["R"] // 2 and (st2["chunks"][1] > 0) == expect_phase_b
    assert torch.equal(img1, img2)
    e1 = raster.export_state(B * V, P, W, H, 0, st1["geom"], st1["binning"], st1["img"])
    e2 = raster.export_state(B * V, P, W, H, 0, st2["geom"], st2["binning"], st2["img"])
    assert torch.equal(e1["final_T"], e2["final_T"]) and torch.equal(e1["n_contrib"], e2["n_contrib"])
    g = torch.randn(img1.shape, device=DEV, generator=torch.Generator(DEV).manual_seed(3))
    d1 = raster.render_batch_backward(st1, g)
    d2 = raster.render_batch_backward(st2, g)
    for a_, b_ in zip(d1, d2):
        assert rel_l2(b_.cpu().numpy(), a_.cpu().numpy()) < 2e-5
    # adaptive near fraction (near_log2 = -1, the default): 1/16 for the dense scene, 1/8 for the sparse one -- same images
    img3, st3 = raster.render_batch_forward(*t, H, W, T(c2w), T(fx), near_log2=-1)
    print(f"[{dist}] adaptive chunks={st3['chunks']}")
    assert torch.equal(img1, img3)
    e3 = raster.export_state(B * V, P, W, H, 0, st3["geom"], st3["binning"], st3["img"])
    assert torch.equal(e1["final_T"], e3["final_T"]) and torch.equal(e1["n_contrib"], e3["n_contrib"])
    d3 = raster.render_batch_backward(st3, g)
    for a_, b_ in zip(d1, d3):
        assert rel_l2(b_.cpu().numpy(), a_.cpu().numpy()) < 2e-5
    if dist == "init":
        assert st3["chunks"][0] < st2["chunks"][0]      # the dense scene took the smaller near fraction
    else:
        assert st3["chunks"] == st2["chunks"]           # the sparse one stayed at 1/8
