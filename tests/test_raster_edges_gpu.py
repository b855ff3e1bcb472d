"""The rasterizer away from the synthetic orbit, against the CPU oracle's fp64 build:
  * the batched renderer's parameter space (Renderer.forward, forward_mse, forward_buffers): SH degrees 1-3 with the
    per-channel clamp, the scaling modifier, off-centre principal points with fx != fy and a rolled camera, ragged and
    sub-tile images;
  * hostile geometry (raster_edge_scenes.py: near plane, camera inside the cloud, frustum edge, needles and pancakes,
    sub-pixel splats, opaque layers, opacities at the 1/255 threshold, bitwise depth ties, extreme quaternion norms), through
    the single-view C ABI and through the batched renderer;
  * the single-view path with a coloured background and with a scale modifier.
Bound of every quantity: max(1e-4, 2 x the oracle's own fp32 build's distance from fp64), the noise-floor rule of
test_raster_gpu.check_grads and test_raster_depth_alpha_gpu._oracle_case (FloorCheck); in single-view cases, where oracle/_ref
is built, also 2 x the reference's own kernels' distance from fp64 on the same inputs.  Colours are compared as colour - background, so
that the background does not dilute the error of the splats.  Integer outputs (radii, num_rendered, n_contrib, and on the
tie scene the sorted lists) are compared with the fp32 oracle, up to the threshold flips test_raster_gpu.py bounds."""
import math

import numpy as np
import pytest
import torch

import raster_edge_scenes as es
from test_raster_gpu import DEV, GRAD_NAMES, TOL, T, _batch_inputs
from util import rel_l2, scene_c1

pytestmark = pytest.mark.gpu
NAMES = ("xyz", "features", "scaling", "rotation", "opacity")


def _np(x):
    return x.detach().cpu().numpy() if torch.is_tensor(x) else np.asarray(x)


class FloorCheck:
    """Each quantity within max(1e-4, 2 x the fp32 oracle's rel_l2 from the fp64 oracle) of the fp64 oracle.  Every
    quantity is printed (with the reference kernels' own error where given) before the failures are raised."""

    def __init__(self, case):
        self.case, self.bad = case, []

    def __call__(self, tag, ours, exact, fp32, ref=None):
        exact = _np(exact)
        floor = rel_l2(_np(fp32), exact)
        e = rel_l2(_np(ours), exact)
        # the fp32 oracle accumulates in fp64 and in a fixed order; the reference's kernels, where built, also measure the
        # atomics-order noise of fp32 kernels (up to 5e-4 in dL_dcov3D on the needle scene, measured on an H100)
        ref_e = None if ref is None else rel_l2(_np(ref), exact)
        tol = max(TOL, 2.0 * floor, 0.0 if ref_e is None else 2.0 * ref_e)
        r = "" if ref is None else f", reference kernels {ref_e:.3e}"
        print(f"  [{self.case}] {tag}: rel_l2={e:.3e} (fp32 oracle {floor:.3e}{r}, tol {tol:.1e})")
        if not e < tol:
            self.bad.append((tag, e, tol))

    def done(self):
        assert not self.bad, (self.case, self.bad)


class Cfg:
    gaussians_sh_degree = 0
    use_gssplat = False


def _grads(outs, leaves, ups):
    loss = sum((o * u.to(o.device, o.dtype)).sum() for o, u in zip(outs, ups) if u is not None)
    g = torch.autograd.grad(loss, leaves, allow_unused=True)
    return [torch.zeros_like(x) if d is None else d for d, x in zip(g, leaves)]


def _oracle_outputs(mode, leaves, H, W, c2w, fx, m, target):
    from oracle import renderer as orr
    from render_buffers_oracle import render_batch_buffers
    if mode == "buffers":
        return list(render_batch_buffers(*leaves, H, W, c2w, fx, scaling_modifier=m))
    img = orr.render_batch(*leaves, H, W, c2w, fx, scaling_modifier=m)
    if mode == "render":
        return [img]
    return [img, ((img - target[:, :, :3]) ** 2).mean(dim=(1, 2, 3, 4))]  # LossComputer's l2 term


def _gpu_outputs(mode, leaves, H, W, c2w, fx, m, target):
    from dgs_b200.renderer import Renderer
    r = Renderer(Cfg())
    r.scaling_modifier = m
    if mode == "buffers":
        d = r.forward_buffers(*leaves, H, W, c2w, fx)
        return [d["render"], d["depth"], d["alpha"]]
    if mode == "render":
        return [r(*leaves, H, W, c2w, fx)]
    return list(r.forward_mse(*leaves, H, W, c2w, fx, target))


OUT_NAMES = dict(render=("render",), buffers=("render", "depth", "alpha"), mse3=("render", "l2"), mse4=("render", "l2"))


def _batched_case(case, raw, c2w, fx, H, W, mode="render", m=None, groups=None, seed=7):
    """Renderer on raw [B, P, *] parameters vs oracle.renderer.render_batch (render_batch_buffers for mode "buffers"):
    every output and the five raw gradients of sum <output, upstream>.  mse3 / mse4: forward_mse with a 3- or 4-channel
    target, differentiated through the l2 loss alone (the gradient image is formed inside the blend backward)."""
    from oracle import raster as orc
    B, V = c2w.shape[:2]
    gen = torch.Generator().manual_seed(seed)
    target = torch.rand(B, V, 4 if mode == "mse4" else 3, H, W, generator=gen)
    if mode == "render":
        ups = [torch.randn(B, V, 3, H, W, generator=gen)]
    elif mode == "buffers":
        ups = [torch.randn(B, V, c, H, W, generator=gen) for c in (3, 1, 1)]
    else:
        ups = [None, torch.tensor([1.0, 2.0][:B])]
    ref = {}
    for f64 in (True, False):
        orc.set_f64(f64)
        try:
            leaves = [torch.tensor(raw[k], requires_grad=True) for k in NAMES]
            outs = _oracle_outputs(mode, leaves, H, W, torch.tensor(c2w), torch.tensor(fx), m, target)
            ref[f64] = ([o.detach() for o in outs], _grads(outs, leaves, ups))
        finally:
            orc.set_f64(False)
    leaves = [T(raw[k]).requires_grad_() for k in NAMES]
    outs = _gpu_outputs(mode, leaves, H, W, T(c2w), T(fx), m, target.to(DEV))
    ours = ([o.detach() for o in outs], _grads(outs, leaves, ups))
    chk = FloorCheck(case)
    for i, name in enumerate(OUT_NAMES[mode]):
        sub = 1.0 if name == "render" else 0.0  # colour - white background
        chk(name, _np(ours[0][i]) - sub, _np(ref[True][0][i]) - sub, _np(ref[False][0][i]) - sub)
    for j, k in enumerate(NAMES):
        chk(f"d{k}", ours[1][j], ref[True][1][j], ref[False][1][j])
        for gname, idx in (groups or {}).items():
            chk(f"d{k}[{gname}]", _np(ours[1][j])[:, idx], _np(ref[True][1][j])[:, idx], _np(ref[False][1][j])[:, idx])
    chk.done()


# ------------------------------------------------------------------------------------------------
# a. the batched renderer's parameter space
# ------------------------------------------------------------------------------------------------
def _sh_inputs(B, V, P, W, H, degree, seed=40):
    """_batch_inputs with SH rest coefficients N(0, 0.3) up to `degree`: a good share of the colour channels clamp at 0."""
    raw, c2w, fx = _batch_inputs(B, V, P, W, H)
    rest = np.random.default_rng(seed).normal(0, 0.3, (B, P, (degree + 1) ** 2 - 1, 3)).astype(np.float32)
    raw["features"] = np.concatenate([raw["features"], rest], axis=2)
    return raw, c2w, fx


@pytest.mark.parametrize("degree,mode", [(1, "render"), (2, "render"), (3, "render"), (3, "mse3"), (3, "mse4"),
                                         (3, "buffers")])
def test_batched_sh_degrees(degree, mode):
    B, V, P, W, H = 2, 3, 2000, 64, 48
    raw, c2w, fx = _sh_inputs(B, V, P, W, H, degree)
    _batched_case(f"sh{degree}/{mode}", raw, c2w, fx, H, W, mode)


@pytest.mark.parametrize("m,mode", [(0.5, "render"), (1.7, "render"), (1.7, "buffers")])
def test_batched_scaling_modifier(m, mode):
    """GaussianModel.get_scaling: S = exp(s) m, so d(scaling) carries the factor m."""
    B, V, P, W, H = 2, 3, 2000, 64, 48
    raw, c2w, fx = _batch_inputs(B, V, P, W, H)
    _batched_case(f"mod{m}/{mode}", raw, c2w, fx, H, W, mode, m=m)


@pytest.mark.parametrize("m", [0.5, 1.7])
def test_batched_scaling_modifier_is_a_log_scale_shift(m):
    """Oracle-free: rendering (scaling, m) and (scaling + ln m, no modifier) on the GPU gives the same images and the same
    gradients with respect to the scaling leaf; they differ only in the rounding of exp."""
    from dgs_b200.renderer import Renderer
    B, V, P, W, H = 2, 3, 2000, 64, 48
    raw, c2w, fx = _batch_inputs(B, V, P, W, H)
    up = torch.randn(B, V, 3, H, W, device=DEV, generator=torch.Generator(DEV).manual_seed(8))
    runs = []
    for shift, mod in ((0.0, m), (math.log(m), None)):
        r = Renderer(Cfg())
        r.scaling_modifier = mod
        leaves = [T(raw[k]).requires_grad_() for k in NAMES]
        img = r(leaves[0], leaves[1], leaves[2] + shift, leaves[3], leaves[4], H, W, T(c2w), T(fx))
        runs.append((img.detach(), _grads([img], leaves, [up])))
    (img_m, g_m), (img_s, g_s) = runs
    errs = {"render": rel_l2(_np(img_m) - 1.0, _np(img_s) - 1.0)}
    errs.update({f"d{k}": rel_l2(_np(a), _np(b)) for k, a, b in zip(NAMES, g_m, g_s)})
    print(f"  [shift m={m}] " + " ".join(f"{k}={e:.2e}" for k, e in errs.items()))
    assert all(e < 1e-5 for e in errs.values()), errs


def test_batched_off_centre_principal_point():
    """cx = 0.31 W, cy = 0.64 H, fy = 0.8 fx in every view, and the last view rolled 30 degrees about its axis."""
    B, V, P, W, H = 2, 3, 2000, 64, 48
    raw, c2w, fx = _batch_inputs(B, V, P, W, H)
    fx[..., 1] = 0.8 * fx[..., 0]
    fx[..., 2], fx[..., 3] = 0.31 * W, 0.64 * H
    c2w[:, -1] = np.stack([es.roll(c, 30.0) for c in c2w[:, -1]])
    _batched_case("off-centre", raw, c2w, fx, H, W)


@pytest.mark.parametrize("W,H", [(100, 70), (33, 17), (16, 16), (9, 13)])
def test_batched_ragged_images(W, H):
    """Tile grids with partial edge tiles, one tile, less than one tile: images and the fused MSE's pixel count."""
    B, V, P = 2, 3, 2000
    raw, c2w, fx = _batch_inputs(B, V, P, W, H)
    _batched_case(f"{W}x{H}", raw, c2w, fx, H, W, "mse3")


# ------------------------------------------------------------------------------------------------
# b. hostile geometry
# ------------------------------------------------------------------------------------------------
def _single_view(sc, bg, mod, dpix, impl):
    """One forward and backward of the single-view ABI (`impl`: dgs_b200.raster or the reference's module)."""
    a = sc["act"]
    e = torch.empty(0, device=DEV)
    args = (T(bg), T(a["means3D"]), e, T(a["opacities"]), T(a["scales"]), T(a["rotations"]), float(mod), e,
            T(sc["view"]), T(sc["proj"]), float(sc["tanx"]), float(sc["tany"]), sc["H"], sc["W"], T(a["shs"]), 0,
            T(sc["campos"]), False, False)
    fwd = impl.rasterize_gaussians(*args)
    R, color, radii, geom, binning, img = fwd
    g = impl.rasterize_gaussians_backward(args[0], args[1], radii, e, args[4], args[5], float(mod), e, args[8], args[9],
                                          args[10], args[11], T(dpix), args[14], 0, args[16], geom, R, binning, img,
                                          False)
    return fwd, [t.cpu().numpy() for t in g]


def _single_view_case(case, sc, bg=(1.0, 1.0, 1.0), mod=1.0, exact_lists=False):
    """The single-view ABI on activated parameters vs the oracle's fp64 build, and the reference's kernels where built."""
    from dgs_b200 import raster
    from oracle import build_ref
    from oracle import raster as orc
    a = sc["act"]
    bg = np.asarray(bg, np.float32)
    dpix = np.random.default_rng(9).normal(0, 1, (3, sc["H"], sc["W"])).astype(np.float32)
    st, g = {}, {}
    for f64 in (True, False):
        orc.set_f64(f64)
        try:
            st[f64] = orc.rasterize_forward(bg, a["means3D"], None, a["opacities"], a["scales"], a["rotations"], mod, None,
                                            sc["view"], sc["proj"], sc["tanx"], sc["tany"], sc["H"], sc["W"], a["shs"],
                                            0, sc["campos"])
            g[f64] = orc.rasterize_backward(st[f64], dpix)
        finally:
            orc.set_f64(False)
    fwd, ours = _single_view(sc, bg, mod, dpix, raster)
    R, color, radii = fwd[0], fwd[1], fwd[2].cpu().numpy()
    refmod = build_ref.load_module()
    ref = _single_view(sc, bg, mod, dpix, refmod) if refmod is not None else None
    s32 = st[False]
    n_rad = int((radii != s32["radii"]).sum())
    print(f"  [{case}] R ours={R} oracle={s32['num_rendered']} radii mismatches={n_rad}"
          + ("" if ref is None else f"; reference R={ref[0][0]} radii mismatches={int((ref[0][2].cpu().numpy() != s32['radii']).sum())}"))
    ex = raster.export_state(1, sc["P"], sc["W"], sc["H"], R, fwd[3], fwd[4], fwd[5])
    if n_rad == 0:
        nc = float((ex["n_contrib"].cpu().numpy().astype(np.int64) != s32["n_contrib"].astype(np.int64)).mean())
        print(f"  [{case}] n_contrib mismatch fraction {nc:.2e}")
    chk = FloorCheck(case)
    bgc = bg[:, None, None]
    chk("colour - bg", color.cpu().numpy() - bgc, st[True]["color"] - bgc, s32["color"] - bgc,
        None if ref is None else ref[0][1].cpu().numpy() - bgc)
    for j, name in enumerate(GRAD_NAMES):
        if g[True][name].size:
            chk(name, ours[j], g[True][name], g[False][name], None if ref is None else ref[1][j])
    assert n_rad <= 2 and abs(R - s32["num_rendered"]) <= 64, (case, n_rad, R, s32["num_rendered"])
    if n_rad == 0:
        assert R == s32["num_rendered"] and nc < 1e-3, (case, R, nc)
    if exact_lists:  # the stable (tile, depth, index) order, bit for bit
        assert np.array_equal(ex["point_list"].cpu().numpy().astype(np.uint32), s32["point_list"])
        ours_r, ref_r = ex["ranges"].cpu().numpy().astype(np.int64), s32["ranges"].astype(np.int64)
        full = ref_r[:, 1] > ref_r[:, 0]  # an empty tile's range is [0, 0] in the oracle, [R, R] past the last list here
        assert np.array_equal(ours_r[:, 1] - ours_r[:, 0], ref_r[:, 1] - ref_r[:, 0])
        assert full.sum() > 0 and np.array_equal(ours_r[full], ref_r[full])
    chk.done()


@pytest.mark.parametrize("name", list(es.SCENES))
def test_hostile_single_view(name):
    _single_view_case(name, es.SCENES[name](), exact_lists=(name == "depth_ties"))


@pytest.mark.parametrize("name", list(es.SCENES))
def test_hostile_batched(name):
    sc = es.SCENES[name]()
    raw = {k: v[None] for k, v in sc["raw"].items()}
    groups = None
    if name == "rotation_norms":  # the 1e-6 quaternions' gradients are 1e10 times the 1e4 ones': check each group
        groups = {"|q|=1e-6": np.arange(0, sc["P"], 2), "|q|=1e4": np.arange(1, sc["P"], 2)}
    _batched_case(name, raw, sc["c2w_batch"], sc["fx_batch"], sc["H"], sc["W"], groups=groups)


def test_single_view_coloured_background():
    """The trained C1 scene over background (0.1, 0.5, 0.9): a channel mix-up in the T bg term shows, where white hides it."""
    _single_view_case("c1 bg", scene_c1(P=10000, dist="trained"), bg=(0.1, 0.5, 0.9))


def test_single_view_scale_modifier():
    """The single-view ABI keeps the reference rasterizer's convention: dL_dscales is d/d(mod scale), without the factor."""
    _single_view_case("c1 mod 1.7", scene_c1(P=3000, dist="trained", W=128, H=128), mod=1.7)
