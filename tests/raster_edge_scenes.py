"""Small hand-built scenes at the rasterizer's numerical edges (TEST INFRASTRUCTURE for test_raster_edges_*.py).

Every constructor returns the scene dict of util.scene_c1 (raw and activated parameters, one camera's matrices, W, H, P)
plus `c2w_batch` [1, 2, 4, 4] / `fx_batch` [1, 2, 4]: the same camera and the same camera rolled 180 degrees about its
optical axis, which keeps every view depth and |x/z|, |y/z| and so each scene's property in both views of the batched
renderer.  test_raster_edges_cpu.py checks on the host that each scene has the property it is named for."""
import math

import numpy as np

from dgs_b200 import synth

W_EDGE, H_EDGE = 128, 96
ROLL_180 = np.diag([-1.0, -1.0, 1.0, 1.0]).astype(np.float32)


def _scene(raw, c2w, W=W_EDGE, H=H_EDGE, fx=None):
    fx = synth.intrinsics(W, H) if fx is None else np.asarray(fx, np.float32)
    c2w = np.asarray(c2w, np.float32)
    view, proj, campos, tanx, tany = synth.camera_matrices(c2w, fx, H, W)
    raw = {k: np.ascontiguousarray(v, dtype=np.float32) for k, v in raw.items()}
    return dict(raw=raw, act=synth.activate(raw), c2w=c2w, fxfycxcy=fx, view=view, proj=proj, campos=campos,
                tanx=tanx, tany=tany, W=W, H=H, P=raw["xyz"].shape[0],
                c2w_batch=np.stack([c2w, c2w @ ROLL_180])[None], fx_batch=np.stack([fx, fx])[None])


def _base(P, seed, dist="trained"):
    return synth.make_gaussians(P, seed, dist)


def _at_origin(az=30.0, el=20.0):
    """An orbit camera's orientation, moved to the origin."""
    c2w = synth.orbit_c2w(3.0, az, el)
    c2w[:3, 3] = 0.0
    return c2w


def _tan(W=W_EDGE, H=H_EDGE):
    fx = synth.intrinsics(W, H)
    return W / (2.0 * fx[0]), H / (2.0 * fx[1])


def _frustum_xy(rng, z, lo, hi, W=W_EDGE, H=H_EDGE):
    """x, y with |x/z| in [lo, hi] tan(fovx) and |y/z| in [lo, hi] tan(fovy), random signs."""
    tx, ty = _tan(W, H)
    u = rng.uniform(lo, hi, (2, z.size)) * rng.choice([-1.0, 1.0], (2, z.size))
    return u[0] * tx * z, u[1] * ty * z


def near_plane(P=1500, seed=21):
    """Camera at the origin looking down +z; view z uniform in [0.15, 0.6] across the 0.2 near plane, inside the frustum."""
    rng = np.random.default_rng(seed)
    g = _base(P, seed)
    z = rng.uniform(0.15, 0.6, P)
    x, y = _frustum_xy(rng, z, 0.0, 0.9)
    g["xyz"] = np.stack([x, y, z], 1)
    g["scaling"] = np.minimum(rng.normal(-4.0, 0.5, (P, 3)), -2.5)
    return _scene(g, np.eye(4))


def camera_inside(P=2000, seed=22):
    """Camera at the centre of the [-1, 1]^3 cloud: about half of it behind the camera, and 1 % of the Gaussians large
    (log-scales up to +0.5) and close, so their splats cover the whole image."""
    rng = np.random.default_rng(seed)
    g = _base(P, seed)
    g["scaling"] = np.minimum(rng.normal(-3.0, 1.0, (P, 3)), 0.5)
    big = rng.choice(P, P // 100, replace=False)
    g["scaling"][big] = rng.uniform(-0.5, 0.5, (big.size, 3))
    return _scene(g, _at_origin())


def frustum_edge(P=900, seed=23):
    """Depth 2-3, and x/z, y/z or both in +-[1.1, 1.5] tan(fov): across the rasterizer's 1.3 tan(fov) clamp of the EWA
    Jacobian.  Splats large enough (log-scales -1.8 .. -0.7) that Gaussians on both sides of the clamp reach the image."""
    rng = np.random.default_rng(seed)
    g = _base(P, seed)
    z = rng.uniform(2.0, 3.0, P)
    xo, yo = _frustum_xy(rng, z, 1.1, 1.5)
    xi, yi = _frustum_xy(rng, z, 0.0, 1.0)
    group = np.arange(P) % 3  # 0: x outside, 1: y outside, 2: both
    x = np.where(group == 1, xi, xo)
    y = np.where(group == 0, yi, yo)
    g["xyz"] = np.stack([x, y, z], 1)
    g["scaling"] = rng.uniform(-1.8, -0.7, (P, 3))
    g["opacity"] = rng.normal(-1.0, 1.0, (P, 1))
    return _scene(g, np.eye(4))


def needles_pancakes(P=800, seed=24):
    """Half needles (log-scales (-1.5, -7, -7)), half pancakes ((-1.5, -1.5, -8)), random rotations: nearly singular
    3D covariances, 2D covariances whose determinant cancels down to the 0.3 px^2 dilation."""
    g = _base(P, seed)
    needle = np.arange(P) % 2 == 0
    g["scaling"] = np.where(needle[:, None], [-1.5, -7.0, -7.0], [-1.5, -1.5, -8.0])
    g["opacity"] = np.random.default_rng(seed).normal(-1.0, 1.5, (P, 1))
    return _scene(g, synth.orbit_c2w())


def sub_pixel(P=3000, seed=25):
    """Every log-scale -8: the 0.3 px^2 dilation dominates the 2D covariance, radii of a few pixels."""
    g = _base(P, seed)
    g["scaling"] = np.full((P, 3), -8.0)
    g["opacity"] = np.random.default_rng(seed).normal(2.0, 1.0, (P, 1))
    return _scene(g, synth.orbit_c2w())


def opaque(P=2000, seed=26):
    """Opacity logits in [6, 12]: alpha clamped at 0.99 and the transmittance below 1e-4 after two or three layers."""
    rng = np.random.default_rng(seed)
    g = _base(P, seed)
    g["opacity"] = rng.uniform(6.0, 12.0, (P, 1))
    g["scaling"] = np.minimum(rng.normal(-3.2, 0.4, (P, 3)), -1.5)
    # With opaque layers the image follows the depth order of nearly tied layers, so the camera must be one whose view
    # matrix every implementation computes bit for bit: axis-aligned, 3 units out (an orbit camera's C2W.inverse() differs
    # in its last bits between the reference's fp32 torch inverse and the batched kernels' fp64 one).
    c2w = np.eye(4)
    c2w[2, 3] = -3.0
    return _scene(g, c2w)


def threshold(P=3000, seed=27):
    """Opacities (1/255)(1 + u), |u| <= 1e-3: whether a pixel passes alpha >= 1/255 is decided within 0.1 % of the
    threshold, where the blend kernels' footprint bound (alpha_extent, with its 0.1 % + 0.01 px margin) is tightest."""
    rng = np.random.default_rng(seed)
    g = _base(P, seed)
    p = (1.0 / 255.0) * (1.0 + rng.uniform(-1e-3, 1e-3, (P, 1)))
    g["opacity"] = np.log(p / (1.0 - p))
    g["scaling"] = rng.normal(-2.0, 0.3, (P, 3))
    return _scene(g, synth.orbit_c2w())


def depth_ties(P=400, seed=28, z=1.5):
    """P overlapping Gaussians at one view depth, bitwise: camera at the origin looking down +z (the view transform is
    exact), every centre at world z = 1.5.  Their order in each tile is the stable (tile, depth, index) order."""
    rng = np.random.default_rng(seed)
    g = _base(P, seed)
    g["xyz"] = np.stack([rng.uniform(-0.2, 0.2, P), rng.uniform(-0.15, 0.15, P), np.full(P, z)], 1)
    g["scaling"] = rng.normal(-3.5, 0.3, (P, 3))
    g["opacity"] = rng.normal(-1.0, 1.0, (P, 1))
    return _scene(g, np.eye(4))


def rotation_norms(P=2000, seed=29):
    """Raw quaternions of norm 1e-6 (even indices) and 1e4 (odd): the normalisation's Jacobian 1/|q| spans ten decades."""
    g = _base(P, seed)
    q = g["rotation"] / np.linalg.norm(g["rotation"], axis=1, keepdims=True)
    g["rotation"] = q * np.where(np.arange(P) % 2 == 0, 1e-6, 1e4)[:, None]
    return _scene(g, synth.orbit_c2w())


SCENES = dict(near_plane=near_plane, camera_inside=camera_inside, frustum_edge=frustum_edge,
              needles_pancakes=needles_pancakes, sub_pixel=sub_pixel, opaque=opaque, threshold=threshold,
              depth_ties=depth_ties, rotation_norms=rotation_norms)


def view_xyz(sc):
    """View-space centres of the scene's (first) camera, fp64."""
    p = sc["act"]["means3D"].astype(np.float64)
    return p @ sc["view"][:3, :3].astype(np.float64) + sc["view"][3, :3].astype(np.float64)


def roll(c2w, degrees):
    """c2w rotated by `degrees` about its own optical (z) axis."""
    a = math.radians(degrees)
    r = np.eye(4, dtype=np.float32)
    r[0, 0], r[0, 1], r[1, 0], r[1, 1] = math.cos(a), -math.sin(a), math.sin(a), math.cos(a)
    return (np.asarray(c2w, np.float32) @ r).astype(np.float32)
