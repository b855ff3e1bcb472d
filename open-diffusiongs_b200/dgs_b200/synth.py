"""Seeded synthetic workloads (configs C1 single-view scenes .. C5 stress sweep): Gaussians, orbit cameras, batches.

Everything is generated with numpy on the host from an explicit seed so that the CPU oracle, the
compiled reference kernels and the sm_90a kernels see bit-identical inputs on any machine.
"""
import math

import numpy as np

SH_C0 = 0.28209479177387814
DEFAULT_FXFY = 1.388889  # reference dGS/data/base.py:55 (`default_fxfy`), in units of image width

DISTRIBUTIONS = {  # (mu, sigma) of the per-axis log-scale
    "init": (-2.3, 0.01),
    "trained": (-4.0, 0.7),
    "fine": (-5.0, 0.5),
}


def orbit_c2w(radius=3.0, az_deg=30.0, el_deg=20.0):
    """OpenCV-convention (x right, y down, z forward) camera-to-world looking at the origin."""
    az, el = math.radians(az_deg), math.radians(el_deg)
    pos = np.array([radius * math.cos(el) * math.cos(az), radius * math.cos(el) * math.sin(az),
                    radius * math.sin(el)], np.float64)
    fwd = -pos / np.linalg.norm(pos)
    up = np.array([0.0, 0.0, 1.0])
    right = np.cross(fwd, up)
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    c2w = np.eye(4)
    c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, down, fwd, pos
    return c2w.astype(np.float32)


def intrinsics(W, H=None):
    H = W if H is None else H
    return np.array([DEFAULT_FXFY * W, DEFAULT_FXFY * W, W / 2.0, H / 2.0], np.float32)


def orbit_cameras(n_views, W, H=None, radius=3.0, el_deg=20.0, az0=0.0, az_step=None):
    az_step = 360.0 / n_views if az_step is None else az_step
    c2w = np.stack([orbit_c2w(radius, az0 + i * az_step, el_deg) for i in range(n_views)])
    fx = np.stack([intrinsics(W, H)] * n_views)
    return c2w, fx


def make_gaussians(P, seed=0, dist="trained", extent=1.0):
    """Raw (pre-activation) parameters in the reference's renderer convention
    (gs_core.py:356-373): scale = exp(scaling), rot = normalize(rotation), opacity = sigmoid(opacity)."""
    mu, sigma = DISTRIBUTIONS[dist]
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(-extent, extent, (P, 3)).astype(np.float32)
    scaling = np.minimum(rng.normal(mu, sigma, (P, 3)), -1.2).astype(np.float32)
    rotation = rng.normal(0, 1, (P, 4)).astype(np.float32)
    rotation /= np.linalg.norm(rotation, axis=1, keepdims=True)
    opacity = rng.normal(0, 2.0, (P, 1)).astype(np.float32)
    features = ((rng.uniform(0, 1, (P, 1, 3)) - 0.5) / SH_C0).astype(np.float32)
    return dict(xyz=xyz, features=features, scaling=scaling, rotation=rotation, opacity=opacity)


def make_shell_gaussians(P, seed=0, dist="trained", radii=(0.6, 0.45, 0.5), thickness=0.02):
    """make_gaussians with the centres on a thin ellipsoidal shell (semi-axes `radii`, relative thickness `thickness`):
    an object-like point set, whose opacity field is a closed surface with empty space inside and out."""
    g = make_gaussians(P, seed, dist)
    rng = np.random.default_rng(seed + 7919)
    d = rng.normal(0, 1, (P, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    r = 1.0 + rng.normal(0, thickness, (P, 1))
    g["xyz"] = (d * r * np.asarray(radii)).astype(np.float32)
    return g


def activate(g):
    """Host-side activations -> the tensors `GaussianRasterizer.forward` receives."""
    return dict(means3D=g["xyz"], shs=g["features"], scales=np.exp(g["scaling"]),
                rotations=g["rotation"] / np.maximum(np.linalg.norm(g["rotation"], axis=1, keepdims=True), 1e-12),
                opacities=1.0 / (1.0 + np.exp(-g["opacity"])))


def camera_matrices(c2w, fxfycxcy, H, W, znear=0.01, zfar=100.0):
    """Host fp32 restatement of the reference `Camera` (gs_core.py:277-316):
    -> viewmatrix (= W2C^T), projmatrix (= (P W2C)^T), campos, tanfovx, tanfovy."""
    c2w = np.asarray(c2w, np.float32)
    w2c = np.linalg.inv(c2w.astype(np.float64)).astype(np.float32)
    fx, fy, cx, cy = [float(v) for v in fxfycxcy]
    Pm = np.zeros((4, 4), np.float32)
    Pm[0, 0] = 2 * fx / W
    Pm[1, 1] = 2 * fy / H
    Pm[0, 2] = 2 * (cx / W) - 1
    Pm[1, 2] = 2 * (cy / H) - 1
    Pm[2, 2] = -(zfar + znear) / (zfar - znear)
    Pm[3, 2] = 1.0
    Pm[2, 3] = -(2 * zfar * znear) / (zfar - znear)
    view = np.ascontiguousarray(w2c.T)
    full = np.ascontiguousarray((view @ Pm.T).astype(np.float32))
    return view, full, np.ascontiguousarray(c2w[:3, 3]), W / (2 * fx), H / (2 * fy)
