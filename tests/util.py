"""Shared helpers of the parity tests: seeded scenes and error metrics."""
import numpy as np
import torch

from dgs_b200 import synth


def scene_c1(P=10000, dist="trained", W=256, H=256, seed=0, az=30.0, el=20.0, radius=3.0):
    g = synth.make_gaussians(P, seed, dist)
    a = synth.activate(g)
    c2w = synth.orbit_c2w(radius, az, el)
    fx = synth.intrinsics(W, H)
    view, proj, campos, tanx, tany = synth.camera_matrices(c2w, fx, H, W)
    return dict(raw=g, act=a, c2w=c2w, fxfycxcy=fx, view=view, proj=proj, campos=campos, tanx=tanx, tany=tany,
                W=W, H=H, P=P)


def oracle_forward(sc, sh=None, degree=0, colors=None, cov3d=None, bg=(1.0, 1.0, 1.0)):
    from oracle import raster as orc
    a = sc["act"]
    return orc.rasterize_forward(np.asarray(bg, np.float32), a["means3D"], colors, a["opacities"],
                                 None if cov3d is not None else a["scales"],
                                 None if cov3d is not None else a["rotations"], 1.0, cov3d, sc["view"], sc["proj"],
                                 sc["tanx"], sc["tany"], sc["H"], sc["W"],
                                 None if colors is not None else (a["shs"] if sh is None else sh), degree,
                                 sc["campos"])


def rel_l2(a, b):
    """||a - b|| / (||b|| + 1e-30) in float64: in torch on a's device when either is a tensor, else in numpy."""
    if isinstance(a, torch.Tensor) or isinstance(b, torch.Tensor):
        a = torch.as_tensor(a).detach().double()
        b = torch.as_tensor(b).detach().to(a.device, torch.float64)
        return float((a - b).norm() / (b.norm() + 1e-30))
    a = np.asarray(a, np.float64).ravel()
    b = np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30))


def max_abs(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max()) if np.size(a) else 0.0
