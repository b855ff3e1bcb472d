"""oracle/renderer.py -- TEST INFRASTRUCTURE: CPU restatement of the reference's Python renderer.

Follows diffusionGS/models/gsrenderer/gs_core.py:
  Camera (277-316), GaussianModel activations (323-373, 545-570), render_opencv_cam (874-945),
  DeferredGaussianRender.forward/backward (949-1060) and renderer.py:34-92 (fp32 cast),
on CPU torch tensors, with the rasterizer itself provided by oracle/raster.py (C restatement).
Never imported by the product path.
"""
import numpy as np
import torch

from . import raster as _r

ZNEAR, ZFAR = 0.01, 100.0  # gs_core.py:286-287


def build_camera(C2W, fxfycxcy, h, w):
    """gs_core.py:277-316 -> (viewmatrix[4,4] = W2C^T, projmatrix[4,4] = (P W2C)^T, campos[3], tanx, tany)"""
    C2W = C2W.detach().clone().float().cpu()
    W2C = C2W.inverse()
    fx, fy, cx, cy = [float(v) for v in fxfycxcy.detach().float().cpu()]
    Pm = torch.zeros(4, 4)
    Pm[0, 0] = 2 * fx / w
    Pm[1, 1] = 2 * fy / h
    Pm[0, 2] = 2 * (cx / w) - 1
    Pm[1, 2] = 2 * (cy / h) - 1
    Pm[2, 2] = -(ZFAR + ZNEAR) / (ZFAR - ZNEAR)
    Pm[3, 2] = 1.0
    Pm[2, 3] = -(2 * ZFAR * ZNEAR) / (ZFAR - ZNEAR)
    view = W2C.transpose(0, 1)
    full = view.unsqueeze(0).bmm(Pm.transpose(0, 1).unsqueeze(0)).squeeze(0)
    return view.contiguous(), full.contiguous(), C2W[:3, 3].contiguous(), w / (2 * fx), h / (2 * fy)


class _Raster(torch.autograd.Function):
    """The binding's autograd contract (DGR/diff_gaussian_rasterization/__init__.py:44-155)."""

    @staticmethod
    def forward(ctx, means3D, shs, opacities, scales, rotations, cam, H, W, degree, bg):
        view, proj, campos, tanx, tany = cam
        st = _r.rasterize_forward(np.asarray(bg, np.float32), means3D.numpy(), None, opacities.numpy(),
                                  scales.numpy(), rotations.numpy(), 1.0, None, view.numpy(), proj.numpy(),
                                  tanx, tany, H, W, shs.numpy(), degree, campos.numpy())
        ctx.st = st
        return torch.from_numpy(st["color"].copy())

    @staticmethod
    def backward(ctx, grad):
        g = _r.rasterize_backward(ctx.st, grad.contiguous().numpy())
        t = torch.from_numpy
        return (t(g["dL_dmeans3D"]), t(g["dL_dsh"]), t(g["dL_dopacity"]), t(g["dL_dscales"]),
                t(g["dL_drotations"]), None, None, None, None, None)


def activated_scales(scaling, scaling_modifier=None):
    """GaussianModel.get_scaling (gs_core.py:545-550): exp(scaling), times the model's scaling_modifier when it has one.
    The rasterizer then runs with scale_modifier = 1, so autograd supplies the modifier's factor in d(scaling)."""
    scales = torch.exp(scaling)                                   # gs_core.py:330,545-550
    return scales if scaling_modifier is None else scales * float(scaling_modifier)


def render_opencv_cam(xyz, features, scaling, rotation, opacity, H, W, C2W, fxfycxcy,
                      bg=(1.0, 1.0, 1.0), scaling_modifier=None):
    """gs_core.py:874-945 on raw (pre-activation) per-sample tensors; differentiable."""
    cam = build_camera(C2W, fxfycxcy, H, W)
    degree = int(round(features.shape[-2] ** 0.5)) - 1
    scales = activated_scales(scaling, scaling_modifier)
    rots = torch.nn.functional.normalize(rotation)                # :332,553
    opac = torch.sigmoid(opacity)                                 # :333,569
    return _Raster.apply(xyz, features, opac, scales, rots, cam, H, W, degree, bg)


def render_batch(xyz, features, scaling, rotation, opacity, H, W, C2W, fxfycxcy, scaling_modifier=None):
    """Renderer.forward + deferred_gaussian_render semantics (renderer.py:34-92,
    gs_core.py:949-1060): [b,P,*] raw params, C2W [b,v,4,4], fxfycxcy [b,v,4] -> [b,v,3,H,W] fp32.
    Differentiable w.r.t. the five parameter tensors (sums over views, like the reference's
    accumulated .grad).  `scaling_modifier`: the GaussianModel's (applied to the scales, see activated_scales)."""
    b, v = C2W.shape[0], C2W.shape[1]
    out = []
    for i in range(b):
        for j in range(v):
            out.append(render_opencv_cam(xyz[i].float(), features[i].float(), scaling[i].float(),
                                         rotation[i].float(), opacity[i].float(), H, W, C2W[i, j],
                                         fxfycxcy[i, j], scaling_modifier=scaling_modifier))
    return torch.stack(out, 0).reshape(b, v, 3, H, W)
