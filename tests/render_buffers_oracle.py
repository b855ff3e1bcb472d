"""CPU oracle of the renderer's depth and alpha maps (TEST INFRASTRUCTURE, on top of oracle/renderer.py and oracle/raster.py).

depth = sum_i w_i z_i and alpha = 1 - T_final = sum_i w_i are linear in the colour's blend weights w_i, so the colour
rasterizer already computes them: a render with colors_precomp = (z_i, 1, 0) and bg = 0 has depth in channel 0 and alpha
in channel 1.  Its backward with dL/dpix = (dD, dA, 0) gives their screen-space gradients, and dL_dcolors[:, 0] is dL/dz,
which reaches the means through W2C's third row.  With oracle.raster.set_f64(True) every call runs in fp64."""
import numpy as np
import torch

from oracle import raster as _r
from oracle.renderer import activated_scales, build_camera, render_opencv_cam


class _AuxRaster(torch.autograd.Function):
    """(means3D, opacities, scales, rotations) activated -> [2, H, W] = (depth, alpha) of one view."""

    @staticmethod
    def forward(ctx, means3D, opacities, scales, rotations, cam, H, W):
        view, proj, campos, tanx, tany = cam

        def render(cols):
            return _r.rasterize_forward(np.zeros(3, np.float32), means3D.numpy(), cols, opacities.numpy(), scales.numpy(),
                                        rotations.numpy(), 1.0, None, view.numpy(), proj.numpy(), tanx, tany, H, W, None,
                                        0, campos.numpy())
        P = means3D.shape[0]
        z = render(np.zeros((P, 3), np.float32))["depths"]  # the oracle's own view-space depths
        st = render(np.stack([z, np.ones_like(z), np.zeros_like(z)], axis=1))
        ctx.st, ctx.row = st, view[:3, 2].numpy()  # view = W2C^T: view[k, 2] = W2C[2, k]
        return torch.from_numpy(st["color"][:2].copy())

    @staticmethod
    def backward(ctx, grad):
        st = ctx.st
        dpix = np.zeros((3, st["H"], st["W"]), grad.numpy().dtype)
        dpix[:2] = grad.numpy()
        g = _r.rasterize_backward(st, dpix)
        dmeans = g["dL_dmeans3D"] + g["dL_dcolors"][:, :1] * ctx.row[None, :].astype(g["dL_dcolors"].dtype)
        t = torch.from_numpy
        return t(dmeans), t(g["dL_dopacity"]), t(g["dL_dscales"]), t(g["dL_drotations"]), None, None, None


def render_batch_buffers(xyz, features, scaling, rotation, opacity, H, W, C2W, fxfycxcy, scaling_modifier=None):
    """oracle.renderer.render_batch plus per-pixel depth and alpha, the buffers of the reference's planned
    edict(render=..., depth=..., alpha=...): -> (render [b,v,3,H,W], depth [b,v,1,H,W], alpha [b,v,1,H,W]) from one colour
    call and one aux call per (sample, view); differentiable w.r.t. the five raw tensors.  `scaling_modifier` is applied
    as oracle.renderer.render_batch applies it."""
    b, v = C2W.shape[0], C2W.shape[1]
    render, aux = [], []
    for i in range(b):
        raw = [t[i].float() for t in (xyz, features, scaling, rotation, opacity)]
        for j in range(v):
            render.append(render_opencv_cam(*raw, H, W, C2W[i, j], fxfycxcy[i, j], scaling_modifier=scaling_modifier))
            cam = build_camera(C2W[i, j], fxfycxcy[i, j], H, W)
            aux.append(_AuxRaster.apply(raw[0], torch.sigmoid(raw[4]), activated_scales(raw[2], scaling_modifier),
                                        torch.nn.functional.normalize(raw[3]), cam, H, W))
    aux = torch.stack(aux, 0).reshape(b, v, 2, H, W)
    return torch.stack(render, 0).reshape(b, v, 3, H, W), aux[:, :, :1], aux[:, :, 1:]
