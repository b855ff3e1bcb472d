"""The geometry terms of the training loss on libdgs_b200.so (dgs_geometry_loss_forward / _backward): the reference's
pointsdist and l2_loss_xyz (diffusionGS/utils/losses.py:286-291, 323-364) over the pixel-aligned Gaussian centres.

    pd, l2 = geometry_losses(img_aligned_xyz, ray_o, gt_img_aligned_xyz, masks)   # [b], [] (None where not asked)

Both are differentiable in img_aligned_xyz only (the reference detaches the pointsdist target; ray_o, the ground truth
and the masks are data).  LossComputer.forward uses this on CUDA tensors.
"""
import torch

from . import _lib
from ._lib import check, f32, ptr, stream


class _GeometryLossFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img_xyz, ray_o, gt_xyz, masks, want_pd, want_xyz):
        B, V, _, H, W = img_xyz.shape
        dev = img_xyz.device
        img, o, gt, m = f32(img_xyz), f32(ray_o), f32(gt_xyz), f32(masks)
        L = _lib.lib()
        pd = torch.empty(B, dtype=torch.float32, device=dev) if want_pd else torch.zeros(B, device=dev)
        l2 = torch.empty((), dtype=torch.float32, device=dev) if want_xyz else torch.zeros((), device=dev)
        state = torch.empty(2 * B * V + 1, dtype=torch.float32, device=dev)
        ws = torch.empty(L.dgs_geometry_loss_workspace_bytes(B, V), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            check(L.dgs_geometry_loss_forward(B, V, H, W, img.data_ptr(), ptr(o), ptr(gt), ptr(m),
                                              pd.data_ptr() if want_pd else None, l2.data_ptr() if want_xyz else None,
                                              state.data_ptr(), ws.data_ptr(), ws.numel(), stream(dev)))
        if not want_pd:
            ctx.mark_non_differentiable(pd)
        if not want_xyz:
            ctx.mark_non_differentiable(l2)
        ctx.set_materialize_grads(False)
        ctx.in_dtype = img_xyz.dtype
        ctx.save_for_backward(img, o, gt, m, state)
        return pd, l2

    @staticmethod
    def backward(ctx, g_pd, g_xyz):
        img, o, gt, m, state = ctx.saved_tensors
        if g_pd is None and g_xyz is None:
            return None, None, None, None, None, None
        B, V, _, H, W = img.shape
        g_pd = None if g_pd is None else g_pd.to(torch.float32).reshape(B).contiguous()
        g_xyz = None if g_xyz is None else g_xyz.to(torch.float32).reshape(1).contiguous()
        d_img = torch.empty_like(img)
        with torch.cuda.device(img.device):
            check(_lib.lib().dgs_geometry_loss_backward(B, V, H, W, img.data_ptr(), ptr(o), ptr(gt), ptr(m),
                                                        state.data_ptr(), ptr(g_pd), ptr(g_xyz), d_img.data_ptr(),
                                                        stream(img.device)))
        return d_img.to(ctx.in_dtype), None, None, None, None, None


def geometry_losses(img_xyz, ray_o=None, gt_xyz=None, masks=None, pointsdist=True):
    """-> (pointsdist [b] or None, l2_xyz [] or None) of img_xyz [b, v, 3, h, w] on a CUDA device.  pointsdist needs ray_o
    [b, v, 3, h, w]; l2_xyz is computed when gt_xyz [b, v, 3, h, w] and masks [b, v, 1, h, w] are both given."""
    if img_xyz.dim() != 5 or img_xyz.shape[2] != 3:
        raise ValueError(f"geometry loss: expected img_xyz [b, v, 3, h, w], got {tuple(img_xyz.shape)}")
    if not img_xyz.is_floating_point():
        raise TypeError(f"geometry loss: expected a floating-point img_xyz, got {img_xyz.dtype}")
    b, v, _, h, w = img_xyz.shape
    want_xyz = gt_xyz is not None and masks is not None
    for name, t, c, need in (("ray_o", ray_o, 3, pointsdist), ("gt_xyz", gt_xyz, 3, want_xyz), ("masks", masks, 1, want_xyz)):
        if not need:
            continue
        if t is None:
            raise ValueError(f"geometry loss: {name} is required")
        if tuple(t.shape) != (b, v, c, h, w):
            raise ValueError(f"geometry loss: expected {name} {(b, v, c, h, w)}, got {tuple(t.shape)}")
        if t.device != img_xyz.device:
            raise _lib.DgsError(f"geometry loss: {name} is on {t.device}, img_xyz on {img_xyz.device}")
    if not img_xyz.is_cuda:
        raise _lib.DgsError("geometry loss needs CUDA tensors (no CPU fallback)")
    if not (pointsdist or want_xyz):
        return None, None
    pd, l2 = _GeometryLossFunction.apply(img_xyz, ray_o if pointsdist else None, gt_xyz if want_xyz else None,
                                         masks if want_xyz else None, bool(pointsdist), want_xyz)
    return (pd if pointsdist else None), (l2 if want_xyz else None)
