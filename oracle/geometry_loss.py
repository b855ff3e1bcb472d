"""fp64 oracle of the geometry loss terms (diffusionGS/utils/losses.py:286-291, 323-364) and of their gradient w.r.t.
img_aligned_xyz, by torch autograd on the reference's formulas.  Runs on any device."""
import torch
import torch.nn.functional as F


def geometry_losses64(img_xyz, ray_o, gt_xyz=None, masks=None, pointsdist=True):
    """-> (pointsdist [b] or None, l2_xyz [] or None) in fp64, differentiable in img_xyz (whatever its dtype)."""
    x = img_xyz if img_xyz.dtype == torch.float64 else img_xyz.double()
    pd = l2 = None
    if pointsdist:
        o = ray_o.double()
        trgt_mean = torch.norm(o, dim=2, p=2, keepdim=True)
        dist = (x - o).norm(dim=2, p=2, keepdim=True)
        dd = dist.detach()
        trgt = (dd - dd.mean(dim=(2, 3, 4), keepdim=True)) / (dd.std(dim=(2, 3, 4), keepdim=True) + 1e-8) * 0.5 + trgt_mean
        pd = ((dist - trgt) ** 2).mean(dim=(1, 2, 3, 4))
    if gt_xyz is not None and masks is not None:
        m = masks.double()
        l2 = F.mse_loss(x * m, gt_xyz.double() * m, reduction="sum") / m.sum()
    return pd, l2


def geometry_grad64(img_xyz, ray_o, gt_xyz=None, masks=None, g_pd=None, g_xyz=None):
    """-> (pointsdist, l2_xyz, d_img) in fp64: the values, and the gradient of sum_b g_pd[b] pointsdist[b] + g_xyz l2_xyz
    w.r.t. img_xyz (g_pd [b] / g_xyz scalar; a term whose weight is None is left out of both)."""
    x = img_xyz.detach().double().requires_grad_(True)
    pd, l2 = geometry_losses64(x, ray_o, gt_xyz if g_xyz is not None else None, masks if g_xyz is not None else None,
                               pointsdist=g_pd is not None)
    loss = 0.0
    if pd is not None:
        loss = loss + (pd * torch.as_tensor(g_pd, dtype=torch.float64, device=x.device)).sum()
    if l2 is not None:
        loss = loss + l2 * float(g_xyz)
    d = torch.autograd.grad(loss, x)[0] if torch.is_tensor(loss) else torch.zeros_like(x)
    return (None if pd is None else pd.detach()), (None if l2 is None else l2.detach()), d
