"""Loss stage of the training step: host-side mirror of `LossComputer`
(diffusionGS/utils/losses.py:239-369) and of the loss weighting in `System.training_step`
(diffusionGS/systems/diffusion_gs_system.py:94-129, schedule function `C`, utils/misc.py:73-94).

What runs where:
* l2 (lambda_diffusion = 1): FUSED into the rasterizer -- `Renderer.forward_mse` returns the per-sample MSE out of the
  blend-forward kernel and the blend-backward kernel forms dL/dpix = lambda * 2 (c - gt) / n itself
  (dgs_render_batch_forward / _backward with a dgs_render_mse).  `LossComputer.forward(..., l2_loss=...)` takes that value; without it
  the l2 term is computed from the images with torch device ops (same numbers, the unfused form).
* lpips (lambda_lpips 0.5 from step 151 in diffusionGS_rel.yaml, 0.1 in diffusionGS_scene.yaml): `dgs_b200.lpips.LPIPS`, the
  LPIPS-VGG16 distance on the library's kernels, with its weights read from the reference's checkpoints
  (`LPIPS.from_checkpoint(path)`); any module with the `lpips.LPIPS(net="vgg")` call convention (`lpips_module(x, y) ->
  [n,1,1,1]`, inputs in [-1,1] at 256 x 256 as in losses.py:300-303) may be passed instead.  Without one the term is zero
  and `combine` refuses a non-zero lambda_lpips.
* ssim: `dgs_b200.ssim.SsimLoss`, the reference's 1 - pytorch_msssim.SSIM(win_size=11, win_sigma=1.5) on the library's
  kernels (`LossComputer(ssim_module=SsimLoss())`).  Every shipped yaml weights it 0: the reference evaluates it anyway
  and multiplies by 0; here the term is skipped unless a module is supplied, and `combine` refuses a non-zero lambda_ssim
  without one.
* pointsdist (diffusionGS_rel.yaml weights it 1 for global steps 0-149, then 0; the other shipped yamls 0): skipped unless
  `compute_pointsdist=True`.  On CUDA tensors it runs on `dgs_b200.geometry_loss` (dgs_geometry_loss_forward /
  _backward), with its gradient flowing into img_aligned_xyz and, through the DiT backward, into the model.
* l2_xyz (lambda_xyz 0.025 from step 151 in diffusionGS_rel.yaml, from step 0 in diffusionGS_rel_512.yaml): the masked
  MSE over img_aligned_xyz (losses.py:286-291), on the same kernels as pointsdist for CUDA tensors.
On CPU tensors both geometry terms are the reference's torch expressions.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .geometry_loss import geometry_losses


def C(value, epoch: int = 0, global_step: int = 0) -> float:
    """Scalar schedule of utils/misc.py:73-94: a number, or [start_step, start_value, end_value, end_step]
    (3 items: start_step = 0); an int end_step interpolates over global steps, a float end_step over epochs."""
    if isinstance(value, (int, float)):
        return value
    value = list(value)
    if len(value) == 3:
        value = [0] + value
    if len(value) != 4:
        raise TypeError(f"Scalar specification only supports a number or a 3/4-item list, got {value!r}")
    start_step, start_value, end_value, end_step = value
    current = global_step if isinstance(end_step, int) else epoch
    return start_value + (end_value - start_value) * max(min(1.0, (current - start_step) / (end_step - start_step)), 0.0)


class LossComputer(nn.Module):
    """Same call signature and return tuple as the reference's LossComputer.forward:
    (l2_loss [b], lpips_loss [], ssim_loss [b], pointsdist_loss [b], l2_loss_xyz [])."""

    def __init__(self, lpips_module=None, ssim_module=None, compute_pointsdist=False):
        super().__init__()
        self.lpips_loss_module = lpips_module
        self.ssim_loss_module = ssim_module
        self.compute_pointsdist = compute_pointsdist
        for m in (lpips_module, ssim_module):
            if m is not None:
                m.eval()
                for p in m.parameters():
                    p.requires_grad = False  # losses.py:244-258

    def forward(self, rendering, target, masks_all, masks, ray_o, img_aligned_xyz=None, gt_img_aligned_xyz=None,
                l2_loss=None):
        b, v, _, h, w = rendering.size()
        rendering = rendering.reshape(b * v, -1, h, w)
        target = target.reshape(b * v, -1, h, w)
        if target.size(1) == 4:
            target, _mask = target.split([3, 1], dim=1)  # losses.py:274-276 (the mask is not used by the l2 term)
        if l2_loss is None:
            per_el = F.mse_loss(rendering, target, reduction="none").reshape(b, v, -1, h, w)
            l2_loss = per_el.mean(dim=(1, 2, 3, 4))  # losses.py:279-281
        if self.lpips_loss_module is not None:
            lp = self.lpips_loss_module(F.interpolate(rendering, size=[256, 256], mode="bilinear") * 2.0 - 1.0,
                                        F.interpolate(target, size=[256, 256], mode="bilinear") * 2.0 - 1.0)
            lpips_loss = lp.mean()  # losses.py:300-305
        else:
            lpips_loss = torch.zeros((), device=rendering.device)
        if self.ssim_loss_module is not None:
            ssim_loss = self.ssim_loss_module(rendering, target).reshape(b, v).mean(dim=1)  # losses.py:314-318
        else:
            ssim_loss = torch.zeros(b, device=rendering.device)
        want_xyz = img_aligned_xyz is not None and gt_img_aligned_xyz is not None
        want_pd = self.compute_pointsdist and img_aligned_xyz is not None
        pointsdist_loss = l2_loss_xyz = None
        if img_aligned_xyz is not None and img_aligned_xyz.is_cuda:  # both terms from one pass of the geometry kernels
            pointsdist_loss, l2_loss_xyz = geometry_losses(img_aligned_xyz, ray_o, gt_img_aligned_xyz if want_xyz else None,
                                                           masks if want_xyz else None, pointsdist=want_pd)
        else:
            if want_xyz:  # losses.py:286-291
                l2_loss_xyz = F.mse_loss(img_aligned_xyz * masks, gt_img_aligned_xyz * masks, reduction="sum") / masks.sum()
            if want_pd:  # losses.py:323-358
                trgt_mean = torch.norm(ray_o, dim=2, p=2, keepdim=True)
                dist = (img_aligned_xyz - ray_o).norm(dim=2, p=2, keepdim=True)
                dd = dist.detach()
                trgt = (dd - dd.mean(dim=(2, 3, 4), keepdim=True)) / (dd.std(dim=(2, 3, 4), keepdim=True) + 1e-8) * 0.5 + trgt_mean
                pointsdist_loss = ((dist - trgt) ** 2).mean(dim=(1, 2, 3, 4))
        if l2_loss_xyz is None:
            l2_loss_xyz = torch.zeros_like(l2_loss)
        if pointsdist_loss is None:
            pointsdist_loss = torch.zeros(b, device=rendering.device)
        return l2_loss, lpips_loss, ssim_loss, pointsdist_loss, l2_loss_xyz

    def combine(self, losses, lambdas, epoch=0, global_step=0):
        """diffusion_gs_system.py:104-129: total = sum_name mean(loss_name) * C(lambda_name)."""
        l2_loss, lpips_loss, ssim_loss, pointsdist_loss, l2_loss_xyz = losses
        out = dict(loss_diffusion=l2_loss.mean(), loss_lpips=lpips_loss.mean(), loss_ssim=ssim_loss.mean(),
                   loss_xyz=l2_loss_xyz.mean(), loss_pointsdist=pointsdist_loss.mean())
        total = 0.0
        for name, value in out.items():
            lam = C(lambdas.get(name.replace("loss_", "lambda_"), 0.0), epoch, global_step)
            if lam != 0.0:
                if name == "loss_lpips" and self.lpips_loss_module is None:
                    raise RuntimeError("lambda_lpips != 0 but no LPIPS module was supplied "
                                       "(e.g. dgs_b200.lpips.LPIPS.from_checkpoint(path))")
                if name == "loss_ssim" and self.ssim_loss_module is None:
                    raise RuntimeError("lambda_ssim != 0 but no SSIM module was supplied")
                if name == "loss_pointsdist" and not self.compute_pointsdist:
                    raise RuntimeError("lambda_pointsdist != 0 needs LossComputer(compute_pointsdist=True) "
                                       "(diffusionGS_rel.yaml weights it 1 for global steps 0-149)")
                total = total + value * lam
        out["loss"] = total
        return out


def fused_render_and_loss(model, gaussians, c2w, fxfycxcy, height, width, target, loss_computer=None, lambdas=None, ray_o=None,
                          masks_all=None, masks=None, img_aligned_xyz=None, gt_img_aligned_xyz=None, epoch=0, global_step=0):
    """render_gaussians + LossComputer + weighting of the reference's System.forward / training_step
    (diffusion_gs_system.py:91-124) with the MSE fused into the rasterizer.  -> (dict of losses incl. "loss", renderings)."""
    g = gaussians
    lc = loss_computer if loss_computer is not None else LossComputer()
    lambdas = lambdas if lambdas is not None else dict(lambda_diffusion=1.0)
    renderings, l2 = model.gs_renderer.forward_mse(g.xyz, g.features, g.scaling, g.rotation, g.opacity, height, width, c2w, fxfycxcy,
                                                   target)
    extra_terms = lc.lpips_loss_module is not None or lc.ssim_loss_module is not None
    losses = lc(renderings if extra_terms else renderings.detach(), target, masks_all, masks, ray_o, img_aligned_xyz,
                gt_img_aligned_xyz, l2_loss=l2)
    return lc.combine(losses, lambdas, epoch, global_step), renderings
