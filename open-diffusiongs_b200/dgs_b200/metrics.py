"""Evaluation metrics of the scene results, PSNR / SSIM / LPIPS on the GPU: `MetricComputer` mirrors the reference's
(diffusionGS/utils/losses.py:373-473) and `compute_metrics` / the command line mirror its eval_scene_result.py.

    python -m dgs_b200.metrics --path RESULTS_DIR [--chunk 8] --lpips-checkpoint CKPT

reads every `*.pt` in RESULTS_DIR ({"render_images": [V, 3, H, W], "image": [V, 3, H, W]}, written by an evaluation run
with save_result_for_eval), prints `psnr: ..., ssim: ..., lpips: ...` and writes RESULTS_DIR/eval_result.json.  SSIM is
skimage's structural_similarity(gaussian_weights=True, win_size=11, channel_axis=0, data_range=1) and PSNR is taken on
the images clamped to [0, 1]; both come from one pass of the SSIM kernel.  LPIPS is the native LPIPS-VGG after a bilinear
resize to 256 x 256, with the weights the reference's checkpoints carry.
"""
import argparse
import json
import os

import torch
import torch.nn as nn
import torch.nn.functional as F

from .ssim import ssim_psnr


class MetricComputer(nn.Module):
    """forward(target, rendering) -> (psnr [n], ssim [n], lpips [n]), fp32, with every leading dimension of the inputs
    flattened into n (the reference's argument order and reshape).  Images must be floating-point and at least 11 x 11,
    for PSNR too (it comes out of the SSIM pass).  `lpips_module` takes the `lpips.LPIPS(net="vgg")`
    call convention, e.g. dgs_b200.lpips.LPIPS.from_checkpoint(path)."""

    def __init__(self, lpips_module):
        super().__init__()
        self.lpips_loss_module = lpips_module
        self.lpips_loss_module.eval()
        for p in self.lpips_loss_module.parameters():
            p.requires_grad = False

    @torch.no_grad()
    def compute_psnr(self, ground_truth, predicted):
        """PSNR of the images clamped to [0, 1], from the SSIM kernel's pass (the same numbers `forward` returns).  Unlike
        the reference's torch expression it therefore needs floating-point images of at least 11 x 11 pixels, as SSIM
        does; smaller or integer images raise ValueError / TypeError."""
        return ssim_psnr(ground_truth, predicted, sample_covariance=True, psnr=True)[1]

    @torch.no_grad()
    def compute_ssim(self, ground_truth, predicted):
        return ssim_psnr(ground_truth, predicted, sample_covariance=True, psnr=False)[0]

    @torch.no_grad()
    def compute_lpips(self, ground_truth, predicted):
        d = self.lpips_loss_module(F.interpolate(predicted, size=[256, 256], mode="bilinear") * 2.0 - 1.0,
                                   F.interpolate(ground_truth, size=[256, 256], mode="bilinear") * 2.0 - 1.0)
        return d.reshape(-1)

    @torch.no_grad()
    def forward(self, target, rendering):
        rendering = rendering.reshape(-1, rendering.shape[-3], rendering.shape[-2], rendering.shape[-1])
        target = target.reshape(-1, target.shape[-3], target.shape[-2], target.shape[-1])
        ssim, psnr = ssim_psnr(target, rendering, sample_covariance=True, psnr=True)
        lpips = self.compute_lpips(target, rendering)
        return psnr, ssim, lpips


def compute_metrics(path, chunk=8, metric_computer=None, lpips_checkpoint=None, device="cuda"):
    """eval_scene_result.py: stacks the "render_images" and "image" of every *.pt file in `path` (in name order), runs
    `metric_computer` over `chunk` scenes at a time, prints the averages and writes `path`/eval_result.json (keys psnr,
    ssim, lpips; indent 4).  Without a `metric_computer`, one is built from `lpips_checkpoint`.  -> the written dict."""
    if metric_computer is None:
        if lpips_checkpoint is None:
            raise ValueError("compute_metrics: pass metric_computer or lpips_checkpoint (the LPIPS-VGG weights)")
        from .lpips import LPIPS
        metric_computer = MetricComputer(LPIPS.from_checkpoint(lpips_checkpoint)).to(device)
    renders, gts = [], []
    for name in sorted(os.listdir(path)):
        if name.endswith(".pt"):
            pkg = torch.load(os.path.join(path, name), map_location="cpu")
            renders.append(pkg["render_images"])
            gts.append(pkg["image"])
    if not renders:
        raise FileNotFoundError(f"compute_metrics: no .pt result files in {path}")
    renders, gts = torch.stack(renders), torch.stack(gts)
    all_psnr, all_ssim, all_lpips = [], [], []
    for i in range(0, len(renders), chunk):
        # the reference passes (render_images, image) as forward(target, rendering); every metric is symmetric
        psnr, ssim, lpips = metric_computer(renders[i:i + chunk].to(device), gts[i:i + chunk].to(device))
        all_psnr.append(psnr)
        all_ssim.append(ssim)
        all_lpips.append(lpips)
    avg_psnr = torch.cat(all_psnr, dim=0).mean()
    avg_ssim = torch.cat(all_ssim, dim=0).mean()
    avg_lpips = torch.cat(all_lpips, dim=0).mean()
    print(f"psnr: {avg_psnr}, ssim: {avg_ssim}, lpips: {avg_lpips}")
    result = {"psnr": avg_psnr.item(), "ssim": avg_ssim.item(), "lpips": avg_lpips.item()}
    with open(os.path.join(path, "eval_result.json"), "w") as f:
        json.dump(result, f, indent=4)
    return result


def main(argv=None):
    ap = argparse.ArgumentParser(description="PSNR / SSIM / LPIPS of a directory of evaluation results (*.pt)")
    ap.add_argument("--path", required=True, help="directory of the .pt result files; eval_result.json is written there")
    ap.add_argument("--chunk", type=int, default=8, help="scenes per metric call (default 8)")
    ap.add_argument("--lpips-checkpoint", required=True,
                    help="checkpoint holding the LPIPS-VGG weights (loss_computer.lpips_loss_module.*)")
    args = ap.parse_args(argv)
    compute_metrics(args.path, chunk=args.chunk, lpips_checkpoint=args.lpips_checkpoint)


if __name__ == "__main__":
    main()
