"""Times the geometry loss terms (pointsdist + l2_xyz) at obj-256 and obj-512 (B = 4, V = 4).

    python tests/perf_geometry_loss.py [--iters 20] [--repeats 5] [--steps 4] [--out perf_geometry_loss.json]

1. The forward + backward kernel pair (dgs_b200.geometry_loss) against the torch-ops path it replaces (the reference's
   expressions in fp32 with autograd), alternating window by window (CUDA events around each window of `iters` calls).
2. One DitTrainer step (recompute mode, the full 24-layer model: DiT forward, fused render + loss, backward, AdamW) with
   the MSE alone and with MSE + pointsdist + 0.025 xyz, alternating step by step over `steps` timed steps each.
Minimum and median per-call times are reported, with the bytes the kernels must move (HBM bound at 3.35 TB/s, the H100
SXM data sheet); the card's name, power limit and max SM clock are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "open-diffusiongs_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

HBM_TBS = 3.35
DEV = "cuda:0"


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def kernel_bytes(B, V, H, W):
    """pass 1 reads img, o, gt (3 ch each) and m; pass 2 img and o; the backward img, o, gt, m and writes d_img"""
    px = B * V * H * W
    return 4 * px * ((3 + 3 + 3 + 1) + (3 + 3) + (3 + 3 + 3 + 1 + 3))


def inputs(B, V, H, W):
    g = torch.Generator(DEV).manual_seed(0)
    o = (torch.randn(B, V, 3, 1, 1, device=DEV, generator=g) * 1.5).expand(B, V, 3, H, W).contiguous()
    d = torch.nn.functional.normalize(torch.randn(B, V, 3, H, W, device=DEV, generator=g), dim=2)
    x = o + d * (2.7 + 0.3 * torch.randn(B, V, 1, H, W, device=DEV, generator=g))
    gt = o + d * (2.7 + 0.3 * torch.rand(B, V, 1, H, W, device=DEV, generator=g))
    m = (torch.rand(B, V, 1, H, W, device=DEV, generator=g) > 0.4).float()
    return x.requires_grad_(True), o, gt, m


def native_pair(x, o, gt, m):
    from dgs_b200.geometry_loss import geometry_losses
    pd, l2 = geometry_losses(x, o, gt, m)
    return torch.autograd.grad(pd.mean() + 0.025 * l2, x)[0]


def torch_pair(x, o, gt, m):
    dist = (x - o).norm(dim=2, p=2, keepdim=True)
    dd = dist.detach()
    trgt = (dd - dd.mean(dim=(2, 3, 4), keepdim=True)) / (dd.std(dim=(2, 3, 4), keepdim=True) + 1e-8) * 0.5 + \
        torch.norm(o, dim=2, p=2, keepdim=True)
    pd = ((dist - trgt) ** 2).mean(dim=(1, 2, 3, 4))
    l2 = torch.nn.functional.mse_loss(x * m, gt * m, reduction="sum") / m.sum()
    return torch.autograd.grad(pd.mean() + 0.025 * l2, x)[0]


def time_window(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def summary(ts):
    return dict(min_ms=min(ts), median_ms=statistics.median(ts))


def bench_kernels(B, V, H, iters, repeats):
    args = inputs(B, V, H, H)
    fns = dict(native=lambda: native_pair(*args), torch=lambda: torch_pair(*args))
    for f in fns.values():
        time_window(f, 3)
    ts = {k: [] for k in fns}
    for _ in range(repeats):
        for k, f in fns.items():
            ts[k].append(time_window(f, iters))
    out = {k: summary(v) for k, v in ts.items()}
    nb = kernel_bytes(B, V, H, H)
    out["native"]["bytes"] = nb
    out["native"]["hbm_bound_ms"] = nb / (HBM_TBS * 1e12) * 1e3
    return out


def bench_step(B, V, H, steps):
    from dgs_b200 import synth
    from dgs_b200.denoiser import DGSDenoiser
    from dgs_b200.losses import LossComputer, fused_render_and_loss
    from dgs_b200.train import DitTrainer
    from dit_regime import dit_inputs
    torch.manual_seed(0)
    model = DGSDenoiser(dict(patch_size=8)).to(DEV)
    trainer = DitTrainer(model, recompute=True)
    model.train()
    images, ray_o, ray_d, t = dit_inputs(B, V, H, H)
    c2w, fx = synth.orbit_cameras(V, H, H)
    c2w = torch.tensor(c2w[None], device=DEV).expand(B, -1, -1, -1).contiguous()
    fx = torch.tensor(fx[None], device=DEV).expand(B, -1, -1).contiguous()
    g = torch.Generator(DEV).manual_seed(1)
    target = torch.rand(B, V, 3, H, H, device=DEV, generator=g)
    gt = ray_o + ray_d * (2.7 + 0.3 * torch.rand(B, V, 1, H, H, device=DEV, generator=g))
    m = (torch.rand(B, V, 1, H, H, device=DEV, generator=g) > 0.4).float()
    variants = dict(mse=(LossComputer(), dict(lambda_diffusion=1.0)),
                    mse_geometry=(LossComputer(compute_pointsdist=True),
                                  dict(lambda_diffusion=1.0, lambda_pointsdist=1.0, lambda_xyz=0.025)))

    def step(lc, lambdas):
        out, img = model.image_to_gaussians(images, ray_o, ray_d, t)
        trainer.zero_grad()
        losses, _ = fused_render_and_loss(model, out, c2w, fx, H, H, target, loss_computer=lc, lambdas=lambdas,
                                          ray_o=ray_o, masks_all=m, masks=m, img_aligned_xyz=img, gt_img_aligned_xyz=gt)
        losses["loss"].backward()
        trainer.optimizer_step(allreduce=False)

    for v in variants.values():
        time_window(lambda: step(*v), 1)
    ts = {k: [] for k in variants}
    for _ in range(steps):
        for k, v in variants.items():
            ts[k].append(time_window(lambda: step(*v), 1))
    del model, trainer
    torch.cuda.empty_cache()
    return {k: summary(v) for k, v in ts.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--out", default="perf_geometry_loss.json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_geometry_loss needs a CUDA device")
    res = dict(card=card())
    print(res["card"])
    for name, H in (("obj-256", 256), ("obj-512", 512)):
        r = dict(kernels=bench_kernels(4, 4, H, a.iters, a.repeats), step=bench_step(4, 4, H, a.steps))
        res[name] = r
        k, s = r["kernels"], r["step"]
        print(f"{name} B=4 V=4: fwd+bwd native {k['native']['median_ms']:.3f} ms (min {k['native']['min_ms']:.3f}, "
              f"HBM bound {k['native']['hbm_bound_ms']:.3f}) vs torch ops {k['torch']['median_ms']:.3f} ms; "
              f"trainer step mse {s['mse']['median_ms']:.1f} ms, mse + geometry {s['mse_geometry']['median_ms']:.1f} ms")
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
