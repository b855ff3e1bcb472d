"""Times SSIM: the training loss (SsimLoss forward + input-gradient backward at 256 x 256) and the evaluation metric
(MetricComputer's SSIM + PSNR at 512 x 512).

    python tests/perf_ssim.py [--iters 20] [--repeats 5] [--cpu-images 4] [--out perf_ssim.json]

For each configuration, the native path (dgs_b200.ssim) and, for comparison only, pytorch_msssim's arithmetic on
torch F.conv2d in fp32 (TF32 off, oracle.ssim.ssim_torch32, autograd for the backward) on the same card.  For the metric,
also skimage's float32 scipy path on the CPU (oracle.ssim.ssim_scipy32, what the reference's evaluation runs), timed on
`--cpu-images` images and scaled to n.  Each GPU configuration is warmed up, then timed in `repeats` windows of `iters`
calls (CUDA events around each window), the implementations alternating window by window; the minimum and median
per-call times are reported.  Bytes and FLOPs are counted from the shapes; the card's name, power limit and max SM clock
are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "open-diffusiongs_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

HBM_TBS, FP32_TFLOPS = 3.35, 67.0  # H100 SXM data sheet (700 W)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def cost(n, H, W, train):
    """-> (bytes, flops) the native kernels need.  Forward: x and y read once; per channel and valid pixel 5 moments x
    11 taps x 2 passes (2 FLOPs each, the horizontal pass over 42/32 of the rows) + ~40 for S.  Training adds 3 fp32 maps
    written; the backward reads x, y and the maps, writes d x, and runs 3 maps x 11 taps x 2 passes per pixel."""
    px, v = n * 3 * H * W, n * 3 * (H - 10) * (W - 10)
    b = 2 * 4 * px
    f = v * (5 * 11 * 2 * (1 + 42 / 32) + 40)
    if train:
        b += 3 * 4 * v + 3 * 4 * v + 3 * 4 * px
        f += px * (3 * 11 * 2 * (1 + 42 / 32) + 6)
    return b, f


def time_window(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def run_config(name, impls, iters, repeats, nbytes, flops):
    for _, fn in impls:
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    windows = {k: [] for k, _ in impls}
    for _ in range(repeats):
        for k, fn in impls:
            windows[k].append(time_window(fn, iters))
    row = dict(config=name, mbytes=nbytes / 1e6, gflop=flops / 1e9)
    floor_ms = max(nbytes / (HBM_TBS * 1e12), flops / (FP32_TFLOPS * 1e12)) * 1e3
    row["bound"] = "HBM" if nbytes / HBM_TBS > flops / FP32_TFLOPS else "fp32"
    row["floor_ms"] = floor_ms
    for k, _ in impls:
        w = sorted(windows[k])
        row[k] = dict(ms_min=w[0], ms_median=w[len(w) // 2], ms_windows=windows[k])
        extra = ""
        if k == "native":
            extra = (f"  {nbytes / w[len(w) // 2] / 1e6:7.1f} GB/s, {flops / w[len(w) // 2] / 1e9:6.2f} TFLOP/s, "
                     f"{100 * floor_ms / w[len(w) // 2]:4.1f} % of the {row['bound']} data-sheet floor")
        print(f"{name:34s} {k:12s} min {w[0]:8.3f} ms  median {w[len(w) // 2]:8.3f} ms{extra}")
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--cpu-images", type=int, default=4)
    ap.add_argument("--out", default="perf_ssim.json")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_ssim.py measures on a GPU"
    from dgs_b200.ssim import SsimLoss, ssim_psnr
    from oracle.ssim import SAMPLE_COV, ssim_scipy32, ssim_torch32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    dev = "cuda"
    res = dict(card=card(), results=[])
    print(f"card: {res['card']}")
    native_loss = SsimLoss()

    def images(n, H, W):
        g = torch.Generator(dev).manual_seed(n)
        y = torch.rand(n, 3, H, W, device=dev, generator=g)
        return (y + 0.1 * torch.randn(n, 3, H, W, device=dev, generator=g)).clamp(0, 1), y

    for n in (32, 128):
        H = W = 256
        x, y = images(n, H, W)

        def train_step(loss_fn):
            def run():
                xg = x.clone().requires_grad_(True)
                loss_fn(xg, y).sum().backward()
            return run
        b, f = cost(n, H, W, True)
        res["results"].append(run_config(f"SsimLoss fwd+bwd 256^2 n={n}", (
            ("native", train_step(native_loss)), ("torch_fp32", train_step(lambda a, c: 1 - ssim_torch32(a, c)))),
            args.iters, args.repeats, b, f))
    n, H, W = 64, 512, 512
    x, y = images(n, H, W)

    def torch_metric():
        with torch.no_grad():
            ssim_torch32(x, y, k=SAMPLE_COV)
            (-10 * torch.log10(((x.clamp(0, 1) - y.clamp(0, 1)) ** 2).mean(dim=(1, 2, 3))))
    b, f = cost(n, H, W, False)
    row = run_config(f"metric SSIM+PSNR 512^2 n={n}", (
        ("native", lambda: ssim_psnr(x, y, sample_covariance=True, psnr=True)), ("torch_fp32", torch_metric)),
        args.iters, args.repeats, b, f)
    k = max(1, min(args.cpu_images, n))
    xc, yc = x[:k].cpu(), y[:k].cpu()
    ts = []
    for _ in range(3):
        t0 = time.perf_counter()
        ssim_scipy32(xc, yc)
        ts.append(time.perf_counter() - t0)
    ms = min(ts) * 1e3 / k * n
    row["scipy_cpu_float32"] = dict(ms_scaled_to_n=ms, images_timed=k, cpu_count=os.cpu_count())
    print(f"{row['config']:34s} scipy (CPU)  {ms:8.1f} ms for n={n} (scaled from {k} images, min of 3, single thread)")
    res["results"].append(row)
    with open(args.out, "w") as fo:
        json.dump(res, fo, indent=1)


if __name__ == "__main__":
    main()
