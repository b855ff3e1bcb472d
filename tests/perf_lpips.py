"""Times the LPIPS-VGG loss term, forward + input-gradient backward, at 256 x 256 (what LossComputer feeds it).

    python tests/perf_lpips.py [--n 40 80] [--iters 20] [--repeats 5] [--out perf_lpips.json]

Reports, for each batch size n, the native module (dgs_b200.lpips.LPIPS) and, for comparison only, the same distance run
by torch/cuDNN (oracle/lpips.py's functional form) in fp32 (TF32 off) and under bf16 autocast with channels-last inputs.
TFLOP/s are computed from the shapes: the 13 convolutions of both inputs' forward plus the input gradient of the first
(3x the forward FLOPs of one input).  Each configuration is warmed up, then timed in `repeats` windows of `iters` calls
(CUDA events around each window); the minimum and median per-call times of the windows are reported, the three
implementations alternating window by window.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "open-diffusiongs_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

CHANNELS = (3, 64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512)
LEVEL = (0, 0, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4)


def forward_flops(H, W):
    """FLOPs of VGG16 features[0:30] on one image (2 per multiply-add)."""
    return sum(2 * (H >> LEVEL[l]) * (W >> LEVEL[l]) * CHANNELS[l + 1] * 9 * CHANNELS[l] for l in range(13))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def time_window(fn, iters):
    """-> ms per call over one window of `iters` calls"""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[40, 80])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default="perf_lpips.json")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_lpips.py measures on a GPU"
    from dgs_b200.lpips import LPIPS
    from lpips_regime import random_lpips_state_dict
    from oracle.lpips import LPIPSOracle
    dev = "cuda"
    H = W = 256
    sd = random_lpips_state_dict(0)
    native = LPIPS.from_state_dict(sd).to(dev)
    ref = LPIPSOracle(sd, dtype=torch.float32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    res = dict(card=card(), H=H, W=W, results=[])
    print(f"card: {res['card']}")
    for n in args.n:
        g = torch.Generator(dev).manual_seed(n)
        in0 = torch.rand(n, 3, H, W, device=dev, generator=g) * 2 - 1
        in1 = torch.rand(n, 3, H, W, device=dev, generator=g) * 2 - 1
        flop = 3 * n * forward_flops(H, W)

        def step(mod, autocast=False, channels_last=False):
            def run():
                x = in0.clone()
                y = in1
                if channels_last:
                    x, y = x.contiguous(memory_format=torch.channels_last), y.contiguous(memory_format=torch.channels_last)
                x.requires_grad_(True)
                with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
                    out = mod(x, y)
                out.sum().backward()
            return run
        row = dict(n=n, gflop=flop / 1e9)
        impls = (("native", step(native)), ("torch_fp32", step(ref)),
                 ("torch_bf16_autocast_channels_last", step(ref, True, True)))
        for _, fn in impls:  # warm-up: module load, cuDNN algorithm choice, allocator
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        windows = {name: [] for name, _ in impls}
        for _ in range(args.repeats):
            for name, fn in impls:
                windows[name].append(time_window(fn, args.iters))
        for name, _ in impls:
            w = sorted(windows[name])
            lo, med = w[0], w[len(w) // 2]
            row[name] = dict(ms_min=lo, ms_median=med, ms_windows=windows[name], tflops_median=flop / med / 1e9)
            print(f"n={n:3d} {name:36s} min {lo:9.2f} ms  median {med:9.2f} ms  ({flop / med / 1e9:6.1f} TFLOP/s at the "
                  f"median, {args.repeats} windows of {args.iters})")
        res["results"].append(row)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
