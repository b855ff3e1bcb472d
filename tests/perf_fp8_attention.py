"""Times the FP8 attention against the bf16 one on the GPU and prints one JSON line (a script, not a test):

    python tests/perf_fp8_attention.py [--windows 5] [--iters 20] [--steps 5]

* kernels, B = 1, 16 heads, N = 4098 (obj-256) and 16386 (obj-512 / scene-512): the bf16 attention forward, the FP8
  attention forward and the quantize pass, each timed with CUDA events over `iters` launches, in `windows` windows that
  alternate bf16 and FP8; reported as the median window and the spread (max - min) over windows, in microseconds;
* the DiT forward (24 layers) at obj-256 and obj-512 in "fp8" against "fp8_attention", alternating, with L2 flushed
  before every step; median and spread of the per-step times, in milliseconds.
The card's name, power limit and maximum SM clock are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "open-diffusiongs_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

DEV = "cuda:0"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (s.strip() for s in q.stdout.strip().splitlines()[0].split(","))
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def _time(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / iters  # us per call


def kernels(N, windows, iters, H=16, B=1):
    from dgs_b200 import _lib
    L, st = _lib.lib(), _lib.stream(DEV)
    g = torch.Generator(DEV).manual_seed(0)
    qkv = (torch.randn(B, N, 3 * H * 64, device=DEV, generator=g) * 1.5).to(torch.bfloat16)
    out = torch.empty(B, N, H * 64, dtype=torch.bfloat16, device=DEV)
    Nk = (N + 127) // 128 * 128
    u8 = lambda *s: torch.empty(*s, dtype=torch.uint8, device=DEV)  # noqa: E731
    q8, k8, vt8 = u8(B, N, H, 64), u8(B, N, H, 64), u8(B, H, 64, Nk)
    sq, sk, sv = (torch.empty(B, H, n, device=DEV) for n in (N, Nk // 128, Nk // 128))
    ops = [p.data_ptr() for p in (q8, k8, vt8, sq, sk, sv)]
    runs = {
        "bf16": lambda: _lib.check(L.dgs_attention_fwd(qkv.data_ptr(), out.data_ptr(), B, N, H, st)),
        "quantize": lambda: _lib.check(L.dgs_attention_quantize_e4m3(qkv.data_ptr(), *ops, B, N, H, st)),
        "fp8": lambda: _lib.check(L.dgs_attention_fwd_fp8(*ops, out.data_ptr(), B, N, H, st)),
    }
    for fn in runs.values():  # warm-up (module load, tensor-map set-up)
        _time(fn, 3)
    t = {k: [] for k in runs}
    for _ in range(windows):
        for k, fn in runs.items():
            t[k].append(_time(fn, iters))
    res = {k: dict(median_us=statistics.median(v), spread_us=max(v) - min(v)) for k, v in t.items()}
    fp8_total = [f + q for f, q in zip(t["fp8"], t["quantize"])]
    flop = 4.0 * B * H * N * N * 64
    res["fp8_plus_quantize"] = dict(median_us=statistics.median(fp8_total), spread_us=max(fp8_total) - min(fp8_total))
    res["bf16_tflops"] = flop / res["bf16"]["median_us"] / 1e6
    res["fp8_tflops"] = flop / res["fp8"]["median_us"] / 1e6
    res["speedup_incl_quantize"] = res["bf16"]["median_us"] / res["fp8_plus_quantize"]["median_us"]
    return res


def dit(res_hw, steps, layers=24):
    from dgs_b200.denoiser import DGSDenoiser
    from dit_regime import dit_inputs
    torch.manual_seed(0)
    model = DGSDenoiser(dict(patch_size=8, num_layers=layers)).to(DEV).eval()
    inputs = dit_inputs(1, 4, res_hw, res_hw, seed=0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)  # > the 50 MB L2
    t = {"fp8": [], "fp8_attention": []}
    with torch.no_grad():
        for mode in t:  # warm-up: weights packed, workspace sized
            model.set_inference_precision(mode)
            model.image_to_gaussians(*inputs)
        for _ in range(steps):
            for mode in t:
                model.set_inference_precision(mode)
                flush.zero_()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                model.image_to_gaussians(*inputs)
                b.record()
                b.synchronize()
                t[mode].append(a.elapsed_time(b))
    del model
    torch.cuda.empty_cache()
    res = {k: dict(median_ms=statistics.median(v), spread_ms=max(v) - min(v)) for k, v in t.items()}
    res["speedup"] = res["fp8"]["median_ms"] / res["fp8_attention"]["median_ms"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--kernels-only", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_fp8_attention.py needs a CUDA GPU")
    out = card()
    out["kernels"] = {str(N): kernels(N, a.windows, a.iters) for N in (4098, 16386)}
    if not a.kernels_only:
        out["dit_forward"] = {"obj-256": dit(256, a.steps), "obj-512": dit(512, a.steps)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
