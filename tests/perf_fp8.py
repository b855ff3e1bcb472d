"""FP8 vs bf16 inference on the H100 (not a pytest file; bench.py keeps measuring the default bf16 path).
    python tests/perf_fp8.py [--out perf_fp8.json]
* per GEMM (qkv, mlp.fc1, mlp.fc2 at N = 4098 tokens, B = 1, with their product epilogues): median time over 200
  launches from CUDA events, bf16 and FP8 alternating in windows of 20, and TFLOP/s against the data-sheet dense peaks
  (989 bf16 / 1,979 FP8 TFLOP/s for an H100 SXM at 700 W; labelled as data-sheet figures, not reached ones);
* the whole obj-256 denoise step (24 blocks, 4 views at 256 x 256 -> 4098 tokens, B = 1): bf16 and FP8 in alternating
  windows of 10 steps, the L2 flushed (a 256 MB write) before every step, events around the step only;
* the card's name, power.limit and clocks.max.sm, read in the same run.
Prints one JSON line."""
import ctypes as C
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "open-diffusiongs_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from dgs_b200 import _lib  # noqa: E402

DEV = "cuda:0"
PEAK = dict(bf16=989.0, fp8=1979.0)  # data sheet, H100 SXM, dense


def st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
        name, pl, clk = [s.strip() for s in r.split(",")]
        return dict(name=name, power_limit=pl, clocks_max_sm=clk)
    except Exception as e:  # noqa: BLE001
        return dict(error=str(e))


def alternate(fns, windows, per_window, flush=None):
    """{name: median ms}: the functions take turns in windows of per_window timed calls each."""
    for f in fns.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    for _ in range(windows):
        for k, f in fns.items():
            ev = []
            for _ in range(per_window):
                if flush is not None:
                    flush()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                f()
                b.record()
                ev.append((a, b))
            torch.cuda.synchronize()
            times[k] += [a.elapsed_time(b) for a, b in ev]
    return {k: sorted(v)[len(v) // 2] for k, v in times.items()}


def gemms(L):
    M, D = 4098, 1024
    Ms = (M + 3) // 4 * 4
    out = {}
    for name, N, K, epi_bf, epi_f8 in (("qkv", 3 * D, D, 0, 0), ("fc1", 4 * D, D, 1, 6), ("fc2", D, 4 * D, 2, 2)):
        A = torch.randn(M, K, device=DEV).to(torch.bfloat16)
        W = (torch.randn(N, K, device=DEV) / K ** 0.5).to(torch.bfloat16)
        bias = torch.randn(N, device=DEV) * 0.1
        gate = torch.randn(1, N, device=DEV) * 0.1
        A8 = torch.randint(0, 120, (M, K), dtype=torch.uint8, device=DEV)
        sa = torch.ones(K // 128, Ms, device=DEV)
        W8 = torch.empty(N, K, dtype=torch.uint8, device=DEV)
        sw = torch.empty(N, device=DEV)
        _lib.check(L.dgs_quantize_rows_e4m3(W.float().contiguous().data_ptr(), N, K, W8.data_ptr(), sw.data_ptr(), st()))
        o_bf = torch.zeros(M, N, dtype=torch.float32 if epi_bf == 2 else torch.bfloat16, device=DEV)
        o_f8 = torch.zeros(M, N, dtype={0: torch.bfloat16, 2: torch.float32, 6: torch.uint8}[epi_f8], device=DEV)
        s_out = torch.empty(N // 128, Ms, device=DEV)
        g = gate.data_ptr() if epi_bf == 2 else None

        def bf():
            _lib.check(L.dgs_gemm_bf16(A.data_ptr(), W.data_ptr(), bias.data_ptr(), g, o_bf.data_ptr(), M, N, K, epi_bf, N, 0,
                                       M, st()))

        def f8():
            _lib.check(L.dgs_gemm_fp8(A8.data_ptr(), sa.data_ptr(), W8.data_ptr(), sw.data_ptr(), bias.data_ptr(), g,
                                      o_f8.data_ptr(), s_out.data_ptr() if epi_f8 == 6 else None, M, N, K, epi_f8, N, 0, M,
                                      st()))
        t = alternate(dict(bf16=bf, fp8=f8), windows=10, per_window=20)
        fl = 2.0 * M * N * K
        out[name] = {k: dict(ms=v, tflops=fl / v / 1e9, of_datasheet_peak=fl / v / 1e9 / PEAK[k]) for k, v in t.items()}
        out[name]["speedup"] = t["bf16"] / t["fp8"]
    return out


def step_times():
    from dgs_b200.denoiser import DGSDenoiser
    from test_dit_gpu import _inputs
    torch.manual_seed(0)
    model = DGSDenoiser(dict(patch_size=8, num_layers=24)).to(DEV).eval()
    inputs = _inputs(1, 4, 256, 256, seed=0)
    scratch = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=DEV)

    def run(prec):
        def f():
            model.set_inference_precision(prec)
            with torch.no_grad():
                model.image_to_gaussians(*inputs)
        return f
    t = alternate(dict(bf16=run("bf16"), fp8=run("fp8")), windows=6, per_window=10, flush=lambda: scratch.fill_(1))
    return dict(t, speedup=t["bf16"] / t["fp8"])


def main():
    L = _lib.lib()
    res = dict(card=card(), gemm_n4098=gemms(L), obj256_step_ms=step_times(), card_after=card())
    line = json.dumps(res)
    print(line, flush=True)
    if "--out" in sys.argv:
        with open(sys.argv[sys.argv.index("--out") + 1], "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
