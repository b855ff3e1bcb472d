"""The DiT block's forward kernels at the obj-256 shapes on the H100 (not a pytest file; bench.py measures the step).
    python tests/perf_dit_linears.py [--baseline-lib PATH] [--out perf_dit_linears.json]
* the four block linears at M = 4098 tokens, B = 1, with their product epilogues (qkv: bias -> bf16, attn.proj and
  mlp.fc2: in-place gate + residual into fp32, mlp.fc1: bias + GELU -> bf16), the attention forward (16 heads), and
  torch.matmul in bf16 at the same GEMM shapes as a cuBLAS point of comparison;
* median time from CUDA events over windows of 20 launches, the variants alternating window by window; with
  --baseline-lib (a libdgs_b200.so of another build) that build's kernels take part as variant "baseline";
* TFLOP/s from the shapes, and the bytes per FLOP that a 128 x BN tile streams from L2 into shared memory
  ((128 + BN) / (128 BN)) with the L2 -> SM bandwidth that implies at the measured rate, for BN = 128 and 256;
* the card's name, power.limit and clocks.sm / clocks.max.sm, read in the same run before and after.
Prints one JSON line."""
import ctypes as C
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "open-diffusiongs_b200"))
from dgs_b200 import _lib  # noqa: E402

DEV = "cuda:0"
M, D, H = 4098, 1024, 16


def st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [s.strip() for s in r.split(",")]))
    except Exception as e:  # noqa: BLE001
        return dict(error=str(e))


def load_lib(path):
    """A second, separately configured handle on the library at path."""
    saved, saved_path = _lib._lib, _lib.LIB_PATH
    try:
        _lib._lib, _lib.LIB_PATH = None, os.path.abspath(path)
        return _lib.lib()
    finally:
        _lib._lib, _lib.LIB_PATH = saved, saved_path


def alternate(fns, windows=10, per_window=20):
    """{name: median ms}: the functions take turns in windows of per_window timed calls each."""
    for f in fns.values():
        for _ in range(5):
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    for _ in range(windows):
        for k, f in fns.items():
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(per_window)]
            for a, b in ev:
                a.record()
                f()
                b.record()
            torch.cuda.synchronize()
            times[k] += [a.elapsed_time(b) for a, b in ev]
    return {k: sorted(v)[len(v) // 2] for k, v in times.items()}


def main():
    libs = dict(this=_lib.lib())
    if "--baseline-lib" in sys.argv:
        libs["baseline"] = load_lib(sys.argv[sys.argv.index("--baseline-lib") + 1])
    g = torch.Generator(DEV).manual_seed(0)
    res = dict(card=card(), shapes=dict(M=M, D=D, heads=H), gemm={})
    mod = torch.randn(1, 6 * D, device=DEV, generator=g) * 0.1  # gate = a row of the adaLN table
    for name, N, K, epi in (("qkv", 3 * D, D, 0), ("proj", D, D, 2), ("fc1", 4 * D, D, 1), ("fc2", D, 4 * D, 2)):
        A = torch.randn(M, K, device=DEV, generator=g).to(torch.bfloat16)
        W = (torch.randn(N, K, device=DEV, generator=g) / K ** 0.5).to(torch.bfloat16)
        bias = torch.randn(N, device=DEV, generator=g) * 0.1
        out = torch.zeros(M, N, dtype=torch.float32 if epi == 2 else torch.bfloat16, device=DEV)
        gate = mod[:, 2 * D:].data_ptr() if epi == 2 else None

        def ours(L):
            return lambda: _lib.check(L.dgs_gemm_bf16(A.data_ptr(), W.data_ptr(), bias.data_ptr(), gate, out.data_ptr(), M,
                                                      N, K, epi, N, mod.stride(0), M, st()))
        fns = {k: ours(L) for k, L in libs.items()}
        fns["torch_matmul_bf16"] = lambda: torch.matmul(A, W.t())
        t = alternate(fns)
        fl = 2.0 * M * N * K
        r = {}
        for k, ms in t.items():
            tf = fl / ms / 1e9
            r[k] = dict(ms=round(ms, 5), tflops=round(tf, 1),
                        l2_to_smem_tb_s={f"128x{bn}": round(tf * (128 + bn) / (128 * bn), 2) for bn in (128, 256)})
        res["gemm"][name] = r
    qkv = (torch.randn(1, M, 3, H, 64, device=DEV, generator=g)).to(torch.bfloat16)
    o = torch.zeros(1, M, H * 64, dtype=torch.bfloat16, device=DEV)

    def att(L):
        return lambda: _lib.check(L.dgs_attention_fwd(qkv.data_ptr(), o.data_ptr(), 1, M, H, st()))
    t = alternate({k: att(L) for k, L in libs.items()})
    fl = 4.0 * M * M * D
    res["attention"] = {k: dict(ms=round(ms, 5), tflops=round(fl / ms / 1e9, 1)) for k, ms in t.items()}
    res["bytes_per_flop"] = {f"128x{bn}": (128 + bn) / (128 * bn) for bn in (128, 256)}
    res["card_after"] = card()
    line = json.dumps(res)
    print(line, flush=True)
    if "--out" in sys.argv:
        with open(sys.argv[sys.argv.index("--out") + 1], "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
