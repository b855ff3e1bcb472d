"""Times screened Poisson reconstruction (dgs_poisson_reconstruct through dgs_b200.mesh.poisson_reconstruction, the
reference's defaults) of the oriented points extract_mesh(method="poisson") builds for the 262,146- and
1,048,578-Gaussian shells (the obj-256 and obj-512 pipelines' counts, as tests/perf_mesh.py) at depth 8 and 9, and
simple_knn's distCUDA2 next to the reference binary (oracle/_ref/simple_knn_ref_C.so, when built) on their centres.

    python tests/perf_poisson.py [--iters 2] [--repeats 5] [--out perf_poisson.json]

Each case is warmed up, then timed in `repeats` windows of `iters` calls (CUDA events around calls that end in a
device synchronise, CUDA tensors in and out); the cases of one size alternate window by window.  The stage split and
the CG iteration count come from the call's own stats (device events between its stages), the peak device memory from
torch's allocator over one call.  The card's name, power limit and SM clocks are read in the same run."""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "open-diffusiongs_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from perf_mesh import card  # noqa: E402


def window(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def alternated(fns, iters, repeats):
    """-> per fn (median, min) ms per call over `repeats` windows, the fns' windows interleaved"""
    for fn in fns.values():
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in fns}
    for _ in range(repeats):
        for k, fn in fns.items():
            ms[k].append(window(fn, iters))
    return {k: (statistics.median(v), min(v)) for k, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default="perf_poisson.json")
    args = ap.parse_args()
    from dgs_b200 import mesh
    from mesh_shapes import shell_model
    from oracle import build_ref_simple_knn
    from simple_knn._C import distCUDA2
    ref = build_ref_simple_knn.load_module()
    free, total = torch.cuda.mem_get_info()
    res = {"card": card(), "device_memory_free_GB": round(free / 1e9, 1), "device_memory_GB": round(total / 1e9, 1),
           "cases": []}
    print(res["card"], res["device_memory_free_GB"], flush=True)
    for P in (262146, 1048578):
        m = shell_model(P, 7, floaters=False)
        c, s = mesh.mesh_frame(m._xyz)
        p, n = mesh.gaussian_points(m._xyz, m._scaling, m._rotation, c, s)
        fns = {f"depth{d}": (lambda d=d: mesh.poisson_reconstruction(p, n, depth=d)) for d in (8, 9)}
        fns["distCUDA2"] = lambda: distCUDA2(m._xyz)
        if ref is not None:
            fns["distCUDA2_reference"] = lambda: ref.distCUDA2(m._xyz)
        times = alternated(fns, args.iters, args.repeats)
        for name, (med, best) in times.items():
            case = {"P": P, "case": name, "median_ms": round(med, 3), "min_ms": round(best, 3)}
            if name.startswith("depth"):
                st = {}
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                v, f = mesh.poisson_reconstruction(p, n, depth=int(name[5:]), stats=st)
                torch.cuda.synchronize()
                case["peak_device_GB"] = round((torch.cuda.max_memory_allocated() - base) / 1e9, 3)
                case["stage_ms"] = {k: round(x, 3) for k, x in st["stage_ms"].items()}
                case.update({k: st[k] for k in ("iterations", "residual", "inliers", "vertices_before", "vertices",
                                                "faces")})
            res["cases"].append(case)
            print(json.dumps(case), flush=True)
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
