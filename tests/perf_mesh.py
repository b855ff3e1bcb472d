"""Times mesh extraction: the opacity field (dgs_mesh_field) and marching cubes (dgs_marching_cubes) at 256^3 with
64 blocks per axis, for 262,146 and 1,048,578 Gaussians on an object-like shell (the obj-256 and obj-512 pipelines'
counts), and, for comparison only, a torch-on-GPU restatement of the reference's per-block loop (gs_core.py:786-852).

    python tests/perf_mesh.py [--iters 5] [--repeats 5] [--ref-blocks 1024] [--out perf_mesh.json]

Each native stage is warmed up, then timed in `repeats` windows of `iters` calls (CUDA events); the median and minimum
per-call times are reported with the pair count and point x Gaussian evaluations per second (every point of a block
against every Gaussian of its list).  The reference loop is timed in full at resolution 128 / 32 blocks; at 256 / 64 it is
timed on `--ref-blocks` random blocks and scaled to all blocks ("extrapolated").  The card's name, power limit and SM
clocks are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "open-diffusiongs_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

NAMES = ("xyz", "scaling", "rotation", "opacity")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def timed(fn, iters, repeats):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b) / iters)
    return statistics.median(ms), min(ms)


def reference_loop(t, resolution, num_blocks, blocks=None, relax_ratio=1.5):
    """The reference's extract_fields loop on the GPU in torch (one iteration per block, host sync per block);
    `blocks`: a subset of (xi, yi, zi) to run, else all."""
    from oracle import mesh as om
    xyz, scaling, rotation, opacity = t
    block_size = 2 / num_blocks
    split = resolution // num_blocks
    center, scale, xyzs, opac, inv = om.normalise(xyz, scaling, rotation, opacity)
    covs = torch.stack(om.covariance6(torch.exp(scaling) * scale, rotation), 1)
    occ = torch.zeros([resolution] * 3, dtype=torch.float32, device=xyz.device)
    X = torch.linspace(-1, 1, resolution).split(split)
    todo = blocks if blocks is not None else [(i, j, k) for i in range(len(X)) for j in range(len(X)) for k in range(len(X))]
    for xi, yi, zi in todo:
        xs, ys, zs = X[xi], X[yi], X[zi]
        xx, yy, zz = torch.meshgrid(xs, ys, zs, indexing="ij")
        pts = torch.cat([xx.reshape(-1, 1), yy.reshape(-1, 1), zz.reshape(-1, 1)], dim=-1).to(xyz.device)
        vmin, vmax = pts.amin(0), pts.amax(0)
        vmin -= block_size * relax_ratio
        vmax += block_size * relax_ratio
        mask = (xyzs < vmax).all(-1) & (xyzs > vmin).all(-1)
        if not mask.any():
            continue
        g_pts = pts.unsqueeze(1) - xyzs[mask].unsqueeze(0)
        a, b, c, d, e, f = covs[mask].unbind(1)
        ia, ib, ic, id_, ie, if_ = om.inverse6([a, b, c, d, e, f])
        x, y, z = g_pts.unbind(-1)
        power = -0.5 * (x ** 2 * ia + y ** 2 * id_ + z ** 2 * if_) - x * y * ib - x * z * ic - y * z * ie
        power[power > 0] = -1e10
        val = (opac[mask].view(1, -1) * torch.exp(power)).sum(-1)
        occ[xi * split: xi * split + len(xs), yi * split: yi * split + len(ys), zi * split: zi * split + len(zs)] = \
            val.reshape(len(xs), len(ys), len(zs))
    return occ


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--ref-blocks", type=int, default=1024)
    ap.add_argument("--out", default="perf_mesh.json")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_mesh.py measures on the GPU"
    from dgs_b200 import mesh, synth
    res = {"card": card(), "cases": []}
    for P in (262146, 1048578):
        g = synth.make_shell_gaussians(P, 11)
        t = [torch.tensor(g[k], device="cuda") for k in NAMES]
        occ, _, _, counts, pairs = mesh.opacity_field(*t, resolution=256, num_blocks=64, return_counts=True)
        split = 256 // 64
        evals = int(counts.long().sum()) * split ** 3
        f_med, f_min = timed(lambda: mesh.opacity_field(*t, resolution=256, num_blocks=64), args.iters, args.repeats)
        m_med, m_min = timed(lambda: mesh.marching_cubes(occ, 0.005), args.iters, args.repeats)
        v, f = mesh.marching_cubes(occ, 0.005)
        case = dict(gaussians=P, resolution=256, num_blocks=64, pairs=pairs, nonempty_blocks=int((counts > 0).sum()),
                    point_gaussian_evals=evals, field_ms_median=f_med, field_ms_min=f_min,
                    evals_per_s=evals / (f_med * 1e-3), mc_ms_median=m_med, mc_ms_min=m_min,
                    vertices=int(v.shape[0]), triangles=int(f.shape[0]))
        # the reference loop: whole at 128 / 32, sampled and extrapolated at 256 / 64
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        reference_loop(t, 128, 32)
        torch.cuda.synchronize()
        case["reference_loop_r128_b32_s"] = time.perf_counter() - t0
        rng = np.random.default_rng(0)
        nb = 64 ** 3
        pick = [tuple(int(x) for x in np.unravel_index(i, (64, 64, 64))) for i in rng.choice(nb, args.ref_blocks,
                                                                                                 replace=False)]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        reference_loop(t, 256, 64, pick)
        torch.cuda.synchronize()
        case["reference_loop_r256_b64_s_extrapolated"] = (time.perf_counter() - t0) * nb / args.ref_blocks
        f128, _ = timed(lambda: mesh.opacity_field(*t, resolution=128, num_blocks=32), args.iters, args.repeats)
        case["field_r128_b32_ms_median"] = f128
        print(json.dumps(case), flush=True)
        res["cases"].append(case)
    print(res["card"])
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
