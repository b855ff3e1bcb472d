"""Times mesh decimation (dgs_mesh_decimate) of the marching-cubes meshes extract_mesh produces for 262,146 and
1,048,578 Gaussians on an object-like shell (the obj-256 and obj-512 pipelines' counts; resolution 256, 64 blocks, iso
0.005) to the reference's 1e5 faces, and, for context, the serial numpy/Python oracle on a small sphere.

    python tests/perf_mesh_decimate.py [--iters 3] [--repeats 5] [--out perf_mesh_decimate.json]

The decimation is warmed up, then timed in `repeats` windows of `iters` calls (CUDA events, CUDA tensors in and out);
the median and minimum per-call times are reported with the rounds, the input and output face counts and faces removed
per ms.  The card's name, power limit and SM clocks are read in the same run."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "open-diffusiongs_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from perf_mesh import NAMES, card, timed  # noqa: E402


def rounds(v, f, target):
    """The round count of one call, through the C ABI"""
    from dgs_b200 import _lib, mesh
    alloc = _lib.Alloc(v.device, mesh._SCRATCH, (str(v.device), "decimate"), cached=1)
    out = [C.c_void_p(), C.c_void_p(), C.c_longlong(), C.c_longlong()]
    n = C.c_int(0)
    _lib.check(_lib.lib().dgs_mesh_decimate(v.data_ptr(), len(v), f.data_ptr(), len(f), int(target), alloc.cb, None,
                                            *[C.byref(o) for o in out], C.byref(n), _lib.stream(v.device)))
    torch.cuda.synchronize()
    return n.value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default="perf_mesh_decimate.json")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_mesh_decimate.py measures on the GPU"
    from dgs_b200 import mesh, synth
    from oracle import mesh as om
    from oracle import mesh_decimate as od
    res = {"card": card(), "cases": []}
    target = 100000
    for P in (262146, 1048578):
        g = synth.make_shell_gaussians(P, 11)
        t = [torch.tensor(g[k], device="cuda") for k in NAMES]
        occ, _, _ = mesh.opacity_field(*t, resolution=256, num_blocks=64)
        v, f = mesh.marching_cubes(occ, 0.005)
        v = (v / 255.0 * 2 - 1).contiguous()
        ms_med, ms_min = timed(lambda: mesh.decimate(v, f, target), args.iters, args.repeats)
        ov, of = mesh.decimate(v, f, target)
        removed = len(f) - len(of)
        case = dict(gaussians=P, in_vertices=len(v), in_faces=len(f), out_vertices=len(ov), out_faces=len(of),
                    rounds=rounds(v, f, target), ms_median=ms_med, ms_min=ms_min,
                    faces_removed_per_ms=removed / ms_med)
        print(json.dumps(case), flush=True)
        res["cases"].append(case)
    x = np.arange(40, dtype=np.float64) - 19.5
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    sv, sf = om.marching_cubes(14.0 - np.sqrt(X ** 2 + Y ** 2 + Z ** 2), 0.0)
    t0 = time.perf_counter()
    _, of, _ = od.decimate(sv, sf, len(sf) // 10)
    oracle_s = time.perf_counter() - t0
    gv, gf = torch.from_numpy(sv.astype(np.float32)).cuda(), torch.from_numpy(sf).cuda()
    g_med, _ = timed(lambda: mesh.decimate(gv, gf, len(sf) // 10), args.iters, args.repeats)
    res["oracle_sphere"] = dict(in_faces=len(sf), out_faces=len(of), oracle_s=oracle_s, native_ms_median=g_med)
    print(json.dumps(res["oracle_sphere"]))
    res["card_after"] = card()
    print(res["card"], "|", res["card_after"])
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
