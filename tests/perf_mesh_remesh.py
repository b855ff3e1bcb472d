"""Times isotropic remeshing (dgs_mesh_remesh at the reference's clean_mesh settings: target_len 0.015, 3 iterations) of
the cleaned marching-cubes meshes extract_mesh produces for 262,146 and 1,048,578 Gaussians on an object-like shell (the
obj-256 and obj-512 pipelines' counts, as tests/perf_mesh_clean.py), extract_mesh with
postprocess=clean_remesh_then_decimate against postprocess=clean_then_decimate end to end, and the serial oracle on the
host CPU on the same meshes.

    python tests/perf_mesh_remesh.py [--iters 3] [--repeats 5] [--out perf_mesh_remesh.json]

The remeshing is warmed up, then timed in `repeats` windows of `iters` calls (CUDA events, CUDA tensors in and out).  A
separate profiled call splits the kernel time by stage (kernel names: grid, split, collapse, flip, smooth, reproject;
the edge sorts and vertex -> face lists, shared by the stages, are their own group).  The stats give the faces after
each split and the collapse and flip rounds per iteration.  The card's name, power limit and SM clocks are read in the
same run."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "open-diffusiongs_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from perf_mesh import card, timed  # noqa: E402

GROUPS = [("grid", ("grid_",)), ("split", ("split_",)), ("collapse", ("collapse_", "m1_kernel", "m2_kernel", "remap_",
                                                                         "DeviceSelect", "DeviceCompact")),
          ("flip", ("flip_", "valence_")), ("smooth", ("smooth_",)), ("reproject", ("reproject_",))]


def stage_ms(fn):
    """Kernel time of one call of fn by stage, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {g: 0.0 for g, _ in GROUPS}
    out["edges_and_lists"] = 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if not t:
            continue
        g = next((g for g, keys in GROUPS if any(k in ev.key for k in keys)), "edges_and_lists")
        out[g] += t / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default="perf_mesh_remesh.json")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_mesh_remesh.py measures on the GPU"
    from dgs_b200 import mesh, synth
    from dgs_b200.renderer import GaussianModel
    from oracle import mesh_remesh as orr
    res = {"card": card(), "cases": []}
    for P in (262146, 1048578):
        g = synth.make_shell_gaussians(P, 11)
        m = GaussianModel(0)
        m._xyz, m._scaling, m._rotation, m._opacity = (torch.tensor(g[k], device="cuda") for k in
                                                       ("xyz", "scaling", "rotation", "opacity"))
        raw = m.extract_mesh()
        cv, cf = mesh.clean(raw.vertices, raw.faces)
        v, f = torch.from_numpy(cv).cuda(), torch.from_numpy(cf).cuda()
        ms_med, ms_min = timed(lambda: mesh.remesh(v, f), args.iters, args.repeats)
        stats = {}
        ov, of = mesh.remesh(v, f, stats=stats)
        stages = stage_ms(lambda: mesh.remesh(v, f))
        t0 = time.perf_counter()
        rv, rf, rs = orr.remesh(cv, cf)
        oracle_s = time.perf_counter() - t0
        equal = (ov.cpu().numpy().tobytes() == rv.tobytes() and np.array_equal(of.cpu().numpy(), rf)
                 and stats["iterations"] == rs)
        e2e_med, e2e_min = timed(lambda: m.extract_mesh(postprocess=mesh.clean_remesh_then_decimate), 1, args.repeats)
        ctd_med, ctd_min = timed(lambda: m.extract_mesh(postprocess=mesh.clean_then_decimate), 1, args.repeats)
        out = m.extract_mesh(postprocess=mesh.clean_remesh_then_decimate)
        case = dict(gaussians=P, in_vertices=len(cv), in_faces=len(cf), out_vertices=len(ov), out_faces=len(of),
                    iterations=stats["iterations"], ms_median=ms_med, ms_min=ms_min, kernel_ms_by_stage=stages,
                    oracle_s=oracle_s, equal_to_oracle=equal, e2e_faces=len(out.faces),
                    extract_mesh_clean_remesh_then_decimate_ms_median=e2e_med,
                    extract_mesh_clean_remesh_then_decimate_ms_min=e2e_min,
                    extract_mesh_clean_then_decimate_ms_median=ctd_med, extract_mesh_clean_then_decimate_ms_min=ctd_min)
        print(json.dumps(case), flush=True)
        res["cases"].append(case)
    res["card_after"] = card()
    print(res["card"], "|", res["card_after"])
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
