"""Times TSDF fusion meshing of the 262,146- and 1,048,578-Gaussian shells (the obj-256 and obj-512 pipelines' counts,
as tests/perf_mesh.py) at resolution 256 and 512 from 100 views at 512 x 512 (extract_mesh(method="tsdf")'s defaults),
next to extract_mesh() (the opacity field at 256) and method="poisson" on the same models.

    python tests/perf_tsdf.py [--iters 1] [--repeats 3] [--out perf_tsdf.json]

A TSDF call is tsdf_fusion + tsdf_mesh + tsdf_colors on the raw mesh's vertices; the extract_mesh calls return the raw
mesh (no postprocess, no colours).  Each case is warmed up, then timed in `repeats` windows of `iters` calls (CUDA
events around calls that end in a device synchronise); the cases of one model alternate window by window.  The stage
split comes from the calls' own stats (device events between the stages), the peak device memory from torch's allocator
over one call, and the voxel-view updates are R^3 * views.  The card's name, power limit and SM clocks are read in the
same run."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "open-diffusiongs_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from perf_mesh import card  # noqa: E402
from perf_poisson import alternated  # noqa: E402

VIEWS, SIZE = 100, 512


def tsdf(m, R, stats=None):
    from dgs_b200 import mesh
    st = {} if stats is None else stats
    vol = mesh.tsdf_fusion(m._xyz, m.get_features, m._scaling, m._rotation, m._opacity, resolution=R,
                           num_views=VIEWS, image_size=SIZE, stats=st)
    v, f = mesh.tsdf_mesh(vol, stats=st)
    rgb = mesh.tsdf_colors(vol, v, stats=st)
    return v, f, rgb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default="perf_tsdf.json")
    args = ap.parse_args()
    from mesh_shapes import shell_model
    free, total = torch.cuda.mem_get_info()
    res = {"card": card(), "device_memory_free_GB": round(free / 1e9, 1), "device_memory_GB": round(total / 1e9, 1),
           "views": VIEWS, "image_size": SIZE, "cases": []}
    print(res["card"], res["device_memory_free_GB"], flush=True)
    for P in (262146, 1048578):
        m = shell_model(P, 7, floaters=False)
        u = m._xyz - (m._xyz.amin(0) + m._xyz.amax(0)) / 2
        m.set_data(m._xyz, (0.4 * u / u.norm(dim=1, keepdim=True) / 0.28209479177387814)[:, None, :], m._scaling,
                   m._rotation, m._opacity)
        fns = {f"tsdf{R}": (lambda R=R: tsdf(m, R)) for R in (256, 512)}
        fns["field256"] = lambda: m.extract_mesh()
        fns["poisson9"] = lambda: m.extract_mesh(method="poisson")
        times = alternated(fns, args.iters, args.repeats)
        for name, (med, best) in times.items():
            case = {"P": P, "case": name, "median_ms": round(med, 2), "min_ms": round(best, 2)}
            st = {}
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            if name.startswith("tsdf"):
                R = int(name[4:])
                v, f, _ = tsdf(m, R, st)
                case["stage_ms"] = {k: round(st[k + "_ms"], 2) for k in ("render", "integrate", "extract", "colors")}
                case["voxel_view_updates"] = float(R ** 3 * VIEWS)
                case["integrate_updates_per_ns"] = round(R ** 3 * VIEWS / (st["integrate_ms"] * 1e6), 2)
                case["vertices"], case["faces"] = len(v), len(f)
            else:
                out = fns[name]()
                case["vertices"], case["faces"] = len(out.vertices), len(out.faces)
            torch.cuda.synchronize()
            case["peak_device_GB"] = round((torch.cuda.max_memory_allocated() - base) / 1e9, 3)
            res["cases"].append(case)
            print(json.dumps(case), flush=True)
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
