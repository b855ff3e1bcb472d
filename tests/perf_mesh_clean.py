"""Times mesh cleaning (dgs_mesh_clean, the reference's clean_mesh without remeshing, at its defaults) of the
marching-cubes meshes extract_mesh produces for 262,146 and 1,048,578 Gaussians on an object-like shell (the obj-256 and
obj-512 pipelines' counts, as tests/perf_mesh_decimate.py; resolution 256, 64 blocks, iso 0.005), and extract_mesh with
postprocess=clean_then_decimate end to end; the serial oracle is timed on the host CPU on the same meshes.

    python tests/perf_mesh_clean.py [--iters 3] [--repeats 5] [--out perf_mesh_clean.json]

The cleaning is warmed up, then timed in `repeats` windows of `iters` calls (CUDA events, CUDA tensors in and out); the
median and minimum per-call times are reported with the merge rounds, stage 7's candidate count and the face and vertex
counts after each stage (the oracle's, which the native output equals bit for bit; checked here too).  The card's name,
power limit and SM clocks are read in the same run."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default="perf_mesh_clean.json")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_mesh_clean.py measures on the GPU"
    from dgs_b200 import mesh, synth
    from dgs_b200.renderer import GaussianModel
    from oracle import mesh_clean as oc
    res = {"card": card(), "cases": []}
    for P in (262146, 1048578):
        g = synth.make_shell_gaussians(P, 11)
        m = GaussianModel(0)
        m._xyz, m._scaling, m._rotation, m._opacity = (torch.tensor(g[k], device="cuda") for k in
                                                       ("xyz", "scaling", "rotation", "opacity"))
        raw = m.extract_mesh()
        v, f = torch.from_numpy(raw.vertices).cuda(), torch.from_numpy(raw.faces).cuda()
        ms_med, ms_min = timed(lambda: mesh.clean(v, f), args.iters, args.repeats)
        # the same call without stage 2's rounds (the later stages then see the unmerged mesh)
        no_merge_med, _ = timed(lambda: mesh.clean(v, f, v_pct=0), args.iters, args.repeats)
        stats = {}
        ov, of = mesh.clean(v, f, stats=stats)
        info = {}
        t0 = time.perf_counter()
        rv, rf, counts = oc.clean(raw.vertices, raw.faces, info=info)
        oracle_s = time.perf_counter() - t0
        equal = (ov.cpu().numpy().tobytes() == rv.tobytes() and np.array_equal(of.cpu().numpy(), rf)
                 and stats["stage_faces"] == counts)
        e2e_med, e2e_min = timed(lambda: m.extract_mesh(postprocess=mesh.clean_then_decimate), 1, args.repeats)
        raw_med, _ = timed(lambda: m.extract_mesh(), 1, args.repeats)
        case = dict(gaussians=P, in_vertices=len(v), in_faces=len(f), out_vertices=len(ov), out_faces=len(of),
                    merge_rounds=stats["merge_rounds"], stage7_candidates=info["candidates"],
                    stage_faces=stats["stage_faces"], stage_vertices=info["stage_vertices"], ms_median=ms_med,
                    ms_min=ms_min, ms_median_v_pct0=no_merge_med, oracle_s=oracle_s, equal_to_oracle=equal,
                    extract_mesh_ms_median=raw_med, extract_mesh_clean_then_decimate_ms_median=e2e_med,
                    extract_mesh_clean_then_decimate_ms_min=e2e_min)
        print(json.dumps(case), flush=True)
        res["cases"].append(case)
    res["card_after"] = card()
    print(res["card"], "|", res["card_after"])
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
