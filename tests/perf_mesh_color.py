"""Times the vertex colour pass (dgs_mesh_vertex_colors: block lists, vertex sort, evaluation, normals) on the meshes
`extract_mesh(postprocess=clean_remesh_then_decimate)` returns for the 262,146- and 1,048,578-Gaussian shells of
perf_mesh.py, at SH degree 0 and 3, and extract_mesh end to end with and without vertex_colors.

    python tests/perf_mesh_color.py [--iters 5] [--repeats 5] [--out perf_mesh_color.json]

Each call is warmed up, then timed in `repeats` windows of `iters` calls (CUDA events), the two extract_mesh variants in
alternated windows; the median and minimum per-call times are reported with the (vertex, Gaussian) pair count (every
vertex against every Gaussian of its block's list) and pairs per second.  The card's name, power limit and SM clocks are
read in the same run."""
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

from perf_mesh import card, timed  # noqa: E402


def pair_count(m, vertices, resolution=256, num_blocks=64):
    """Sum over the vertices of their block's list length"""
    from dgs_b200 import mesh
    _, _, _, counts, _ = mesh.opacity_field(m._xyz, m._scaling, m._rotation, m._opacity, m.scaling_modifier, resolution,
                                            num_blocks, return_counts=True)
    lin = torch.linspace(-1, 1, resolution).cuda()
    v = torch.from_numpy(vertices).cuda()
    i = (torch.searchsorted(lin, v.contiguous(), right=True) - 1).clamp(0, resolution - 1) // (resolution // num_blocks)
    return int(counts.long()[i[:, 0], i[:, 1], i[:, 2]].sum())


def alternated(fns, iters, repeats):
    """Median / min per-call ms of each fn, their windows alternated"""
    for fn in fns:
        fn()
    torch.cuda.synchronize()
    ms = [[] for _ in fns]
    for _ in range(repeats):
        for k, fn in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                fn()
            b.record()
            b.synchronize()
            ms[k].append(a.elapsed_time(b) / iters)
    return [(statistics.median(x), min(x)) for x in ms]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default="perf_mesh_color.json")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_mesh_color.py measures on the GPU"
    from dgs_b200 import mesh, synth
    from dgs_b200.renderer import GaussianModel
    res = {"card": card(), "cases": []}
    for P in (262146, 1048578):
        g = synth.make_shell_gaussians(P, 11)
        for deg in (0, 3):
            m = GaussianModel(deg)
            f = torch.randn(P, (deg + 1) ** 2, 3, generator=torch.Generator().manual_seed(0)) * 0.5
            t = {k: torch.tensor(g[k], device="cuda") for k in ("xyz", "scaling", "rotation", "opacity")}
            m.set_data(t["xyz"], f.cuda(), t["scaling"], t["rotation"], t["opacity"])
            post = mesh.clean_remesh_then_decimate
            out = m.extract_mesh(postprocess=post)
            v, fc = out.vertices, out.faces
            vt, ft = torch.from_numpy(v).cuda(), torch.from_numpy(fc).cuda()
            feats = m.get_features

            def colors():
                return mesh.vertex_colors(m._xyz, feats, m._scaling, m._rotation, m._opacity, vt, ft, m.mesh_center,
                                          m.mesh_scale, None, 256, 64)
            c_med, c_min = timed(colors, args.iters, args.repeats)
            pairs = pair_count(m, v)
            (p_med, p_min), (q_med, q_min) = alternated(
                [lambda: m.extract_mesh(postprocess=post), lambda: m.extract_mesh(postprocess=post, vertex_colors=True)],
                max(1, args.iters // 2), args.repeats)
            case = dict(gaussians=P, sh_degree=deg, vertices=len(v), faces=len(fc), pairs=pairs,
                        colors_ms_median=c_med, colors_ms_min=c_min, pairs_per_s=pairs / (c_med * 1e-3),
                        extract_mesh_ms_median=p_med, extract_mesh_ms_min=p_min,
                        extract_mesh_colors_ms_median=q_med, extract_mesh_colors_ms_min=q_min)
            print(json.dumps(case), flush=True)
            res["cases"].append(case)
    print(res["card"])
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
