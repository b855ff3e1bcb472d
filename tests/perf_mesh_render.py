"""Times dgs_mesh_render on the meshes of the 262,146- and 1,048,578-Gaussian shells (extract_mesh at resolution 256
and 512), raw marching cubes and after clean_remesh_then_decimate: a 150-view turntable at 512 x 512 (colour map, as
render_turntable draws and quantises it, left on the device) and get_render's four views at 224 x 224, with the
frames renderer.render_turntable draws of the same Gaussians (raster.render_frames, also left on the device) at
512 x 512 in alternated windows for scale.

    python tests/perf_mesh_render.py [--iters 3] [--repeats 5] [--out perf_mesh_render.json]

Reported per case: the median and minimum ms per frame over the alternated windows, the peak device memory of one
call (with the mesh renderer's cached scratch dropped first, so the arena is counted) next to its output bytes, and
the per-stage split (setup, coverage, resolve, antialias, mesh edge table) of one call under torch.profiler.  The card's name, power limit and SM clocks are read in the same run."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "open-diffusiongs_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from perf_mesh import card  # noqa: E402
from perf_mesh_color import alternated  # noqa: E402

STAGES = {"setup_kernel": "setup", "cover_small_kernel": "coverage", "cover_tiles_kernel": "coverage",
          "DeviceScan": "coverage", "resolve_kernel": "resolve", "antialias_kernel": "antialias"}


def stages(fn):
    """ms per stage of one call of fn (kernels not named in STAGES: the edge table, the checks and copies)"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        st = next((v for k, v in STAGES.items() if k in e.name), "other")
        out[st] = out.get(st, 0.0) + e.device_time / 1e3
    return out


def peak(fn):
    """-> (peak device bytes of one call of fn over what was allocated before it, bytes of its outputs).  The mesh
    renderer's cached scratch is dropped first, so the peak counts the arena the call allocates."""
    from dgs_b200 import mesh_render as mr
    mr._SCRATCH.clear()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    outs = out.values() if isinstance(out, dict) else out if isinstance(out, tuple) else [out]
    return torch.cuda.max_memory_allocated() - base, sum(t.numel() * t.element_size() for t in outs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default="perf_mesh_render.json")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_mesh_render.py measures on the GPU"
    from dgs_b200 import mesh, mesh_render as mr, raster, renderer, synth
    from dgs_b200.cameras import get_turntable_cameras
    res = {"card": card(), "cases": []}
    for P, R in ((262146, 256), (1048578, 512)):
        g = synth.make_shell_gaussians(P, 11)
        m = renderer.GaussianModel(0)
        t = {k: torch.tensor(g[k], device="cuda") for k in ("xyz", "scaling", "rotation", "opacity")}
        m.set_data(t["xyz"], torch.full((P, 1, 3), 0.5, device="cuda"), t["scaling"], t["rotation"], t["opacity"])
        for post in (None, mesh.clean_remesh_then_decimate):
            out = m.extract_mesh(resolution=R, postprocess=post, vertex_colors=True)
            world = out.vertices / np.float32(m.mesh_scale) + m.mesh_center.cpu().numpy()
            v, f = torch.from_numpy(world).cuda(), torch.from_numpy(out.faces).cuda()
            col = torch.from_numpy(out.vertex_colors).cuda()
            nv = 150
            w, h, _, K, c2w = get_turntable_cameras(num_views=nv, w=512, h=512)
            clip = mr.clip_from_opencv(c2w, K, h, w)
            c2w_t, K_t = torch.tensor(c2w, dtype=torch.float32), torch.tensor(K, dtype=torch.float32)

            def mesh_turntable():  # uint8 frames on the device, as render_turntable quantises them
                rgb = mr.render_clip(v, f, clip, h, w, colors=col, color_bg=(1.0, 1.0, 1.0), outputs=("rgb",))["rgb"]
                return rgb.mul_(255.0).clamp_(0.0, 255.0).to(torch.uint8)

            def gauss_turntable():  # renderer.render_turntable's frames, on the device (no host copy)
                with torch.no_grad():
                    return raster.render_frames(m._xyz[None], m.get_features[None], m._scaling[None],
                                                m._rotation[None], m._opacity[None], h, w, c2w_t.cuda()[None],
                                                K_t.cuda()[None], m.scaling_modifier)

            def four_views():
                return mr.get_render(world, out.faces.astype(np.int32), "cuda", 224)
            (mt, mt_min), (gt, gt_min), (fv, fv_min) = alternated([mesh_turntable, gauss_turntable, four_views],
                                                                   args.iters, args.repeats)
            case = dict(gaussians=P, resolution=R, postprocess=post.__name__ if post else "raw", faces=len(out.faces),
                        mesh_turntable_ms_per_frame=mt / nv, mesh_turntable_ms_per_frame_min=mt_min / nv,
                        gaussian_turntable_ms_per_frame=gt / nv, gaussian_turntable_ms_per_frame_min=gt_min / nv,
                        get_render_224_ms=fv, get_render_224_ms_min=fv_min,
                        mesh_turntable_peak_and_output_bytes=peak(mesh_turntable),
                        get_render_peak_and_output_bytes=peak(four_views),
                        mesh_turntable_stages_ms=stages(mesh_turntable), get_render_stages_ms=stages(four_views))
            print(json.dumps(case), flush=True)
            res["cases"].append(case)
    print(res["card"])
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
