"""Validation-video rendering on the GPU: dgs_b200.raster.render_frames (the blend kernel writes the uint8 frames, views
in arena-bounded chunks, one host copy) vs

  (a) the reference's loop on this library: one render_batch_forward per view into an fp32 [v,3,h,w] tensor, then a
      torch quantise, (x * 255).clamp(0, 255).to(uint8), and one host copy (gs_core.py:1201-1219, 1300-1316);
  (b) the UNMODIFIED reference rasterizer (oracle/_ref/dgr_ref_C.so, when build() made it), one view per call, with
      the same quantise and copy.

Workloads: the object turntable (150 views at 512^2 of a shell-like obj-512 set, P = 1,048,578 before
apply_all_filters with save_guassians_ply's arguments) and a scene fly-through (4 keyframes closed into a loop,
240 frames, at 256^2 and 512^2).  For each: ms per frame, frames/s and the peak device memory of the render.  Timing
windows of the methods alternate, each repeated; the median and the spread (min, max) are reported.  The card's name,
power limit and SM clock are read in the same run.  Not a pytest file (name perf_*).

    python tests/perf_render_video.py OUT.json [--reps N]
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "open-diffusiongs_b200")):
    sys.path.insert(0, p)

from dgs_b200 import raster, synth  # noqa: E402
from dgs_b200.cameras import get_interpolated_poses_many, get_turntable_cameras  # noqa: E402
from dgs_b200.renderer import GaussianModel  # noqa: E402
from oracle import build_ref  # noqa: E402

DEV = "cuda:0"
NAMES = ("xyz", "features", "scaling", "rotation", "opacity")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [s.strip() for s in r.split(",")]))
    except Exception as e:  # noqa: BLE001
        return dict(error=str(e))


def T(x):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float32, device=DEV)


def object_workload():
    g = synth.make_shell_gaussians(1_048_578, 0, "trained")
    pc = GaussianModel(0, None).set_data(*(T(g[k]) for k in NAMES))
    pc.apply_all_filters(opacity_thres=0.02, crop_bbx=[-0.91, 0.91, -0.91, 0.91, -0.91, 0.91], cam_origins=None,
                         nearfar_percent=(0.0001, 1.0))  # save_guassians_ply (utils/saving.py:452-469)
    w, h, v, fx, c2w = get_turntable_cameras(w=512, h=512, num_views=150)
    return pc, T(c2w), T(fx), h, w


def scene_workload(res, P):
    """prune(0.05)-ed scene Gaussians and save_guassians_ply_scene's path through 4 keyframes (saving.py:472-504)."""
    g = synth.make_gaussians(P, 1, "trained")
    pc = GaussianModel(0, None).set_data(*(T(g[k]) for k in NAMES)).prune(opacity_thres=0.05)
    key = torch.tensor(np.stack([synth.orbit_c2w(3.0, az, 15.0 + 10.0 * i) for i, az in enumerate((0, 80, 170, 260))]),
                       dtype=torch.float32)
    f = synth.intrinsics(res, res)
    Ks = torch.zeros(4, 3, 3)
    Ks[:, 0, 0], Ks[:, 1, 1], Ks[:, 0, 2], Ks[:, 1, 2] = float(f[0]), float(f[1]), float(f[2]), float(f[3])
    c2ws, Ks = get_interpolated_poses_many(torch.cat([key, key[:1]])[:, :3, :4], torch.cat([Ks, Ks[:1]]), 60)
    c2ws = torch.cat([c2ws, torch.tensor([[[0.0, 0.0, 0.0, 1.0]]]).repeat(c2ws.shape[0], 1, 1)], dim=1)
    fx = torch.stack([Ks[:, 0, 0], Ks[:, 1, 1], Ks[:, 0, 2], Ks[:, 1, 2]], dim=1)
    return pc, c2ws.to(DEV), fx.to(DEV), res, res


def methods(pc, c2w, fx, h, w, ref):
    """name -> callable returning the uint8 frames [v, h, w, 3] on the host."""
    feats = pc.get_features
    raw = [pc._xyz[None], feats[None], pc._scaling[None], pc._rotation[None], pc._opacity[None]]
    v = c2w.shape[0]
    cache_ours, cache_a = {}, {}

    def ours():
        return raster.render_frames(*raw, h, w, c2w[None], fx[None], arena_cache=cache_ours)[0].cpu().numpy()

    def quantised(images):
        return (images * 255).clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).cpu().numpy()

    def per_view():
        images = torch.empty(v, 3, h, w, device=DEV)
        for j in range(v):
            images[j] = raster.render_batch_forward(*raw, h, w, c2w[None, j:j + 1], fx[None, j:j + 1],
                                                    arena_cache=cache_a)[0][0, 0]
        return quantised(images)
    out = {"ours_render_frames": ours, "a_render_batch_forward_per_view": per_view}
    if ref is not None:
        act = dict(m3=pc._xyz, sh=feats, op=pc.get_opacity, sc=pc.get_scaling, ro=pc.get_rotation)
        cams = [synth.camera_matrices(c2w[j].cpu().numpy(), fx[j].cpu().numpy(), h, w) for j in range(v)]
        cams = [(T(c[0]), T(c[1]), T(c[2]), float(c[3]), float(c[4])) for c in cams]
        bg, e = T(np.ones(3)), torch.empty(0, device=DEV)

        def reference():
            images = torch.empty(v, 3, h, w, device=DEV)
            for j, c in enumerate(cams):
                images[j] = ref.rasterize_gaussians(bg, act["m3"], e, act["op"], act["sc"], act["ro"], 1.0, e, c[0],
                                                    c[1], c[3], c[4], h, w, act["sh"], 0, c[2], False, False)[1]
            return quantised(images)
        out["b_reference_rasterizer_per_view"] = reference
    return out


def run(name, pc, c2w, fx, h, w, ref, reps):
    fns = methods(pc, c2w, fx, h, w, ref)
    v = c2w.shape[0]
    res = dict(workload=name, P=int(pc._xyz.shape[0]), views=v, h=h, w=w)
    frames = {}
    for m, fn in fns.items():  # warm-up, outputs, peak memory
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        frames[m] = fn()
        torch.cuda.synchronize()
        res[f"{m}/peak_mem_GiB"] = (torch.cuda.max_memory_allocated() - base) / 2**30
    ours = frames["ours_render_frames"]
    for m, f in frames.items():
        d = np.abs(f.astype(np.int32) - ours.astype(np.int32))
        res[f"{m}/max_lsb_vs_ours"], res[f"{m}/frac_differ_vs_ours"] = int(d.max()), float((d != 0).mean())
    assert res["a_render_batch_forward_per_view/max_lsb_vs_ours"] == 0  # the same quantisation of the same images
    times = {m: [] for m in fns}
    for _ in range(reps):
        for m, fn in fns.items():  # alternating windows
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()  # ends in a host copy, which synchronises
            times[m].append((time.perf_counter() - t0) * 1e3)
    for m, ts in times.items():
        med = float(np.median(ts))
        res[f"{m}/ms_per_frame"] = med / v
        res[f"{m}/ms_per_frame_min_max"] = (min(ts) / v, max(ts) / v)
        res[f"{m}/frames_per_s"] = v / med * 1e3
    for m in fns:
        if m != "ours_render_frames":
            res[f"speedup_vs_{m}"] = res[f"{m}/ms_per_frame"] / res["ours_render_frames/ms_per_frame"]
    print(json.dumps(res), flush=True)
    return res


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 and not sys.argv[1].startswith("--") else "perf_render_video.json"
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 5
    assert torch.cuda.is_available(), "perf_render_video.py measures on the GPU"
    ref = build_ref.load_module()
    before = card()
    print(json.dumps(dict(card=before, torch=torch.__version__, reference_rasterizer=ref is not None)), flush=True)
    results = [run("object_turntable_512", *object_workload(), ref, reps)]
    results.append(run("scene_flythrough_256", *scene_workload(256, 2 + 4 * 256 * 256), ref, reps))
    results.append(run("scene_flythrough_512", *scene_workload(512, 2 + 4 * 512 * 512), ref, reps))
    json.dump(dict(card_before=before, card_after=card(), reps=reps, results=results), open(out_path, "w"), indent=1)


if __name__ == "__main__":
    main()
