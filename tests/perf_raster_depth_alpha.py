"""Cost of the rasterizer's depth and alpha maps on the H100 (not a pytest file).
    python tests/perf_raster_depth_alpha.py [--baseline-lib PATH] [--out perf_raster_depth_alpha.json]
* workloads: obj-256 init-like (P = 262,146, 4 views at 256^2) and the "fine" P = 400,000 scene (phase B not empty), both at
  the adaptive near fraction: the plain render (render_batch_forward / render_batch_backward) against the same render with
  the depth and alpha maps (aux=True, the launch set Renderer.forward_buffers runs), whose backward receives gradients on all
  three maps; median forward and backward ms from CUDA events, the two alternating window by window, and their spread;
  whether the render is bitwise equal with and without the maps;
* with --baseline-lib (a libdgs_b200.so of another build of the same ABI version): every workload of
  tests/perf_raster.py, this build against that one (bitwise equality of the outputs, gradient differences, timings);
* the card's name, power.limit and clocks.sm / clocks.max.sm, read in the same run before and after.
Prints one JSON line."""
import contextlib
import io
import json
import sys

import torch

import perf_raster as pr
from dgs_b200 import raster


def run_aux(name, wl):
    gen = torch.Generator(pr.DEV).manual_seed(4)
    gd = torch.randn(wl.B, wl.V, 1, wl.H, wl.W, device=pr.DEV, generator=gen)
    ga = torch.randn(wl.B, wl.V, 1, wl.H, wl.W, device=pr.DEV, generator=gen)

    def fwd(aux):
        return raster.render_batch_forward(*wl.t, wl.H, wl.W, wl.c2w, wl.fx, near_log2=wl.near_log2, aux=aux)
    plain, buffers = fwd(False), fwd(True)
    r = dict(R=plain[1]["R"], chunks=list(plain[1]["chunks"]),
             render_bitwise_equal=bool(torch.equal(plain[0], buffers[0])))
    tf = pr.alternate(dict(plain=lambda: fwd(False), aux=lambda: fwd(True)))
    tb = pr.alternate(dict(plain=lambda: raster.render_batch_backward(plain[1], wl.g),
                           aux=lambda: raster.render_batch_backward(buffers[3], wl.g, grad_depth=gd, grad_alpha=ga)))
    r["forward"] = {k: pr.summary(v) for k, v in tf.items()}
    r["backward"] = {k: pr.summary(v) for k, v in tb.items()}
    for p in ("forward", "backward"):
        r[p]["aux_over_plain"] = round(r[p]["aux"]["ms"] / r[p]["plain"]["ms"], 4)
    print(f"[perf_raster_depth_alpha] {name}: {json.dumps(r)}", file=sys.stderr, flush=True)
    return r


def main():
    out = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
    res = dict(card=pr.card(), workloads={})
    if "--baseline-lib" in sys.argv:
        saved_argv = sys.argv
        sys.argv = [a for i, a in enumerate(saved_argv) if a != "--out" and (i == 0 or saved_argv[i - 1] != "--out")]
        buf = io.StringIO()
        try:
            with contextlib.redirect_stdout(buf):
                pr.main()
        finally:
            sys.argv = saved_argv
        res["existing_vs_baseline"] = json.loads(buf.getvalue().strip().splitlines()[-1])
    obj = dict(B=1, V=4, P=2 + 4 * 256 * 256, W=256, H=256, dist="init", near_log2=-1)
    for name, kw in (("obj256_depth_alpha", obj), ("fine400k_depth_alpha", dict(obj, P=400000, dist="fine"))):
        res["workloads"][name] = run_aux(name, pr.Batch(**kw))
        torch.cuda.empty_cache()
    res["card_after"] = pr.card()
    line = json.dumps(res)
    print(line, flush=True)
    if out:
        with open(out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
