"""The rasterizer's binning paths on the H100, this build against another (not a pytest file; bench.py measures the step).
    python tests/perf_raster.py [--baseline-lib PATH] [--out perf_raster.json]
* workloads: a single-view C1 scene and the crowded C1 scene whose long tile lists send the small-scene binning to the
  global path (rasterize_gaussians + backward); the batched B=2, V=3, P=1500 scene; obj-256 init-like (P = 262,146,
  4 views at 256^2) at near_log2 0, 3 and -1; the "fine" P = 400,000 scene at 3 and -1 (phase B not empty); obj-256
  with the fused MSE loss, forward and backward (render_batch_forward / render_batch_backward);
* per workload and build: the binning path, read from the profile span counts of one forward (the small-scene path
  records no raster.tile_ranges span, a second raster.scan span marks its fallback, two raster.blend_fwd spans phase B);
* with --baseline-lib (a libdgs_b200.so of another build): whether images, radii, R, the chunk instance counts, the
  first pass's point list and ranges, final_T and n_contrib are bitwise equal between the builds, and the gradients' and
  loss_sum's relative difference between the builds next to this build's own run-to-run difference;
* median forward and backward ms from CUDA events over windows of timed calls, the builds alternating window by window,
  and the spread of the per-window medians of each build ((max - min) / median);
* the card's name, power.limit and clocks.sm / clocks.max.sm, read in the same run before and after.
Prints one JSON line."""
import contextlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "open-diffusiongs_b200"))
from dgs_b200 import _lib, raster, synth  # noqa: E402
from perf_dit_linears import card, load_lib  # noqa: E402
from util import rel_l2 as rel, scene_c1  # noqa: E402

DEV = "cuda:0"


@contextlib.contextmanager
def using(L):
    saved = _lib._lib
    _lib._lib = L
    try:
        yield
    finally:
        _lib._lib = saved


def T(x):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float32, device=DEV)


class Single:
    """One view through rasterize_gaussians(_backward), the reference's drop-in API."""

    def __init__(self, **kw):
        self.sc = sc = scene_c1(**kw)
        a, e = sc["act"], torch.empty(0, device=DEV)
        self.args = (T(np.ones(3)), T(a["means3D"]), e, T(a["opacities"]), T(a["scales"]), T(a["rotations"]), 1.0, e,
                     T(sc["view"]), T(sc["proj"]), sc["tanx"], sc["tany"], sc["H"], sc["W"], T(a["shs"]), 0,
                     T(sc["campos"]), False, False)
        self.dpix = torch.randn(3, sc["H"], sc["W"], device=DEV, generator=torch.Generator(DEV).manual_seed(1))

    def forward(self):
        return raster.rasterize_gaussians(*self.args)

    def backward(self, fwd):
        R, _, radii, geom, binning, img = fwd
        bg, m3, _, _, sc_, ro, mod, cov, vm, pm, tx, ty, _, _, sh, deg, cp, _, _ = self.args
        return raster.rasterize_gaussians_backward(bg, m3, radii, cov, sc_, ro, mod, cov, vm, pm, tx, ty, self.dpix, sh,
                                                   deg, cp, geom, R, binning, img, False)

    def outputs(self, fwd):
        R, color, radii, geom, binning, img = fwd
        ex = raster.export_state(1, self.sc["P"], self.sc["W"], self.sc["H"], R, geom, binning, img)
        return dict(R=R, image=color, radii=radii, point_list=ex["point_list"], ranges=ex["ranges"],
                    final_T=ex["final_T"], n_contrib=ex["n_contrib"])

    def chunks(self, fwd):
        return (fwd[0], 0)


class Batch:
    """All (sample, view) pairs through render_batch_forward / render_batch_backward."""

    def __init__(self, B, V, P, W, H, dist, near_log2, mse=False):
        gs = [synth.make_gaussians(P, 10 + i, dist) for i in range(B)]
        raw = {k: np.stack([g[k] for g in gs]) for k in gs[0]}
        c2w, fx = zip(*[synth.orbit_cameras(V, W, H, az0=15.0 * i) for i in range(B)])
        self.t = [T(raw[k]) for k in ("xyz", "features", "scaling", "rotation", "opacity")]
        self.c2w, self.fx = T(np.stack(c2w)), T(np.stack(fx))
        self.B, self.V, self.P, self.W, self.H, self.near_log2 = B, V, P, W, H, near_log2
        gen = torch.Generator(DEV).manual_seed(3)
        self.g = torch.randn(B, V, 3, H, W, device=DEV, generator=gen)
        self.target = torch.rand(B, V, 3, H, W, device=DEV, generator=gen) if mse else None
        self.loss = torch.zeros(B, dtype=torch.float64, device=DEV)
        self.coef = torch.full((B,), 1.0 / (V * 3 * H * W), device=DEV)

    def forward(self):
        self.loss.zero_()
        img, st = raster.render_batch_forward(*self.t, self.H, self.W, self.c2w, self.fx, near_log2=self.near_log2,
                                              mse_target=self.target,
                                              mse_loss_sum=None if self.target is None else self.loss)
        return img, st, self.loss.clone()

    def backward(self, fwd):
        if self.target is not None:
            return raster.render_batch_backward(fwd[1], None, mse_coef=self.coef)
        return raster.render_batch_backward(fwd[1], self.g)

    def outputs(self, fwd):
        img, st, loss = fwd
        ex = raster.export_state(self.B * self.V, self.P, self.W, self.H, st["chunks"][0], st["geom"], st["binning"],
                                 st["img"])
        o = dict(R=st["R"], chunks=st["chunks"], image=img, point_list=ex["point_list"], ranges=ex["ranges"],
                 final_T=ex["final_T"], n_contrib=ex["n_contrib"])
        if self.target is not None:
            o["loss_sum"] = loss
        return o

    def chunks(self, fwd):
        return fwd[1]["chunks"]


def path_of(spans, R, chunks):
    if spans["raster.tile_ranges"][1] == 0:
        return "small"
    phase_b = spans["raster.blend_fwd"][1] > 1  # phase B records one more raster.scan span (its open-tile counts)
    p = "small->global" if spans["raster.scan"][1] - phase_b > 1 else "global"
    if chunks[0] < R:
        p += " two-phase A" + ("+B" if phase_b else "")
    return p


def alternate(fns, windows=10, per_window=10):
    """{name: per-window median ms}: the functions take turns in windows of per_window timed calls each."""
    for f in fns.values():
        for _ in range(10):
            f()
    torch.cuda.synchronize()
    med = {k: [] for k in fns}
    for _ in range(windows):
        for k, f in fns.items():
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(per_window)]
            for a, b in ev:
                a.record()
                f()
                b.record()
            torch.cuda.synchronize()
            t = sorted(a.elapsed_time(b) for a, b in ev)
            med[k].append(t[len(t) // 2])
    return med


def summary(w):
    s = sorted(w)
    m = s[len(s) // 2]
    return dict(ms=round(m, 4), window_spread=round((s[-1] - s[0]) / m, 4))


def same(a, b):
    if isinstance(a, torch.Tensor):
        return bool(a.shape == b.shape and torch.equal(a, b))
    return a == b


def run(name, wl, libs):
    r = dict(path={})
    outs, grads = {}, {}
    for k, L in libs.items():
        with using(L):
            L.dgs_profile_enable(1)
            _lib.profile_read()
            fwd = wl.forward()
            spans = _lib.profile_read()
            L.dgs_profile_enable(0)
            o = wl.outputs(fwd)
            r["path"][k] = path_of(spans, o["R"], wl.chunks(fwd))
            outs[k] = o
            grads[k] = [wl.backward(fwd), wl.backward(fwd)]
            if "loss_sum" in o:
                grads[k].append(wl.outputs(wl.forward())["loss_sum"])  # a second forward: loss_sum run to run
    r["R"], r["chunks"] = outs["this"]["R"], list(wl.chunks(fwd))
    if "baseline" in libs:
        a, b = outs["this"], outs["baseline"]
        r["bitwise_equal"] = {f: same(a[f], b[f]) for f in a if f != "loss_sum"}
        ga, gb = grads["this"], grads["baseline"]
        r["grad_rel_vs_baseline"] = max(rel(x, y) for x, y in zip(ga[0], gb[0]))
        r["grad_rel_run_to_run"] = max(max(rel(x, y) for x, y in zip(g[0], g[1])) for g in (ga, gb))
        if "loss_sum" in a:
            r["loss_rel_vs_baseline"] = rel(a["loss_sum"], b["loss_sum"])
            r["loss_rel_run_to_run"] = max(rel(o["loss_sum"], g[2]) for o, g in ((a, ga), (b, gb)))
    del outs, grads

    def fwd_fn(L):
        def f():
            with using(L):
                wl.forward()
        return f
    states = {}
    for k, L in libs.items():
        with using(L):
            states[k] = wl.forward()

    def bwd_fn(k, L):
        def f():
            with using(L):
                wl.backward(states[k])
        return f
    tf = alternate({k: fwd_fn(L) for k, L in libs.items()})
    tb = alternate({k: bwd_fn(k, L) for k, L in libs.items()})
    r["forward"] = {k: summary(v) for k, v in tf.items()}
    r["backward"] = {k: summary(v) for k, v in tb.items()}
    print(f"[perf_raster] {name}: {json.dumps(r)}", file=sys.stderr, flush=True)
    return r


def main():
    libs = dict(this=_lib.lib())
    if "--baseline-lib" in sys.argv:
        libs["baseline"] = load_lib(sys.argv[sys.argv.index("--baseline-lib") + 1])
    res = dict(card=card(), workloads={})
    obj = dict(B=1, V=4, P=2 + 4 * 256 * 256, W=256, H=256, dist="init")
    fine = dict(obj, P=400000, dist="fine")
    workloads = [
        ("c1_trained", lambda: Single(P=10000, dist="trained")),
        ("c1_crowded", lambda: Single(P=10000, dist="init", W=48, H=48)),
        ("batch_b2v3_p1500", lambda: Batch(2, 3, 1500, 64, 48, "trained", -1)),
        ("obj256_near0", lambda: Batch(**obj, near_log2=0)),
        ("obj256_near3", lambda: Batch(**obj, near_log2=3)),
        ("obj256_adaptive", lambda: Batch(**obj, near_log2=-1)),
        ("fine400k_near3", lambda: Batch(**fine, near_log2=3)),
        ("fine400k_adaptive", lambda: Batch(**fine, near_log2=-1)),
        ("obj256_mse", lambda: Batch(**obj, near_log2=-1, mse=True)),
    ]
    for name, make in workloads:
        res["workloads"][name] = run(name, make(), libs)
        torch.cuda.empty_cache()
    res["card_after"] = card()
    line = json.dumps(res)
    print(line, flush=True)
    if "--out" in sys.argv:
        with open(sys.argv[sys.argv.index("--out") + 1], "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
