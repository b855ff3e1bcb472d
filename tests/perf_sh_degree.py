"""What view-dependent colour costs: the obj-256 model at gaussians_sh_degree 0, 1 and 3 on the H100 (not a pytest
file).
    python tests/perf_sh_degree.py [--out perf_sh_degree.json] [--windows N]
* the DiT forward (inference, 24 layers, 4 views 256x256, B = 1), and the heads' share of it from the library's
  profiler (dit.heads: the two heads' LayerNorm + modulate, the upsampler and decoder products, the Gaussian epilogue);
* the batched render forward, and forward + backward, of those 262,146 Gaussians into the 4 views (the rasterizer
  evaluates degree-d SH per view and differentiates it);
* one training step: image_to_gaussians -> Renderer.forward_mse -> backward -> DitTrainer.optimizer_step (recompute
  mode, B = 1);
* median times from CUDA events, the degrees alternating window by window in one process; the decoder GEMM's FLOPs
  (2 x 4096 x 64 C x 3072) beside them; the card's name, power.limit and clocks read in the same run.
Prints one JSON line (and writes it to --out)."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "open-diffusiongs_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from dgs_b200 import _lib, synth  # noqa: E402
from dgs_b200.denoiser import DGSDenoiser  # noqa: E402
from dgs_b200.train import DitTrainer  # noqa: E402

DEV = "cuda:0"
DEGREES = (0, 1, 3)
B, V, H, W = 1, 4, 256, 256


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [s.strip() for s in r.split(",")]))
    except Exception as e:  # noqa: BLE001
        return dict(error=str(e))


def timed(fn, n):
    """median ms of n calls, each between two CUDA events"""
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    t = sorted(a.elapsed_time(b) for a, b in ev)
    return t[len(t) // 2]


def setup(degree):
    torch.manual_seed(0)
    model = DGSDenoiser(dict(patch_size=8, gaussians_sh_degree=degree)).to(DEV)
    g = torch.Generator(DEV).manual_seed(1)
    images = torch.rand(B, V, 3, H, W, device=DEV, generator=g)
    ray_o = torch.randn(B, V, 3, 1, 1, device=DEV, generator=g).expand(B, V, 3, H, W).contiguous() * 1.5
    ray_d = torch.nn.functional.normalize(torch.randn(B, V, 3, H, W, device=DEV, generator=g), dim=2)
    t = torch.tensor([500] * B, device=DEV)
    c2w, fx = synth.orbit_cameras(V, W, H)
    c2w, fx = torch.tensor(c2w[None], device=DEV), torch.tensor(fx[None], device=DEV)
    target = torch.rand(B, V, 3, H, W, device=DEV, generator=g)
    trainer = DitTrainer(model, lr=1e-5)
    trainer.recompute = True
    inp = (images, ray_o, ray_d, t)
    with torch.no_grad():
        out, _ = model.image_to_gaussians(*inp)
    leaves = {k: out[k].detach().clone().requires_grad_(True) for k in ("xyz", "features", "scaling", "rotation",
                                                                         "opacity")}
    r = model.gs_renderer

    def dit_forward():
        with torch.no_grad():
            model.image_to_gaussians(*inp)

    def render_forward():
        with torch.no_grad():
            r(*(leaves[k] for k in leaves), H, W, c2w, fx)

    def render_fwd_bwd():
        _, l2 = r.forward_mse(*(leaves[k] for k in leaves), H, W, c2w, fx, target)
        l2.sum().backward()

    def train_step():
        model.train()
        o, _ = model.image_to_gaussians(*inp)
        _, l2 = r.forward_mse(o.xyz, o.features, o.scaling, o.rotation, o.opacity, H, W, c2w, fx, target)
        trainer.zero_grad()
        l2.mean().backward()
        trainer.optimizer_step(allreduce=False)
        model.eval()

    return dict(dit_forward=dit_forward, render_forward=render_forward, render_fwd_bwd=render_fwd_bwd,
                train_step=train_step)


def heads_share(fns, n=10):
    L = _lib.lib()
    torch.cuda.synchronize()
    L.dgs_profile_enable(1)
    _lib.profile_read()
    for _ in range(n):
        fns["dit_forward"]()
    fam = _lib.profile_read()
    L.dgs_profile_enable(0)
    return fam["dit.heads"][0] / n, sum(v[0] for k, v in fam.items() if k.startswith("dit.")) / n


def main():
    windows = int(sys.argv[sys.argv.index("--windows") + 1]) if "--windows" in sys.argv else 5
    res = dict(card_before=card(), shape=dict(B=B, V=V, H=H, W=W, layers=24, patch=8), degrees={})
    runs = {d: setup(d) for d in DEGREES}
    for fns in runs.values():  # warm up every shape
        for f in fns.values():
            for _ in range(3):
                f()
    torch.cuda.synchronize()
    times = {d: {k: [] for k in runs[d]} for d in DEGREES}
    reps = dict(dit_forward=10, render_forward=10, render_fwd_bwd=10, train_step=3)
    for _ in range(windows):
        for d in DEGREES:
            for k, f in runs[d].items():
                times[d][k].append(timed(f, reps[k]))
    for d in DEGREES:
        C_ = 11 + 3 * (d + 1) ** 2
        heads_ms, dit_prof_ms = heads_share(runs[d])
        med = {k: sorted(v)[len(v) // 2] for k, v in times[d].items()}
        res["degrees"][d] = dict(channels=C_, decoder_gemm_gflop=2 * 4096 * 64 * C_ * 3072 / 1e9,
                                 ms={k: round(v, 3) for k, v in med.items()},
                                 spread_ms={k: round(max(v) - min(v), 3) for k, v in times[d].items()},
                                 heads_ms_profiled=round(heads_ms, 3), dit_ms_profiled=round(dit_prof_ms, 3))
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    out = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else "perf_sh_degree.json"
    with open(out, "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
