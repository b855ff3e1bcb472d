"""Validation videos on sm_90a: dgs_render_frames (the blend kernel's uint8 frames epilogue) through
dgs_b200.raster.render_frames and the reference-named render_turntable / render_generic.

* Exactness: the frames equal the reference's quantisation, (image * 255).clip(0, 255).astype(uint8), of
  render_batch_forward's fp32 images for the same inputs, bit for bit, on every binning path.
* Chunking: the frames do not depend on how the views are chunked, and the arenas do not grow with the frame count.
* Against the reference: the frames of render_turntable / render_generic vs tests/golden/render_video_ref.npz, the
  reference's own frames (written by make_render_video_golden.py)."""
import os

import numpy as np
import pytest
import torch

from dgs_b200 import _lib, raster, synth
from dgs_b200.cameras import get_turntable_cameras
from dgs_b200.renderer import GaussianModel, render_generic, render_turntable

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NAMES = ("xyz", "features", "scaling", "rotation", "opacity")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "render_video_ref.npz")


def T(x):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float32, device=DEV)


def scene(P, V, W, H, degree=0, dist="trained", seed=0, turntable=False):
    """Gaussians [1, P, ...] with SH degree `degree` and V cameras -> (list of 5 tensors, C2W [1,V,4,4], fx [1,V,4])."""
    g = synth.make_gaussians(P, seed, dist)
    rest = np.random.default_rng(seed + 1).normal(0, 0.3, (P, (degree + 1) ** 2 - 1, 3)).astype(np.float32)
    g["features"] = np.concatenate([g["features"], rest], axis=1)
    if turntable:
        _, _, _, fx, c2w = get_turntable_cameras(w=W, h=H, num_views=V)
    else:
        c2w, fx = synth.orbit_cameras(V, W, H, az0=7.0 * seed)
    return [T(g[k][None]) for k in NAMES], T(c2w[None]), T(fx[None])


def quantise(images):
    """The reference's frames (gs_core.py:1215-1216) of fp32 images [B,V,3,H,W] -> uint8 numpy [B,V,H,W,3]."""
    return (images.cpu().numpy() * 255).clip(0, 255).astype(np.uint8).transpose(0, 1, 3, 4, 2)


def arenas(V, P, H, W):
    L = _lib.lib()
    return L.dgs_raster_geom_bytes(V, P) + L.dgs_raster_image_bytes(V, W, H)


# name -> (P, V, W, H, SH degree, distribution, near_log2)
CASES = {
    "small_sh0_1view": (3000, 1, 64, 48, 0, "trained", -1),          # small-scene binning
    "small_sh3_7views": (3000, 7, 64, 48, 3, "trained", -1),
    "global_single_pass_ragged": (40000, 7, 200, 136, 3, "trained", 0),  # 7 * 40000 view-Gaussians: global binning
    "two_phase_fixed": (400000, 4, 256, 256, 0, "fine", 3),          # phase A and phase B
    "two_phase_adaptive": (400000, 4, 256, 256, 3, "fine", -1),
    "turntable_150views": (3000, 150, 64, 64, 3, "trained", -1),
}


@pytest.mark.parametrize("case", list(CASES))
def test_frames_equal_quantised_images(case):
    P, V, W, H, degree, dist, near_log2 = CASES[case]
    g, c2w, fx = scene(P, V, W, H, degree, dist, turntable=V == 150)
    images, state = raster.render_batch_forward(*g, H, W, c2w, fx, near_log2=near_log2)
    R = state["R"]
    frames = raster.render_frames(*g, H, W, c2w, fx, near_log2=near_log2)
    assert frames.dtype == torch.uint8 and tuple(frames.shape) == (1, V, H, W, 3)
    assert raster.LAST_NUM_RENDERED == R
    expect = quantise(images)
    got = frames.cpu().numpy()
    print(f"[{case}] R={R} chunks={state['chunks']} frames mean={got.mean():.2f}")
    assert np.array_equal(got, expect), f"{int((got != expect).sum())} values differ"


def test_frames_do_not_depend_on_chunking():
    """7 ragged views rendered in chunks of 1 and of 3 views (budgets of exactly that many views' arenas) and in one
    chunk: the same frames, bit for bit."""
    P, V, W, H = 3000, 7, 200, 136
    g, c2w, fx = scene(P, V, W, H, degree=1, seed=3)
    whole = raster.render_frames(*g, H, W, c2w, fx)
    for n in (1, 3):
        budget = arenas(n, P, H, W)
        assert raster.frames_chunk_views(V, P, H, W, budget) == n
        cache = {}
        chunked = raster.render_frames(*g, H, W, c2w, fx, max_arena_bytes=budget, arena_cache=cache)
        assert torch.equal(chunked, whole), n
        assert cache[("geom", 0)].numel() < arenas(n + 1, P, H, W)  # the arenas held n views, not 7


def test_frames_halve_chunks_past_the_instance_limit(monkeypatch):
    """A chunk whose instance count would pass 2^31-1 is rendered in halves (the status is injected for every call of
    more than 2 views): the same frames."""
    P, V, W, H = 3000, 5, 64, 48
    g, c2w, fx = scene(P, V, W, H, seed=4)
    whole = raster.render_frames(*g, H, W, c2w, fx)
    L = _lib.lib()
    real = L.dgs_render_frames
    views = []

    class Lib:
        def __getattr__(self, name):
            return getattr(L, name)

        @staticmethod
        def dgs_render_frames(args, *rest):
            views.append(args._obj.V)
            if args._obj.V > 2:
                raise _lib.DgsError("libdgs_b200 status 4: instance count 3000000000 exceeds 2^31-1")
            return real(args, *rest)
    monkeypatch.setattr(_lib, "lib", lambda: Lib())
    halved = raster.render_frames(*g, H, W, c2w, fx)
    assert views == [5, 2, 2, 1]
    assert torch.equal(halved, whole)


def test_arena_memory_does_not_grow_with_frames():
    """With a budget of 8 views, 64 views need no more device memory than 8 beyond their larger output: the chunks
    re-use one arena set.  The slack covers the binning arena, which grows (by 1.25x) to the largest chunk's lists."""
    P, W, H = 20000, 96, 96
    budget = arenas(8, P, H, W)

    def peak(V):
        g, c2w, fx = scene(P, V, W, H, degree=1, seed=5, turntable=True)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        frames = raster.render_frames(*g, H, W, c2w, fx, max_arena_bytes=budget)
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base, frames.numel()
    p8, out8 = peak(8)
    p64, out64 = peak(64)
    slack = (p8 - out8) // 4
    print(f"peak 8 views {p8 / 2**20:.1f} MiB, 64 views {p64 / 2**20:.1f} MiB, output difference "
          f"{(out64 - out8) / 2**20:.1f} MiB, slack {slack / 2**20:.1f} MiB")
    assert p64 - p8 <= (out64 - out8) + slack


def test_empty_model_gives_black_frames():
    """P = 0: the reference's rasterizer returns its zero-filled image for an empty model, not the white background."""
    g, c2w, fx = scene(0, 3, 40, 24)
    frames = raster.render_frames(*g, 24, 40, c2w, fx)
    assert tuple(frames.shape) == (1, 3, 24, 40, 3) and int(frames.count_nonzero()) == 0
    pc = GaussianModel(1, None).set_data(*(t[0] for t in scene(0, 1, 8, 8, degree=1)[0]))
    strip = render_turntable(pc, rendering_resolution=32, num_views=4)
    assert strip.shape == (32, 128, 3) and strip.dtype == np.uint8 and not strip.any()


def _compare(name, ours, ref):
    d = np.abs(ours.astype(np.int32) - ref.astype(np.int32))
    rel = float(np.linalg.norm(d) / np.linalg.norm(ref.astype(np.float64)))
    print(f"[{name}] max |diff| = {d.max()} LSB, {(d != 0).mean():.2e} of values differ, rel_l2 = {rel:.2e}")
    assert d.max() <= 2 and rel < 2e-3


def test_turntable_and_generic_vs_reference():
    """render_turntable (96^2, 8 views) and render_generic (136 x 200, frames of the keyframe loop) of the fixture's
    1,000 SH-degree-1 Gaussians vs the reference's own frames: within the renderer's 1e-4 plus one quantisation step."""
    z = np.load(GOLDEN)
    pc = GaussianModel(1, None).set_data(*(T(z["in/" + k]) for k in NAMES))
    strip = render_turntable(pc, rendering_resolution=96, num_views=8)
    assert strip.shape == (96, 8 * 96, 3) and strip.dtype == np.uint8
    _compare("turntable", strip, z["turntable/frames"])
    frames = render_generic(pc, torch.from_numpy(z["generic/c2ws"]), torch.from_numpy(z["generic/fxfycxcy"]), 136, 200)
    assert frames.shape == (2, 136, 200, 3) and frames.dtype == np.uint8
    _compare("generic", frames, z["generic/frames"])
