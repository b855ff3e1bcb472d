"""Validation videos on the host: the camera paths of dgs_b200.cameras against the reference's own (fixture
tests/golden/render_video_ref.npz, written by make_render_video_golden.py), the reference's frame quantisation on the
CPU oracle's renders, the argument checks of dgs_render_frames, and render_frames' chunk planner.  No GPU."""
import ctypes
import os

import numpy as np
import pytest
import torch

from dgs_b200 import _lib, raster
from dgs_b200.cameras import get_interpolated_poses_many, get_turntable_cameras
from oracle import renderer as orr

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "render_video_ref.npz")
NAMES = ("xyz", "features", "scaling", "rotation", "opacity")


@pytest.fixture(scope="module")
def ref():
    return dict(np.load(GOLDEN))


def quantise(images):
    """The reference's frames from fp32 images [v, 3, h, w] (gs_core.py:1215-1216) -> uint8 [v, h, w, 3]."""
    return (images * 255).clip(0, 255).astype(np.uint8).transpose(0, 2, 3, 1)


def keyframe_path(c2ws_key, fx_key, steps=60):
    """save_guassians_ply_scene's loop (saving.py:479-496) on dgs_b200's get_interpolated_poses_many."""
    Ks = torch.zeros((c2ws_key.shape[0], 3, 3))
    Ks[:, 0, 0], Ks[:, 1, 1], Ks[:, 0, 2], Ks[:, 1, 2] = fx_key[:, 0], fx_key[:, 1], fx_key[:, 2], fx_key[:, 3]
    c2ws = torch.cat([c2ws_key, c2ws_key[[0], :]], dim=0)
    Ks = torch.cat([Ks, Ks[[0], :]], dim=0)
    return get_interpolated_poses_many(c2ws[:, :3, :4], Ks, steps, order_poses=False)


@pytest.mark.parametrize("n, res", [(8, 384), (150, 512)])
def test_turntable_cameras_equal_reference(ref, n, res):
    w, h, v, fxfycxcy, c2ws = get_turntable_cameras(w=res, h=res, num_views=n)
    assert (w, h, v) == tuple(ref[f"turntable{n}/whv"])
    assert fxfycxcy.dtype == c2ws.dtype == np.float64
    np.testing.assert_array_equal(fxfycxcy, ref[f"turntable{n}/fxfycxcy"])
    np.testing.assert_array_equal(c2ws, ref[f"turntable{n}/c2ws"])


def test_interpolated_poses_equal_reference(ref):
    """A closed loop of four keyframes with their own intrinsics, whose transitions take the slerp's plain, flipped
    (negative quaternion dot product) and equal-rotation branches: poses and intrinsics to the last bit."""
    poses, Ks = keyframe_path(torch.from_numpy(ref["path/key_c2ws"]), torch.from_numpy(ref["path/key_fxfycxcy"]))
    assert poses.dtype == Ks.dtype == torch.float32
    assert poses.shape == (240, 3, 4) and Ks.shape == (240, 3, 3)
    np.testing.assert_array_equal(poses.numpy(), ref["path/poses"])
    np.testing.assert_array_equal(Ks.numpy(), ref["path/Ks"])
    # linspace(0, 1, steps) includes both ends: every keyframe after the first appears twice in a row
    for b in (60, 120, 180):
        assert torch.equal(poses[b - 1], poses[b]) and torch.equal(Ks[b - 1], Ks[b])


def test_interpolated_poses_refuse_reordering():
    poses, Ks = torch.eye(4)[None, :3].repeat(2, 1, 1), torch.eye(3)[None].repeat(2, 1, 1)
    with pytest.raises(NotImplementedError):
        get_interpolated_poses_many(poses, Ks, 4, order_poses=True)


def _oracle_images(ref, c2ws, fxfycxcy, h, w):
    g = {k: torch.from_numpy(ref["in/" + k]) for k in NAMES}
    with torch.no_grad():
        return np.stack([orr.render_opencv_cam(*(g[k] for k in NAMES), h, w, c2ws[j], fxfycxcy[j]).numpy()
                         for j in range(c2ws.shape[0])])


def test_oracle_frames_reproduce_reference_turntable(ref):
    """render_turntable at 96^2, 8 views: the oracle's images, quantised as the reference quantises them and put side
    by side, are the reference's frame strip bit for bit."""
    w, h, v, fxfycxcy, c2ws = get_turntable_cameras(w=96, h=96, num_views=8)
    images = _oracle_images(ref, torch.from_numpy(c2ws).float(), torch.from_numpy(fxfycxcy).float(), h, w)
    strip = quantise(images).transpose(1, 0, 2, 3).reshape(h, v * w, 3)
    np.testing.assert_array_equal(strip, ref["turntable/frames"])


def test_oracle_frames_reproduce_reference_generic(ref):
    """render_generic at 136 x 200 on frames of the keyframe loop.  The oracle builds the projection in fp64 where the
    reference's Camera uses fp32 tensors, so the images differ in the last bits and a frame value may sit one LSB away
    where the two straddle a quantisation step."""
    images = _oracle_images(ref, torch.from_numpy(ref["generic/c2ws"]), torch.from_numpy(ref["generic/fxfycxcy"]),
                            136, 200)
    d = np.abs(quantise(images).astype(np.int32) - ref["generic/frames"])
    assert d.max() <= 1 and (d != 0).mean() < 1e-3


def test_render_frames_argument_validation_without_gpu():
    """dgs_render_frames: invalid arguments -> status code + message before any device work; P = 0 is legal and
    touches nothing (the caller's zero-filled frames are the result)."""
    L = _lib.lib()
    fake = 256
    n = ctypes.c_longlong(-1)

    def call(args, frames=fake, alloc=True, num=n):
        cb = _lib.ALLOC_FN(lambda nbytes, user: None) if alloc else _lib.ALLOC_FN()  # (a NULL function pointer)
        return L.dgs_render_frames(None if args is None else ctypes.byref(args), cb, None, cb, None, cb, None, frames,
                                   None if num is None else ctypes.byref(num), None)

    def args(**kw):
        a = dict(B=1, V=2, P=10, M=1, D=0, W=16, H=16, xyz=fake, features=fake, scaling=fake, rotation=fake,
                 opacity=fake, c2w=fake, fxfycxcy=fake, scale_modifier=1.0)
        a.update(kw)
        return _lib.RenderBatchArgs(**a)
    assert call(None) == 1 and b"args is NULL" in L.dgs_last_error()
    assert call(args(D=5)) == 1 and b"SH degree" in L.dgs_last_error()
    assert call(args(D=1, M=3)) == 1 and b"SH degree" in L.dgs_last_error()
    assert call(args(W=0)) == 1 and b"bad sizes" in L.dgs_last_error()
    assert call(args(P=-1)) == 1 and b"bad sizes" in L.dgs_last_error()
    assert call(args(xyz=None)) == 1 and b"NULL input" in L.dgs_last_error()
    assert call(args(), frames=None) == 1 and b"NULL output" in L.dgs_last_error()
    assert call(args(), alloc=False) == 1 and b"allocator" in L.dgs_last_error()
    # the empty model: sizes still checked, input pointers may be NULL, nothing rendered
    empty = dict(P=0, xyz=None, features=None, scaling=None, rotation=None, opacity=None)
    assert call(args(H=0, **empty)) == 1 and b"bad sizes" in L.dgs_last_error()
    assert call(args(**empty), frames=None) == 1 and b"NULL output" in L.dgs_last_error()
    assert call(args(**empty)) == 0 and n.value == 0


@pytest.mark.parametrize("V, P, H, W, budget", [
    (150, 1_048_578, 512, 512, 2 << 30),   # the object turntable at the default budget
    (240, 200_000, 256, 256, 2 << 30),     # a scene fly-through
    (64, 20_000, 96, 96, 6 << 20),         # a budget of a few views
    (7, 3000, 136, 200, 1 << 40),          # everything in one chunk
    (150, 1_048_578, 512, 512, 1),         # below one view: still one view per chunk
])
def test_frames_chunk_planner(V, P, H, W, budget):
    """Views per chunk = the largest n <= V whose geometry + image arenas fit the budget, and at least 1."""
    L = _lib.lib()

    def arenas(n):
        return L.dgs_raster_geom_bytes(n, P) + L.dgs_raster_image_bytes(n, W, H)
    n = raster.frames_chunk_views(V, P, H, W, budget)
    assert 1 <= n <= V
    assert n == 1 or arenas(n) <= budget
    assert n == V or arenas(n + 1) > budget
    if budget == 2 << 30 and P > 1_000_000:
        assert 10 <= n <= 30  # ~100 B of geometry state per (view, Gaussian): about 20 views of the obj-512 model
