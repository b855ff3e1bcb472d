"""Writes tests/golden/render_video_ref.npz: the camera paths and video frames of the REFERENCE's own code --
gs_core.py's get_turntable_cameras, render_turntable and render_generic, cam_utils.py's get_interpolated_poses_many on a
keyframe loop closed as utils/saving.py:479-496 closes it -- executed by path from the reference checkout on CPU
tensors, with the compiled `_C` underneath replaced by the CPU oracle (see ref_import.py).  Also stored: the Gaussians
(1,000 on a shell, SH degree 1).  The fp32 render_opencv_cam images the frames are quantised from are checked here, not
stored: quantising each view's image as gs_core.py:1215-1216 does must give the reference's frames.

cam_utils.py imports jaxtyping (annotations only; stubbed when absent) and was written for numpy 1.x, where
np.array(x, dtype, copy=False) copies when it must; numpy 2 raises instead, so the module runs with a numpy whose
`array` keeps the 1.x meaning.

    python tests/golden/make_render_video_golden.py        # needs the reference checkout (DGS_REFERENCE_ROOT)

The file is written with fixed zip timestamps, so a rerun reproduces it byte for byte.
"""
import io
import os
import sys
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [HERE, ROOT, os.path.join(ROOT, "open-diffusiongs_b200")]
import ref_import as ri  # noqa: E402
from dgs_b200 import synth  # noqa: E402


class _Subscriptable:
    def __getitem__(self, _):
        return object


class _Numpy1:
    """numpy with the 1.x meaning of np.array(..., copy=False): copy when needed."""

    def __getattr__(self, name):
        return getattr(np, name)

    @staticmethod
    def array(obj, dtype=None, copy=True, **kw):
        return np.asarray(obj, dtype=dtype, **kw) if copy is False else np.array(obj, dtype=dtype, copy=copy, **kw)


def load_cam_utils():
    """The reference's cam_utils.py, loaded by path into the package skeleton ref_import sets up."""
    ri.load("oracle")
    if "jaxtyping" not in sys.modules:
        try:
            import jaxtyping  # noqa: F401
        except ImportError:
            ri._mod("jaxtyping", Float=_Subscriptable())
    cu = ri._load("diffusionGS.models.gsrenderer.cam_utils",
                  os.path.join(ri.REF, "diffusionGS", "models", "gsrenderer", "cam_utils.py"))
    cu.np = _Numpy1()
    return cu

OUT = os.path.join(HERE, "render_video_ref.npz")
P, SH_DEGREE, SEED = 1000, 1, 31
TURNTABLE_RES, TURNTABLE_VIEWS = 96, 8
GENERIC_H, GENERIC_W = 136, 200
STEPS = 60  # frames per keyframe transition (save_guassians_ply_scene's num_frames)


def gaussians():
    """A trained-like object: 1,000 Gaussians on a shell, SH degree 1 (the rest coefficients small, as trained)."""
    g = synth.make_shell_gaussians(P, SEED, "trained")
    rest = np.random.default_rng(SEED + 1).normal(0, 0.3, (P, (SH_DEGREE + 1) ** 2 - 1, 3)).astype(np.float32)
    g["features"] = np.concatenate([g["features"], rest], axis=1)
    return g


def look_at(pos, target=(0.0, 0.0, 0.0), up=(0.0, 0.0, 1.0)):
    """OpenCV camera-to-world [4, 4] at pos looking at target (columns right, down, forward)."""
    pos = np.asarray(pos, np.float64)
    f = np.asarray(target, np.float64) - pos
    f /= np.linalg.norm(f)
    r = np.cross(f, up)
    r /= np.linalg.norm(r)
    d = np.cross(f, r)
    c2w = np.eye(4)
    c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = r, d, f, pos
    return c2w


def keyframes():
    """Four keyframes, each transition a case of the slerp: 0 -> 1 a plain arc; 1 -> 2 two orientations whose
    quaternions have a negative dot product (the shortest-path flip); 2 -> 3 the same rotation, the camera dollying in
    (the |d| = 1 branch); 3 -> 0 closes the loop.  Every keyframe has its own intrinsics."""
    az = np.deg2rad([0.0, 60.0, 200.0, 200.0])
    radius = [2.6, 2.4, 2.8, 2.1]
    c2ws = np.stack([look_at([r * np.cos(a), r * np.sin(a), 0.5]) for a, r in zip(az, radius)])
    c2ws[3, :3, :3] = c2ws[2, :3, :3]
    c2ws[3, :3, 3] = c2ws[2, :3, 3] + 0.7 * c2ws[2, :3, 2]
    fx = np.array([[190.0, 188.0, 100.0, 68.0], [210.0, 214.0, 97.5, 70.0], [170.0, 169.0, 103.0, 66.5],
                   [230.0, 231.0, 100.5, 67.5]])
    return torch.tensor(c2ws, dtype=torch.float32), torch.tensor(fx, dtype=torch.float32)


def keyframe_path(cam_utils, c2ws_key, fx_key):
    """save_guassians_ply_scene's camera path (saving.py:479-496) -> c2ws [n, 4, 4], fxfycxcy [n, 4], fp32."""
    Ks = torch.zeros((c2ws_key.shape[0], 3, 3))
    Ks[:, 0, 0], Ks[:, 1, 1], Ks[:, 0, 2], Ks[:, 1, 2] = fx_key[:, 0], fx_key[:, 1], fx_key[:, 2], fx_key[:, 3]
    c2ws = torch.cat([c2ws_key, c2ws_key[[0], :]], dim=0)
    Ks = torch.cat([Ks, Ks[[0], :]], dim=0)
    poses, k = cam_utils.get_interpolated_poses_many(c2ws[:, :3, :4], Ks, STEPS, order_poses=False)
    frame_c2ws = torch.cat([poses, torch.tensor([[[0, 0, 0, 1]]]).repeat(poses.shape[0], 1, 1)], dim=1)
    fxfycxcy = torch.stack([k[:, 0, 0], k[:, 1, 1], k[:, 0, 2], k[:, 1, 2]], dim=1)
    return poses, k, frame_c2ws, fxfycxcy


def quantise(image):
    """gs_core.py:1215-1216 on one fp32 image [3, h, w] -> uint8 [h, w, 3]."""
    return (image * 255).clip(0, 255).astype(np.uint8).transpose(1, 2, 0)


def savez_fixed(path, arrays):
    """np.savez_compressed with a fixed timestamp on every member, so equal arrays give an equal file."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for name, a in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(a), allow_pickle=False)
            info = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def main():
    gs, cu = ri.load("oracle").gs_core, load_cam_utils()
    rec = {}
    for n, res in ((8, 384), (150, 512)):
        w, h, v, fxfycxcy, c2ws = gs.get_turntable_cameras(w=res, h=res, num_views=n)
        rec[f"turntable{n}/fxfycxcy"], rec[f"turntable{n}/c2ws"], rec[f"turntable{n}/whv"] = fxfycxcy, c2ws, (w, h, v)
    c2ws_key, fx_key = keyframes()
    q = [cu.quaternion_from_matrix(c[:3, :3].numpy()) for c in c2ws_key]
    assert np.dot(q[1], q[2]) < 0 and abs(abs(np.dot(q[2], q[3])) - 1) < cu._EPS  # the cases keyframes() promises
    poses, k, frame_c2ws, frame_fx = keyframe_path(cu, c2ws_key, fx_key)
    rec.update({"path/key_c2ws": c2ws_key.numpy(), "path/key_fxfycxcy": fx_key.numpy(), "path/poses": poses.numpy(),
                "path/Ks": k.numpy()})

    g = gaussians()
    rec.update({"in/" + key: val for key, val in g.items()})
    pc = gs.GaussianModel(SH_DEGREE, None)
    pc.set_data(*(torch.from_numpy(g[key]) for key in ("xyz", "features", "scaling", "rotation", "opacity")))
    with ri.cpu_device_shim(), torch.no_grad():
        rec["turntable/frames"] = gs.render_turntable(pc, rendering_resolution=TURNTABLE_RES, num_views=TURNTABLE_VIEWS)
        _, _, _, fxfycxcy, c2ws = gs.get_turntable_cameras(w=TURNTABLE_RES, h=TURNTABLE_RES, num_views=TURNTABLE_VIEWS)
        c2ws, fxfycxcy = torch.from_numpy(c2ws).float(), torch.from_numpy(fxfycxcy).float()  # as render_turntable
        images = [gs.render_opencv_cam(pc, TURNTABLE_RES, TURNTABLE_RES, c2ws[j], fxfycxcy[j])["render"].numpy()
                  for j in range(TURNTABLE_VIEWS)]
        strip = np.concatenate([quantise(im) for im in images], axis=1)
        assert np.array_equal(strip, rec["turntable/frames"])
        pick = np.array([1, 2], dtype=np.int64) * STEPS + STEPS // 3  # inside the flipped and the equal-rotation transition
        c2ws, fxfycxcy = frame_c2ws[pick], frame_fx[pick]
        rec["generic/pick"], rec["generic/c2ws"], rec["generic/fxfycxcy"] = pick, c2ws.numpy(), fxfycxcy.numpy()
        rec["generic/frames"] = gs.render_generic(pc, c2ws, fxfycxcy, GENERIC_H, GENERIC_W)
        for j in range(len(pick)):
            image = gs.render_opencv_cam(pc, GENERIC_H, GENERIC_W, c2ws[j], fxfycxcy[j])["render"].numpy()
            assert np.array_equal(quantise(image), rec["generic/frames"][j])
    savez_fixed(OUT, rec)
    for key in ("turntable/frames", "generic/frames"):
        print(key, rec[key].shape, rec[key].dtype, f"mean={rec[key].mean():.2f}")
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
