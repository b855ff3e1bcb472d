"""Mesh decimation without a GPU: the serial quadric edge-collapse oracle on marching-cubes spheres and tori (face
count, closed and oriented, topology, distance to the analytic surface), argument checks of dgs_mesh_decimate with fake
pointers, the Python wrapper's shape / dtype checks and the command line's --decimate-target."""
import ctypes

import numpy as np
import pytest

from mesh_shapes import closed_and_oriented, euler, grid, volume
from oracle import mesh as om
from oracle import mesh_decimate as od


@pytest.mark.parametrize("shape", ["sphere", "torus"])
def test_oracle_decimates_closed_surfaces(shape):
    X, Y, Z = grid(28)
    if shape == "sphere":
        r = 9.0
        field, chi = r - np.sqrt(X ** 2 + Y ** 2 + Z ** 2), 2
        dist = lambda p: np.abs(np.linalg.norm(p, axis=1) - r)  # noqa: E731
    else:
        R0, r0 = 8.0, 3.5
        field, chi = r0 - np.sqrt((np.sqrt(X ** 2 + Y ** 2) - R0) ** 2 + Z ** 2), 0
        dist = lambda p: np.abs(np.hypot(np.hypot(p[:, 0], p[:, 1]) - R0, p[:, 2]) - r0)  # noqa: E731
    v, f = om.marching_cubes(field, 0.0)
    target = len(f) // 8
    ov, of, n = od.decimate(v, f, target)
    c = (np.array(field.shape) - 1) / 2
    d = dist(ov.astype(np.float64) - c)
    vol0, vol1 = volume(v, f), volume(ov, of)
    print(f"{shape}: {len(f)} -> {len(of)} faces ({n} collapses), distance mean {d.mean():.3f} max {d.max():.3f}, "
          f"volume {vol1 / vol0:.4f} of the raw mesh's")
    assert len(of) in (target - 1, target) and n == (len(f) - len(of)) // 2
    assert ov.dtype == np.float32 and of.dtype == np.int64 and len(np.unique(of)) == len(ov)
    assert (of[:, 0] != of[:, 1]).all() and (of[:, 1] != of[:, 2]).all() and (of[:, 0] != of[:, 2]).all()
    closed_and_oriented(of)
    assert euler(of) == chi
    assert d.max() < 0.5 and abs(vol1 / vol0 - 1) < 0.03


def test_oracle_keeps_small_meshes():
    X, Y, Z = grid(12)
    v, f = om.marching_cubes(4.0 - np.sqrt(X ** 2 + Y ** 2 + Z ** 2), 0.0)
    ov, of, n = od.decimate(v, f, len(f))
    assert n == 0 and np.array_equal(ov, v.astype(np.float32)) and np.array_equal(of, f)


def test_decimate_entry_point_validates_without_gpu():
    from dgs_b200 import _lib
    L = _lib.lib()
    cb = _lib.ALLOC_FN(lambda n, u: None)
    fake = ctypes.c_void_p(256)
    outs = [ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_longlong(), ctypes.c_longlong()]
    rounds = ctypes.c_int(0)

    def call(V=100, F=196, target=10, out=None):
        o = [ctypes.byref(x) for x in outs] if out is None else out
        return L.dgs_mesh_decimate(fake, V, fake, F, target, cb, None, *o, ctypes.byref(rounds), None)
    assert call(out=[None, ctypes.byref(outs[1]), ctypes.byref(outs[2]), ctypes.byref(outs[3])]) == 1
    assert b"must not be NULL" in L.dgs_last_error()
    assert call(target=-1) == 1 and b"target_faces" in L.dgs_last_error()
    assert call(V=-1) == 1 and b"negative" in L.dgs_last_error()
    assert call(F=-5) == 1 and b"negative" in L.dgs_last_error()
    assert call(F=1 << 30) == 1 and b"too many" in L.dgs_last_error()
    assert L.dgs_mesh_decimate(None, 100, fake, 196, 10, cb, None, *[ctypes.byref(x) for x in outs], None, None) == 1
    assert b"vertices and faces" in L.dgs_last_error()


def test_decimate_wrapper_rejects_bad_input():
    import torch
    from dgs_b200 import mesh
    v, f = np.zeros((4, 3), np.float32), np.array([[0, 1, 2], [0, 2, 3]], np.int64)
    with pytest.raises(ValueError, match=r"\[V, 3\]"):
        mesh.decimate(v[:, :2], f, 1)
    with pytest.raises(ValueError, match=r"\[F, 3\]"):
        mesh.decimate(v, f.reshape(-1), 1)
    with pytest.raises(TypeError, match="floating point"):
        mesh.decimate(v.astype(np.int32), f, 1)
    with pytest.raises(TypeError, match="integer"):
        mesh.decimate(v, f.astype(np.float32), 1)
    with pytest.raises(ValueError, match="target_faces"):
        mesh.decimate(v, f, -1)
    with pytest.raises(ValueError, match="target_faces"):
        mesh.decimate(v, f, float("nan"))
    with pytest.raises(ValueError, match="int32"):
        mesh.decimate(v, f + (1 << 31), 1)
    with pytest.raises(TypeError, match="CUDA"):
        mesh.decimate(torch.from_numpy(v), torch.from_numpy(f), 1)


def test_cli_decimate_target_flag():
    from dgs_b200 import mesh
    a = mesh.parser().parse_args(["g.ply", "m.obj", "--decimate-target", "100000"])
    assert a.decimate_target == 100000
    assert mesh.parser().parse_args(["g.ply", "m.obj"]).decimate_target is None
