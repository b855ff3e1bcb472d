"""Mesh cleaning without a GPU: the serial oracle (oracle/mesh_clean.py) against hand-worked answers, one behaviour each,
its result on a marching-cubes sphere with a floater, argument checks of dgs_mesh_clean and of the Python wrapper, and
the command line's --clean."""
import ctypes

import numpy as np
import pytest

from mesh_clean_cases import cases
from oracle import mesh as om
from oracle import mesh_clean as oc


@pytest.mark.parametrize("case", cases(), ids=lambda c: c[0])
def test_oracle_hand_cases(case):
    _, v, f, kw, ev, ef, counts = case
    ov, of, c = oc.clean(v, f, **kw)
    assert ov.dtype == np.float32 and of.dtype == np.int64
    assert np.array_equal(ov, ev.reshape(-1, 3)) and np.array_equal(of, ef.reshape(-1, 3))
    assert c == counts


def test_distance_exactly_r_is_the_radius():
    # the case's radius is exactly 1.0, so its pair at distance 1 tests the strict comparison
    v = next(c for c in cases() if c[0] == "distance_exactly_r")[1]
    d = v.max(0).astype(np.float64) - v.min(0).astype(np.float64)
    assert (20 / 100.0) * float(np.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2])) == 1.0


def test_oracle_sphere_with_floater():
    x = np.arange(40, dtype=np.float64) - 19.5
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    field = np.maximum(14.0 - np.sqrt(X ** 2 + Y ** 2 + Z ** 2), 1.5 - np.sqrt((X - 17) ** 2 + (Y - 17) ** 2 + (Z - 17) ** 2))
    v, f = om.marching_cubes(field, 0.0)
    v = v.astype(np.float32)
    ov, of, counts = oc.clean(v, f)
    print(f"sphere + floater: {len(v)} -> {len(ov)} vertices, stage faces {counts}")
    assert counts[0] == len(f) and counts[1] < 0.7 * len(f)  # r = 1 % of the diagonal is ~0.5 grid units here
    assert counts[4] < counts[3]  # the floater
    assert len(np.unique(np.sort(of, axis=1), axis=0)) == len(of)
    assert (oc.doubled_area(ov, of) > 0).all()
    c = np.linalg.norm(ov.astype(np.float64) - 19.5, axis=1)  # index coordinates
    assert c.min() > 12 and c.max() < 16  # only the sphere is left
    assert set(map(tuple, ov.tolist())) <= set(map(tuple, v.tolist()))  # positions are copies


def test_oracle_large_indices():
    # referenced indices above 2^21: the duplicate test must compare full indices
    base = 1 << 22
    v = np.zeros((base + 8, 3), np.float32)
    v[base:base + 4] = [(0, 0, 0), (1, 0, 0), (0, 1, 0), (1, 1, 0)]
    v[base + 4] = (0, 0, 1)
    f = np.array([(base, base + 1, base + 2), (base + 2, base + 1, base), (base + 1, base + 3, base + 2),
                  (base, base + 1, base + 4)])
    ov, of, counts = oc.clean(v, f, v_pct=0, min_f=0, min_d=0)
    assert counts == [4, 4, 3, 3, 3, 3, 3, 3, 3]
    assert np.array_equal(ov, v[base:base + 5]) and np.array_equal(of, [(0, 1, 2), (1, 3, 2), (0, 1, 4)])


def test_argument_checks_without_gpu():
    from dgs_b200 import _lib
    L = _lib.lib()
    fake = ctypes.c_void_p(256)
    out = [ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_longlong(), ctypes.c_longlong()]
    refs = [ctypes.byref(o) for o in out]
    alloc = _lib.ALLOC_FN(lambda n, u: None)

    def call(V=3, F=1, v_pct=1.0, min_d=20.0, alloc_fn=alloc, v=fake, f=fake, outs=refs):
        return L.dgs_mesh_clean(v, V, f, F, v_pct, 64, min_d, 1, alloc_fn, None, *outs, None, None, None)
    assert call(alloc_fn=_lib.ALLOC_FN()) == 1 and b"must not be NULL" in L.dgs_last_error()
    assert call(outs=[None] * 4) == 1 and b"must not be NULL" in L.dgs_last_error()
    assert call(V=-1) == 1 and b"negative" in L.dgs_last_error()
    assert call(V=1 << 30, F=1 << 29) == 1 and b"too many" in L.dgs_last_error()
    assert call(v=None) == 1 and b"NULL" in L.dgs_last_error()
    assert call(v_pct=float("nan")) == 1 and b"finite" in L.dgs_last_error()
    assert call(min_d=float("inf")) == 1 and b"finite" in L.dgs_last_error()
    # no faces: an empty result, before any device work
    assert call(F=0, f=None) == 0 and out[2].value == 0 and out[3].value == 0 and not out[0].value


def test_wrapper_checks():
    torch = pytest.importorskip("torch")
    from dgs_b200 import mesh
    v, f = np.zeros((3, 3), np.float32), np.array([(0, 1, 2)])
    with pytest.raises(ValueError, match=r"clean: expected vertices \[V, 3\]"):
        mesh.clean(v[:, :2], f)
    with pytest.raises(TypeError, match="clean: vertices must be floating point"):
        mesh.clean(v, f.astype(np.float32))
    with pytest.raises(ValueError, match="finite"):
        mesh.clean(v, f, v_pct=float("nan"))
    with pytest.raises(ValueError, match="int32"):
        mesh.clean(v, f + (1 << 31))
    with pytest.raises(TypeError, match="CUDA"):
        mesh.clean(torch.from_numpy(v), torch.from_numpy(f))


def test_cli_clean_flag():
    from dgs_b200 import mesh
    a = mesh.parser().parse_args(["g.ply", "m.obj", "--clean", "--decimate-target", "1000"])
    assert a.clean and mesh._postprocess(a) == dict(postprocess=mesh.clean_then_decimate, decimate_target=1000)
    a = mesh.parser().parse_args(["g.ply", "m.obj", "--clean"])
    assert a.clean and a.decimate_target is None and "postprocess" in mesh._postprocess(a)
    a = mesh.parser().parse_args(["g.ply", "m.obj", "--decimate-target", "10"])
    assert not a.clean and mesh._postprocess(a) == dict(postprocess=mesh.decimate, decimate_target=10)
    assert mesh._postprocess(mesh.parser().parse_args(["g.ply", "m.obj"])) == {}
