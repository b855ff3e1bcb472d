"""Isotropic remeshing without a GPU: the serial oracle (oracle/mesh_remesh.py) on marching-cubes spheres and tori and on
an open patch (orientation, topology, boundary loops, face validity, edge lengths), its closest-point query against
brute force, the Python wrapper's argument checks and the command line's --remesh."""
import numpy as np
import pytest

from mesh_shapes import check_remeshed, edges, grid, patch
from oracle import mesh as om
from oracle import mesh_clean as oc
from oracle import mesh_remesh as orr


def _mc(field):
    v, f = om.marching_cubes(field, 0.0)
    v, f, _ = oc.clean(v.astype(np.float32), f, min_f=0, min_d=0)
    return v, f


def _sphere(n=28, r=10.0):
    X, Y, Z = grid(n)
    return _mc(r - np.sqrt(X * X + Y * Y + Z * Z))


def _torus(n=36):
    X, Y, Z = grid(n)
    return _mc(4.5 - np.sqrt((np.sqrt(X * X + Y * Y) - 10) ** 2 + Z * Z))


@pytest.mark.parametrize("shape", ["sphere", "torus"])
@pytest.mark.parametrize("L", [1.0, 1.6])
def test_oracle_closed_surfaces(shape, L):
    v, f = _sphere() if shape == "sphere" else _torus()
    ov, of, stats = orr.remesh(v, f, L, 3)
    ln = check_remeshed(v, f, ov, of, L)
    e, cnt = edges(of)
    assert (cnt == 2).all(), "not closed"
    val = np.bincount(e.reshape(-1))
    print(f"{shape} L={L}: {len(f)} -> {len(of)} faces, in [lo, hi] {np.mean((ln >= 0.8 * L) & (ln <= 4 * L / 3)):.3f}, "
          f"mean |valence - 6| {np.abs(val - 6).mean():.3f}, stats {stats}")
    assert np.abs(val - 6).mean() < 0.6
    _, d2, _ = orr.closest_points(v, f, ov.astype(np.float64))
    assert np.sqrt(d2).max() < 1e-5


def test_oracle_open_patch_keeps_its_boundary():
    v, f = patch()
    ov, of, _ = orr.remesh(v, f, 0.7, 3)
    check_remeshed(v, f, ov, of, 0.7)
    e, cnt = edges(f)
    b_in = {tuple(v[x]) for x in np.unique(e[cnt == 1])}
    oe, ocnt = edges(of)
    b_out = {tuple(ov[x]) for x in np.unique(oe[ocnt == 1])}
    assert b_in <= b_out, "a boundary vertex moved or went"
    # the boundary is split, never collapsed: its new vertices are midpoints on the old boundary segments
    assert len(b_out) >= len(b_in)


def test_oracle_feature_crease_is_kept():
    # a strip folded by 90 degrees along x = 0: the crease edges are feature edges, so its vertices stay put
    n = 8
    xs = np.arange(-n, n + 1, dtype=np.float64)
    pts = [(x, y, 0.0) if x <= 0 else (0.0, y, -x) for x in xs for y in range(4)]
    v = np.asarray(pts, np.float32)
    f = []
    for i in range(len(xs) - 1):
        for j in range(3):
            a = 4 * i + j
            f += [[a, a + 4, a + 1], [a + 1, a + 4, a + 5]]
    f = np.asarray(f)
    ov, of, _ = orr.remesh(v, f, 0.8, 2)
    crease = {tuple(v[4 * n + j]) for j in range(4)}
    assert crease <= {tuple(p) for p in ov}


def test_iterations_zero_and_empty():
    v, f = _sphere(12, 4.0)
    v = np.concatenate([v, [[9, 9, 9]]]).astype(np.float32)  # an unreferenced vertex stays with iterations=0
    ov, of, st = orr.remesh(v, f, 1.0, 0)
    assert ov.tobytes() == v.tobytes() and np.array_equal(of, f) and st == []
    ov, of, st = orr.remesh(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64), 1.0, 2)
    assert ov.shape == (0, 3) and of.shape == (0, 3) and st == [[0, 0, 0, 0]] * 2


def test_closest_points_against_brute_force():
    v, f = _torus(24)
    rng = np.random.default_rng(3)
    q = rng.uniform(-14, 14, (400, 3))
    q[:50] = v[rng.integers(0, len(v), 50)]  # queries on vertices: ties between the faces around them
    p, d2, t = orr.closest_points(v, f, q)
    P = v.astype(np.float64)
    for i in range(len(q)):
        qq, dd = orr.closest_on_triangles(np.repeat(q[i:i + 1], len(f), 0), P[f[:, 0]], P[f[:, 1]], P[f[:, 2]])
        j = np.lexsort((np.arange(len(f)), dd))[0]
        assert d2[i] == dd[j] and t[i] == j and np.array_equal(p[i], qq[j])


def test_closest_on_triangle_regions():
    a, b, c = np.array([[0.0, 0, 0]]), np.array([[2.0, 0, 0]]), np.array([[0.0, 2, 0]])
    for p, want in [((-1, -1, 0), (0, 0, 0)), ((3, -1, 0), (2, 0, 0)), ((-1, 3, 0), (0, 2, 0)),
                    ((1, -1, 0), (1, 0, 0)), ((-1, 1, 0), (0, 1, 0)), ((2, 2, 0), (1, 1, 0)),
                    ((0.5, 0.5, 3), (0.5, 0.5, 0))]:
        q, d2 = orr.closest_on_triangles(np.array([p], np.float64), a, b, c)
        assert np.allclose(q[0], want, atol=1e-15)


@pytest.mark.parametrize("kw, match", [(dict(target_len=0), "target_len"), (dict(target_len=-1), "target_len"),
                                       (dict(target_len=float("nan")), "target_len"),
                                       (dict(target_len=float("inf")), "target_len"),
                                       (dict(iterations=-1), "iterations"), (dict(iterations=1.5), "iterations"),
                                       (dict(feature_deg=float("nan")), "feature_deg"),
                                       (dict(max_surf_dist=-1.0), "max_surf_dist")])
def test_wrapper_argument_checks(kw, match):
    from dgs_b200 import mesh
    v = np.zeros((3, 3), np.float32)
    f = np.array([[0, 1, 2]])
    with pytest.raises(ValueError, match=match):
        mesh.remesh(v, f, **kw)


def test_wrapper_rejects_bad_inputs():
    from dgs_b200 import mesh
    v = np.zeros((3, 3), np.float32)
    with pytest.raises(ValueError, match="int32"):
        mesh.remesh(v, np.array([[0, 1, 1 << 40]]))
    with pytest.raises(TypeError):
        mesh.remesh(v.astype(np.int32), np.array([[0, 1, 2]]))
    with pytest.raises(ValueError, match="expected vertices"):
        mesh.remesh(v[:, :2], np.array([[0, 1, 2]]))


def test_cli_remesh_flag():
    from dgs_b200 import mesh
    ap = mesh.parser()
    assert ap.parse_args(["a.ply", "b.obj"]).remesh is None
    assert ap.parse_args(["a.ply", "b.obj", "--remesh"]).remesh == 0.015
    args = ap.parse_args(["a.ply", "b.obj", "--clean", "--remesh", "0.02", "--decimate-target", "500"])
    assert args.remesh == 0.02 and args.clean and args.decimate_target == 500
    kw = mesh._postprocess(args)
    assert kw["decimate_target"] == 500 and callable(kw["postprocess"])
    calls = []
    orig = (mesh.clean, mesh.remesh, mesh.decimate)
    try:
        mesh.clean = lambda v, f: (calls.append("clean"), (v, f))[1]
        mesh.remesh = lambda v, f, L: (calls.append(("remesh", L)), (v, f))[1]
        mesh.decimate = lambda v, f, t: (calls.append(("decimate", t)), (v, f[:t]))[1]
        kw["postprocess"](np.zeros((3, 3)), np.zeros((900, 3)), 500)
        assert calls == ["clean", ("remesh", 0.02), ("decimate", 500)]
        calls.clear()
        kw2 = mesh._postprocess(ap.parse_args(["a.ply", "b.obj", "--remesh"]))
        kw2["postprocess"](np.zeros((3, 3)), np.zeros((900, 3)), kw2["decimate_target"])
        assert calls == [("remesh", 0.015)]
    finally:
        mesh.clean, mesh.remesh, mesh.decimate = orig


def test_closest_points_wrapper_checks():
    from dgs_b200 import mesh
    v = np.zeros((3, 3), np.float32)
    with pytest.raises(ValueError, match="no faces"):
        mesh.closest_points(v, np.zeros((0, 3), np.int64), np.zeros((1, 3)))
    with pytest.raises(ValueError, match="queries"):
        mesh.closest_points(v, np.array([[0, 1, 2]]), np.zeros((4, 2)))
