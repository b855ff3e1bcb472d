"""Isotropic remeshing on the H100 (dgs_mesh_remesh through dgs_b200.mesh.remesh): bit-for-bit equality with the serial
oracle (vertices, faces and stats) on hand-built meshes and on marching-cubes spheres, tori and sphere pairs; the
properties of the remeshed obj-256 mesh; the clean-remesh-decimate postprocess; determinism, numpy / CUDA-tensor
agreement and the edge cases."""
import time

import numpy as np
import pytest
import torch

from mesh_shapes import check_remeshed, components, cuda_grid, edges, mc, patch, shell_model
from oracle import mesh_clean as oc
from oracle import mesh_remesh as orr

pytestmark = pytest.mark.gpu


def _same_as_oracle(v, f, L, iterations=3, **kw):
    from dgs_b200 import mesh
    st = {}
    ov, of = mesh.remesh(v, f, L, iterations, stats=st, **kw)
    rv, rf, rs = orr.remesh(v, f, L, iterations, **kw)
    assert st["iterations"] == rs, f"stats {st['iterations']} != oracle {rs}"
    assert ov.dtype == np.float32 and of.dtype == np.int64
    assert ov.tobytes() == rv.tobytes() and np.array_equal(of, rf)
    return ov, of, rs


def _tetra():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    return v, np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]])


def _crease_strip():
    n = 8
    xs = np.arange(-n, n + 1, dtype=np.float64)
    v = np.asarray([(x, y, 0.0) if x <= 0 else (0.0, y, -x) for x in xs for y in range(4)], np.float32)
    f = [[4 * i + j, 4 * i + j + 4, 4 * i + j + 1] for i in range(len(xs) - 1) for j in range(3)]
    f += [[4 * i + j + 1, 4 * i + j + 4, 4 * i + j + 5] for i in range(len(xs) - 1) for j in range(3)]
    return v, np.asarray(f)


@pytest.mark.parametrize("case, L, it", [("tetra", 0.4, 3), ("tetra", 3.0, 2), ("crease_strip", 0.8, 3),
                                         ("crease_strip", 1.7, 2), ("patch", 0.7, 3), ("patch", 1.5, 3)])
def test_hand_cases_equal_oracle(case, L, it):
    v, f = {"tetra": _tetra, "crease_strip": _crease_strip, "patch": patch}[case]()
    ov, of, st = _same_as_oracle(v, f, L, it)
    print(f"{case} L={L}: {len(f)} -> {len(of)} faces, stats {st}")
    assert components(f) == components(of)


def _surface(shape):
    X, Y, Z = cuda_grid(44)
    if shape == "sphere":
        return mc(16 - torch.sqrt(X * X + Y * Y + Z * Z), clean=True)
    if shape == "torus":
        return mc(6 - torch.sqrt((torch.sqrt(X * X + Y * Y) - 13) ** 2 + Z * Z), clean=True)
    a = 9 - torch.sqrt((X - 10) ** 2 + Y * Y + Z * Z)
    b = 8 - torch.sqrt((X + 10) ** 2 + Y * Y + Z * Z)
    return mc(torch.maximum(a, b), clean=True)


@pytest.mark.parametrize("shape", ["sphere", "torus", "two_spheres"])
@pytest.mark.parametrize("L, it", [(1.0, 1), (1.0, 3), (1.8, 1), (1.8, 3)])
def test_surfaces_equal_oracle(shape, L, it):
    v, f = _surface(shape)
    ov, of, st = _same_as_oracle(v, f, L, it)
    print(f"{shape} L={L} it={it}: {len(f)} -> {len(of)} faces, stats {st}")
    if it == 3:
        check_remeshed(v, f, ov, of, L)


def test_obj256_properties():
    from dgs_b200 import mesh
    m = shell_model(262146, 11)
    raw = m.extract_mesh()
    v, f = mesh.clean(raw.vertices, raw.faces)
    L = 0.015
    st = {}
    ov, of = mesh.remesh(v, f, L, 3, stats=st)
    ln = check_remeshed(v, f, ov, of, L, nondegenerate=False)
    _, d2, _ = orr.closest_points(v, f, ov.astype(np.float64))
    share = float(np.mean((ln >= 0.8 * L) & (ln <= 4 * L / 3)))
    e, _ = edges(of)
    dval = float(np.abs(np.bincount(e.reshape(-1)) - 6).mean())
    print(f"obj-256 cleaned: {len(f)} -> {len(of)} faces, stats {st['iterations']}, max distance to S "
          f"{np.sqrt(d2).max():.2e}, edges in [lo, hi] {share:.3f}, mean |valence - 6| {dval:.3f}, zero-area faces "
          f"{int((oc.doubled_area(ov, of) == 0).sum())}")
    assert np.sqrt(d2).max() <= 1e-6
    # about twice the first H100 run's distance from ideal (0.842 of the edges in [lo, hi], mean |valence - 6| 0.284)
    assert share >= 0.68 and dval <= 0.57
    # determinism and CUDA-tensor input
    for _ in range(3):
        ov2, of2 = mesh.remesh(v, f, L, 3)
        assert ov2.tobytes() == ov.tobytes() and np.array_equal(of2, of)
    tv, tf = mesh.remesh(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), L, 3)
    assert tv.is_cuda and tv.dtype == torch.float32 and tf.dtype == torch.int64
    assert tv.cpu().numpy().tobytes() == ov.tobytes() and np.array_equal(tf.cpu().numpy(), of)
    # the oracle at this size
    t0 = time.perf_counter()
    rv, rf, rs = orr.remesh(v, f, L, 3)
    print(f"  oracle {time.perf_counter() - t0:.1f} s")
    assert rs == st["iterations"] and rv.tobytes() == ov.tobytes() and np.array_equal(rf, of)


def _boundary_loops(f):
    """-> the number of connected pieces of the edges with one face"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    e, cnt = edges(f)
    b = e[cnt == 1]
    if not len(b):
        return 0
    ids, inv = np.unique(b, return_inverse=True)
    inv = inv.reshape(-1, 2)
    n, _ = connected_components(coo_matrix((np.ones(len(b)), (inv[:, 0], inv[:, 1])), shape=(len(ids),) * 2),
                                directed=False)
    return n


def _sphere_field(n, r):
    x = torch.linspace(-1, 1, n, device="cuda")
    X, Y, Z = torch.meshgrid(x, x, x, indexing="ij")
    return (r - torch.sqrt(X * X + Y * Y + Z * Z)).contiguous()


def test_clean_remesh_then_decimate_closed_sphere():
    # a closed cleaned mesh comes back closed through the whole chain: a sphere of radius 0.6 in extract_mesh's frame.
    # At 96 grid points `clean` keeps it closed (checked first); at 128 its non-manifold edge repair opens 50 edges, so
    # there the remeshing is checked on the raw (closed) marching-cubes mesh instead.
    from dgs_b200 import mesh
    field = _sphere_field(96, 0.6)
    raw = mesh.extract_mesh(field, 0.0, 96)
    cv, cf = mesh.clean(raw.vertices, raw.faces)
    assert (edges(cf)[1] == 2).all(), "the cleaned sphere is not closed"
    out = mesh.extract_mesh(field, 0.0, 96, postprocess=mesh.clean_remesh_then_decimate, decimate_target=20000)
    _, cnt = edges(out.faces)
    print(f"sphere through clean_remesh_then_decimate: {len(cf)} cleaned -> {len(out.faces)} faces")
    assert 0 < len(out.faces) <= 20000 and (cnt == 2).all(), "not closed"
    assert components(out.faces) == [(2, False)]
    raw = mesh.extract_mesh(_sphere_field(128, 0.6), 0.0, 128)
    rv, rf = mesh.remesh(raw.vertices, raw.faces)
    assert (edges(rf)[1] == 2).all() and components(rf) == [(2, False)]


def test_clean_remesh_then_decimate_postprocess():
    from dgs_b200 import mesh
    m = shell_model(262146, 11)
    out = m.extract_mesh(postprocess=mesh.clean_remesh_then_decimate)
    raw = m.extract_mesh()
    cv, cf = mesh.clean(raw.vertices, raw.faces)
    _, cnt = edges(out.faces)
    _, ccnt = edges(cf)
    print(f"clean_remesh_then_decimate: {len(out.faces)} faces, {int((cnt == 1).sum())} boundary edges in "
          f"{_boundary_loops(out.faces)} loops (the cleaned input {int((ccnt == 1).sum())} in {_boundary_loops(cf)})")
    assert len(out.faces) <= 1e5 and (cnt <= 2).all()
    # This shell's cleaned mesh is not closed: the non-manifold edge repair of `clean` drops faces and leaves holes.
    # Remeshing only splits boundary edges and decimation keeps boundary loops, so the holes are neither closed nor
    # grown: the output has exactly the input's boundary loops (closed iff the input is; see the sphere test above).
    assert _boundary_loops(out.faces) == _boundary_loops(cf)
    rv, rf = mesh.remesh(cv, cf)
    if len(rf) <= 1e5:
        assert np.array_equal(out.vertices, rv) and np.array_equal(out.faces, rf)
    small = m.extract_mesh(postprocess=mesh.clean_remesh_then_decimate, decimate_target=len(rf) // 2)
    assert len(small.faces) <= len(rf) // 2


def test_edge_cases():
    from dgs_b200 import _lib, mesh
    v, f = _surface("sphere")
    bad = f.copy()
    bad[7, 1] = len(v)
    with pytest.raises(_lib.DgsError, match="face 7 "):
        mesh.remesh(v, bad, 1.0)
    bad[7, 1] = bad[7, 0]
    with pytest.raises(_lib.DgsError, match="face 7 .* repeated"):
        mesh.remesh(v, bad, 1.0)
    ov, of = mesh.remesh(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64), 1.0)
    assert ov.shape == (0, 3) and of.shape == (0, 3)
    ov, of = mesh.remesh(np.ones((5, 3), np.float32), np.zeros((0, 3), np.int64), 1.0, 0)
    assert ov.shape == (5, 3) and of.shape == (0, 3)
    vu = np.concatenate([v, [[99, 99, 99]]]).astype(np.float32)  # an unreferenced vertex
    st = {}
    ov, of = mesh.remesh(vu, f, 1.0, 0, stats=st)
    assert ov.tobytes() == vu.tobytes() and np.array_equal(of, f) and st["iterations"] == []
    # a mesh already at the target length changes little
    rv, rf = mesh.remesh(v, f, 1.2, 3)
    st = {}
    r2v, r2f = mesh.remesh(rv, rf, 1.2, 1, stats=st)
    print(f"at target: {len(rf)} -> {len(r2f)} faces, stats {st['iterations']}")
    assert st["iterations"][0][0] <= 1.05 * len(rf) and abs(len(r2f) - len(rf)) <= 0.05 * len(rf)
    _same_as_oracle(rv, rf, 1.2, 1)


@pytest.mark.parametrize("shape", ["sphere", "torus", "two_spheres"])
def test_closest_points_equal_oracle(shape):
    # the reprojection's grid query on its own: random points around and far outside the grid box, points on the
    # surface's vertices (ties between the faces around them) and on its edges
    from dgs_b200 import mesh
    v, f = _surface(shape)
    rng = np.random.default_rng(7)
    lo, hi = v.min(0).astype(np.float64), v.max(0).astype(np.float64)
    span = hi - lo
    q = np.concatenate([rng.uniform(lo - 0.3 * span, hi + 0.3 * span, (3000, 3)),
                        rng.uniform(lo - 5 * span, hi + 5 * span, (200, 3)),
                        v[rng.integers(0, len(v), 300)].astype(np.float64),
                        0.5 * (v[f[:300, 0]].astype(np.float64) + v[f[:300, 1]])])
    p, d2, t = mesh.closest_points(v, f, q)
    rp, rd2, rt = orr.closest_points(v, f, q)
    assert p.dtype == np.float64 and t.dtype == np.int64
    assert p.tobytes() == rp.tobytes() and d2.tobytes() == rd2.tobytes() and np.array_equal(t, rt)
    tp, td2, tt = mesh.closest_points(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), torch.from_numpy(q).cuda())
    assert tp.is_cuda and tp.cpu().numpy().tobytes() == p.tobytes() and np.array_equal(tt.cpu().numpy(), t)


def test_iterations_zero_cuda_output_is_the_callers():
    # the outputs of an iterations=0 call are fresh buffers: later calls on the device must not write into them
    from dgs_b200 import mesh
    v, f = _surface("sphere")
    tv, tf = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()
    ov, of = mesh.remesh(tv, tf, 1.0, 0)
    keep_v, keep_f = ov.cpu().numpy().copy(), of.cpu().numpy().copy()
    assert keep_v.tobytes() == v.tobytes() and np.array_equal(keep_f, f)
    mesh.remesh(tv, tf, 1.0, 2)
    mesh.remesh(tv * 2, tf, 1.0, 0)
    mesh.remesh(tv[:, [2, 0, 1]].contiguous(), tf, 0.7, 1)
    torch.cuda.synchronize()
    assert ov.cpu().numpy().tobytes() == keep_v.tobytes() and np.array_equal(of.cpu().numpy(), keep_f)
