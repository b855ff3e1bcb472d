"""Mesh decimation on the H100 (dgs_mesh_decimate through dgs_b200.mesh.decimate): face counts, closed and oriented
output, topology per component, distance to the analytic surface, boundary loops of open surfaces, quality against the
serial oracle, the extract_mesh pipeline at the obj-256 size, determinism and the edge cases."""
import numpy as np
import pytest
import torch

from mesh_shapes import closed_and_oriented, cuda_grid, directed, euler_per_component, mc, shell_model, volume
from oracle import mesh_decimate as od

pytestmark = pytest.mark.gpu

# Bounds, from the first H100 run (measured values in the comments; each bound has about 2x margin over them).
SPHERE_DIST = {5000: 0.1, 500: 0.7}  # max | |x - c| - r | in grid units, r = 40: measured 0.046 / 0.361
SPHERE_VOL = {5000: 0.002, 500: 0.02}  # |volume / raw volume - 1|: measured 0.0008 / 0.0097
PIPELINE_DIST = 7e-3  # max distance of a decimated vertex to the raw surface (extract_mesh units): measured 3.6e-3


def _clean(faces):
    assert (faces[:, 0] != faces[:, 1]).all() and (faces[:, 1] != faces[:, 2]).all() and (faces[:, 0] != faces[:, 2]).all()
    assert len(np.unique(np.sort(faces, axis=1), axis=0)) == len(faces), "a duplicate face"


def _sphere(n, r):
    X, Y, Z = cuda_grid(n)
    return mc(r - torch.sqrt(X * X + Y * Y + Z * Z))


def _torus(n, R0, r0):
    X, Y, Z = cuda_grid(n)
    return mc(r0 - torch.sqrt((torch.sqrt(X * X + Y * Y) - R0) ** 2 + Z * Z))


def _sphere_dist(v, n, r):
    return np.abs(np.linalg.norm(v.astype(np.float64) - (n - 1) / 2, axis=1) - r)


def _torus_dist(v, n, R0, r0):
    p = v.astype(np.float64) - (n - 1) / 2
    return np.abs(np.hypot(np.hypot(p[:, 0], p[:, 1]) - R0, p[:, 2]) - r0)


def _decimate(v, f, target):
    from dgs_b200 import mesh
    return mesh.decimate(v, f, target)


@pytest.mark.parametrize("target", [5000, 500])
def test_sphere(target):
    n, r = 128, 40.0
    v, f = _sphere(n, r)
    ov, of = _decimate(v, f, target)
    d = _sphere_dist(ov, n, r)
    vol = volume(ov, of) / volume(v, f)
    print(f"sphere r={r}: {len(f)} -> {len(of)} faces, {len(ov)} vertices, distance mean {d.mean():.4f} max "
          f"{d.max():.4f}, volume / raw {vol:.5f}")
    assert ov.dtype == np.float32 and of.dtype == np.int64
    assert len(of) in (target - 1, target)
    _clean(of)
    closed_and_oriented(of)
    assert euler_per_component(of) == [2]
    assert len(np.unique(of)) == len(ov)
    assert d.max() <= SPHERE_DIST[target] and abs(vol - 1) <= SPHERE_VOL[target]


def test_torus_and_two_spheres_keep_topology():
    v, f = _torus(128, 36.0, 14.0)
    ov, of = _decimate(v, f, 2000)
    print(f"torus: {len(f)} -> {len(of)} faces, distance max {_torus_dist(ov, 128, 36.0, 14.0).max():.4f}")
    assert len(of) in (1999, 2000) and euler_per_component(of) == [0]
    _clean(of)
    closed_and_oriented(of)
    X, Y, Z = cuda_grid(128)
    two = torch.maximum(20 - torch.sqrt((X - 30) ** 2 + Y * Y + Z * Z), 15 - torch.sqrt((X + 30) ** 2 + Y * Y + Z * Z))
    v, f = mc(two)
    ov, of = _decimate(v, f, 1000)
    print(f"two spheres: {len(f)} -> {len(of)} faces, components {euler_per_component(of)}")
    assert len(of) in (999, 1000) and euler_per_component(of) == [2, 2]
    _clean(of)
    closed_and_oriented(of)


def test_open_surface_keeps_boundary_loops():
    g = torch.Generator("cuda").manual_seed(0)
    rnd = torch.rand(1, 1, 48, 44, 40, device="cuda", generator=g)
    field = torch.nn.functional.avg_pool3d(rnd, 5, 1, 2, count_include_pad=False)[0, 0]
    v, f = mc(field - field.mean())  # not zeroed at the grid's faces: the surface is cut open there
    ov, of = _decimate(v, f, len(f) // 3)

    def boundary(v, f):
        d = directed(f)
        fwd = {tuple(e) for e in d.tolist()}
        return {(tuple(v[a]), tuple(v[b])) for a, b in fwd if (b, a) not in fwd}
    b0, b1 = boundary(v, f), boundary(ov, of)
    print(f"open surface: {len(f)} -> {len(of)} faces, {len(b0)} boundary edges")
    assert len(b0) > 100 and b1 == b0  # the same directed edges between bit-identical positions
    assert len(of) < 0.5 * len(f)
    _clean(of)
    d = directed(of)
    assert len({tuple(e) for e in d.tolist()}) == len(d), "a directed edge is used twice"


@pytest.mark.parametrize("shape", ["sphere", "torus"])
def test_quality_against_serial_oracle(shape):
    if shape == "sphere":
        n, args = 40, (14.0,)
        v, f = _sphere(n, *args)
        dist = _sphere_dist
    else:
        n, args = 40, (11.0, 4.5)
        v, f = _torus(n, *args)
        dist = _torus_dist
    target = len(f) // 10
    gv, gf = _decimate(v, f, target)
    rv, rf, _ = od.decimate(v, f, target)
    dg, dr = dist(gv, n, *args), dist(rv, n, *args)
    print(f"{shape}: {len(f)} -> {len(gf)} (GPU) / {len(rf)} (oracle) faces; distance mean {dg.mean():.4f} / "
          f"{dr.mean():.4f}, max {dg.max():.4f} / {dr.max():.4f}")
    assert len(gf) in (target - 1, target) and len(rf) in (target - 1, target)
    closed_and_oriented(gf)
    assert dg.mean() <= 2 * dr.mean() and dg.max() <= 2 * dr.max()


def test_extract_mesh_pipeline():
    from scipy.spatial import cKDTree
    from dgs_b200 import mesh
    m = shell_model(262146, 11, "fine", floaters=False)
    raw = m.extract_mesh()
    dec = m.extract_mesh(postprocess=mesh.decimate)
    again = m.extract_mesh(postprocess=mesh.decimate)
    F = len(dec.faces)
    assert F in (99999, 100000)
    _clean(dec.faces)
    closed_and_oriented(dec.faces)
    chi_raw, chi_dec = euler_per_component(raw.faces), euler_per_component(dec.faces)
    assert chi_dec == chi_raw
    assert np.array_equal(dec.vertices, again.vertices) and np.array_equal(dec.faces, again.faces)
    tv, tf = mesh.decimate(torch.from_numpy(raw.vertices).cuda(), torch.from_numpy(raw.faces).cuda(), 1e5)
    assert tv.is_cuda and tf.dtype == torch.int64
    assert np.array_equal(tv.cpu().numpy(), dec.vertices) and np.array_equal(tf.cpu().numpy(), dec.faces)
    # distance of the decimated vertices to dense samples of the raw surface (3 x 3 barycentric grid per triangle)
    rv, rf = raw.vertices.astype(np.float64), raw.faces
    w = np.array([(i, j, 4 - i - j) for i in range(5) for j in range(5 - i)], np.float64) / 4
    samples = np.einsum("sk,fkd->fsd", w, rv[rf]).reshape(-1, 3)
    dist, _ = cKDTree(samples).query(dec.vertices.astype(np.float64))
    print(f"extract_mesh: {len(raw.faces)} -> {F} faces, {len(dec.vertices)} vertices, {len(chi_raw)} components, "
          f"distance to the raw surface mean {dist.mean():.2e} max {dist.max():.2e}")
    assert dist.max() <= PIPELINE_DIST


def test_edge_cases():
    from dgs_b200 import _lib, mesh
    v, f = _sphere(24, 8.0)
    ov, of = mesh.decimate(v, f, len(f))
    assert np.array_equal(ov, v) and np.array_equal(of, f)
    ov, of = mesh.decimate(v, f, 1e9)
    assert np.array_equal(ov, v) and np.array_equal(of, f)
    ev, ef = mesh.decimate(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64), 0)
    assert ev.shape == (0, 3) and ef.shape == (0, 3)
    ov, of = mesh.decimate(v, f, 0)
    print(f"target 0: {len(f)} -> {len(of)} faces")
    assert 4 <= len(of) < len(f) // 10
    _clean(of)
    closed_and_oriented(of)
    assert euler_per_component(of) == [2]
    bad = f.copy()
    bad[7, 1] = len(v)
    with pytest.raises(_lib.DgsError, match="face 7 .* outside"):
        mesh.decimate(v, bad, 10)
    bad = f.copy()
    bad[3, 2] = bad[3, 0]
    with pytest.raises(_lib.DgsError, match="face 3 .* repeated"):
        mesh.decimate(v, bad, 10)
