"""Point-cloud reconstruction on the H100: dgs_knn bit for bit against the brute-force oracle, simple_knn's distCUDA2
against the oracle and the reference binary, the outlier mask, normals and solution of dgs_poisson_reconstruct against
oracle/poisson.py, the geometry of reconstructed spheres and tori, and extract_mesh(method="poisson") on the shell
model."""
import numpy as np
import pytest
import torch

from mesh_shapes import closed_and_oriented, directed, euler, shell_model, volume
from oracle import poisson as opo

pytestmark = pytest.mark.gpu


def _sphere(n, r=0.5, seed=0):
    d = np.random.default_rng(seed).normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return (r * d).astype(np.float32), d.astype(np.float32)


def _clouds():
    rng = np.random.default_rng(5)
    plane = rng.uniform(-1, 1, (6000, 3))
    plane[:, 2] = 0.25
    return {
        "uniform": rng.uniform(-1, 1, (20000, 3)),
        "clustered": np.concatenate([rng.normal(0, 1e-4, (4000, 3)), 50 + rng.normal(0, 5, (4000, 3)),
                                     rng.normal(0, 1, (2000, 3))]),
        "coplanar": plane,
        "duplicates": np.round(rng.uniform(-1, 1, (8000, 3)) * 4) / 4,
    }


_CLOUDS = {k: v.astype(np.float32) for k, v in _clouds().items()}
_ORACLE = {}


def _oracle_knn(name):
    if name not in _ORACLE:
        _ORACLE[name] = opo.knn(_CLOUDS[name], 32)
    return _ORACLE[name]


@pytest.mark.parametrize("k", [1, 4, 20, 32])
@pytest.mark.parametrize("name", sorted(_CLOUDS))
def test_knn_is_the_oracle_bit_for_bit(name, k):
    from dgs_b200 import mesh
    p = torch.tensor(_CLOUDS[name], device="cuda")
    idx, d2 = mesh.knn(p, k)
    ri, rd = _oracle_knn(name)
    assert idx.dtype == torch.int32 and d2.dtype == torch.float32
    assert np.array_equal(idx.cpu().numpy(), ri[:, :k])
    assert d2.cpu().numpy().tobytes() == np.ascontiguousarray(rd[:, :k]).tobytes()
    idx2, d22 = mesh.knn(p, k)
    assert torch.equal(idx, idx2) and d2.cpu().numpy().tobytes() == d22.cpu().numpy().tobytes()


@pytest.mark.parametrize("k", [1, 4, 20, 32])
def test_knn_small_clouds(k):
    from dgs_b200 import mesh
    rng = np.random.default_rng(k)
    for P in sorted({0, 1, k - 1}):
        p = rng.normal(size=(P, 3)).astype(np.float32)
        idx, d2 = mesh.knn(p, k)
        assert idx.shape == (P, k) and d2.shape == (P, k)
        if P:
            ri, rd = opo.knn(p, k)
            assert np.array_equal(idx, ri) and d2.tobytes() == rd.tobytes()
    with pytest.raises(Exception, match="non-finite"):
        mesh.knn(torch.tensor([[0.0, 0.0, float("nan")]] * 4, device="cuda"), 2)


def test_distcuda2():
    from oracle import build_ref_simple_knn
    from simple_knn._C import distCUDA2
    p = _CLOUDS["clustered"]
    ours = distCUDA2(torch.tensor(p, device="cuda")).cpu().numpy()
    assert ours.tobytes() == opo.distcuda2(p).tobytes()
    for P in (1, 2, 3):
        small = np.random.default_rng(P).normal(size=(P, 3)).astype(np.float32)
        got = distCUDA2(torch.tensor(small, device="cuda")).cpu().numpy()
        assert got.tobytes() == opo.distcuda2(small).tobytes()
        assert np.isinf(got).all() == (P <= 2)
    ref = build_ref_simple_knn.load_module()
    if ref is None:
        pytest.skip("oracle/_ref/simple_knn_ref_C.so was not built")
    for q in (p, _CLOUDS["uniform"], np.random.default_rng(9).normal(size=(3, 3)).astype(np.float32)):
        t = torch.tensor(q, device="cuda")
        a, b = distCUDA2(t).cpu().numpy(), ref.distCUDA2(t).cpu().numpy()
        fin = np.isfinite(b)
        assert np.array_equal(np.isfinite(a), fin)
        ulp = np.abs(a[fin].view(np.int32).astype(np.int64) - b[fin].view(np.int32).astype(np.int64))
        # each of the three squared distances may differ by up to 2 ulp (the reference contracts two of its products
        # to FMAs), so their mean by a little more: on the clustered cloud 15 of 10,000 values differ by 3 ulp
        assert ulp.max() <= 4 and (ulp > 2).mean() < 0.01, f"{int((ulp > 2).sum())} values more than 2 ulp off"


def _with_outliers(n=6000, seed=0):
    p, d = _sphere(n, seed=seed)
    far = np.random.default_rng(seed + 1).normal(size=(8, 3))
    far = (10 * far / np.linalg.norm(far, axis=1, keepdims=True)).astype(np.float32)
    return np.concatenate([p, far]), np.concatenate([d, far / 10])


@pytest.mark.parametrize("given", [True, False])
def test_outliers_and_normals_match_the_oracle(given):
    from dgs_b200 import mesh
    p, n = _with_outliers()
    tr, st = {}, {}
    mesh.poisson_reconstruction(p, n if given else None, depth=5, density_quantile=0, stats=st, trace=tr)
    mask, a, thr = opo.outliers(p, 20, 10.0)
    near = np.abs(a - thr) <= 1e-12 * abs(thr)
    got = tr["inliers"].cpu().numpy()
    assert np.array_equal(got[~near], mask[~near]) and not got[-8:].any()
    assert st["inliers"] == got.sum()
    ip = p[got]
    ref = opo.unit(n[got]) if given else opo.pca_normals(ip, 20)
    out = tr["normals"].cpu().numpy()
    if given:
        assert out.tobytes() == ref.tobytes()
    else:
        np.testing.assert_allclose(out, ref, rtol=0, atol=1e-5)


@pytest.mark.parametrize("depth", [5, 6])
def test_solution_matches_the_oracle(depth):
    from dgs_b200 import mesh
    p, n = _sphere(5000, seed=depth)
    tr, st = {}, {}
    mesh.poisson_reconstruction(p, n, depth=depth, density_quantile=0, tol=1e-8, max_iters=200, stats=st, trace=tr)
    o = opo.reconstruct(p, n, depth=depth, density_quantile=0, direct=depth <= 5)
    chi = tr["chi"].cpu().numpy().astype(np.float64)
    rel = np.linalg.norm(chi - o["chi"]) / np.linalg.norm(o["chi"])
    print(f"depth {depth}: {st['iterations']} iterations, residual {st['residual']:.2e}, chi rel {rel:.2e}")
    assert st["residual"] <= 1e-8 and rel <= 1e-5
    tr2 = {}
    mesh.poisson_reconstruction(p, n, depth=depth, density_quantile=0, tol=1e-8, max_iters=200, trace=tr2)
    assert tr2["chi"].cpu().numpy().tobytes() == tr["chi"].cpu().numpy().tobytes()


def _check_sphere(v, f, h, r=0.5):
    closed_and_oriented(f)
    assert euler(f) == 2
    rad = np.linalg.norm(v.astype(np.float64), axis=1)
    assert np.abs(rad - r).max() <= h, f"a vertex {np.abs(rad - r).max() / h:.2f} cells off the sphere"
    vol = volume(v, f) / (4 / 3 * np.pi * r ** 3)
    assert abs(vol - 1) < 0.01, f"volume ratio {vol}"


@pytest.mark.parametrize("given", [True, False])
def test_sphere_geometry(given):
    from dgs_b200 import mesh
    p, n = _sphere(200000, seed=11)
    st = {}
    v, f = mesh.poisson_reconstruction(torch.tensor(p, device="cuda"), torch.tensor(n, device="cuda") if given else None,
                                       depth=8, density_quantile=0, stats=st)
    assert v.is_cuda and f.dtype == torch.int64
    print(st)
    _check_sphere(v.cpu().numpy(), f.cpu().numpy(), 1.1 / 256)


def test_torus_is_genus_one():
    from dgs_b200 import mesh
    rng = np.random.default_rng(3)
    u, w = rng.uniform(0, 2 * np.pi, (2, 150000))
    Rm, rm = 0.6, 0.2
    c = np.stack([np.cos(u), np.sin(u), np.zeros_like(u)], 1)
    n = np.stack([np.cos(w) * np.cos(u), np.cos(w) * np.sin(u), np.sin(w)], 1)
    p = Rm * c + rm * n
    v, f = mesh.poisson_reconstruction(p.astype(np.float32), n.astype(np.float32), depth=7, density_quantile=0)
    closed_and_oriented(f)
    assert euler(f) == 0
    assert volume(v, f) > 0


def test_density_trim_follows_the_quantile_rule():
    from dgs_b200 import mesh
    p, n = _sphere(50000, seed=4)
    tr, st = {}, {}
    v, f = mesh.poisson_reconstruction(p, n, depth=7, stats=st, trace=tr)
    dens = tr["density"].cpu().numpy()
    assert len(dens) == st["vertices_before"]
    assert len(v) == st["vertices"] == int((dens >= np.quantile(dens, 0.1)).sum()) < len(dens)
    assert len(f) == st["faces"] and f.max() < len(v)
    v0, f0 = mesh.poisson_reconstruction(p, n, depth=7, density_quantile=0)
    keep = dens >= np.quantile(dens, 0.1)
    np.testing.assert_array_equal(v, v0[keep])  # the kept vertices, in order


def test_depth9_converges_on_a_million_points():
    from dgs_b200 import mesh
    m = shell_model(1048578, 7, floaters=False)
    c, s = mesh.mesh_frame(m._xyz)
    p, n = mesh.gaussian_points(m._xyz, m._scaling, m._rotation, c, s)
    st = {}
    v, f = mesh.poisson_reconstruction(p, n, depth=9, stats=st)
    print(st)
    assert st["residual"] <= 1e-6 and st["iterations"] < 100
    assert len(f) > 0 and f.max() < len(v)


def test_extract_mesh_poisson_on_the_shell_model():
    from dgs_b200 import mesh
    m = shell_model(262146, 11, floaters=False)
    field = m.extract_mesh()
    assert np.array_equal(m.extract_mesh(method="field").vertices, field.vertices)
    pm = m.extract_mesh(method="poisson")
    d = directed(pm.faces)
    assert len(np.unique(d, axis=0)) == len(d), "a directed edge twice"
    # the untrimmed surface of the same points is closed
    p, n = mesh.gaussian_points(m._xyz, m._scaling, m._rotation, m.mesh_center, m.mesh_scale)
    v0, f0 = mesh.poisson_reconstruction(p, n, density_quantile=0)
    closed_and_oriented(f0.cpu().numpy())
    _, d2, _ = mesh.closest_points(field.vertices, field.faces, pm.vertices)
    cell = 2 / 255
    dist = np.sqrt(d2) / cell
    far = dist.max()
    print(f"poisson vertices: {len(pm.vertices)}, distance to the field mesh in field cells: median "
          f"{np.median(dist):.2f}, 99 % {np.quantile(dist, 0.99):.2f}, max {far:.2f}")
    # The synthetic shell's Gaussians have random rotations, so their shortest axes carry little more than the radial
    # sign the orientation gives them, and 262,146 points leave most depth-9 cells empty: the surface follows the
    # points' noise rather than the field's iso-surface.  Measured on an H100: median 8.1, max 11.1 field cells.
    assert far <= 16, f"a vertex {far:.1f} field cells (2 / 255) from the field mesh"
    m._features_dc = torch.rand(len(m._xyz), 1, 3, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    post = m.extract_mesh(method="poisson", postprocess=mesh.clean_remesh_then_decimate, vertex_colors=True)
    assert len(post.faces) <= 1e5 and post.vertex_colors.shape == post.vertices.shape
