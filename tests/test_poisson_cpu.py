"""Point-cloud reconstruction without a GPU: the oracle's brute-force kNN against a k-d tree, its outlier rule, its
direct solve and its depth-5 reconstruction of a sphere (closed, outward, within a cell), and the Python wrappers'
argument checks."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

from mesh_shapes import closed_and_oriented, euler, volume
from oracle import poisson as opo


def sphere(n, r=0.5, seed=0):
    d = np.random.default_rng(seed).normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return (r * d).astype(np.float32), d.astype(np.float32)


def clouds():
    rng = np.random.default_rng(1)
    uniform = rng.uniform(-1, 1, (1500, 3)).astype(np.float32)
    clustered = np.concatenate([rng.normal(0, 1e-3, (700, 3)), 100 + rng.normal(0, 10, (700, 3)),
                                rng.uniform(-1, 1, (100, 3))]).astype(np.float32)
    duplicates = np.round(rng.uniform(-1, 1, (1500, 3)) * 3).astype(np.float32) / 3  # 343 distinct positions
    return {"uniform": uniform, "clustered": clustered, "duplicates": duplicates}


@pytest.mark.parametrize("name", ["uniform", "clustered", "duplicates"])
@pytest.mark.parametrize("k", [1, 4, 20])
def test_oracle_knn_is_the_kdtree_query(name, k):
    p = clouds()[name]
    idx, d2 = opo.knn(p, k)
    dd, _ = cKDTree(p.astype(np.float64)).query(p.astype(np.float64), k)
    dd = dd.reshape(len(p), k)
    exact = (p[idx].astype(np.float64) - p[:, None].astype(np.float64)) ** 2
    np.testing.assert_allclose(exact.sum(-1), dd ** 2, rtol=1e-6, atol=1e-12)  # the same neighbour distances
    np.testing.assert_allclose(d2, dd ** 2, rtol=1e-5, atol=1e-12)
    # (distance, index) order: ties go to the smaller index
    assert ((d2[:, 1:] > d2[:, :-1]) | ((d2[:, 1:] == d2[:, :-1]) & (idx[:, 1:] > idx[:, :-1]))).all()
    assert (d2[:, 0] == 0).all() and (idx[:, 0] <= np.arange(len(p))).all()


def test_oracle_knn_pads_missing_neighbours():
    idx, d2 = opo.knn(np.zeros((2, 3), np.float32), 4)
    assert (idx[:, 2:] == -1).all() and np.isinf(d2[:, 2:]).all()
    # a missing neighbour counts as FLT_MAX: two of them overflow to inf, one leaves FLT_MAX / 3
    assert np.isinf(opo.distcuda2(np.zeros((2, 3), np.float32))).all()
    assert (opo.distcuda2(np.zeros((3, 3), np.float32)) == opo.FLT_MAX / np.float32(3)).all()


def test_oracle_outlier_rule():
    p, _ = sphere(3000)
    mask, _, _ = opo.outliers(p, 20, 10.0)
    assert mask.all()
    far = np.random.default_rng(2).normal(size=(5, 3))
    far = (10 * far / np.linalg.norm(far, axis=1, keepdims=True)).astype(np.float32)  # 10x the cloud's extent away
    mask, _, _ = opo.outliers(np.concatenate([p, far]), 20, 10.0)
    assert mask[:3000].all() and not mask[3000:].any()


@pytest.fixture(scope="module")
def depth5():
    p, n = sphere(4000)
    return p, opo.reconstruct(p, n, depth=5, density_quantile=0)


def test_oracle_solve_is_exact(depth5):
    assert depth5[1]["residual"] <= 1e-10


def test_oracle_reconstructs_a_sphere(depth5):
    _, o = depth5
    v, f = o["vertices"], o["faces"]
    closed_and_oriented(f)
    assert euler(f) == 2
    r = np.linalg.norm(v.astype(np.float64), axis=1)
    assert np.abs(r - 0.5).max() <= o["h"], "a vertex more than one cell off the sphere"
    assert abs(volume(v, f) / (4 / 3 * np.pi * 0.125) - 1) < 0.01  # positive: outward


def test_oracle_trim_removes_the_low_density_tail():
    p, n = sphere(2000, seed=3)
    o = opo.reconstruct(p, n, depth=4, density_quantile=0.1)
    t = np.quantile(o["density"], 0.1)
    assert len(o["vertices"]) == int((o["density"] >= t).sum()) < o["vertices_before"]
    assert o["faces"].max() < len(o["vertices"])


def test_argument_checks():
    from dgs_b200 import mesh
    p, n = sphere(100)
    with pytest.raises(ValueError, match="fewer than nb_neighbors"):
        mesh.poisson_reconstruction(p[:19], depth=5)
    bad = p.copy()
    bad[7, 1] = np.nan
    with pytest.raises(ValueError, match="non-finite"):
        mesh.poisson_reconstruction(bad, depth=5)
    with pytest.raises(ValueError, match="do not match"):
        mesh.poisson_reconstruction(p, n[:50], depth=5)
    for depth in (3, 10, 5.5):
        with pytest.raises(ValueError, match="depth"):
            mesh.poisson_reconstruction(p, n, depth=depth)
    with pytest.raises(ValueError, match="scale"):
        mesh.poisson_reconstruction(p, n, scale=0.9)
    with pytest.raises(ValueError, match="k must be"):
        mesh.knn(p, 33)
    with pytest.raises(ValueError, match=r"\[P, 3\]"):
        mesh.knn(p[:, :2], 4)


def test_command_line_selects_poisson():
    from dgs_b200 import mesh
    assert mesh.parser().parse_args(["a.ply", "b.obj"]).poisson is None
    assert mesh.parser().parse_args(["a.ply", "b.obj", "--poisson"]).poisson == 9
    assert mesh.parser().parse_args(["a.ply", "b.obj", "--poisson", "7"]).poisson == 7
