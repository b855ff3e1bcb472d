"""TSDF fusion without a GPU: the oracle (oracle/tsdf.py) on ray-cast maps of analytic surfaces (a sphere fuses to a
closed outward mesh within a grid spacing of it, a plane seen from one side to an open sheet, constant colours come back
exactly), the observed-mask rules, the sphere cameras' coverage of the grid, and the argument checks."""
import numpy as np
import pytest
import torch

from mesh_shapes import closed_and_oriented, directed, volume
from oracle import tsdf as ot
from tsdf_cases import plane_maps, sphere_maps


def _fuse(R, maps_fn, views=100, size=96, keep=None):
    from dgs_b200.cameras import sphere_cameras
    K, c2w = sphere_cameras(views, size)
    if keep is not None:
        K, c2w = K[keep(c2w)], c2w[keep(c2w)]
    vol = ot.volume(R)
    ot.integrate(vol, c2w, K, *maps_fn(c2w, K, size, size), trunc=8.0 / (R - 1))
    return vol


def test_sphere_fuses_to_a_closed_outward_mesh_on_the_sphere():
    R, r = 48, 0.6
    vol = _fuse(R, lambda c2w, K, H, W: sphere_maps(c2w, K, H, W, r))
    v, f = ot.extract(vol)
    v = ot.to_frame(v, R)
    assert len(f) > 1000
    closed_and_oriented(f)
    assert volume(v, f) > 0, "faces must point outwards"
    err = np.abs(np.linalg.norm(v.astype(np.float64), axis=1) - r)
    assert err.max() <= 2.0 / (R - 1), err.max()
    assert len(np.unique(f)) == len(v)


def test_plane_seen_from_one_side_is_an_open_sheet():
    R, z0 = 32, 0.1
    vol = _fuse(R, lambda c2w, K, H, W: plane_maps(c2w, K, H, W, z0), keep=lambda c2w: c2w[:, 2, 3] > 1.0)
    v, f = ot.extract(vol)
    v = ot.to_frame(v, R)
    assert len(f) > 100
    d = directed(f)
    assert len(np.unique(d, axis=0)) == len(d), "consistently oriented"
    e, cnt = np.unique(np.sort(d, 1), axis=0, return_counts=True)
    assert (cnt == 1).any() and cnt.max() == 2, "an open, edge-manifold sheet"
    assert np.abs(v[:, 2] - z0).max() <= 2.0 / (R - 1)
    n = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    assert (n[:, 2] > 0).mean() > 0.99, "oriented towards the cameras"


def test_constant_colours_come_back_exactly():
    R, c = 40, (0.25, 0.5, 0.125)
    vol = _fuse(R, lambda c2w, K, H, W: sphere_maps(c2w, K, H, W, 0.55, c), views=40, size=80)
    rw = vol["rgb_weight"]
    assert (rw > 0).sum() > 1000
    got = vol["rgb_sum"][rw > 0] / rw[rw > 0][:, None].astype(np.float32)
    assert (got == np.float32(c)).all()
    v, _ = ot.extract(vol)
    rgb = ot.colors(vol, ot.to_frame(v, R))
    assert (rgb == np.float32(c)).all()
    assert (ot.colors(vol, np.full((1, 3), 0.99, np.float32)) == 1).all(), "no coloured corner: white"


def test_observed_mask_rules():
    rng = np.random.default_rng(3)
    R = 14
    vol = ot.volume(R)
    vol["weight"][:] = rng.integers(1, 4, (R, R, R)) * (rng.random((R, R, R)) > 0.06)
    vol["tsdf_sum"][:] = rng.uniform(0.05, 1.0, (R, R, R)).astype(np.float32) * rng.choice([-1, 1], (R, R, R))
    obs = vol["weight"] > 0
    v, f = ot.extract(vol)
    assert len(f) > 50
    assert np.array_equal(np.unique(f), np.arange(len(v))), "every vertex is referenced"
    lo = np.floor(v).astype(np.int64)
    axis = np.argmax(v != lo, axis=1)
    assert ((v != lo).sum(1) == 1).all()
    hi = lo.copy()
    hi[np.arange(len(v)), axis] += 1
    assert obs[tuple(lo.T)].all() and obs[tuple(hi.T)].all(), "a vertex on an unobserved point's edge"
    for tri in f:
        ends = np.concatenate([lo[tri], hi[tri]])
        o, e = ends.min(0), ends.max(0)
        assert (e - o <= 1).all()
        assert obs[o[0]:o[0] + 2, o[1]:o[1] + 2, o[2]:o[2] + 2].all(), "a face on an unobserved point"
    # without the mask the same volume's unobserved points (value 0, outside) would make more surface
    full = ot.marching_cubes_observed(ot.field(vol), np.ones_like(obs))
    assert len(full[1]) > len(f)


def test_sphere_cameras_see_the_whole_grid():
    from dgs_b200.cameras import sphere_cameras
    for n, size in ((100, 512), (7, 33)):
        K, c2w = sphere_cameras(n, size)
        assert K.shape == (n, 4) and c2w.shape == (n, 4, 4)
        assert np.allclose(np.linalg.norm(c2w[:, :3, 3], axis=1), 4)
        corners = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float64)
        for k in range(n):
            R, t = c2w[k, :3, :3], c2w[k, :3, 3]
            assert np.allclose(R.T @ R, np.eye(3))
            pc = (corners - t) @ R
            assert (pc[:, 2] > 0.2).all()
            u = K[k, 0] * pc[:, 0] / pc[:, 2] + K[k, 2]
            v = K[k, 1] * pc[:, 1] / pc[:, 2] + K[k, 3]
            assert ((u > 0) & (u < size) & (v > 0) & (v < size)).all()
            assert np.allclose(-R[:, 2] * 4, t), "looking at the origin"


def test_argument_checks():
    from dgs_b200 import _lib, mesh
    g = [torch.zeros(4, 3), torch.zeros(4, 1, 3), torch.zeros(4, 3), torch.ones(4, 4), torch.zeros(4, 1)]
    for res in (1, 513, 64.5):
        with pytest.raises(ValueError, match="resolution"):
            mesh.tsdf_fusion(*g, resolution=res)
    with pytest.raises(ValueError, match="both c2ws and fxfycxcy"):
        mesh.tsdf_fusion(*g, c2ws=np.eye(4)[None])
    with pytest.raises(ValueError, match=r"c2ws \[n, 4, 4\]"):
        mesh.tsdf_fusion(*g, c2ws=np.eye(4)[None], fxfycxcy=np.ones((2, 4)))
    with pytest.raises(ValueError, match="square"):
        mesh.tsdf_fusion(*g, image_size=(64, 32))
    with pytest.raises(ValueError, match="alpha_thresh"):
        mesh.tsdf_fusion(*g, alpha_thresh=0)
    with pytest.raises(ValueError, match="sdf_trunc"):
        mesh.tsdf_fusion(*g, sdf_trunc=-1.0)
    with pytest.raises(_lib.DgsError, match="CUDA"):
        mesh.tsdf_fusion(*g)
    L = _lib.lib()
    rc = L.dgs_tsdf_extract(None, None, 1, _lib.ALLOC_FN(lambda n, u: None), None, None, None, None, None, None)
    assert rc != 0 and b"resolution" in L.dgs_last_error()
    rc = L.dgs_tsdf_integrate(1, None, None, 8, 8, None, None, None, None, 16, 0.1, 0.5, None, None, None, None,
                              _lib.ALLOC_FN(lambda n, u: None), None, None)
    assert rc != 0 and b"four volume arrays" in L.dgs_last_error()
    rc = L.dgs_tsdf_colors(None, None, 16, None, -1, None, None)
    assert rc != 0 and b"negative size" in L.dgs_last_error()
    with pytest.raises(SystemExit):
        mesh.parser().parse_args(["a.ply", "b.obj", "--tsdf", "--poisson"])
    assert mesh.parser().parse_args(["a.ply", "b.obj", "--tsdf"]).tsdf
