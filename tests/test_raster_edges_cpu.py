"""Host checks behind test_raster_edges_gpu.py, no GPU needed:
  * the oracle's scaling-modifier semantics (GaussianModel.get_scaling: S = exp(s) m outside a rasterizer run with mod = 1):
    rendering (scaling, m) equals rendering (scaling + ln m, None), images and every gradient, d(scaling) included;
  * each hostile scene of raster_edge_scenes.py has the property it is named for, measured with the oracle's own
    depths, radii, conic_opacity, final_T and n_contrib."""
import math

import numpy as np
import pytest
import torch

import raster_edge_scenes as es
from util import oracle_forward, rel_l2

NAMES = ("xyz", "features", "scaling", "rotation", "opacity")


@pytest.mark.parametrize("m", [0.5, 1.7])
def test_oracle_scaling_modifier_is_a_log_scale_shift(m):
    from dgs_b200 import synth
    from oracle import raster as orc
    from oracle import renderer as orr
    B, V, P, W, H = 1, 2, 600, 48, 32
    raw = {k: v[None] for k, v in synth.make_gaussians(P, 5, "trained").items()}
    c2w, fx = synth.orbit_cameras(V, W, H)
    c2w, fx = torch.tensor(c2w[None]), torch.tensor(fx[None])
    up = torch.tensor(np.random.default_rng(6).normal(0, 1, (B, V, 3, H, W)).astype(np.float32))
    orc.set_f64(True)  # no fp32 threshold flips between the two runs: they differ only in the rounding of exp
    try:
        outs = []
        for shift, mod in ((0.0, m), (math.log(m), None)):
            leaves = [torch.tensor(raw[k], requires_grad=True) for k in NAMES]
            scaling = leaves[2] + shift
            img = orr.render_batch(leaves[0], leaves[1], scaling, leaves[3], leaves[4], H, W, c2w, fx,
                                   scaling_modifier=mod)
            (img * up).sum().backward()
            outs.append((img.detach(), [t.grad for t in leaves]))
    finally:
        orc.set_f64(False)
    (img_m, g_m), (img_s, g_s) = outs
    e = rel_l2(img_m.numpy(), img_s.numpy())
    print(f"m={m}: image rel_l2={e:.2e}")
    assert e < 1e-6
    for k, a, b in zip(NAMES, g_m, g_s):
        e = rel_l2(a.numpy(), b.numpy())
        print(f"  d{k}: rel_l2={e:.2e}")
        assert e < 1e-5, k
    # the factor m is really in d(scaling): without it the two would differ by |1 - 1/m|
    assert rel_l2(g_m[2].numpy() / m, g_s[2].numpy()) > 0.2


def _scene_state(name):
    sc = es.SCENES[name]()
    return sc, oracle_forward(sc), es.view_xyz(sc)


def test_near_plane_scene():
    sc, st, pv = _scene_state("near_plane")
    z = st["depths"]
    near = (pv[:, 2] > 0.2) & (pv[:, 2] <= 0.25)
    culled = pv[:, 2] <= 0.2
    print(f"near_plane: {near.sum()} in (0.2, 0.25], {culled.sum()} <= 0.2, max radius {st['radii'].max()}")
    assert near.sum() >= 100 and culled.sum() >= 100
    assert np.all(st["radii"][culled] == 0)
    assert np.all(st["radii"][near] > 0) and np.allclose(z[near], pv[near, 2], rtol=1e-6)
    assert st["radii"].max() >= 100  # J ~ 1/z^2: splats of hundreds of pixels


def test_camera_inside_scene():
    sc, st, pv = _scene_state("camera_inside")
    behind = pv[:, 2] <= 0.2
    print(f"camera_inside: {behind.mean():.2f} behind the near plane, max radius {st['radii'].max()}, "
          f"min final_T {st['final_T'].min():.2e}")
    assert 0.4 < behind.mean() < 0.7 and np.all(st["radii"][behind] == 0)
    assert (st["radii"] > max(sc["W"], sc["H"])).sum() >= 3  # splats wider than the image
    ranges = st["ranges"].astype(np.int64)
    assert (ranges[:, 1] - ranges[:, 0]).min() >= 3  # every tile has the large splats in its list


def test_frustum_edge_scene():
    sc, st, pv = _scene_state("frustum_edge")
    lim_x, lim_y = 1.3 * sc["tanx"], 1.3 * sc["tany"]
    vis = st["radii"] > 0
    ax, ay = np.abs(pv[:, 0] / pv[:, 2]), np.abs(pv[:, 1] / pv[:, 2])
    counts = dict(x_in=(vis & (ax < lim_x) & (ax > sc["tanx"])).sum(), x_out=(vis & (ax > lim_x)).sum(),
                  y_in=(vis & (ay < lim_y) & (ay > sc["tany"])).sum(), y_out=(vis & (ay > lim_y)).sum())
    print(f"frustum_edge: rendered {vis.sum()} of {sc['P']}, {counts}")
    assert np.all((ax >= 1.1 * sc["tanx"] - 1e-6) | (ay >= 1.1 * sc["tany"] - 1e-6))
    assert all(v >= 10 for v in counts.values()), counts


def test_needles_pancakes_scene():
    sc, st, _ = _scene_state("needles_pancakes")
    A, B, C = (st["conic_opacity"][:, k].astype(np.float64) for k in range(3))
    vis = st["radii"] > 0
    needle = np.arange(sc["P"]) % 2 == 0
    rel_det = np.ones(sc["P"])
    rel_det[vis] = (A * C - B * B)[vis] / (A * C)[vis]  # the splat is a sliver where A C ~ B^2
    rn, rp = rel_det[vis & needle], rel_det[vis & ~needle]
    print(f"needles_pancakes: rendered {vis.sum()}, det/(AC) of the conic: needles median {np.median(rn):.2e}, "
          f"pancakes 10th percentile {np.percentile(rp, 10):.2e}")
    assert rn.size >= 300 and rp.size >= 300
    assert np.median(rn) < 0.05 and np.percentile(rp, 10) < 0.2  # pancakes seen edge-on are slivers too


def test_sub_pixel_scene():
    sc, st, _ = _scene_state("sub_pixel")
    vis = st["radii"] > 0
    A, C = st["conic_opacity"][vis, 0], st["conic_opacity"][vis, 2]
    print(f"sub_pixel: rendered {vis.sum()}, radii {np.unique(st['radii'][vis])}, conic A in [{A.min():.4f}, {A.max():.4f}]")
    assert vis.sum() >= 2000 and st["radii"].max() <= 3
    assert np.allclose(A, 1 / 0.3, rtol=1e-2) and np.allclose(C, 1 / 0.3, rtol=1e-2)  # the dilation alone


def test_opaque_scene():
    sc, st, _ = _scene_state("opaque")
    op = st["conic_opacity"][st["radii"] > 0, 3]
    sat = st["final_T"] < 1e-3
    # the blend stops once T would fall below 1e-4: a saturated pixel's last contributor comes before its tile list ends
    H, W = sc["H"], sc["W"]
    tile = ((np.arange(H) // 16)[:, None] * ((W + 15) // 16) + (np.arange(W) // 16)[None, :]).ravel()
    ranges = st["ranges"].astype(np.int64)
    stopped = st["n_contrib"].astype(np.int64) < (ranges[tile, 1] - ranges[tile, 0])
    print(f"opaque: opacity >= {op.min():.4f}, saturated pixels {sat.mean():.2f}, "
          f"{stopped[sat].mean():.2f} of them stopped before their tile list ends")
    assert op.min() > 0.99 and sat.mean() > 0.2 and stopped[sat].mean() > 0.9


def test_threshold_scene():
    sc, st, _ = _scene_state("threshold")
    op = st["conic_opacity"][st["radii"] > 0, 3].astype(np.float64)
    lit = (st["n_contrib"] > 0).sum()
    print(f"threshold: 255 opacity - 1 in [{(255 * op - 1).min():.2e}, {(255 * op - 1).max():.2e}], "
          f"{(255 * op >= 1).mean():.2f} above, {lit} pixels with a contributor")
    assert op.size >= 1000 and np.all(np.abs(255 * op - 1) <= 1.001e-3)
    assert 0.3 < (255 * op >= 1).mean() < 0.7 and lit >= 50


def test_depth_ties_scene():
    sc, st, pv = _scene_state("depth_ties")
    z = st["depths"]
    print(f"depth_ties: distinct depths {np.unique(z).size}, R={st['num_rendered']}")
    assert np.unique(z).size == 1 and np.unique(z.view(np.uint32)).size == 1 and np.all(st["radii"] > 0)
    ranges = st["ranges"].astype(np.int64)
    assert (ranges[:, 1] - ranges[:, 0]).max() >= 100  # the ties overlap: long equal-depth runs in one tile


def test_rotation_norms_scene():
    sc, st, _ = _scene_state("rotation_norms")
    n = np.linalg.norm(sc["raw"]["rotation"].astype(np.float64), axis=1)
    print(f"rotation_norms: |q| in {np.unique(np.round(np.log10(n)))}")
    assert np.allclose(n[0::2], 1e-6, rtol=1e-5) and np.allclose(n[1::2], 1e4, rtol=1e-5)
    assert np.allclose(np.linalg.norm(sc["act"]["rotations"], axis=1), 1.0, atol=1e-6)
    assert (st["radii"] > 0).sum() > 1000
