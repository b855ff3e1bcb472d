"""The oracle's depth and alpha maps (render_buffers_oracle.render_batch_buffers: a colour render with colors_precomp = (z, 1, 0)
and bg = 0) against a direct fp64 restatement of their definitions, per pixel:
    depth = sum_i alpha_i T_i z_i,   alpha = 1 - T_final,
over the tile's depth-sorted list with the colour blend's alpha >= 1/255, power <= 0, 0.99 clamp and T < 1e-4 stop.
This checks the colour-channel construction the GPU depth / alpha tests compare against."""
import numpy as np
import torch

from util import rel_l2


def _restated(st):
    """depth, alpha [H, W] in fp64 from the oracle's projected state (xy, conic_opacity, depths, sorted tile lists)."""
    H, W = st["H"], st["W"]
    gx = (W + 15) // 16
    depth, alpha = np.zeros((H, W)), np.zeros((H, W))
    xy, co, z = st["xy"].astype(np.float64), st["conic_opacity"].astype(np.float64), st["depths"].astype(np.float64)
    for t, (s, e) in enumerate(st["ranges"].astype(np.int64)):
        ty, tx = divmod(t, gx)
        py, px = np.meshgrid(np.arange(ty * 16, min(ty * 16 + 16, H)), np.arange(tx * 16, min(tx * 16 + 16, W)), indexing="ij")
        T, D = np.ones(px.shape), np.zeros(px.shape)
        done = np.zeros(px.shape, bool)
        for g in st["point_list"][s:e].astype(np.int64):
            dx, dy = xy[g, 0] - px, xy[g, 1] - py
            A, B, C, o = co[g]
            power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy
            a = np.minimum(0.99, o * np.exp(power))
            ok = ~done & (power <= 0) & (a >= 1.0 / 255.0)
            test_T = T * (1 - a)
            done |= ok & (test_T < 1e-4)
            ok &= test_T >= 1e-4
            D = np.where(ok, D + a * T * z[g], D)
            T = np.where(ok, test_T, T)
        depth[py, px], alpha[py, px] = D, 1 - T
    return depth, alpha


def test_oracle_depth_alpha_match_the_definitions():
    from dgs_b200 import synth
    from oracle import raster as orc
    from oracle import renderer as orr
    from render_buffers_oracle import render_batch_buffers
    B, V, P, W, H = 1, 2, 200, 32, 32
    g = synth.make_gaussians(P, 5, "trained")
    c2w, fx = synth.orbit_cameras(V, W, H)
    names = ("xyz", "features", "scaling", "rotation", "opacity")
    raw = [torch.tensor(g[k][None]) for k in names]
    C2W, FX = torch.tensor(c2w[None]), torch.tensor(fx[None])
    render, depth, alpha = render_batch_buffers(*raw, H, W, C2W, FX)
    assert render.shape == (B, V, 3, H, W) and depth.shape == alpha.shape == (B, V, 1, H, W)
    assert torch.equal(render, orr.render_batch(*raw, H, W, C2W, FX))
    act = synth.activate(g)
    for v in range(V):
        view, proj, campos, tanx, tany = orr.build_camera(C2W[0, v], FX[0, v], H, W)
        st = orc.rasterize_forward(np.zeros(3, np.float32), act["means3D"], None, act["opacities"], act["scales"],
                                   act["rotations"], 1.0, None, view.numpy(), proj.numpy(), tanx, tany, H, W,
                                   act["shs"], 0, campos.numpy())
        d_ref, a_ref = _restated(st)
        assert a_ref.max() > 0.5 and d_ref.max() > 0  # the scene covers the view
        e_d, e_a = rel_l2(depth[0, v, 0].numpy(), d_ref), rel_l2(alpha[0, v, 0].numpy(), a_ref)
        print(f"view {v}: depth rel_l2={e_d:.2e} alpha rel_l2={e_a:.2e}")
        assert e_d < 1e-4 and e_a < 1e-4
