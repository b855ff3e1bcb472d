"""Depth, alpha and colour maps of analytic surfaces for the TSDF tests: fp64 ray casting through pixel centres (pinhole
coordinate x + 1/2 for pixel x, as the rasterizer places them), accumulated depth = view-space z of the hit, alpha 1 on
the surface and 0 off it, and a constant colour on a white background."""
import numpy as np


def _rays(c2w, K, H, W):
    """-> (origins [n, 3], world directions [n, H, W, 3] whose camera-space z is 1)"""
    c2w, K = np.asarray(c2w, np.float64), np.asarray(K, np.float64)
    u, v = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)
    d = np.stack([(u[None] - K[:, 2, None, None]) / K[:, 0, None, None],
                  (v[None] - K[:, 3, None, None]) / K[:, 1, None, None], np.ones((len(K), H, W))], -1)
    return c2w[:, :3, 3], np.einsum("nij,nhwj->nhwi", c2w[:, :3, :3], d)


def _maps(s, hit, colour):
    """hit parameter s (= view-space z) and mask -> (image [n, 3, H, W], depth [n, H, W], alpha [n, H, W]) fp32"""
    alpha = hit.astype(np.float32)
    depth = np.where(hit, s, 0.0).astype(np.float32)
    image = np.where(hit[:, None], np.asarray(colour, np.float32)[None, :, None, None], np.float32(1))
    return image.astype(np.float32), depth, alpha


def sphere_maps(c2w, K, H, W, radius, colour=(0.25, 0.5, 0.125)):
    o, d = _rays(c2w, K, H, W)
    a = (d * d).sum(-1)
    b = 2 * (d * o[:, None, None]).sum(-1)
    c = (o * o).sum(-1)[:, None, None] - radius * radius
    disc = b * b - 4 * a * c
    s = (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a)
    return _maps(s, (disc > 0) & (s > 0), colour)


def plane_maps(c2w, K, H, W, z0, colour=(0.5, 0.25, 1.0)):
    """The plane z = z0, seen from either side"""
    o, d = _rays(c2w, K, H, W)
    with np.errstate(all="ignore"):
        s = (z0 - o[:, None, None, 2]) / d[..., 2]
    return _maps(s, np.isfinite(s) & (s > 0), colour)
