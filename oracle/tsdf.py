"""Oracle of TSDF fusion (dgs_tsdf_integrate / dgs_tsdf_extract / dgs_tsdf_colors, open-diffusiongs_b200/csrc/tsdf.cu).

The contract of tsdf.cu's header in numpy fp32, operation for operation and in its order, so the kernels (compiled with
-fmad=false) match it bit for bit: `integrate` fuses views into a volume, `extract` marches the mean tsdf at 0 over the
observed points (`marching_cubes_observed`: oracle/mesh.py's case tables, vertex and triangle order, with the observed
mask), and `colors` reads vertex colours back from the volume.
"""
import numpy as np
import torch

from oracle.mesh import load_tables

F32 = np.float32


def volume(R):
    """An empty volume: the dict of numpy arrays tsdf_sum fp32 [R, R, R], weight int32, rgb_sum fp32 [R, R, R, 3],
    rgb_weight int32, and lin, the fp32 linspace(-1, 1, R) the library uses"""
    return dict(tsdf_sum=np.zeros((R, R, R), F32), weight=np.zeros((R, R, R), np.int32),
                rgb_sum=np.zeros((R, R, R, 3), F32), rgb_weight=np.zeros((R, R, R), np.int32),
                lin=torch.linspace(-1, 1, R).numpy())


def integrate(vol, c2w, fxfycxcy, image, depth, alpha, trunc, alpha_thresh=0.5):
    """Fuses views into vol in place: c2w fp32 [n, 4, 4], fxfycxcy fp32 [n, 4], image fp32 [n, 3, H, W], depth and
    alpha fp32 [n, H, W]; trunc and alpha_thresh are rounded to fp32 as the C ABI takes them."""
    c2w, K = np.asarray(c2w, F32), np.asarray(fxfycxcy, F32)
    image, depth, alpha = (np.asarray(a, F32) for a in (image, depth, alpha))
    trunc, thr = F32(trunc), F32(alpha_thresh)
    n, _, H, W = image.shape
    lin = vol["lin"]
    px, py, pz = (a.reshape(-1) for a in np.meshgrid(lin, lin, lin, indexing="ij"))
    ts, w = vol["tsdf_sum"].reshape(-1), vol["weight"].reshape(-1)
    rgb, rw = vol["rgb_sum"].reshape(-1, 3), vol["rgb_weight"].reshape(-1)
    with np.errstate(all="ignore"):
        for k in range(n):
            m = c2w[k]
            dx, dy, dz = px - m[0, 3], py - m[1, 3], pz - m[2, 3]
            xc, yc, zc = ((m[0, c] * dx + m[1, c] * dy) + m[2, c] * dz for c in range(3))
            u = K[k, 0] * xc / zc + K[k, 2]
            v = K[k, 1] * yc / zc + K[k, 3]
            ok = ~(zc <= F32(0.2)) & (u >= 0) & (u < F32(W)) & (v >= 0) & (v < F32(H))
            sel = np.flatnonzero(ok)
            iu, iv = np.floor(u[sel]).astype(np.int64), np.floor(v[sel]).astype(np.int64)
            a = alpha[k, iv, iu]
            bg = a < thr
            carve = sel[bg]
            ts[carve] += F32(1)
            w[carve] += 1
            fg, a, iu, iv = sel[~bg], a[~bg], iu[~bg], iv[~bg]
            sdf = depth[k, iv, iu] / a - zc[fg]
            keep = ~(sdf < -trunc)
            fg, a, iu, iv, sdf = fg[keep], a[keep], iu[keep], iv[keep], sdf[keep]
            ts[fg] += np.minimum(F32(1), sdf / trunc)
            w[fg] += 1
            col = sdf < trunc
            fg, a, iu, iv = fg[col], a[col], iu[col], iv[col]
            for ch in range(3):
                rgb[fg, ch] += (image[k, ch, iv, iu] - (F32(1) - a)) / a
            rw[fg] += 1
    return vol


def field(vol):
    """-(tsdf_sum / weight) where weight > 0, else 0: the function extract marches at 0"""
    w = vol["weight"]
    with np.errstate(all="ignore"):
        return np.where(w > 0, -(vol["tsdf_sum"] / w.astype(F32)), F32(0)).astype(F32)


def marching_cubes_observed(f, observed):
    """Marching cubes of fp32 f [nx, ny, nz] at 0 (inside iff f > 0) over the observed points -> (vertices fp32 [V, 3]
    in index coordinates, triangles int64 [F, 3]): a voxel emits triangles only when its 8 corners are observed, an edge
    a vertex only when it changes sign, both its ends are observed and a voxel containing it is.  Vertices in
    owning-edge order (grid point in C order, then axis), triangles by voxel then table order, as oracle/mesh.py."""
    edges, ntri, tri = load_tables()
    nx, ny, nz = f.shape
    inside, obs = f > 0, np.asarray(observed, bool)
    full = np.ones((nx - 1, ny - 1, nz - 1), bool)
    for c in range(8):
        dx, dy, dz = c & 1, (c >> 1) & 1, c >> 2
        full &= obs[dx:nx - 1 + dx, dy:ny - 1 + dy, dz:nz - 1 + dz]
    fp = np.zeros((nx + 1, ny + 1, nz + 1), bool)  # fp[o + 1]: the voxel of origin o is fully observed
    fp[1:nx, 1:ny, 1:nz] = full
    cross = np.zeros(f.shape + (3,), bool)
    cross[:-1, :, :, 0] = (inside[:-1] != inside[1:]) & obs[:-1] & obs[1:] & (
        fp[1:nx, 0:ny, 0:nz] | fp[1:nx, 1:ny + 1, 0:nz] | fp[1:nx, 0:ny, 1:nz + 1] | fp[1:nx, 1:ny + 1, 1:nz + 1])
    cross[:, :-1, :, 1] = (inside[:, :-1] != inside[:, 1:]) & obs[:, :-1] & obs[:, 1:] & (
        fp[0:nx, 1:ny, 0:nz] | fp[1:nx + 1, 1:ny, 0:nz] | fp[0:nx, 1:ny, 1:nz + 1] | fp[1:nx + 1, 1:ny, 1:nz + 1])
    cross[:, :, :-1, 2] = (inside[:, :, :-1] != inside[:, :, 1:]) & obs[:, :, :-1] & obs[:, :, 1:] & (
        fp[0:nx, 0:ny, 1:nz] | fp[1:nx + 1, 0:ny, 1:nz] | fp[0:nx, 1:ny + 1, 1:nz] | fp[1:nx + 1, 1:ny + 1, 1:nz])
    flat = cross.reshape(-1)
    vid = np.cumsum(flat) - 1
    idx = np.nonzero(flat)[0]
    p, a = idx // 3, idx % 3
    step = np.array([ny * nz, nz, 1])
    pos = np.stack(np.unravel_index(p, f.shape), 1).astype(F32)
    va, vb = f.reshape(-1)[p], f.reshape(-1)[p + step[a]]
    pos[np.arange(len(p)), a] += (F32(0) - va) / (vb - va)
    case = np.zeros((nx - 1, ny - 1, nz - 1), np.int64)
    for c in range(8):
        dx, dy, dz = c & 1, (c >> 1) & 1, c >> 2
        case |= inside[dx:nx - 1 + dx, dy:ny - 1 + dy, dz:nz - 1 + dz].astype(np.int64) << c
    case = np.where(full, case, 0)
    vox = np.nonzero(ntri[case.reshape(-1)] > 0)[0]
    vx, vy, vz = np.unravel_index(vox, case.shape)
    origin = (vx * ny + vy) * nz + vz
    rows = tri[case.reshape(-1)[vox]]
    valid = rows >= 0
    e = np.where(valid, rows, 0)
    c0 = edges[e, 0]
    q = origin[:, None] + (c0 & 1) * step[0] + ((c0 >> 1) & 1) * step[1] + (c0 >> 2) * step[2]
    ids = vid[q * 3 + (e >> 2)]
    return pos, ids[valid].reshape(-1, 3)


def extract(vol):
    """-> (vertices fp32 [V, 3] in index coordinates, triangles int64 [F, 3]) as dgs_tsdf_extract returns them"""
    return marching_cubes_observed(field(vol), vol["weight"] > 0)


def to_frame(vertices, R):
    """Index coordinates -> the grid's [-1, 1] frame, v / (R - 1) * 2 - 1 in fp64 rounded to fp32 (tsdf_mesh)"""
    return (np.asarray(vertices, np.float64) / (R - 1.0) * 2 - 1).astype(F32)


def colors(vol, vertices):
    """vertices fp32 [V, 3] in the grid's [-1, 1] frame -> rgb fp32 [V, 3] as dgs_tsdf_colors computes it"""
    v = np.asarray(vertices, F32).reshape(-1, 3)
    R = vol["weight"].shape[0]
    s, hi = F32(R - 1) * F32(0.5), F32(R - 1)
    g = np.fmin(np.fmax((v + F32(1)) * s, F32(0)), hi)
    i0 = np.minimum(np.floor(g).astype(np.int64), R - 2)
    t = g - i0.astype(F32)
    acc, wsum = np.zeros((len(v), 3), F32), np.zeros(len(v), F32)
    rgb, rw = vol["rgb_sum"].reshape(-1, 3), vol["rgb_weight"].reshape(-1)
    with np.errstate(all="ignore"):
        for c in range(8):
            cx, cy, cz = c & 1, (c >> 1) & 1, c >> 2
            q = ((i0[:, 0] + cx) * R + (i0[:, 1] + cy)) * R + (i0[:, 2] + cz)
            ok = rw[q] > 0
            wx, wy, wz = (t[:, k] if on else F32(1) - t[:, k] for k, on in enumerate((cx, cy, cz)))
            wt = (wx * wy) * wz
            col = rgb[q] / rw[q].astype(F32)[:, None]
            acc = np.where(ok[:, None], acc + wt[:, None] * col, acc)
            wsum = np.where(ok, wsum + wt, wsum)
        out = np.fmin(np.fmax(acc / wsum[:, None], F32(0)), F32(1))
    return np.where((wsum == 0)[:, None], F32(1), out).astype(F32)
