"""Oracle of the per-vertex normals and colours (dgs_mesh_vertex_colors, open-diffusiongs_b200/csrc/mesh_color.cu; the
semantics are include/dgs_b200.h's).

The records and block lists are oracle/mesh.py's own (`normalise`, `chunks`, `membership`), so a vertex is evaluated
against exactly the Gaussians the field sums for its block.  Normals are fp64 with no fused operation, faces added in
face order (np.add.at); weights and colour sums are fp64 from the fp32 records (the kernel's: the power's coefficients
scaled to the log2 domain and rounded to fp32), relative to each vertex's largest weight as the kernel keeps them.
"""
import numpy as np
import torch

from oracle import mesh as om

SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435)


def sh_basis(d, deg):
    """The 3DGS real SH basis of directions d [N, 3] -> fp64 [N, (deg + 1)^2]"""
    x, y, z = (d[:, k].astype(np.float64) for k in range(3))
    b = [np.full_like(x, SH_C0)]
    if deg > 0:
        b += [-SH_C1 * y, SH_C1 * z, -SH_C1 * x]
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        b += [SH_C2[0] * xy, SH_C2[1] * yz, SH_C2[2] * (2 * zz - xx - yy), SH_C2[3] * xz, SH_C2[4] * (xx - yy)]
        if deg > 2:
            b += [SH_C3[0] * y * (3 * xx - yy), SH_C3[1] * xy * z, SH_C3[2] * y * (4 * zz - xx - yy),
                  SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy), SH_C3[4] * x * (4 * zz - xx - yy), SH_C3[5] * z * (xx - yy),
                  SH_C3[6] * x * (xx - 3 * yy)]
    return np.stack(b, 1)


def normals(vertices, faces):
    """-> float32 [V, 3]: per vertex the fp64 sum of (b - a) x (c - a) over its faces in face order, over its length;
    0 without faces or for a zero sum"""
    v = np.asarray(vertices, np.float32).astype(np.float64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    a = v[f[:, 0]]
    u, w = v[f[:, 1]] - a, v[f[:, 2]] - a
    n = np.stack([u[:, 1] * w[:, 2] - u[:, 2] * w[:, 1], u[:, 2] * w[:, 0] - u[:, 0] * w[:, 2],
                  u[:, 0] * w[:, 1] - u[:, 1] * w[:, 0]], 1)
    s = np.zeros((len(v), 3))
    np.add.at(s, f.reshape(-1), np.repeat(n, 3, axis=0))  # incidence 3 f + k: face order
    length = np.sqrt(s[:, 0] * s[:, 0] + s[:, 1] * s[:, 1] + s[:, 2] * s[:, 2])
    out = np.zeros_like(s)
    ok = length > 0
    out[ok] = s[ok] / length[ok, None]
    return out.astype(np.float32)


def vertex_chunks(p, lin, split):
    """-> int64 [N]: the chunk of the grid point at or below each fp32 coordinate (the largest i with lin[i] <= p,
    clamped to [0, R - 1]; 0 for NaN) over split"""
    p = np.asarray(p, np.float32)
    i = np.searchsorted(np.asarray(lin, np.float32), p, side="right") - 1
    i = np.where(np.isnan(p), 0, np.clip(i, 0, len(lin) - 1))
    return i // split


def vertex_colors(xyz, features, scaling, rotation, opacity, vertices, faces, resolution=256, num_blocks=64,
                  relax_ratio=1.5, scaling_modifier=None, subset=None, device="cpu"):
    """-> dict(rgb float64 [N, 3], normals float32 [V, 3], unweighted bool [N], cmin / cmax float64 [N, 3] (the range of
    the colours of the Gaussians with nonzero weight; +inf / -inf where none), count int64 [N] (the list length)) for
    the vertices `subset` (indices; default all, N = V).  The Gaussian arrays are CPU torch tensors or numpy, raw as
    the field takes them; mesh_center / mesh_scale are the field's (from xyz, as extract_fields sets them).  The records
    are formed on the torch `device`: a thin Gaussian's cofactor inverse turns one ulp of a scale into about 1e-3 of its
    power, so records that must be the kernels' own come from torch's CUDA exp ("cuda")."""
    t = [torch.as_tensor(np.asarray(a, np.float32)).to(device) for a in (xyz, scaling, rotation, opacity)]
    _, _, xyz_n, opac, inv = om.normalise(*t, scaling_modifier=scaling_modifier)
    lin, bounds, vmin, vmax = om.chunks(resolution, num_blocks, relax_ratio, device)
    m = [a.cpu().numpy() for a in om.membership(xyz_n, vmin, vmax)]
    xyz_n, opac, inv, lin = xyz_n.cpu(), opac.cpu(), [a.cpu() for a in inv], lin.cpu()
    split = resolution // num_blocks
    g = xyz_n.numpy().astype(np.float64)
    op = opac.numpy().astype(np.float64)
    # the kernel's record: the power's coefficients times -log2(e) / 2 (squares) and -log2(e) (products), rounded to fp32
    h, l2e = np.float32(-0.5 * 1.4426950408889634), np.float32(-1.4426950408889634)
    ia, id_, if_ = ((h * a.numpy()).astype(np.float64) for a in (inv[0], inv[3], inv[5]))
    ib, ic, ie = ((l2e * a.numpy()).astype(np.float64) for a in (inv[1], inv[2], inv[4]))
    sh = np.asarray(features, np.float32).astype(np.float64)
    deg = int(round(sh.shape[1] ** 0.5)) - 1
    v = np.asarray(vertices, np.float32)
    nrm = normals(v, faces)
    idx = np.arange(len(v)) if subset is None else np.asarray(subset, np.int64)
    p = v[idx]
    blk = np.stack([vertex_chunks(p[:, k], lin.numpy(), split) for k in range(3)], 1)
    basis = sh_basis(-nrm[idx], deg)
    N = len(idx)
    num, den = np.zeros((N, 3)), np.zeros(N)
    cmin, cmax = np.full((N, 3), np.inf), np.full((N, 3), -np.inf)
    count = np.zeros(N, np.int64)
    keys, inverse = np.unique(blk, axis=0, return_inverse=True)
    for b, (bx, by, bz) in enumerate(keys):
        sel = np.flatnonzero(m[0][:, bx] & m[1][:, by] & m[2][:, bz])  # the block's list, in Gaussian order
        rows = np.flatnonzero(inverse.reshape(-1) == b)
        count[rows] = len(sel)
        if len(sel) == 0:
            continue
        d = [p[rows, k].astype(np.float64)[:, None] - g[None, sel, k] for k in range(3)]
        power = (d[0] * d[0] * ia[sel] + d[1] * d[1] * id_[sel] + d[2] * d[2] * if_[sel] + d[0] * d[1] * ib[sel]
                 + d[0] * d[2] * ic[sel] + d[1] * d[2] * ie[sel])  # log2 of exp(power)
        # weights relative to the vertex's largest (the ratio is the same), so none underflows
        with np.errstate(divide="ignore"):
            lw = np.where(power > 0, -np.inf, power + np.log2(op[sel])[None])
        top = lw.max(1, keepdims=True)
        w = np.where(np.isfinite(lw), np.exp2(lw - np.where(np.isfinite(top), top, 0.0)), 0.0)
        c = np.maximum(0.5 + np.einsum("vk,gkc->vgc", basis[rows], sh[sel]), 0.0)  # [rows, list, 3]
        num[rows] = np.einsum("vg,vgc->vc", w, c)
        den[rows] = w.sum(1)
        live = (w > 0)[:, :, None]
        cmin[rows] = np.where(live, c, np.inf).min(1)
        cmax[rows] = np.where(live, c, -np.inf).max(1)
    unweighted = den == 0
    rgb = np.ones((N, 3))
    rgb[~unweighted] = np.clip(num[~unweighted] / den[~unweighted, None], 0.0, 1.0)
    return dict(rgb=rgb, normals=nrm, unweighted=unweighted, cmin=cmin, cmax=cmax, count=count)
