"""Oracle of the mesh extraction (dgs_mesh_field / dgs_marching_cubes, open-diffusiongs_b200/csrc/mesh.cu).

`field` restates GaussianModel.extract_fields (gs_core.py:786-852): the normalisation, covariance and cofactor inverse
in the reference's fp32 arithmetic (elementwise torch ops in its evaluation order, so CPU and CUDA agree), block
membership in fp32 exactly as its mask, and the density accumulated in fp64.  It runs on CPU or CUDA tensors.

`marching_cubes` is a plain numpy marching cubes over the committed case table (csrc/mc_tables.h), with the vertex and
triangle order the kernel documents.
"""
import os
import re

import numpy as np
import torch

TABLES_H = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "open-diffusiongs_b200", "csrc",
                        "mc_tables.h")


# --------------------------------------------------------------------------------------------------------- field
def _rotation(r):  # build_rotation (gs_core.py:112-135): the raw quaternion over its Euclidean norm
    norm = torch.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    return [[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
            [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
            [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]]


def covariance6(stds, rotation):
    """(R S)(R S)^T as (xx, xy, xz, yy, yz, zz), summed in the order of torch's CPU bmm for 3 x 3 operands."""
    R = _rotation(rotation)
    L = [[R[i][j] * stds[:, j] for j in range(3)] for i in range(3)]

    def dot(i, k):
        return (L[i][0] * L[k][0] + L[i][1] * L[k][1]) + L[i][2] * L[k][2]
    return [dot(0, 0), dot(0, 1), dot(0, 2), dot(1, 1), dot(1, 2), dot(2, 2)]


def inverse6(cov):  # gaussian_3d_coeff (gs_core.py:27-46), fp32
    a, b, c, d, e, f = cov
    inv_det = 1 / (a * d * f + 2 * e * c * b - e ** 2 * a - c ** 2 * d - b ** 2 * f + 1e-24)
    return [(d * f - e ** 2) * inv_det, (e * c - b * f) * inv_det, (e * b - c * d) * inv_det,
            (a * f - c ** 2) * inv_det, (b * c - e * a) * inv_det, (a * d - b ** 2) * inv_det]


def normalise(xyz, scaling, rotation, opacity, scaling_modifier=None):
    """-> (mesh_center fp32 [3], mesh_scale Python float, xyz_n [P,3], opacity [P], inverse covariance: 6 x [P]),
    all fp32 as extract_fields forms them."""
    stds = torch.exp(scaling)
    if scaling_modifier is not None:
        stds = stds * scaling_modifier
    mn, mx = xyz.amin(0), xyz.amax(0)
    center = (mn + mx) / 2
    scale = 1.8 / (mx - mn).amax().item()
    xyz_n = (xyz - center) * scale
    stds = stds * scale
    return center, scale, xyz_n, torch.sigmoid(opacity).reshape(-1), inverse6(covariance6(stds, rotation))


def chunks(resolution, num_blocks, relax_ratio, device="cpu"):
    """-> (lin fp32 [R], list of (first, last + 1) point ranges per chunk, vmin fp32 [nc], vmax fp32 [nc])"""
    block_size = 2 / num_blocks
    assert resolution % block_size == 0
    split = resolution // num_blocks
    lin = torch.linspace(-1, 1, resolution).to(device)
    bounds = [(s, min(s + split, resolution)) for s in range(0, resolution, split)]
    vmin = torch.stack([lin[s] for s, _ in bounds]) - block_size * relax_ratio
    vmax = torch.stack([lin[e - 1] for _, e in bounds]) + block_size * relax_ratio
    return lin, bounds, vmin, vmax


def membership(xyz_n, vmin, vmax):
    """-> per axis a bool [P, nc]: vmin < x < vmax, strictly, in fp32"""
    return [(xyz_n[:, k:k + 1] > vmin[None]) & (xyz_n[:, k:k + 1] < vmax[None]) for k in range(3)]


def block_counts(m):
    """-> int64 [nc, nc, nc]: Gaussians per block from the per-axis memberships"""
    mx, my, mz = (t.to(torch.float64) for t in m)
    return torch.einsum("gi,gj,gk->ijk", mx, my, mz).round().to(torch.int64)


def field(xyz, scaling, rotation, opacity, resolution=128, num_blocks=16, relax_ratio=1.5, scaling_modifier=None,
          blocks=None):
    """-> dict(occ fp64 [R, R, R], counts int64 [nc, nc, nc], center, scale).  blocks: None = every block, else a list of
    (bx, by, bz); the other blocks of occ are left 0."""
    dev = xyz.device
    center, scale, xyz_n, opac, inv = normalise(xyz, scaling, rotation, opacity, scaling_modifier)
    lin, bounds, vmin, vmax = chunks(resolution, num_blocks, relax_ratio, dev)
    m = membership(xyz_n, vmin, vmax)
    counts = block_counts(m)
    occ = torch.zeros([resolution] * 3, dtype=torch.float64, device=dev)
    nc = len(bounds)
    if blocks is None:
        blocks = [tuple(b) for b in torch.nonzero(counts).tolist()]
    g64 = xyz_n.double()
    inv64 = [t.double() for t in inv]
    lin64 = lin.double()
    for bx, by, bz in blocks:
        assert 0 <= bx < nc and 0 <= by < nc and 0 <= bz < nc
        sel = torch.nonzero(m[0][:, bx] & m[1][:, by] & m[2][:, bz]).reshape(-1)
        if sel.numel() == 0:
            continue
        (x0, x1), (y0, y1), (z0, z1) = bounds[bx], bounds[by], bounds[bz]
        px, py, pz = torch.meshgrid(lin64[x0:x1], lin64[y0:y1], lin64[z0:z1], indexing="ij")
        d = [p.reshape(-1, 1) - g64[sel, k][None] for k, p in enumerate((px, py, pz))]
        ia, ib, ic, id_, ie, if_ = (t[sel][None] for t in inv64)
        power = (-0.5 * (d[0] ** 2 * ia + d[1] ** 2 * id_ + d[2] ** 2 * if_) - d[0] * d[1] * ib - d[0] * d[2] * ic
                 - d[1] * d[2] * ie)
        w = torch.where(power > 0, torch.zeros_like(power), torch.exp(power))
        val = (w * opac[sel].double()[None]).sum(1)
        occ[x0:x1, y0:y1, z0:z1] = val.reshape(x1 - x0, y1 - y0, z1 - z0)
    return dict(occ=occ, counts=counts, center=center, scale=scale)


# ------------------------------------------------------------------------------------------------ marching cubes
def load_tables(path=TABLES_H):
    """-> (edge corners int [12, 2], triangles per case int [256], triangle edges int [256, 3 * max]) from the header"""
    txt = open(path).read()

    def array(name):
        body = re.search(name + r"\[[^=]*=\s*\{(.*?)\};", txt, re.S).group(1)
        return np.array([int(v) for v in re.findall(r"-?\d+", body)], np.int64)
    ntri = array("kMcNumTris")
    edges = array("kMcEdgeCorners").reshape(12, 2)
    tri = array("kMcTriEdges").reshape(256, -1)
    return edges, ntri, tri


def marching_cubes(field, iso):
    """field [nx, ny, nz] -> (vertices fp64 [V, 3] in index coordinates, triangles int64 [F, 3]); a point is inside iff
    value > iso.  Vertices in owning-edge order (grid point in C order, then axis), triangles by voxel then table order."""
    f = np.asarray(field, np.float64)
    nx, ny, nz = f.shape
    edges, ntri, tri = load_tables()
    inside = f > iso
    cross = np.zeros(f.shape + (3,), bool)
    cross[:-1, :, :, 0] = inside[:-1] != inside[1:]
    cross[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    cross[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    flat = cross.reshape(-1)
    vid = np.cumsum(flat) - 1  # vertex id of crossing (point, axis)
    idx = np.nonzero(flat)[0]
    p, a = idx // 3, idx % 3
    pos = np.stack(np.unravel_index(p, f.shape), 1).astype(np.float64)
    step = np.array([ny * nz, nz, 1])
    va, vb = f.reshape(-1)[p], f.reshape(-1)[p + step[a]]
    pos[np.arange(len(p)), a] += (iso - va) / (vb - va)
    # voxel cases, voxels in C order of their origin point
    case = np.zeros((nx - 1, ny - 1, nz - 1), np.int64)
    for c in range(8):
        dx, dy, dz = c & 1, (c >> 1) & 1, c >> 2
        case |= inside[dx:nx - 1 + dx, dy:ny - 1 + dy, dz:nz - 1 + dz].astype(np.int64) << c
    vox = np.nonzero(ntri[case.reshape(-1)] > 0)[0]
    vx, vy, vz = np.unravel_index(vox, case.shape)
    origin = (vx * ny + vy) * nz + vz
    rows = tri[case.reshape(-1)[vox]]          # [n, 3 * max]
    valid = rows >= 0
    e = np.where(valid, rows, 0)
    c0 = edges[e, 0]
    q = origin[:, None] + (c0 & 1) * step[0] + ((c0 >> 1) & 1) * step[1] + (c0 >> 2) * step[2]
    ids = vid[q * 3 + (e >> 2)]
    return pos, ids[valid].reshape(-1, 3)
