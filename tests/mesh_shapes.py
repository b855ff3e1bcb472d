"""Shapes and mesh properties the tests/test_mesh_*.py files share: sampling grids, marching-cubes meshes, a shell
model, and checks of orientation, topology (Euler characteristics, components) and volume."""
import numpy as np
import torch
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from oracle import mesh_clean as oc


def grid(n):
    x = np.arange(n, dtype=np.float64) - (n - 1) / 2
    return np.meshgrid(x, x, x, indexing="ij")


def cuda_grid(n):
    x = torch.arange(n, device="cuda", dtype=torch.float32) - (n - 1) / 2
    return torch.meshgrid(x, x, x, indexing="ij")


def mc(field, clean=False):
    """GPU marching cubes at 0 -> numpy (vertices float32 [V, 3] in index coordinates, faces int64 [F, 3]); with
    `clean`, then mesh.clean without its component removal"""
    from dgs_b200 import mesh
    v, f = mesh.marching_cubes(field.contiguous(), 0.0)
    v, f = v.cpu().numpy(), f.cpu().numpy().astype(np.int64)
    return mesh.clean(v, f, min_f=0, min_d=0) if clean else (v, f)


def shell_model(P, seed, dist="fine", floaters=True):
    """A GaussianModel on cuda of P shell Gaussians; with `floaters`, plus three small clusters of 400 off the shell"""
    from dgs_b200 import synth
    from dgs_b200.renderer import GaussianModel
    g = synth.make_shell_gaussians(P, seed, dist)
    if floaters:
        rng = np.random.default_rng(seed)
        k = 400
        for c in [(0.8, 0.7, 0.0), (-0.7, -0.75, 0.6), (0.1, -0.8, -0.7)]:
            extra = {key: g[key][:k].copy() for key in g}
            extra["xyz"] = (np.asarray(c) + rng.normal(0, 0.01, (k, 3))).astype(np.float32)
            g = {key: np.concatenate([g[key], extra[key]]) for key in g}
    m = GaussianModel(0)
    m._xyz, m._scaling, m._rotation, m._opacity = (torch.tensor(g[k], device="cuda") for k in
                                                   ("xyz", "scaling", "rotation", "opacity"))
    return m


def directed(faces):
    return np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])


def closed_and_oriented(faces):
    d = directed(faces)
    fwd = {tuple(e) for e in d.tolist()}
    assert len(fwd) == len(d), "a directed edge is used twice (inconsistent orientation)"
    assert all((b, a) in fwd for a, b in fwd), "an edge without its opposite (open surface)"


def euler(faces):
    e = np.sort(directed(faces), axis=1)
    return len(np.unique(faces)) - len(np.unique(e, axis=0)) + len(faces)


def euler_per_component(faces):
    """-> sorted Euler characteristics V - E + F of the edge-connected components"""
    n = int(faces.max()) + 1 if len(faces) else 0
    d = directed(faces)
    _, lab = connected_components(coo_matrix((np.ones(len(d)), (d[:, 0], d[:, 1])), shape=(n, n)), directed=False)
    out = []
    for c in np.unique(lab[faces[:, 0]]):
        f = faces[lab[faces[:, 0]] == c]
        e = np.unique(np.sort(directed(f), axis=1), axis=0)
        out.append(len(np.unique(f)) - len(e) + len(f))
    return sorted(out)


def volume(v, f, f64=True):
    """The signed volume, summed in float64 (f64) or in the vertices' own dtype"""
    if f64:
        v = v.astype(np.float64)
    return float(np.einsum("ij,ij->i", v[f[:, 0]], np.cross(v[f[:, 1]], v[f[:, 2]])).sum() / 6.0)


def patch(n=14):
    """An open, gently curved grid patch (a boundary loop of 4 (n - 1) vertices)"""
    x = np.arange(n, dtype=np.float64)
    X, Y = np.meshgrid(x, x, indexing="ij")
    v = np.stack([X, Y, 0.02 * (X - n / 2) ** 2], -1).reshape(-1, 3).astype(np.float32)
    i = np.arange(n - 1)
    a = (i[:, None] * n + i[None, :]).reshape(-1)
    f = np.concatenate([np.stack([a, a + n, a + 1], 1), np.stack([a + 1, a + n, a + n + 1], 1)])
    return v, f


def edges(f):
    e = np.sort(directed(f), 1)
    return np.unique(e, axis=0, return_counts=True)


def components(f):
    """-> per edge-connected component: (Euler characteristic V - E + F, whether it has a boundary), sorted"""
    d = directed(f)
    key = np.sort(d, 1)
    fid = np.tile(np.arange(len(f)), 3)
    order = np.lexsort((fid, key[:, 1], key[:, 0]))
    ks = key[order]
    same = np.flatnonzero((ks[1:] == ks[:-1]).all(1)) + 1
    _, lab = connected_components(coo_matrix((np.ones(len(same)), (fid[order][same], fid[order][same - 1])),
                                             shape=(len(f), len(f))), directed=False)
    out = []
    for c in np.unique(lab):
        fc = f[lab == c]
        e, cnt = edges(fc)
        out.append((len(np.unique(fc)) - len(e) + len(fc), bool((cnt == 1).any())))
    return sorted(out)


def check_remeshed(v, f, ov, of, L, nondegenerate=True):
    """The properties every remeshed closed or open surface keeps.  Reprojection may land two vertices of a face on
    one point of the input (at creases of a coarse input), so large meshes skip the zero-area check."""
    assert ov.dtype == np.float32 and of.dtype == np.int64 and np.isfinite(ov).all()
    assert of.min() >= 0 and of.max() < len(ov) and len(np.unique(of)) == len(ov)
    assert (of[:, 0] != of[:, 1]).all() and (of[:, 1] != of[:, 2]).all() and (of[:, 0] != of[:, 2]).all()
    assert len(np.unique(np.sort(of, 1), axis=0)) == len(of), "a duplicate face"
    assert not nondegenerate or (oc.doubled_area(ov, of) > 0).all(), "a zero-area face"
    # oriented where the input is: no directed edge twice.  An input edge that two faces run in one direction is
    # blocked: never collapsed or flipped, but each iteration's split may halve it into two such edges
    def twice(t):
        d = directed(t)
        return len(d) - len(np.unique(d, axis=0))
    assert twice(of) <= 8 * twice(f), f"{twice(of)} edges run twice in one direction (input: {twice(f)})"
    assert components(f) == components(of), "topology changed"
    e, _ = edges(of)
    ln = np.linalg.norm(ov[e[:, 0]].astype(np.float64) - ov[e[:, 1]], axis=1)
    med = float(np.median(ln))
    assert 4 * L / 5 <= med <= 4 * L / 3, f"median edge {med} outside [{4 * L / 5}, {4 * L / 3}]"
    return ln
