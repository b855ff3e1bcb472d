"""Oracle of the point-cloud passes (dgs_knn, open-diffusiongs_b200/csrc/knn.cu, and dgs_poisson_reconstruct,
csrc/poisson.cu): numpy / scipy restatements of their contracts, with no Open3D.

`knn` is brute force in fp32 with the kernel's squared distance (dx*dx + dy*dy) + dz*dz and its (distance, index)
order; `distcuda2` is simple_knn's distCUDA2 over it.  `outliers`, `pca_normals` and `reconstruct` follow poisson.cu's
header step by step: the statistical outlier rule, PCA normals oriented away from the centroid, the trilinear splat of
D and V over the scaled bounding cube, the screened system (L + point_weight (R^2 / N) B^T B) chi = -div V assembled as
a scipy.sparse matrix and solved directly (spsolve; fp64 CG where that is too slow), the iso value, marching cubes (oracle.mesh) and the density trim.
The sums are fp64 in numpy's order, so values the kernels sum in their own fixed order agree to rounding, not bits.
"""
import numpy as np
import scipy.sparse as sp
from scipy.sparse.linalg import cg, spsolve

from oracle import mesh as om

FLT_MAX = np.float32(3.4028234663852886e38)


def knn(points, k):
    """-> (idx int32 [P, k], d2 float32 [P, k]): the k nearest points in (squared distance, index) order, the point
    itself included; slots beyond P are (-1, inf)"""
    p = np.ascontiguousarray(points, np.float32)
    P = len(p)
    idx = np.full((P, k), -1, np.int32)
    d2 = np.full((P, k), np.inf, np.float32)
    kk = min(k, P)
    for a in range(0, P, 256):
        q = p[a:a + 256]
        dx, dy, dz = (p[None, :, c] - q[:, None, c] for c in range(3))
        d = (dx * dx + dy * dy) + dz * dz
        kth = np.partition(d, kk - 1, axis=1)[:, kk - 1]
        for r in range(len(q)):
            cand = np.flatnonzero(d[r] <= kth[r])  # every tie of the k-th value, in index order
            order = cand[np.argsort(d[r, cand], kind="stable")][:kk]
            idx[a + r, :kk] = order
            d2[a + r, :kk] = d[r, order]
    return idx, d2


def distcuda2(points):
    """simple_knn's distCUDA2: the mean of the three smallest squared distances to other indices (FLT_MAX when
    missing), summed (b0 + b1) + b2 and divided by 3 in fp32"""
    P = len(points)
    idx, d2 = knn(points, 4)
    other = idx != np.arange(P)[:, None]
    other[:, 3] &= ~other.all(1)
    d = np.where(idx < 0, FLT_MAX, d2)[other].reshape(P, 3)
    with np.errstate(over="ignore"):
        return ((d[:, 0] + d[:, 1]) + d[:, 2]) / np.float32(3.0)


def outliers(points, k, std_ratio):
    """-> (inlier mask bool [P], a_i float64 [P], threshold): a_i the mean of the square roots of the k nearest squared
    distances (in neighbour order), kept iff 0 < a_i < mean + std_ratio * sample std over the a_i > 0"""
    _, d2 = knn(points, k)
    s = np.zeros(len(points))
    for j in range(k):
        s = s + np.sqrt(d2[:, j].astype(np.float64))
    a = s / k
    v = a[a > 0]
    m = v.sum() / len(v) if len(v) else 0.0
    sd = np.sqrt(((v - m) ** 2).sum() / (len(v) - 1)) if len(v) >= 2 else 0.0
    thr = m + std_ratio * sd
    return (a > 0) & (a < thr), a, thr


def pca_normals(points, k):
    """Unit normals (float32 [N, 3]): the smallest-eigenvalue eigenvector of the fp64 covariance of each point's k
    nearest points (fewer when N < k), with n . (p - centroid) >= 0"""
    p = np.asarray(points, np.float32)
    idx, _ = knn(p, k)
    q = p.astype(np.float64)
    valid = idx >= 0
    nb = q[np.maximum(idx, 0)] * valid[..., None]
    cnt = valid.sum(1)[:, None]
    mean = nb.sum(1) / cnt
    d = (nb - mean[:, None]) * valid[..., None]
    cov = np.einsum("nki,nkj->nij", d, d) / cnt[..., None]
    _, vec = np.linalg.eigh(cov)
    n = vec[:, :, 0]
    c = q.sum(0) / len(q)
    o = (n[:, 0] * (q[:, 0] - c[0]) + n[:, 1] * (q[:, 1] - c[1])) + n[:, 2] * (q[:, 2] - c[2])
    n = np.where((o < 0)[:, None], -n, n)
    ln = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
    return (n / ln[:, None]).astype(np.float32)


def unit(normals):
    """Given normals over their fp64 length, rounded to fp32"""
    n = np.asarray(normals, np.float32).astype(np.float64)
    ln = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
    return (n / ln[:, None]).astype(np.float32)


def grid(points, depth, scale):
    """-> (origin float64 [3], h, R): the points' bounding cube scaled by `scale`, 2^depth + 1 nodes per axis"""
    p = np.asarray(points, np.float32)
    lo, hi = p.min(0).astype(np.float64), p.max(0).astype(np.float64)
    R = 2 ** depth + 1
    side = (hi - lo).max() * scale
    return 0.5 * (lo + hi) - 0.5 * side, side / (R - 1), R


def interpolation(points, origin, h, R):
    """B: the trilinear interpolation matrix (N x R^3, csr) at the points, weights as fp32 roundings of fp64 products"""
    g = (np.asarray(points, np.float32).astype(np.float64) - origin) / h
    c = np.clip(np.floor(g), 0, R - 2).astype(np.int64)
    f = g - c
    rows, cols, vals = [], [], []
    N = len(g)
    for cc in range(8):
        dx, dy, dz = (cc >> 2) & 1, (cc >> 1) & 1, cc & 1
        w = np.where(dx, f[:, 0], 1 - f[:, 0]) * np.where(dy, f[:, 1], 1 - f[:, 1])
        w = w * np.where(dz, f[:, 2], 1 - f[:, 2])
        rows.append(np.arange(N))
        cols.append(((c[:, 0] + dx) * R + c[:, 1] + dy) * R + c[:, 2] + dz)
        vals.append(w.astype(np.float32).astype(np.float64))
    return sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(N, R ** 3))


def laplacian(R):
    """The 7-point negative Laplacian on the interior nodes ((R - 2)^3 unknowns, h = 1, Dirichlet 0 outside)"""
    n = R - 2
    e = np.ones(n)
    T1 = sp.diags([-e[:-1], 2 * e, -e[:-1]], [-1, 0, 1])
    I1 = sp.identity(n)
    return (sp.kron(sp.kron(T1, I1), I1) + sp.kron(sp.kron(I1, T1), I1) + sp.kron(sp.kron(I1, I1), T1)).tocsr()


def interior(R):
    x = np.arange(R)
    m = (x > 0) & (x < R - 1)
    return (m[:, None, None] & m[None, :, None] & m[None, None, :]).reshape(-1)


def reconstruct(points, normals=None, depth=5, nb_neighbors=20, std_ratio=10.0, scale=1.1, point_weight=4.0,
                density_quantile=0.1, direct=True):
    """poisson.cu's contract, step by step -> dict: inliers (bool [P]), a, threshold, normals (float32 [N, 3]),
    origin, h, R, D (fp64 [R^3]), chi (fp64 [R, R, R]), residual (||A chi - b|| / ||b||), iso, vertices_before,
    density (float32 [vertices_before]), threshold_density, vertices (float32 [V, 3]) and faces (int64 [F, 3])"""
    p = np.asarray(points, np.float32)
    mask, a, thr = outliers(p, nb_neighbors, std_ratio)
    ip = p[mask]
    N = len(ip)
    n = unit(np.asarray(normals)[mask]) if normals is not None else pca_normals(ip, nb_neighbors)
    origin, h, R = grid(ip, depth, scale)
    B = interpolation(ip, origin, h, R)
    r2n = R * R / N
    D = np.asarray(B.sum(0)).reshape(-1)
    V = [r2n * (B.T @ n[:, c].astype(np.float64)) for c in range(3)]
    Vg = [v.reshape(R, R, R) for v in V]
    div = np.zeros((R, R, R))
    div[1:-1, 1:-1, 1:-1] = (0.5 * (Vg[0][2:, 1:-1, 1:-1] - Vg[0][:-2, 1:-1, 1:-1]) +
                             0.5 * (Vg[1][1:-1, 2:, 1:-1] - Vg[1][1:-1, :-2, 1:-1]) +
                             0.5 * (Vg[2][1:-1, 1:-1, 2:] - Vg[2][1:-1, 1:-1, :-2]))
    inner = interior(R)
    Bi = B[:, inner]
    A = (laplacian(R) + (point_weight * r2n) * (Bi.T @ Bi)).tocsc()
    b = -div.reshape(-1)[inner]
    # spsolve's fill-in grows fast with depth (minutes at depth 6): direct=False solves by unpreconditioned fp64 CG to a
    # relative residual of 1e-13 instead
    x = spsolve(A, b) if direct else cg(A, b, rtol=1e-13, atol=0.0, maxiter=100000)[0]
    residual = float(np.linalg.norm(A @ x - b) / np.linalg.norm(b))
    chi = np.zeros(R ** 3)
    chi[inner] = x
    iso = float((B @ chi).sum() / N)
    field = (-chi).astype(np.float32).reshape(R, R, R)
    v, f = om.marching_cubes(field, np.float32(-iso))
    Df = D.astype(np.float32).reshape(R, R, R)
    dens = vertex_density(v, Df)
    out = dict(inliers=mask, a=a, threshold=thr, normals=n, origin=origin, h=h, R=R, D=D, chi=chi.reshape(R, R, R),
               residual=residual, iso=iso, vertices_before=len(v), density=dens)
    keep = np.ones(len(v), bool)
    if density_quantile > 0 and len(v):
        t = np.quantile(dens, density_quantile)
        out["threshold_density"] = t
        keep = ~(dens < t)
    vertices, faces = trim(v, f, keep)
    out["vertices"] = (origin + h * vertices.astype(np.float64)).astype(np.float32)
    out["faces"] = faces
    return out


def vertex_density(v, D):
    """D (float32 [R, R, R]) interpolated trilinearly in fp32 at vertices in index coordinates"""
    R = D.shape[0]
    v = np.asarray(v, np.float32)
    c = np.clip(np.floor(v).astype(np.int64), 0, R - 2)
    f = v - c.astype(np.float32)
    acc = np.zeros(len(v), np.float32)
    one = np.float32(1)
    for cc in range(8):
        dx, dy, dz = (cc >> 2) & 1, (cc >> 1) & 1, cc & 1
        w = (np.where(dx, f[:, 0], one - f[:, 0]) * np.where(dy, f[:, 1], one - f[:, 1])) * np.where(dz, f[:, 2],
                                                                                                   one - f[:, 2])
        acc = acc + w * D[c[:, 0] + dx, c[:, 1] + dy, c[:, 2] + dz]
    return acc


def trim(v, f, keep):
    """Open3D's remove_vertices_by_mask: the kept vertices in order (referenced or not), the faces whose three vertices
    are kept, renumbered"""
    new = np.cumsum(keep) - 1
    f = np.asarray(f, np.int64)
    fk = keep[f].all(1) if len(f) else np.zeros(0, bool)
    return np.asarray(v)[keep], new[f[fk]].astype(np.int64).reshape(-1, 3)
