"""Serial oracle of the isotropic remeshing (dgs_mesh_remesh, open-diffusiongs_b200/csrc/mesh_remesh.cu): VCG's
IsotropicRemeshing as pymeshlab's meshing_isotropic_explicit_remeshing runs it inside the reference's clean_mesh
(utils/mesh_utils.py:88-147, remesh=True), restated as the exact contract of include/dgs_b200.h.  Each iteration splits
long edges, collapses short ones, flips edges towards valence 6, smooths tangentially and reprojects onto the input.

All arithmetic is fp64 from the fp32 positions with every product and sum rounded on its own (numpy's elementwise
float64 operations; sums over a vertex's faces run slot by slot in face order, never through np.sum or @, which
reorder), so the kernels, compiled without FMA contraction, must equal this bit for bit: vertices, faces and stats.
Collapse and flip rounds are vectorised over the round's edges; their selections are independent sets, so applying
them together is the same as applying them one by one.
"""
import math

import numpy as np
from scipy.sparse import csr_matrix
from scipy.spatial import cKDTree

ROUND_CAP = 256  # rounds per collapse / flip stage and iteration
NO_KEY = np.uint64(0xFFFFFFFFFFFFFFFF)


def _dot(u, w):
    return u[:, 0] * w[:, 0] + u[:, 1] * w[:, 1] + u[:, 2] * w[:, 2]


def _cross(u, w):
    return np.stack([u[:, 1] * w[:, 2] - u[:, 2] * w[:, 1], u[:, 2] * w[:, 0] - u[:, 0] * w[:, 2],
                     u[:, 0] * w[:, 1] - u[:, 1] * w[:, 0]], 1)


def _normal(p0, p1, p2):
    """(p1 - p0) x (p2 - p0): twice the area-weighted normal"""
    return _cross(p1 - p0, p2 - p0)


def _dist(p, q):
    d = q - p
    return np.sqrt(_dot(d, d))


def _diag(p):
    d = p.max(0).astype(np.float64) - p.min(0).astype(np.float64)
    return float(np.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]))


def closest_on_triangles(p, a, b, c):
    """Ericson's ClosestPtPointTriangle (Real-Time Collision Detection, 5.1.5), rows of fp64 [n, 3] -> (closest point
    [n, 3], squared distance [n]).  Regions are tested in the book's order: a, b, edge ab, c, edge ac, edge bc, face."""
    with np.errstate(all="ignore"):
        ab, ac, ap = b - a, c - a, p - a
        d1, d2 = _dot(ab, ap), _dot(ac, ap)
        bp = p - b
        d3, d4 = _dot(ab, bp), _dot(ac, bp)
        vc = d1 * d4 - d3 * d2
        cp = p - c
        d5, d6 = _dot(ab, cp), _dot(ac, cp)
        vb = d5 * d2 - d1 * d6
        va = d3 * d6 - d5 * d4
        e43, e56 = d4 - d3, d5 - d6
        region = np.select([(d1 <= 0) & (d2 <= 0), (d3 >= 0) & (d4 <= d3), (vc <= 0) & (d1 >= 0) & (d3 <= 0),
                            (d6 >= 0) & (d5 <= d6), (vb <= 0) & (d2 >= 0) & (d6 <= 0),
                            (va <= 0) & (e43 >= 0) & (e56 >= 0)], np.arange(6), 6)
        denom = 1.0 / (va + vb + vc)
        choices = [a, b, a + (d1 / (d1 - d3))[:, None] * ab, c, a + (d2 / (d2 - d6))[:, None] * ac,
                   b + (e43 / (e43 + e56))[:, None] * (c - b), a + ab * (vb * denom)[:, None] + ac * (vc * denom)[:, None]]
        q = np.select([(region == k)[:, None] for k in range(6)], choices[:6], choices[6])
        dq = p - q
        return q, _dot(dq, dq)


def closest_points(pos, faces, queries):
    """The closest point of the surface (pos fp32 [V, 3], faces [F, 3], F > 0) to each query (fp64 [m, 3]) ->
    (points fp64 [m, 3], squared distances [m], faces [m]): the smallest (squared distance, face index) over all faces,
    a face whose result is not a number never winning.  Exact, not a grid walk: every face within the distance to the
    nearest referenced vertex, plus the largest centre-to-corner radius, is evaluated."""
    P = np.asarray(pos, np.float32).astype(np.float64)
    faces = np.asarray(faces, np.int64)
    Q = np.asarray(queries, np.float64).reshape(-1, 3)
    A, B, C = P[faces[:, 0]], P[faces[:, 1]], P[faces[:, 2]]
    cen = (A + B + C) / 3.0
    rmax = float(max(_dist(cen, A).max(), _dist(cen, B).max(), _dist(cen, C).max()))
    ub, _ = cKDTree(P[np.unique(faces)]).query(Q)
    r = (ub + rmax) * (1 + 1e-9) + 1e-12
    lists = cKDTree(cen).query_ball_point(Q, r)
    cnt = np.fromiter((len(x) for x in lists), np.int64, len(lists))
    tri = np.fromiter((t for x in lists for t in x), np.int64, int(cnt.sum()))
    qi = np.repeat(np.arange(len(Q)), cnt)
    q, d2 = closest_on_triangles(Q[qi], A[tri], B[tri], C[tri])
    d2 = np.where(np.isnan(d2), np.inf, d2)
    order = np.lexsort((tri, d2, qi))
    best = order[np.searchsorted(qi[order], np.arange(len(Q)))]
    return q[best], d2[best], tri[best]


class _Edges:
    """The unique undirected edges of a face list, in (min, max) order, with half-edge h = 3 f + k running from corner
    k to corner k + 1 of face f."""

    def __init__(self, pos, f, cos_t):
        F = len(f)
        self.u = f.reshape(-1)
        self.w = f[:, [1, 2, 0]].reshape(-1)
        lo, hi = np.minimum(self.u, self.w), np.maximum(self.u, self.w)
        order = np.lexsort((np.arange(3 * F), hi, lo))
        head = np.ones(3 * F, bool)
        head[1:] = (lo[order][1:] != lo[order][:-1]) | (hi[order][1:] != hi[order][:-1])
        starts = np.flatnonzero(head)
        self.E = len(starts)
        self.nf = np.diff(np.append(starts, 3 * F))
        self.eid = np.empty(3 * F, np.int64)
        self.eid[order] = np.cumsum(head) - 1
        self.a, self.b = lo[order[starts]], hi[order[starts]]
        self.h0 = order[starts]
        self.h1 = order[np.minimum(starts + 1, 3 * F - 1)]
        fv = f.reshape(-1)
        self.c = fv[3 * (self.h0 // 3) + (self.h0 % 3 + 2) % 3]
        self.d = fv[3 * (self.h1 // 3) + (self.h1 % 3 + 2) % 3]
        # an edge of two faces that run it in opposite directions; anything else blocks it like a boundary
        manifold = (self.nf == 2) & (self.u[self.h0] == self.w[self.h1])
        P = pos.astype(np.float64)
        n0 = _face_normals(P, f[self.h0 // 3])
        n1 = _face_normals(P, f[self.h1 // 3])
        feature = _dot(n0, n1) < cos_t * np.sqrt(_dot(n0, n0)) * np.sqrt(_dot(n1, n1))
        self.blocked = ~manifold | feature
        self.length = _dist(P[self.a], P[self.b])
        self.key = self.a * (1 << 32) + self.b


def _face_normals(P, f):
    return _normal(P[f[:, 0]], P[f[:, 1]], P[f[:, 2]])


def _vertex_faces(f, V):
    """-> (start [V + 1], faces of the sorted (vertex, face) incidences, the vertex's corner in each)"""
    v = f.reshape(-1)
    order = np.argsort(v, kind="stable")
    return np.searchsorted(v[order], np.arange(V + 1)), order // 3, order % 3


def _split(pos, f, lock, ed, hi):
    V = len(pos)
    split = ed.length > hi
    ns = int(split.sum())
    new_id = np.full(ed.E, -1, np.int64)
    new_id[split] = V + np.arange(ns)
    P = pos.astype(np.float64)
    mid = (0.5 * (P[ed.a[split]] + P[ed.b[split]])).astype(np.float32)
    pos = np.concatenate([pos, mid])
    lock = np.concatenate([lock, ed.blocked[split]])
    P = pos.astype(np.float64)
    m = new_id[ed.eid.reshape(-1, 3)]  # the midpoint of edge k (corner k -> k + 1), -1 if not split
    cnt = (m >= 0).sum(1)
    out = np.full((len(f), 4, 3), -1, np.int64)
    out[:, 0] = f
    r = np.arange(len(f))
    s1 = cnt == 1
    k = np.argmax(m >= 0, 1)
    a, b, c, mm = f[r, k], f[r, (k + 1) % 3], f[r, (k + 2) % 3], m[r, k]
    out[s1, 0] = np.stack([a, mm, c], 1)[s1]
    out[s1, 1] = np.stack([mm, b, c], 1)[s1]
    s2 = cnt == 2
    k = np.argmin(m >= 0, 1)  # the edge that is not split: (c, a)
    c, a, b = f[r, k], f[r, (k + 1) % 3], f[r, (k + 2) % 3]
    mab, mbc = m[r, (k + 1) % 3], m[r, (k + 2) % 3]
    other = np.zeros(len(f), bool)
    other[s2] = _dist(P[mab[s2]], P[c[s2]]) < _dist(P[a[s2]], P[mbc[s2]])  # diagonal (m_ab, c) strictly shorter
    out[s2, 0] = np.stack([mab, b, mbc], 1)[s2]
    out[s2, 1] = np.where(other[:, None], np.stack([a, mab, c], 1), np.stack([a, mab, mbc], 1))[s2]
    out[s2, 2] = np.where(other[:, None], np.stack([mab, mbc, c], 1), np.stack([a, mbc, c], 1))[s2]
    s3 = cnt == 3
    v0, v1, v2, m0, m1, m2 = f[:, 0], f[:, 1], f[:, 2], m[:, 0], m[:, 1], m[:, 2]
    out[s3, 0] = np.stack([v0, m0, m2], 1)[s3]
    out[s3, 1] = np.stack([m0, v1, m1], 1)[s3]
    out[s3, 2] = np.stack([m2, m1, v2], 1)[s3]
    out[s3, 3] = np.stack([m0, m1, m2], 1)[s3]
    extra = out[:, 1:][np.arange(3)[None, :] < cnt[:, None]]
    return pos, np.concatenate([out[:, 0], extra]), lock


def _keeps_orientation(P, f, vs, others, p, start, vfaces, vcorner):
    """Per candidate: moving vertex vs[i] to p[i] keeps every face around it that does not contain others[i] facing the
    same way (new normal . old normal > 0); faces of zero area before are exempt."""
    cnt = start[vs + 1] - start[vs]
    ci = np.repeat(np.arange(len(vs)), cnt)
    inc = np.repeat(start[vs], cnt) + (np.arange(int(cnt.sum())) - np.repeat(np.cumsum(cnt) - cnt, cnt))
    t = f[vfaces[inc]]
    live = (t != others[ci][:, None]).all(1)
    q = [P[t[:, j]] for j in range(3)]
    n0 = _normal(*q)
    live &= ~((n0[:, 0] == 0) & (n0[:, 1] == 0) & (n0[:, 2] == 0))
    k = vcorner[inc]
    q = [np.where((k == j)[:, None], p[ci], q[j]) for j in range(3)]
    bad = live & ~(_dot(n0, _normal(*q)) > 0)
    ok = np.ones(len(vs), bool)
    ok[ci[bad]] = False
    return ok, ci, t


def _collapse_round(pos, f, lock, ed, lo, hi, surf, msd):
    """One round of collapses -> (pos, f, lock, taken)"""
    V = len(pos)
    P = pos.astype(np.float64)
    cand = np.flatnonzero(~ed.blocked & (ed.length < lo) & ~(lock[ed.a] & lock[ed.b]))
    a, b, c, d = ed.a[cand], ed.b[cand], ed.c[cand], ed.d[cand]
    mid = (0.5 * (P[a] + P[b])).astype(np.float32).astype(np.float64)
    p = np.where(lock[a][:, None], P[a], np.where(lock[b][:, None], P[b], mid))
    # link condition: the common neighbours are exactly c != d, and not both (a, c, d) and (b, c, d) are faces
    adj = csr_matrix((np.ones(2 * ed.E), (np.concatenate([ed.a, ed.b]), np.concatenate([ed.b, ed.a]))), shape=(V, V))
    common = np.asarray(adj[a].multiply(adj[b]).sum(1)).ravel()
    fs = np.sort(f, 1)
    fkey = np.sort((fs[:, 0] * V + fs[:, 1]) * V + fs[:, 2])

    def is_face(x, y, z):
        s = np.sort(np.stack([x, y, z], 1), 1)
        k = (s[:, 0] * V + s[:, 1]) * V + s[:, 2]
        i = np.minimum(np.searchsorted(fkey, k), len(fkey) - 1)
        return fkey[i] == k
    ok = (c != d) & (common == 2) & ~(is_face(a, c, d) & is_face(b, c, d))
    # fold-over, then no edge longer than hi at the new position
    start, vfaces, vcorner = _vertex_faces(f, V)
    for vs, others in ((a, b), (b, a)):
        keep, ci, t = _keeps_orientation(P, f, vs, others, p, start, vfaces, vcorner)
        ok &= keep
        for j in range(3):
            x = t[:, j]
            far = (x != a[ci]) & (x != b[ci]) & (_dist(p[ci], P[x]) > hi)
            ok[ci[far]] = False
    idx = np.flatnonzero(ok)
    if len(idx):
        _, d2, _ = closest_points(*surf, p[idx])
        ok[idx[np.sqrt(d2) > msd]] = False
    key = np.full(ed.E, NO_KEY, np.uint64)
    lens = ed.length[cand[ok]].astype(np.float32).view(np.uint32).astype(np.uint64)
    key[cand[ok]] = (lens << np.uint64(32)) | cand[ok].astype(np.uint64)
    m1 = np.full(V, NO_KEY, np.uint64)
    np.minimum.at(m1, ed.a, key)
    np.minimum.at(m1, ed.b, key)
    m2 = m1.copy()
    np.minimum.at(m2, ed.a, m1[ed.b])
    np.minimum.at(m2, ed.b, m1[ed.a])
    take = (key != NO_KEY) & (m2[ed.a] == key) & (m2[ed.b] == key)
    if not take.any():
        return pos, f, lock, 0
    pos = pos.copy()
    pe = np.zeros((ed.E, 3))
    pe[cand] = p
    ta, tb = ed.a[take], ed.b[take]
    pos[ta] = pe[take].astype(np.float32)
    lock = lock.copy()
    lock[ta] |= lock[tb]
    to = np.arange(V)
    to[tb] = ta
    f = to[f]
    f = f[(f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 0] != f[:, 2])]
    return pos, f, lock, int(take.sum())


def _flip_round(pos, f, ed, surf, msd):
    """One round of flips -> (f, taken)"""
    V = len(pos)
    P = pos.astype(np.float64)
    val = np.bincount(ed.a, minlength=V) + np.bincount(ed.b, minlength=V)
    bnd = np.zeros(V, bool)
    one = ed.nf == 1
    bnd[ed.a[one]] = bnd[ed.b[one]] = True
    tgt = np.where(bnd, 4, 6)
    cand = np.flatnonzero(~ed.blocked & (ed.c != ed.d))
    a, b, c, d = ed.a[cand], ed.b[cand], ed.c[cand], ed.d[cand]
    ck = np.minimum(c, d) * (1 << 32) + np.maximum(c, d)
    i = np.minimum(np.searchsorted(ed.key, ck), ed.E - 1)
    ok = ed.key[i] != ck

    def e(x, dv):
        return (val[x] + dv - tgt[x]) ** 2
    gain = e(a, 0) + e(b, 0) + e(c, 0) + e(d, 0) - (e(a, -1) + e(b, -1) + e(c, 1) + e(d, 1))
    ok &= gain > 0
    h0, h1 = ed.h0[cand], ed.h1[cand]
    u, w = ed.u[h0], ed.w[h0]
    n0, n1 = _face_normals(P, f[h0 // 3]), _face_normals(P, f[h1 // 3])
    m0, m1 = _normal(P[c], P[u], P[d]), _normal(P[d], P[w], P[c])
    ok &= (_dot(m0, n0) > 0) & (_dot(m0, n1) > 0) & (_dot(m1, n0) > 0) & (_dot(m1, n1) > 0)
    idx = np.flatnonzero(ok)
    if len(idx):
        _, d2, _ = closest_points(*surf, 0.5 * (P[c[idx]] + P[d[idx]]))
        ok[idx[np.sqrt(d2) > msd]] = False
    cand, a, b, c, d, h0, h1, u, w = (x[ok] for x in (cand, a, b, c, d, h0, h1, u, w))
    key = ((np.uint64(0x7FFFFFFF) - gain[ok].astype(np.uint64)) << np.uint64(32)) | cand.astype(np.uint64)
    vmin = np.full(V, NO_KEY, np.uint64)
    for x in (a, b, c, d):
        np.minimum.at(vmin, x, key)
    take = (vmin[a] == key) & (vmin[b] == key) & (vmin[c] == key) & (vmin[d] == key)
    if not take.any():
        return f, 0
    f = f.copy()
    f[h0[take] // 3] = np.stack([c, u, d], 1)[take]
    f[h1[take] // 3] = np.stack([d, w, c], 1)[take]
    return f, int(take.sum())


def _smooth(pos, f, lock):
    """One Jacobi pass of tangential smoothing of the free vertices"""
    V = len(pos)
    P = pos.astype(np.float64)
    start, vf, vc = _vertex_faces(f, V)
    deg = np.diff(start)
    nxt = f[vf, (vc + 1) % 3]
    prv = f[vf, (vc + 2) % 3]
    fn = _face_normals(P, f)[vf]
    s = np.zeros((V, 3))
    ns = np.zeros((V, 3))
    for j in range(int(deg.max()) if V else 0):
        sel = np.flatnonzero(deg > j)
        i = start[sel] + j
        s[sel] += P[nxt[i]]
        s[sel] += P[prv[i]]
        ns[sel] += fn[i]
    with np.errstate(all="ignore"):
        c = s / (2.0 * deg)[:, None]
        nl = np.sqrt(_dot(ns, ns))
        n = ns / nl[:, None]
        dv = c - P
        t = _dot(dv, n)
        q = P + (dv - t[:, None] * n)
    free = ~lock & (deg > 0) & (nl > 0)
    pos = pos.copy()
    pos[free] = q[free].astype(np.float32)
    return pos, deg


def remesh(vertices, faces, target_len=0.015, iterations=3, feature_deg=30.0, max_surf_dist=None):
    """-> (vertices float32 [V', 3], faces int64 [F', 3], stats [iterations][4]: faces after the split, collapse
    rounds, flip rounds, 1 if a stage stopped at ROUND_CAP rounds).  max_surf_dist None or < 0: 1 % of the bounding-box
    diagonal of the referenced input vertices."""
    pos = np.ascontiguousarray(vertices, np.float32).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    V = len(pos)
    assert len(f) == 0 or (f.min() >= 0 and f.max() < V), "face index out of range"
    assert ((f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 0] != f[:, 2])).all(), "repeated index in a face"
    if iterations == 0:
        return pos.copy(), f.copy(), []
    stats = [[0, 0, 0, 0] for _ in range(iterations)]
    if len(f) == 0:
        return np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64), stats
    L = float(target_len)
    lo, hi = 4.0 * L / 5.0, 4.0 * L / 3.0
    cos_t = math.cos(float(feature_deg) * (math.pi / 180.0))
    msd = _diag(pos[np.unique(f)]) / 100.0 if max_surf_dist is None or max_surf_dist < 0 else float(max_surf_dist)
    surf = (pos.copy(), f.copy())
    for it in range(iterations):
        if not len(f):
            break
        ed = _Edges(pos, f, cos_t)
        lock = np.zeros(len(pos), bool)
        lock[ed.a[ed.blocked]] = lock[ed.b[ed.blocked]] = True
        pos, f, lock = _split(pos, f, lock, ed, hi)
        stats[it][0] = len(f)
        for _ in range(ROUND_CAP if len(f) else 0):
            pos, f, lock, taken = _collapse_round(pos, f, lock, _Edges(pos, f, cos_t), lo, hi, surf, msd)
            if not taken:
                break
            stats[it][1] += 1
        for _ in range(ROUND_CAP if len(f) else 0):
            f, taken = _flip_round(pos, f, _Edges(pos, f, cos_t), surf, msd)
            if not taken:
                break
            stats[it][2] += 1
        stats[it][3] = int(stats[it][1] == ROUND_CAP or stats[it][2] == ROUND_CAP)
        if not len(f):
            break
        pos, deg = _smooth(pos, f, lock)
        ref = np.flatnonzero(deg > 0)
        q, _, _ = closest_points(*surf, pos[ref].astype(np.float64))
        pos = pos.copy()
        pos[ref] = q.astype(np.float32)
    used = np.unique(f)
    remap = np.full(len(pos), -1, np.int64)
    remap[used] = np.arange(len(used))
    return pos[used], remap[f], stats
