"""Serial oracle of the quadric edge-collapse decimation (dgs_mesh_decimate, open-diffusiongs_b200/csrc/mesh_decimate.cu).

Plain Garland-Heckbert with a heap: the globally cheapest collapsible edge is collapsed, one at a time, and the edges
around the survivor are re-evaluated.  The quadrics, the placement and its fallback, the locked vertices, the link
condition and the fold-over test are the kernel's rules, restated in fp64 Python; only the order of the collapses
differs (the kernel takes rounds of independent local minima), so the result is the quality reference, not a bitwise
one.  Meant for meshes of a few thousand faces.
"""
import heapq
import math

import numpy as np

MAX_CONDITION = 1e7  # as the kernel: above this Frobenius condition number the 3 x 3 system is not solved


def _f32(x):
    return float(np.float32(x))


def _sub(u, v):
    return (u[0] - v[0], u[1] - v[1], u[2] - v[2])


def _dot(u, v):
    return u[0] * v[0] + u[1] * v[1] + u[2] * v[2]


def _cross(u, v):
    return (u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0])


def face_quadric(p0, p1, p2):
    """Area-weighted plane quadric A p p^T, p = (n, -n.p0), as its 10 unique entries (xx xy xz xw yy yz yw zz zw ww)."""
    n = _cross(_sub(p1, p0), _sub(p2, p0))
    ln = math.sqrt(_dot(n, n))
    if not (ln > 0) or not math.isfinite(ln):
        return [0.0] * 10
    p = (n[0] / ln, n[1] / ln, n[2] / ln, -_dot(n, p0) / ln)
    w = 0.5 * ln
    return [w * p[i] * p[j] for i in range(4) for j in range(i, 4)]


def quadric_cost(q, v):
    x, y, z = v
    return (q[0] * x * x + 2 * q[1] * x * y + 2 * q[2] * x * z + 2 * q[3] * x + q[4] * y * y + 2 * q[5] * y * z
            + 2 * q[6] * y + q[7] * z * z + 2 * q[8] * z + q[9])


def placement(q, pa, pb):
    """-> (fp32 position, cost): the minimiser of v^T Q v, or the best of midpoint, a, b when the system is singular or
    ill-conditioned, the solution not finite or farther than |a - b| from the midpoint."""
    mid = tuple(_f32(0.5 * (pa[k] + pb[k])) for k in range(3))
    a00, a01, a02, a11, a12, a22 = q[0], q[1], q[2], q[4], q[5], q[7]
    c00, c01, c02 = a11 * a22 - a12 * a12, a02 * a12 - a01 * a22, a01 * a12 - a02 * a11
    c11, c12, c22 = a00 * a22 - a02 * a02, a01 * a02 - a00 * a12, a00 * a11 - a01 * a01
    det = a00 * c00 + a01 * c01 + a02 * c02
    nA = math.sqrt(a00 ** 2 + a11 ** 2 + a22 ** 2 + 2 * (a01 ** 2 + a02 ** 2 + a12 ** 2))
    nC = math.sqrt(c00 ** 2 + c11 ** 2 + c22 ** 2 + 2 * (c01 ** 2 + c02 ** 2 + c12 ** 2))
    if det != 0 and nA * nC <= MAX_CONDITION * abs(det):
        b0, b1, b2 = q[3], q[6], q[8]
        with np.errstate(over="ignore"):
            v = (_f32(-(c00 * b0 + c01 * b1 + c02 * b2) / det), _f32(-(c01 * b0 + c11 * b1 + c12 * b2) / det),
                 _f32(-(c02 * b0 + c12 * b1 + c22 * b2) / det))
        dm, ab = _sub(v, mid), _sub(pa, pb)
        if all(math.isfinite(c) for c in v) and _dot(dm, dm) <= _dot(ab, ab):
            return v, quadric_cost(q, v)
    best = min(((quadric_cost(q, c), i, c) for i, c in enumerate((mid, tuple(pa), tuple(pb)))))
    return best[2], best[0]


def decimate(vertices, faces, target):
    """-> (vertices float32 [V', 3], faces int64 [F', 3], collapses).  Surviving vertices in index order, faces in face
    order; the lower index of a collapsed edge survives."""
    pos = [tuple(float(c) for c in p) for p in np.asarray(vertices, np.float32)]
    tri = [list(map(int, f)) for f in np.asarray(faces, np.int64)]
    V, F = len(pos), len(tri)
    assert all(0 <= x < V for f in tri for x in f) and all(len(set(f)) == 3 for f in tri)
    if F <= target:
        return np.asarray(vertices, np.float32).reshape(-1, 3), np.asarray(faces, np.int64).reshape(-1, 3), 0
    vf = [set() for _ in range(V)]
    Q = [[0.0] * 10 for _ in range(V)]
    edge_count = {}
    for i, f in enumerate(tri):
        K = face_quadric(*(pos[x] for x in f))
        for x in f:
            vf[x].add(i)
            Q[x] = [s + k for s, k in zip(Q[x], K)]
        for k in range(3):
            e = tuple(sorted((f[k], f[(k + 1) % 3])))
            edge_count[e] = edge_count.get(e, 0) + 1
    locked = {x for e, n in edge_count.items() if n != 2 for x in e}

    def nbrs(v):
        return {x for i in vf[v] for x in tri[i]} - {v}

    def keeps_orientation(v, other, p):
        for i in vf[v]:
            f = tri[i]
            if other in f:
                continue
            P = [pos[x] for x in f]
            n0 = _cross(_sub(P[1], P[0]), _sub(P[2], P[0]))
            if n0 == (0.0, 0.0, 0.0):
                continue
            P[f.index(v)] = p
            if not _dot(n0, _cross(_sub(P[1], P[0]), _sub(P[2], P[0]))) > 0:
                return False
        return True

    def evaluate(a, b):
        if a in locked or b in locked:
            return None
        both = vf[a] & vf[b]
        if len(both) != 2:
            return None
        c, d = ((set(tri[i]) - {a, b}).pop() for i in sorted(both))
        if c == d or nbrs(a) & nbrs(b) != {c, d}:
            return None
        if (any({c, d} <= set(tri[i]) and b not in tri[i] for i in vf[a])
                and any({c, d} <= set(tri[i]) and a not in tri[i] for i in vf[b])):
            return None
        q = [x + y for x, y in zip(Q[a], Q[b])]
        v, cost = placement(q, pos[a], pos[b])
        if not math.isfinite(cost) or not keeps_orientation(a, b, v) or not keeps_orientation(b, a, v):
            return None
        return _f32(max(cost, 0.0)), v

    heap, stamp = [], {}

    def push(a, b):
        e = (min(a, b), max(a, b))
        stamp[e] = stamp.get(e, 0) + 1
        r = evaluate(*e)
        if r is not None:
            heapq.heappush(heap, (r[0], e, stamp[e]))

    for e in edge_count:
        push(*e)
    live, collapses = F, 0
    while live > target and heap:
        _, (a, b), st = heapq.heappop(heap)
        if stamp[(a, b)] != st:
            continue
        r = evaluate(a, b)
        if r is None:
            continue
        pos[a] = r[1]
        Q[a] = [x + y for x, y in zip(Q[a], Q[b])]
        for i in vf[a] & vf[b]:
            for x in tri[i]:
                vf[x].discard(i)
            tri[i] = None
        for i in vf[b]:
            tri[i][tri[i].index(b)] = a
            vf[a].add(i)
        vf[b] = set()
        live -= 2
        collapses += 1
        # the edges whose cost or tests read a's new position or faces: every edge of a and of its neighbours
        for e in {(min(x, y), max(x, y)) for x in nbrs(a) | {a} for y in nbrs(x)}:
            push(*e)
    alive = [f for f in tri if f is not None]
    used = sorted({x for f in alive for x in f})
    new = {v: i for i, v in enumerate(used)}
    out_v = np.array([pos[v] for v in used], np.float32).reshape(-1, 3)
    out_f = np.array([[new[x] for x in f] for f in alive], np.int64).reshape(-1, 3)
    return out_v, out_f, collapses
