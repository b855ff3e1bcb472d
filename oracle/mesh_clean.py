"""Serial oracle of the mesh cleaning (dgs_mesh_clean, open-diffusiongs_b200/csrc/mesh_clean.cu): the reference's
clean_mesh (utils/mesh_utils.py:88-147) with remesh=False, as the nine stages the header states, in the same fp64
arithmetic (numpy's elementwise float64 operations round each product and sum, as the kernels compiled without FMA
contraction do).  The native path must equal this bit for bit: vertices, faces and the face count after each stage.

The vertex merge is the plain greedy loop (a vertex is a seed iff no earlier seed is within r; otherwise it goes to the
lowest-index seed within r), and the non-manifold edge repair the plain walk over the sorted candidates; everything
else is vectorised numpy / scipy, so the obj-256 marching-cubes mesh (341 k vertices, 682 k faces) runs in seconds.
"""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components
from scipy.spatial import cKDTree

STAGES = ("unreferenced", "merge", "duplicate", "null", "diameter", "face_count", "nonmanifold_edges",
          "nonmanifold_vertices", "compact")


def _diag(p):
    """fp64 norm of max - min over the rows of p (fp32 [n, 3], n > 0)"""
    d = p.max(0).astype(np.float64) - p.min(0).astype(np.float64)
    return float(np.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]))


def doubled_area(pos, faces):
    """|(b - a) x (c - a)| in fp64 from the fp32 positions, per face"""
    a, b, c = (pos[faces[:, k]].astype(np.float64) for k in range(3))
    u, w = b - a, c - a
    n0 = u[:, 1] * w[:, 2] - u[:, 2] * w[:, 1]
    n1 = u[:, 2] * w[:, 0] - u[:, 0] * w[:, 2]
    n2 = u[:, 0] * w[:, 1] - u[:, 1] * w[:, 0]
    return np.sqrt(n0 * n0 + n1 * n1 + n2 * n2)


def merge_close(pos, faces, r):
    """-> rep [V]: every referenced vertex's seed (itself for a seed).  Seeds are the lexicographically-first maximal
    independent set of the graph of pairs at distance < r."""
    V = len(pos)
    rep = np.arange(V, dtype=np.int64)
    if not r > 0:
        return rep
    used = np.unique(faces)
    p = pos[used].astype(np.float64)
    pairs = cKDTree(p).query_pairs(r * (1 + 1e-6), output_type="ndarray")  # a superset; the exact test follows
    if len(pairs):
        d = p[pairs[:, 0]] - p[pairs[:, 1]]
        keep = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]) < r
        lo, hi = used[pairs[keep].min(1)], used[pairs[keep].max(1)]
    else:
        lo = hi = np.zeros(0, np.int64)
    order = np.lexsort((lo, hi))
    lo, hi = lo[order], hi[order]
    start = np.searchsorted(hi, np.arange(V + 1))
    seed = np.zeros(V, bool)
    for v in used.tolist():
        nb = lo[start[v]:start[v + 1]]
        s = nb[seed[nb]]
        if len(s):
            rep[v] = s[0]
        else:
            seed[v] = True
    return rep


def _edge_runs(faces):
    """-> (half-edge ids sorted by undirected edge, in half-edge order within an edge; True where a sorted half-edge
    starts a new edge)"""
    u = faces.reshape(-1)
    w = faces[:, [1, 2, 0]].reshape(-1)
    a, b = np.minimum(u, w), np.maximum(u, w)
    order = np.lexsort((np.arange(len(a)), b, a))
    a, b = a[order], b[order]
    head = np.ones(len(a), bool)
    head[1:] = (a[1:] != a[:-1]) | (b[1:] != b[:-1])
    return order, head


def _components(n, i, j):
    """-> for each of n nodes the smallest node of its component in the graph with edges (i, j)"""
    _, lab = connected_components(coo_matrix((np.ones(len(i)), (i, j)), shape=(n, n)), directed=False)
    low = np.full(lab.max() + 1 if n else 0, n, np.int64)
    np.minimum.at(low, lab, np.arange(n))
    return low[lab]


def clean(vertices, faces, v_pct=1, min_f=64, min_d=20, repair=True, info=None):
    """-> (vertices float32 [V', 3], faces int64 [F', 3], face count after each of the nine stages).  `info`, a dict,
    receives "stage_vertices" (the referenced vertex count after each stage) and "candidates" (stage 7's)."""
    pos = np.ascontiguousarray(vertices, np.float32).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    V = len(pos)
    assert len(f) == 0 or (f.min() >= 0 and f.max() < V), "face index out of range"
    counts = []
    if info is not None:
        info.update(stage_vertices=[], candidates=0)

    def done(n=1):  # the stage(s) leave f
        counts.extend([len(f)] * n)
        if info is not None:
            info["stage_vertices"] += [len(np.unique(f))] * n
    done()  # 1: unreferenced vertices are never read below; compaction at the end drops them
    # 2. merge close vertices
    if v_pct > 0 and len(f):
        r = (v_pct / 100.0) * _diag(pos[np.unique(f)])
        f = merge_close(pos, f, r)[f]
        f = f[(f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 0] != f[:, 2])]
    done()
    # 3. duplicate faces: the same sorted index triple; the lowest face index stays
    s = np.sort(f, axis=1)
    order = np.lexsort((np.arange(len(f)), s[:, 2], s[:, 1], s[:, 0]))
    ss = s[order]
    dup = np.zeros(len(f), bool)
    dup[order[1:]] = (ss[1:] == ss[:-1]).all(1)
    f = f[~dup]
    done()
    # 4. null faces
    f = f[doubled_area(pos, f) != 0]
    done()
    # 5, 6. small components (faces connected through shared edges) by diameter, then by face count
    if len(f) and (min_d > 0 or min_f > 0):
        order, head = _edge_runs(f)
        same = np.flatnonzero(~head)
        comp = _components(len(f), order[same] // 3, order[same - 1] // 3)
        if min_d > 0:
            thr = (min_d / 100.0) * _diag(pos[np.unique(f)])
            corner = pos[f].reshape(-1, 3)
            cc = np.repeat(comp, 3)
            mn = np.full((len(f), 3), np.inf, np.float32)
            mx = np.full((len(f), 3), -np.inf, np.float32)
            np.minimum.at(mn, cc, corner)
            np.maximum.at(mx, cc, corner)
            with np.errstate(invalid="ignore"):  # rows of labels no face has: inf - inf
                d = mx.astype(np.float64) - mn.astype(np.float64)
                cdiag = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])
            keep5 = ~(cdiag[comp] < thr)
            f, comp = f[keep5], comp[keep5]
        done()
        if min_f > 0:
            f = f[~(np.bincount(comp)[comp] < min_f)]
        done()
    else:
        done(2)
    if repair and len(f):
        # 7. non-manifold edges: candidates in (doubled area, face index) order; one goes while an edge of it still
        #    has more than two live faces
        order, head = _edge_runs(f)
        eid = np.empty(len(order), np.int64)
        eid[order] = np.cumsum(head) - 1
        live = np.bincount(eid)
        fe = eid.reshape(-1, 3)
        cand = np.flatnonzero((live[fe] > 2).any(1))
        alive = np.ones(len(f), bool)
        if info is not None:
            info["candidates"] = len(cand)
        if len(cand):
            area = doubled_area(pos, f[cand])
            for c in cand[np.lexsort((cand, area))].tolist():
                e = fe[c]
                if (live[e] > 2).any():
                    live[e] -= 1
                    alive[c] = False
        f = f[alive]
        done()
        # 8. non-manifold vertices: corners 3 f + k of a vertex joined through the edges at that vertex; each fan but
        #    the one holding the vertex's lowest face gets a copy
        if len(f):
            order, head = _edge_runs(f)
            same = np.flatnonzero(~head)
            h1, h0 = order[same], order[same - 1]  # two half-edges of one edge: corners k and k + 1 of their faces

            def nxt(h):
                return 3 * (h // 3) + (h % 3 + 1) % 3
            fv = f.reshape(-1)
            # the corner of the same vertex: h0's start is h1's start or h1's end
            s0 = fv[h0] == fv[h1]
            i = np.concatenate([h0, nxt(h0)])
            j = np.concatenate([np.where(s0, h1, nxt(h1)), np.where(s0, nxt(h1), h1)])
            fan = _components(3 * len(f), i, j)  # the fan's lowest corner, 3 * its lowest face + k
            first = np.full(V, 3 * len(f), np.int64)
            np.minimum.at(first, fv, np.arange(3 * len(f)))  # the vertex's corner in its lowest face
            roots = np.flatnonzero((fan == np.arange(3 * len(f))) & (first[fv] != np.arange(3 * len(f))))
            roots = roots[np.lexsort((roots, fv[roots]))]
            new_id = np.full(3 * len(f), -1, np.int64)
            new_id[roots] = V + np.arange(len(roots))
            src = fv[roots]
            ids = new_id[fan]
            fv = np.where(ids >= 0, ids, fv)
            f = fv.reshape(-1, 3)
            pos = np.concatenate([pos, pos[src]])
        done()
    else:
        done(2)
    # 9. compact
    used = np.unique(f)
    remap = np.full(len(pos), -1, np.int64)
    remap[used] = np.arange(len(used))
    done()
    return pos[used].reshape(-1, 3), remap[f].reshape(-1, 3), counts
