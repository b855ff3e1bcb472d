"""Small meshes for the mesh-cleaning tests, one behaviour each, with the result worked out by hand: (name, vertices
float32 [V, 3], faces int64 [F, 3], clean() keyword arguments, expected vertices, expected faces, expected face count
after each of the nine stages or None)."""
import numpy as np

OFF = dict(v_pct=0, min_f=0, min_d=0, repair=False)  # every optional stage off


def _far(n):
    """2 n vertices far from the origin and from each other: the other two corners of n thin triangles"""
    return [p for i in range(n) for p in ((10.0 * i, 20.0, 0.0), (10.0 * i, 0.0, 20.0))]


def _fans(n, base):
    return [(k, base + 2 * k, base + 2 * k + 1) for k in range(n)]


def cases():
    out = []
    P = np.array([(0, 0, 0), (9, 9, 9), (1, 0, 0), (0, 1, 0), (7, 7, 7)], np.float32)
    out.append(("unreferenced", P, np.array([(0, 2, 3)]), OFF, P[[0, 2, 3]], np.array([(0, 1, 2)]), [1] * 9))

    # A - B and B - C within r = 1.5, A - C not: the greedy order decides whether C survives
    chain = [(0.0, 0, 0), (1.0, 0, 0), (2.0, 0, 0)] + _far(3)
    V = np.array(chain, np.float32)
    diag = float(np.linalg.norm(V.max(0).astype(np.float64) - V.min(0).astype(np.float64)))
    kw = dict(v_pct=150.0 / diag, min_f=0, min_d=0, repair=False)
    F = np.array(_fans(3, 3))
    # A (0) a seed, B (1) -> A, C (2): its only neighbour B is merged, so a seed
    out.append(("chain_abc", V, F, kw, V[[0, 2, 3, 4, 5, 6, 7, 8]], np.array([(0, 2, 3), (0, 4, 5), (1, 6, 7)]),
                [3] * 9))
    # the same points in the order B, A, C: B a seed, A -> B and C -> B
    V2 = V[[1, 0, 2] + list(range(3, 9))]
    out.append(("chain_bac", V2, F, kw, V2[[0, 3, 4, 5, 6, 7, 8]], np.array([(0, 1, 2), (0, 3, 4), (0, 5, 6)]),
                [3] * 9))

    # box (0..3, 0..4, 0): diag 5, v_pct 20 -> r = 1.0 exactly; 0 - 1 at distance exactly r stays, 2 - 3 at 0.5 merges
    Q = np.array([(0, 0, 0), (1, 0, 0), (3, 4, 0), (3, 3.5, 0), (0, 4, 0), (3, 0, 0)], np.float32)
    Fq = np.array([(0, 1, 4), (1, 5, 2), (1, 5, 3)])
    # vertex 3 -> 2: faces (0, 1, 4), (1, 5, 2), (1, 5, 2) -> the duplicate goes in stage 3
    out.append(("distance_exactly_r", Q, Fq, dict(v_pct=20, min_f=0, min_d=0, repair=False), Q[[0, 1, 2, 4, 5]],
                np.array([(0, 1, 3), (1, 4, 2)]), [3, 3, 2, 2, 2, 2, 2, 2, 2]))

    # merging makes a face repeat a vertex: it goes in stage 2
    Q2 = np.array([(0, 0, 0), (3, 0, 0), (0, 4, 0), (2.8, 0.1, 0), (3, 4, 0)], np.float32)
    out.append(("degenerate_by_merge", Q2, np.array([(0, 1, 2), (1, 3, 4), (1, 4, 2)]),
                dict(v_pct=20, min_f=0, min_d=0, repair=False), Q2[[0, 1, 2, 4]], np.array([(0, 1, 2), (1, 3, 2)]),
                [3, 2, 2, 2, 2, 2, 2, 2, 2]))

    T = np.array([(0, 0, 0), (1, 0, 0), (0, 1, 0), (1, 1, 0)], np.float32)
    out.append(("duplicates", T, np.array([(1, 3, 2), (0, 1, 2), (0, 1, 2), (2, 1, 0), (1, 2, 0), (2, 3, 1)]), OFF, T,
                np.array([(1, 3, 2), (0, 1, 2)]), [6, 6, 2, 2, 2, 2, 2, 2, 2]))

    L = np.array([(0, 0, 0), (1, 0, 0), (2, 0, 0), (0, 1, 0)], np.float32)
    out.append(("null_face", L, np.array([(0, 1, 2), (0, 1, 3), (3, 3, 1)]), OFF, L[[0, 1, 3]],
                np.array([(0, 1, 2)]), [3, 3, 3, 1, 1, 1, 1, 1, 1]))

    # a 10 x 1 strip of 20 faces, a tiny triangle (under 20 % of the diagonal) and a long 2-face strip (under min_f)
    strip = [(float(x), float(y), 0.0) for x in range(11) for y in (0, 1)]
    sf = [(2 * x, 2 * x + 2, 2 * x + 1) for x in range(10)] + [(2 * x + 1, 2 * x + 2, 2 * x + 3) for x in range(10)]
    n = len(strip)
    tiny = [(5.0, 5.0, 0.0), (5.1, 5.0, 0.0), (5.0, 5.1, 0.0)]
    long2 = [(0.0, 3.0, 0.0), (8.0, 3.0, 0.0), (0.0, 3.5, 0.0), (8.0, 3.5, 0.0)]
    S = np.array(strip + tiny + long2, np.float32)
    Sf = np.array(sf + [(n, n + 1, n + 2), (n + 3, n + 4, n + 5), (n + 5, n + 4, n + 6)])
    out.append(("small_components", S, Sf, dict(v_pct=0, min_f=10, min_d=20, repair=False), S[:n], np.array(sf),
                [23, 23, 23, 23, 22, 20, 20, 20, 20]))

    bow = np.array([(0, 0, 0), (1, 0, 0), (1, 1, 0), (-1, 0, 0), (-1, -1, 0)], np.float32)
    bf = np.array([(0, 1, 2), (0, 3, 4)])
    # faces that share only a vertex are two components: one face each, both under min_f = 2
    out.append(("vertex_only_components", bow, bf, dict(v_pct=0, min_f=2, min_d=0, repair=False),
                np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64), [2, 2, 2, 2, 2, 0, 0, 0, 0]))
    # the bow-tie vertex is split: the fan of face 1 gets a copy of vertex 0, appended
    out.append(("bowtie_split", bow, bf, dict(v_pct=0, min_f=0, min_d=0, repair=True), bow[[0, 1, 2, 3, 4, 0]],
                np.array([(0, 1, 2), (5, 3, 4)]), [2] * 9))
    out.append(("bowtie_no_repair", bow, bf, OFF, bow, bf, [2] * 9))

    # edge (0, 1) with 3 faces (apexes at heights 3, 1, 2) and edge (5, 6) with 4 (heights 2, 4, 1, 3): the smallest
    # faces go until 2 are left
    E = np.array([(0, 0, 0), (1, 0, 0), (0.5, 3, 0), (0.5, 0, 1), (0.5, -2, 0),
                  (5, 0, 0), (6, 0, 0), (5.5, 2, 0), (5.5, 0, 4), (5.5, -1, 0), (5.5, 0, -3)], np.float32)
    Ef = np.array([(0, 1, 2), (0, 1, 3), (1, 0, 4), (5, 6, 7), (5, 6, 8), (6, 5, 9), (5, 6, 10)])
    keep = [0, 2, 4, 6]
    used = sorted({x for k in keep for x in Ef[k]})
    remap = {v: i for i, v in enumerate(used)}
    out.append(("nonmanifold_edges", E, Ef, dict(v_pct=0, min_f=0, min_d=0, repair=True), E[used],
                np.array([[remap[x] for x in Ef[k]] for k in keep]), [7, 7, 7, 7, 7, 7, 4, 4, 4]))

    # the defaults on a closed mesh with nothing to do but merge: a tetrahedron far larger than r
    tet = np.array([(0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1)], np.float32)
    tf = np.array([(0, 2, 1), (0, 1, 3), (0, 3, 2), (1, 2, 3)])
    out.append(("all_zero_options", tet, tf, dict(v_pct=0, min_f=0, min_d=0, repair=True), tet, tf, [4] * 9))
    out.append(("defaults_remove_small", tet, tf, {}, np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64),
                [4, 4, 4, 4, 4, 0, 0, 0, 0]))
    out.append(("empty", np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64), {}, np.zeros((0, 3), np.float32),
                np.zeros((0, 3), np.int64), [0] * 9))
    return out
