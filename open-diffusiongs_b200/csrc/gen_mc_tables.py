"""Generates mc_tables.h, the marching-cubes case tables of mesh.cu, from first principles.

    python open-diffusiongs_b200/csrc/gen_mc_tables.py            # rewrites mc_tables.h next to this file
    python open-diffusiongs_b200/csrc/gen_mc_tables.py --check    # exit 1 if the committed header differs

Conventions (shared with mesh.cu and oracle/mesh.py):
  corner c = dx + 2 dy + 4 dz, (dx, dy, dz) in {0, 1}^3, offsets along (x, y, z) = the field's (i, j, k) axes;
  edge a * 4 + j runs along axis a from corner EDGE_CORNERS[e][0] (bit a clear) to EDGE_CORNERS[e][1] (bit a set);
  case index = sum over inside corners of 1 << c, a corner being inside iff its value > iso.

For each case every cube face is cut into segments between the crossings on its four edges.  Walking the face's
boundary counter-clockwise as seen from outside the cube, each maximal run of inside boundary is closed off by one
segment from the crossing where the run starts to the crossing where it ends.  On a face with two diagonally opposite
inside corners this always SEPARATES the inside corners; the rule depends only on the face's four corner values, so the
two cubes sharing a face cut it the same way and the surface is watertight.  Each crossing is then the head of one
segment and the tail of one other, on the two faces sharing its edge, so the segments chain into closed loops.  Each
loop is triangulated without a chord between two crossings of one face (such a chord would lie in the face, where the
neighbouring cube may use it too, and the surface would fold onto itself); of those triangulations the one closest to a
fan from the loop's first crossing is taken.  The loop direction makes each triangle's right-hand-rule normal point from
the inside (values above iso) to the outside.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "mc_tables.h")


def _corner(d):
    return d[0] + 2 * d[1] + 4 * d[2]


def edges():
    out = []
    for a in range(3):
        u, v = (a + 1) % 3, (a + 2) % 3
        for j in range(4):
            d = [0, 0, 0]
            d[u], d[v] = j & 1, j >> 1
            c0 = _corner(d)
            out.append((c0, c0 | (1 << a)))
    return out


EDGE_CORNERS = edges()
EDGE_OF = {frozenset(e): i for i, e in enumerate(EDGE_CORNERS)}


def faces():
    """-> six lists of 4 corners, counter-clockwise as seen from outside the cube."""
    out = []
    for a in range(3):
        u, v = (a + 1) % 3, (a + 2) % 3  # e_u x e_v = e_a
        for s in (0, 1):
            ring = [(0, 0), (1, 0), (1, 1), (0, 1)]
            if s == 0:  # outward normal -e_a: the same square seen from the other side
                ring = ring[::-1]
            cs = []
            for pu, pv in ring:
                d = [0, 0, 0]
                d[a], d[u], d[v] = s, pu, pv
                cs.append(_corner(d))
            out.append(cs)
    return out


FACES = faces()


def case_loops(case):
    inside = [(case >> c) & 1 for c in range(8)]
    nxt = {}  # crossing edge -> the crossing edge its segment leads to
    for ring in FACES:
        crossings = []  # (edge, kind) in counter-clockwise order; kind 1 = run of inside boundary starts here
        for k in range(4):
            c0, c1 = ring[k], ring[(k + 1) % 4]
            if inside[c0] != inside[c1]:
                crossings.append((EDGE_OF[frozenset((c0, c1))], inside[c1]))
        if not crossings:
            continue
        start = next(i for i, (_, kind) in enumerate(crossings) if kind == 1)
        crossings = crossings[start:] + crossings[:start]
        for i in range(0, len(crossings), 2):  # (start of an inside run, its end)
            (e_in, _), (e_out, _) = crossings[i], crossings[i + 1]
            assert e_in not in nxt
            nxt[e_in] = e_out
    loops, seen = [], set()
    for e in sorted(nxt):
        if e in seen:
            continue
        loop = [e]
        seen.add(e)
        while nxt[loop[-1]] != e:
            loop.append(nxt[loop[-1]])
            seen.add(loop[-1])
        loops.append(loop)
    return loops


FACE_EDGES = [{EDGE_OF[frozenset((r[k], r[(k + 1) % 4]))] for k in range(4)} for r in FACES]


def _on_common_face(e0, e1):
    return any(e0 in f and e1 in f for f in FACE_EDGES)


def triangulate(loop):
    """Triangles of a loop, each in loop order, whose chords (triangle sides that are not loop sides) never join two
    crossings of one cube face: such a chord lies in the face, where the neighbouring cube could use it as well."""
    n = len(loop)
    if n == 3:
        return [tuple(loop)]
    for k in range(n - 2, 0, -1):  # apex of the triangle on the side (loop[0], loop[n-1]); k = n-2 first: a fan
        chords = ([(loop[0], loop[k])] if k > 1 else []) + ([(loop[k], loop[n - 1])] if k < n - 2 else [])
        if any(_on_common_face(a, b) for a, b in chords):
            continue
        left = triangulate(loop[:k + 1]) if k > 1 else []
        right = triangulate(loop[k:]) if k < n - 2 else []
        if left is not None and right is not None:
            return left + [(loop[0], loop[k], loop[n - 1])] + right
    return None


def tables():
    """-> 256 flat lists of edge indices, 3 per triangle, in loop order"""
    tris = []
    for case in range(256):
        t = []
        for loop in case_loops(case):
            tri = triangulate(loop)
            assert tri is not None, (case, loop)
            t += [e for tr in tri for e in tr]
        tris.append(t)
    return tris


def render():
    tris = tables()
    max_t = max(len(t) for t in tris) // 3
    lines = ["// mc_tables.h -- generated by gen_mc_tables.py; do not edit.  Conventions are in that script's docstring.",
             "#pragma once", "", f"#define DGS_MC_MAX_TRIS {max_t}", "",
             "// edge e runs from corner kMcEdgeCorners[e][0] to kMcEdgeCorners[e][1] (corner c = dx + 2 dy + 4 dz)",
             "static __constant__ signed char kMcEdgeCorners[12][2] = {"]
    lines.append("    " + ", ".join(f"{{{a}, {b}}}" for a, b in EDGE_CORNERS) + "};")
    lines += ["", "// triangles of each case", "static __constant__ signed char kMcNumTris[256] = {"]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(len(t) // 3) for t in tris[r:r + 32]) + ",")
    lines += ["};", "", "// edge indices of each case's triangles, 3 per triangle, -1 padded",
              f"static __constant__ signed char kMcTriEdges[256][{3 * max_t}] = {{"]
    for t in tris:
        row = t + [-1] * (3 * max_t - len(t))
        lines.append("    {" + ", ".join(str(x) for x in row) + "},")
    lines += ["};", ""]
    return "\n".join(lines)


def main(argv):
    text = render()
    if "--check" in argv:
        with open(OUT) as f:
            ok = f.read() == text
        print("mc_tables.h is up to date" if ok else "mc_tables.h differs from the generator's output")
        return 0 if ok else 1
    with open(OUT, "w") as f:
        f.write(text)
    print(OUT)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
