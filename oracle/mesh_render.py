"""oracle/mesh_render.py -- TEST INFRASTRUCTURE: the serial specification of dgs_mesh_render (mesh_render.cu), in numpy
float32 / int64, operation for operation as the kernels round them (no np.dot, no @ on fp32 data).  Never imported by
the product path.

Conventions.  clip [n_views, 4, 4] are row-major world -> clip matrices.  A corner becomes (X, Y, w) =
((x_c + w_c) W / 2, (y_c + w_c) H / 2, w_c) (each product rounded to fp32; x_c = ((m0 x + m1 y) + m2 z) + m3), so pixel
(i, j) (column i, row j) has its centre at X / w = i + 0.5, Y / w = j + 0.5.

1. Setup, per (view, face).  Sutherland-Hodgman clipping of the corner polygon against, in order, w >= near,
   X >= -G w, X <= (W + G) w, Y >= -G w, Y <= (H + G) w with G = 8192 (a plane no corner is outside of is skipped).  An
   edge crossing a plane gives the point I + s (O - I), s = d_I / (d_I - d_O), from its inside end I (d >= 0) to its
   outside end O, so both faces of a shared edge make the same point; a polygon that would exceed 8 corners (possible
   only when rounding alternates the signs of d on a near-degenerate face) is culled.  Corners snap to
   rint(X / w * 256), rint(Y / w * 256) (1/256 pixel); a polygon of negative area is reversed, one of zero area or with an empty pixel box (pixel i is a
   candidate when 256 i + 128 lies within the snapped range, clamped to the image) is culled.  The facing of the face
   is the sign of det[(X, Y, w) of its unclipped corners]: (X0 (Y1 w2 - w1 Y2) - Y0 (X1 w2 - w1 X2)) + w0 (X1 Y2 - Y1 X2).
2. Coverage.  Pixel (i, j), at p = (256 i + 128, 256 j + 128), is covered when for every edge a -> b of the snapped
   polygon with b != a, e = (bx - ax)(py - ay) - (by - ay)(px - ax) (int64) is > 0, or = 0 and the edge is top-left
   (by - ay < 0, or by = ay and bx > ax).  Its barycentrics are those of the unclipped face: with ex_k = X_k - px w_k,
   ey_k = Y_k - py w_k (px = i + 0.5 in fp32), b0 = ex1 ey2 - ex2 ey1, b1 = ex2 ey0 - ex0 ey2, b2 = ex0 ey1 - ex1 ey0,
   d = (b0 + b1) + b2, u = b / d (d = 0: not covered), and depth = (u0 w0 + u1 w1) + u2 w2.  The pixel keeps the
   smallest key (fkey(depth) << 32) | face, fkey the order-preserving map of float bits.
3. Resolve.  Background (no key): face_id -1, depth 0, normal_bg, color_bg.  Otherwise the winning face's u gives depth,
   n = (u0 n0 + u1 n1) + u2 n2 per channel over its length sqrt((n0 n0 + n1 n1) + n2 n2) (0 where that is 0) and
   rgb = (u0 c0 + u1 c1) + u2 c2.
4. Antialias (silhouette edges, after Laine et al. 2020, "Modular primitives for high-performance differentiable
   rendering", in gather form).  Alpha is 1 on faces and 0 on background, then alpha, normal and rgb of each pixel are
   updated from its left, right, upper and lower neighbour in this order, each from the values before antialiasing:
   acc = acc + weight * (v_neighbour - v_self), where weight != 0.  For a pair of pixels with different faces (or face
   and background) the occluder is the one with the smaller key.  With the occluder face's homogeneous edge functions
   b_o at its centre and b_f at the far centre (as in 2) and d its sum at the occluder's centre, edge k is left through
   when the far centre is outside it (b_f < 0 for d > 0, > 0 for d < 0) and the occluder's centre is not
   (b_o >= 0, resp. <= 0); t_k = b_o / (b_o - b_f), and the first edge by t (ties: lower k) is taken, at distance t in
   pixels from the occluder's centre.  It contributes only when it is steeper than 45 degrees for a horizontal pair
   (|a| > |b| with a = w2 Y1 - w1 Y2, b = w1 X2 - w2 X1 for the edge between corners 1 and 2) or not for a vertical
   pair, and when it is a silhouette edge: a boundary or non-manifold edge (not exactly two half-edges) or one whose
   neighbour across has another facing in this view.  Then the far pixel's weight is t - 1/2 when t > 1/2, and the
   occluder's 1/2 - t when t < 1/2.  The edge opposite corner k is half-edge (k + 1) mod 3 of the face, the half-edge
   from corner k to corner k + 1 being half-edge k.  Depth and face_id are not antialiased.
"""
import numpy as np

F32 = np.float32
GUARD = F32(8192.0)
SUB = F32(256.0)
TILE = 8
NOKEY = np.uint64(0xFFFFFFFFFFFFFFFF)


def fkey(x):
    """Order-preserving uint32 key of float32 values (mesh_common.cuh's fkey)."""
    u = np.asarray(x, F32).view(np.uint32)
    return np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def homogeneous(vertices, M, H, W):
    """-> X, Y, w float32 [V] of every vertex under the row-major clip matrix M."""
    x, y, z = (vertices[:, k].astype(F32) for k in range(3))
    M = np.asarray(M, F32)
    cx = ((M[0, 0] * x + M[0, 1] * y) + M[0, 2] * z) + M[0, 3]
    cy = ((M[1, 0] * x + M[1, 1] * y) + M[1, 2] * z) + M[1, 3]
    cw = ((M[3, 0] * x + M[3, 1] * y) + M[3, 2] * z) + M[3, 3]
    hw, hh = F32(0.5) * F32(W), F32(0.5) * F32(H)
    return (cx + cw) * hw, (cy + cw) * hh, cw


def _plane_dist(p, X, Y, w, near, gx, gy):
    return (w - near, X + GUARD * w, gx * w - X, Y + GUARD * w, gy * w - Y)[p]


def _clip_polygon(corners, near, gx, gy):
    """Scalar Sutherland-Hodgman of one face's [(X, Y, w)] -> the clipped polygon (may have < 3 corners)."""
    a = list(corners)
    for p in range(5):
        d = [_plane_dist(p, *v, near, gx, gy) for v in a]
        if all(dk >= 0 for dk in d):
            continue
        b = []
        n = len(a)
        for k in range(n):
            k1 = 0 if k + 1 == n else k + 1
            in0, in1 = bool(d[k] >= 0), bool(d[k1] >= 0)
            if len(b) + in0 + (in0 != in1) > 8:  # more than 8 corners: only from alternating signs, culled
                return []
            if in0:
                b.append(a[k])
            if in0 != in1:
                I, O = (a[k], a[k1]) if in0 else (a[k1], a[k])
                di, do = (d[k], d[k1]) if in0 else (d[k1], d[k])
                s = di / (di - do)
                b.append(tuple(I[c] + s * (O[c] - I[c]) for c in range(3)))
        a = b
        if len(a) < 3:
            return []
    return a


def setup(X, Y, w, faces, H, W, near):
    """-> polygons: n int [F] (0: culled), px, py int64 [F, 8] (snapped, positive orientation), box i0, i1, j0, j1,
    and facing int8 [F]."""
    near = F32(near)
    gx, gy = F32(W) + GUARD, F32(H) + GUARD
    F = len(faces)
    tX, tY, tw = X[faces], Y[faces], w[faces]                                 # [F, 3]
    det = (tX[:, 0] * (tY[:, 1] * tw[:, 2] - tw[:, 1] * tY[:, 2]) - tY[:, 0] * (tX[:, 1] * tw[:, 2] - tw[:, 1] * tX[:, 2])) \
        + tw[:, 0] * (tX[:, 1] * tY[:, 2] - tY[:, 1] * tX[:, 2])
    facing = ((det > 0).astype(np.int8) - (det < 0).astype(np.int8))
    inside = np.ones(F, bool)
    for p in range(5):
        inside &= np.all(_plane_dist(p, tX, tY, tw, near, gx, gy) >= 0, axis=1)
    n = np.zeros(F, np.int64)
    px = np.zeros((F, 8), np.int64)
    py = np.zeros((F, 8), np.int64)
    with np.errstate(all="ignore"):
        px[:, :3] = np.rint((tX / tw) * SUB).astype(np.int64)
        py[:, :3] = np.rint((tY / tw) * SUB).astype(np.int64)
    n[inside] = 3
    for f in np.nonzero(~inside)[0]:
        poly = _clip_polygon([(tX[f, k], tY[f, k], tw[f, k]) for k in range(3)], near, gx, gy)
        n[f] = len(poly)
        for k, (pX, pY, pw) in enumerate(poly):
            px[f, k] = int(np.rint((pX / pw) * SUB))
            py[f, k] = int(np.rint((pY / pw) * SUB))
    px[n == 0] = 0
    py[n == 0] = 0
    k = np.arange(8)
    nxt = np.where(k[None, :] + 1 >= n[:, None], 0, k[None, :] + 1)
    live = k[None, :] < n[:, None]
    xn, yn = np.take_along_axis(px, nxt, 1), np.take_along_axis(py, nxt, 1)
    area = np.where(live, px * yn - xn * py, 0).sum(1)
    n[area == 0] = 0
    for f in np.nonzero(area < 0)[0]:
        px[f, :n[f]] = px[f, :n[f]][::-1].copy()
        py[f, :n[f]] = py[f, :n[f]][::-1].copy()
    big, small = np.int64(1 << 40), np.int64(-(1 << 40))
    xmin = np.where(live, px, big).min(1)
    xmax = np.where(live, px, small).max(1)
    ymin = np.where(live, py, big).min(1)
    ymax = np.where(live, py, small).max(1)
    i0 = np.maximum((xmin - 128 + 255) >> 8, 0)
    i1 = np.minimum((xmax - 128) >> 8, W - 1)
    j0 = np.maximum((ymin - 128 + 255) >> 8, 0)
    j1 = np.minimum((ymax - 128) >> 8, H - 1)
    n[(i0 > i1) | (j0 > j1)] = 0
    return dict(n=n, px=px, py=py, i0=i0, i1=i1, j0=j0, j1=j1, facing=facing)


def tile_counts(prim):
    """Tiles of each prim's pixel box (8 x 8, aligned to the box), 0 for culled prims: 1 is the one-thread path."""
    t = ((prim["i1"] - prim["i0"]) // TILE + 1) * ((prim["j1"] - prim["j0"]) // TILE + 1)
    return np.where(prim["n"] > 0, t, 0)


def edge_fns(tX, tY, tw, px, py):
    """Homogeneous edge functions b [.., 3] and their sum d at screen points (px, py), float32."""
    ex = tX - px[..., None] * tw
    ey = tY - py[..., None] * tw
    b0 = ex[..., 1] * ey[..., 2] - ex[..., 2] * ey[..., 1]
    b1 = ex[..., 2] * ey[..., 0] - ex[..., 0] * ey[..., 2]
    b2 = ex[..., 0] * ey[..., 1] - ex[..., 1] * ey[..., 0]
    return np.stack([b0, b1, b2], -1), (b0 + b1) + b2


def _lerp3(u, a):
    return (u[..., 0] * a[..., 0] + u[..., 1] * a[..., 1]) + u[..., 2] * a[..., 2]


def coverage(prim, fids, X, Y, w, faces, H, W):
    """Depth-tested keys uint64 [H * W] of one view (NOKEY: background)."""
    keys = np.full(H * W, NOKEY, np.uint64)
    live = np.nonzero(prim["n"] > 0)[0]
    if len(live) == 0:
        return keys
    bw = prim["i1"][live] - prim["i0"][live] + 1
    bh = prim["j1"][live] - prim["j0"][live] + 1
    cnt = bw * bh
    rep = np.repeat(np.arange(len(live)), cnt)
    local = np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    f = live[rep]
    i = prim["i0"][f] + local % bw[rep]
    j = prim["j0"][f] + local // bw[rep]
    pX, pY = 256 * i + 128, 256 * j + 128
    n = prim["n"][f]
    ok = np.ones(len(f), bool)
    for k in range(8):
        k1 = np.where(k + 1 >= n, 0, k + 1)
        ax, ay = prim["px"][f, k], prim["py"][f, k]
        bx, by = prim["px"][f, k1], prim["py"][f, k1]
        dx, dy = bx - ax, by - ay
        e = dx * (pY - ay) - dy * (pX - ax)
        tl = (dy < 0) | ((dy == 0) & (dx > 0))
        ok &= ~((k < n) & ~((dx == 0) & (dy == 0)) & (e < np.where(tl, 0, 1)))
    f, i, j = f[ok], i[ok], j[ok]
    c = faces[f]
    with np.errstate(all="ignore"):
        b, d = edge_fns(X[c], Y[c], w[c], i.astype(F32) + F32(0.5), j.astype(F32) + F32(0.5))
        good = d != 0
        u = b[good] / d[good][:, None]
    f, i, j, c = f[good], i[good], j[good], c[good]
    depth = _lerp3(u, w[c])
    key = (fkey(depth).astype(np.uint64) << np.uint64(32)) | fids[f].astype(np.uint64)
    np.minimum.at(keys, j * W + i, key)
    return keys


def opposite_faces(faces):
    """int64 [3F]: the face across half-edge 3 f + k (corner k -> k + 1) when its undirected edge has exactly two
    half-edges, else -1."""
    F = len(faces)
    a = faces.reshape(-1)
    b = faces[:, [1, 2, 0]].reshape(-1)
    lo, hi = np.minimum(a, b).astype(np.int64), np.maximum(a, b).astype(np.int64)
    order = np.lexsort((np.arange(3 * F), hi, lo))
    lo, hi = lo[order], hi[order]
    head = np.ones(3 * F, bool)
    head[1:] = (lo[1:] != lo[:-1]) | (hi[1:] != hi[:-1])
    eid = np.cumsum(head) - 1
    count = np.bincount(eid, minlength=eid[-1] + 1 if len(eid) else 0)
    opp = np.full(3 * F, -1, np.int64)
    two = np.nonzero(count[eid] == 2)[0]
    first = two[head[two]]
    opp[order[first]] = order[first + 1] // 3
    opp[order[first + 1]] = order[first] // 3
    return opp


def _aa_weight(kp, kq, ip, jp, iq, jq, horizontal, X, Y, w, faces, opp, facing):
    """Vectorised pair weight of the pixels p (self) from their pairs with q, as in 4."""
    self_occ = kp < kq
    ko = np.where(self_occ, kp, kq)
    f = (ko & np.uint64(0xFFFFFFFF)).astype(np.int64)
    ci, cj = np.where(self_occ, ip, iq), np.where(self_occ, jp, jq)
    fi, fj = np.where(self_occ, iq, ip), np.where(self_occ, jq, jp)
    c = faces[f]
    tX, tY, tw = X[c], Y[c], w[c]
    bo, d = edge_fns(tX, tY, tw, ci.astype(F32) + F32(0.5), cj.astype(F32) + F32(0.5))
    bf, _ = edge_fns(tX, tY, tw, fi.astype(F32) + F32(0.5), fj.astype(F32) + F32(0.5))
    ke = np.full(len(f), -1)
    te = np.zeros(len(f), F32)
    pos = d > 0
    with np.errstate(all="ignore"):
        for k in range(3):
            out_f = np.where(pos, bf[:, k] < 0, bf[:, k] > 0)
            in_o = np.where(pos, bo[:, k] >= 0, bo[:, k] <= 0)
            tk = bo[:, k] / (bo[:, k] - bf[:, k])
            take = out_f & in_o & ((ke < 0) | (tk < te))
            ke = np.where(take, k, ke)
            te = np.where(take, tk, te)
    found = ke >= 0
    kk = np.maximum(ke, 0)
    r = np.arange(len(f))
    p1, p2 = (kk + 1) % 3, (kk + 2) % 3
    a = tw[r, p2] * tY[r, p1] - tw[r, p1] * tY[r, p2]
    b = tw[r, p1] * tX[r, p2] - tw[r, p2] * tX[r, p1]
    cls = (np.abs(a) > np.abs(b)) == horizontal
    nb = opp[3 * f + p1]
    sil = (nb < 0) | (facing[np.maximum(nb, 0)] != facing[f])
    wgt = np.where(self_occ, np.where(te < F32(0.5), F32(0.5) - te, F32(0)),
                   np.where(te > F32(0.5), te - F32(0.5), F32(0)))
    return np.where(found & cls & sil, wgt, F32(0)).astype(F32)


def render(vertices, faces, clip, H, W, near=0.01, normals=None, colors=None, normal_bg=(0, 0, 0), color_bg=(0, 0, 0),
           with_bary=False):
    """dgs_mesh_render's outputs for every view -> dict(face_id int32 [v, H, W], depth, alpha fp32 [v, H, W], normal
    [v, H, W, 3] when normals are given, rgb [v, H, W, 3] when colors are given, tiles int64 [v, F] (the tile count of
    each (view, face), 0 when culled); with_bary also bary [v, H, W, 3], the winning face's u (0 on background)."""
    vertices = np.asarray(vertices, F32).reshape(-1, 3)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    clip = np.asarray(clip, F32).reshape(-1, 4, 4)
    V, F, nv = len(vertices), len(faces), len(clip)
    if F and (faces.min() < 0 or faces.max() >= V):
        raise ValueError("face index out of range")
    opp = opposite_faces(faces) if F else np.zeros(0, np.int64)
    fids = np.arange(F, dtype=np.int64)
    nbg, cbg = np.asarray(normal_bg, F32), np.asarray(color_bg, F32)
    out = {k: [] for k in ("face_id", "depth", "alpha", "normal", "rgb", "tiles", "bary")}
    for v in range(nv):
        X, Y, w = homogeneous(vertices, clip[v], H, W)
        prim = setup(X, Y, w, faces, H, W, near)
        out["tiles"].append(tile_counts(prim))
        keys = coverage(prim, fids, X, Y, w, faces, H, W)
        fg = keys != NOKEY
        pix = np.nonzero(fg)[0]
        fid = np.full(H * W, -1, np.int64)
        fid[pix] = (keys[pix] & np.uint64(0xFFFFFFFF)).astype(np.int64)
        c = faces[fid[pix]]
        jj, ii = pix // W, pix % W
        b, d = edge_fns(X[c], Y[c], w[c], ii.astype(F32) + F32(0.5), jj.astype(F32) + F32(0.5))
        u = b / d[:, None]
        depth = np.zeros(H * W, F32)
        depth[pix] = _lerp3(u, w[c])
        pre = np.empty((H * W, 6), F32)
        pre[:, :3] = nbg
        pre[:, 3:] = cbg
        if normals is not None:
            N = np.asarray(normals, F32)
            nn = np.stack([_lerp3(u, N[c][..., k]) for k in range(3)], -1)
            ln = np.sqrt((nn[:, 0] * nn[:, 0] + nn[:, 1] * nn[:, 1]) + nn[:, 2] * nn[:, 2])
            with np.errstate(all="ignore"):
                pre[pix, :3] = np.where(ln[:, None] > 0, nn / ln[:, None], F32(0))
        if colors is not None:
            Cc = np.asarray(colors, F32)
            pre[pix, 3:] = np.stack([_lerp3(u, Cc[c][..., k]) for k in range(3)], -1)
        a0 = fg.astype(F32)
        acc = np.concatenate([a0[:, None], pre], 1)
        vals = acc.copy()
        jg, ig = np.divmod(np.arange(H * W), W)
        for s, (di, dj) in enumerate(((-1, 0), (1, 0), (0, -1), (0, 1))):
            qi, qj = ig + di, jg + dj
            valid = (qi >= 0) & (qi < W) & (qj >= 0) & (qj < H)
            p = np.nonzero(valid)[0]
            q = qj[p] * W + qi[p]
            diff = (keys[p] & np.uint64(0xFFFFFFFF)) != (keys[q] & np.uint64(0xFFFFFFFF))
            p, q = p[diff], q[diff]
            if len(p) == 0:
                continue
            wgt = _aa_weight(keys[p], keys[q], ig[p], jg[p], ig[q], jg[q], s < 2, X, Y, w, faces, opp,
                             prim["facing"])
            nz = wgt != 0
            p, q, wgt = p[nz], q[nz], wgt[nz]
            acc[p] = acc[p] + wgt[:, None] * (vals[q] - vals[p])
        out["face_id"].append(fid.astype(np.int32).reshape(H, W))
        out["depth"].append(depth.reshape(H, W))
        out["alpha"].append(acc[:, 0].reshape(H, W))
        out["normal"].append(acc[:, 1:4].reshape(H, W, 3))
        out["rgb"].append(acc[:, 4:7].reshape(H, W, 3))
        bary = np.zeros((H * W, 3), F32)
        bary[pix] = u
        out["bary"].append(bary.reshape(H, W, 3))
    res = {k: np.stack(out[k]) if nv else np.zeros((0, H, W) + ((3,) if k in ("normal", "rgb", "bary") else ()),
                                                    np.int32 if k == "face_id" else F32)
           for k in ("face_id", "depth", "alpha", "normal", "rgb", "bary")}
    res["tiles"] = np.stack(out["tiles"]) if nv else np.zeros((0, F), np.int64)
    if normals is None:
        del res["normal"]
    if colors is None:
        del res["rgb"]
    if not with_bary:
        del res["bary"]
    return res
