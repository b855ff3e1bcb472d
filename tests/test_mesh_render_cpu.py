"""oracle/mesh_render.py against geometry, without a GPU: exact coverage of shared edges, no cracks in closed meshes,
depth and barycentrics against fp64 ray casting (near-plane clipping included), the antialiased area of straight
edges, untouched interior edges, cameras that line up with the Gaussian rasterizer's and the reference's, and the
argument checks."""
import ctypes

import numpy as np
import pytest
import torch
from scipy.spatial import ConvexHull, Delaunay

from mesh_render_cases import icosphere, look_at
from oracle import mesh as omesh
from oracle import mesh_render as om
from oracle import renderer as orr


def _screen_clip(W, H):
    """A clip matrix under which world (x, y) is the screen position in pixels (w = 1, depth 1)"""
    M = np.zeros((4, 4), np.float32)
    M[0, 0], M[0, 3] = 2.0 / W, -1.0
    M[1, 1], M[1, 3] = 2.0 / H, -1.0
    M[3, 3] = 1.0
    return M[None]


def _opencv_clip(c2w, K, h, w):
    from dgs_b200 import mesh_render as mr
    return mr.clip_from_opencv(np.asarray(c2w)[None], np.asarray(K, np.float64)[None], h, w).numpy()


@pytest.mark.parametrize("seed", range(6))
def test_shared_edge_is_covered_exactly_once(seed):
    rng = np.random.default_rng(seed)
    H, W = 48, 64
    c = np.array([W / 2, H / 2])
    a = rng.uniform(0, 2 * np.pi)
    d = np.array([np.cos(a), np.sin(a)]) * rng.uniform(10, 20)
    p = c + d, c - d  # the shared edge, through the image centre at any angle
    side = np.array([-d[1], d[0]]) / np.linalg.norm(d) * rng.uniform(5, 15)
    q = c + side + rng.normal(0, 3, 2), c - side + rng.normal(0, 3, 2)
    v = np.array([[*p[0], 0], [*p[1], 0], [*q[0], 0], [*q[1], 0]], np.float32)
    if seed % 2:  # snap the shared edge to pixel centres, so centres lie exactly on it
        v[:2, :2] = np.floor(v[:2, :2]) + 0.5
    f = np.array([[0, 1, 2], [1, 0, 3]])
    clip = _screen_clip(W, H)
    both = om.render(v, f, clip, H, W)["face_id"][0]
    one = [om.render(v, f[k:k + 1], clip, H, W)["face_id"][0] >= 0 for k in range(2)]
    assert not (one[0] & one[1]).any()
    assert np.array_equal(one[0] | one[1], both >= 0)
    assert np.array_equal(both == 0, one[0]) and np.array_equal(both == 1, one[1])


def test_centre_on_a_shared_edge_goes_to_the_top_left_owner():
    H, W = 16, 16
    v = np.array([[8.5, 2, 0], [8.5, 14, 0], [3, 8, 0], [14, 8, 0]], np.float32)  # vertical edge through centres x=8.5
    f = np.array([[0, 1, 2], [1, 0, 3]])  # face 0 to the left of the edge, face 1 to the right
    fid = om.render(v, f, _screen_clip(W, H), H, W)["face_id"][0]
    rows = np.arange(3, 14)
    assert (fid[rows, 8] == 1).all()  # the edge is face 1's left edge
    h = np.array([[2, 8.5, 0], [14, 8.5, 0], [8, 3, 0], [8, 14, 0]], np.float32)  # horizontal edge through y=8.5
    fid = om.render(h, np.array([[0, 1, 2], [1, 0, 3]]), _screen_clip(W, H), H, W)["face_id"][0]
    assert (fid[8, 3:14] == 1).all()  # face 1 lies below: the edge is its top edge


def _mc_sphere():
    n = 20
    x = np.arange(n, dtype=np.float32) - (n - 1) / 2
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    v, f = omesh.marching_cubes(7.0 - np.sqrt(X * X + 1.4 * Y * Y + 0.7 * Z * Z) + np.sin(0.5 * X), 0.0)
    return (np.asarray(v, np.float32) / (n - 1) * 2 - 1).astype(np.float32), np.asarray(f, np.int64)


@pytest.mark.parametrize("shape", ["icosphere", "marching_cubes"])
def test_closed_meshes_have_no_cracks(shape):
    from dgs_b200.cameras import get_turntable_cameras
    v, f = icosphere(3) if shape == "icosphere" else _mc_sphere()
    H, W = 64, 96
    _, _, _, K, c2w = get_turntable_cameras(num_views=4, w=W, h=H, radius=2.5, elevation=25)
    for c, k in zip(c2w, K):
        clip = _opencv_clip(c, k, H, W)
        fid = om.render(v, f, clip, H, W)["face_id"][0]
        X, Y, w = om.homogeneous(v, clip[0], H, W)
        pts = np.stack([X / w, Y / w], 1).astype(np.float64)
        hull = Delaunay(pts[ConvexHull(pts).vertices]) if shape == "icosphere" else None
        jj, ii = np.mgrid[0:H, 0:W]
        centres = np.stack([ii.ravel() + 0.5, jj.ravel() + 0.5], 1)
        if hull is not None:
            inside = hull.find_simplex(centres) >= 0
        else:  # a non-convex silhouette: the filled outline of the covered pixels' 4-connected interior
            from scipy.ndimage import binary_fill_holes
            inside = binary_fill_holes(fid >= 0).ravel()
        assert (fid.ravel()[inside] >= 0).all(), f"{int((fid.ravel()[inside] < 0).sum())} holes"


def _ray_cast(v, f, c2w, K, i, j):
    """fp64: the first hit of the ray through pixel centre (i, j) -> (view z, point) or None"""
    fx, fy, cx, cy = K
    d = c2w[:3, :3] @ np.array([(i + 0.5 - cx) / fx, (j + 0.5 - cy) / fy, 1.0])
    o = c2w[:3, 3]
    best = None
    for a, b, c in v[f].astype(np.float64):
        e1, e2 = b - a, c - a
        p = np.cross(d, e2)
        det = e1 @ p
        if abs(det) < 1e-15:
            continue
        s = o - a
        u = s @ p / det
        q = np.cross(s, e1)
        vv = d @ q / det
        t = e2 @ q / det
        if u >= -1e-9 and vv >= -1e-9 and u + vv <= 1 + 1e-9 and t > 0 and (best is None or t < best[0]):
            best = (t, o + t * d)
    return best


# fp32 bound: the clip transform and the edge functions round a few times at the magnitude of the coordinates, and
# the barycentrics' quotient amplifies it by at most the ratio of the triangle's size to the pixel's distance from
# its edges; 1e-4 of the depth covers the scenes here with a margin of about 10.
DEPTH_REL = 1e-4


@pytest.mark.parametrize("scene", ["sphere", "floor"])
def test_depth_and_barycentrics_match_fp64_ray_casting(scene):
    H, W = 40, 56
    K = np.array([40.0, 42.0, 27.0, 21.5])
    if scene == "sphere":
        v, f = icosphere(2)
        c2w = look_at((1.9, -0.8, 0.7), (0.1, 0.0, 0.0))
    else:  # a floor plane z = -0.5 running behind the camera: the near plane clips it
        g = np.linspace(-6, 6, 7)
        X, Y = np.meshgrid(g, g, indexing="ij")
        v = np.stack([X.ravel(), Y.ravel(), np.full(X.size, -0.5)], 1).astype(np.float32)
        a = (np.arange(6)[:, None] * 7 + np.arange(6)[None, :]).ravel()
        f = np.concatenate([np.stack([a, a + 7, a + 1], 1), np.stack([a + 1, a + 7, a + 8], 1)])
        c2w = look_at((0.2, 0.1, 0.0), (3.0, 0.6, -0.6))
    out = om.render(v, f, _opencv_clip(c2w, K, H, W), H, W, with_bary=True)
    fid, depth, bary = out["face_id"][0], out["depth"][0], out["bary"][0]
    assert (fid >= 0).any() and (fid < 0).any()
    worst = 0.0
    for j in range(H):
        for i in range(W):
            hit = _ray_cast(v, f, c2w, K, i, j)
            if fid[j, i] < 0:
                continue
            assert hit is not None, (i, j)
            z = (np.linalg.inv(c2w) @ np.append(hit[1], 1.0))[2]
            assert z > 0
            p = (bary[j, i, :, None].astype(np.float64) * v[f[fid[j, i]]]).sum(0)
            worst = max(worst, abs(depth[j, i] - z) / z, np.linalg.norm(p - hit[1]) / z)
    print(f"{scene}: worst relative depth / position error {worst:.2e}")
    assert worst < DEPTH_REL


def _crossings(P, c, axis):
    """The boundary of the convex polygon P [n, 2] along the line {axis} = c -> ((low, edge), (high, edge)) of the two
    crossings, each with the edge's direction, or None"""
    hits = []
    for k in range(len(P)):
        a, b = P[k], P[(k + 1) % len(P)]
        if (a[axis] - c) * (b[axis] - c) < 0:
            s = (c - a[axis]) / (b[axis] - a[axis])
            hits.append((a[1 - axis] + s * (b[1 - axis] - a[1 - axis]), b - a))
    return sorted(hits, key=lambda h: h[0]) if len(hits) == 2 else None


def _exact_lines(P, alpha, axis, margin=3.0):
    """(line sum of alpha, exact chord length) of every row (axis 1) or column (axis 0) whose two boundary crossings are
    on edges steeper than 45 degrees from the line's direction (by a margin) and whose strip lies more than `margin`
    pixels from every corner.  Across such a strip each edge stays within the pixel pair that straddles its crossing
    at the strip's centre, and the pair's antialiased alpha sums to the covered length of the pair exactly, so the
    line's sum is the chord at the strip's centre (the covered area of a strip cut by two straight lines)."""
    out = []
    for j in range(alpha.shape[1 - axis]):
        c = j + 0.5
        if np.abs(P[:, axis] - c).min() <= margin + 0.5:
            continue
        hit = _crossings(P, c, axis)
        if hit is None or any(abs(d[1 - axis]) >= 0.9 * abs(d[axis]) for _, d in hit):
            continue
        line = alpha[j] if axis == 1 else alpha[:, j]
        out.append((float(line.astype(np.float64).sum()), hit[1][0] - hit[0][0]))
    return out


@pytest.mark.parametrize("seed", range(4))
def test_antialiased_lines_sum_to_the_exact_chord(seed):
    """Rows crossed by two steep edges and columns crossed by two shallow ones, away from corners, sum to the exact
    chord of the polygon to fp32 rounding; hard coverage (the same pixels without antialiasing) misses it by up to a
    pixel per edge.  The corners sit on the 1/256-pixel grid, so snapping does not move the edges."""
    H, W = 64, 128  # powers of two: the screen clip matrix maps x to X without rounding
    rng = np.random.default_rng(seed)
    c = np.array([64.0, 32.0])
    ang = np.sort(rng.uniform(0, 2 * np.pi, 6))
    r = rng.uniform(18, 29, 6)
    pts = np.round((c + np.stack([r * np.cos(ang) * 1.8, r * np.sin(ang)], 1)) * 256) / 256
    P = pts[ConvexHull(pts).vertices]
    n = len(P)
    ctr = np.round(P.mean(0) * 256) / 256
    v = np.concatenate([np.c_[P, np.zeros(n)], [[*ctr, 0]]]).astype(np.float32)
    f = np.array([[n, k, (k + 1) % n] for k in range(n)])
    out = om.render(v, f, _screen_clip(W, H), H, W)
    alpha, hard = out["alpha"][0], (out["face_id"][0] >= 0).astype(np.float32)
    lines = _exact_lines(P, alpha, 1) + _exact_lines(P, alpha, 0)
    hard_lines = _exact_lines(P, hard, 1) + _exact_lines(P, hard, 0)
    err = np.array([abs(s - L) for s, L in lines])
    hard_err = np.array([abs(s - L) for s, L in hard_lines])
    print(f"{n} corners: {len(lines)} lines, antialiased error max {err.max():.2e}, hard coverage error max "
          f"{hard_err.max():.3f} mean {hard_err.mean():.3f}")
    assert len(lines) >= 12
    assert err.max() < 1e-4
    assert (hard_err > 1e-2).mean() > 0.5  # without antialiasing most of these lines miss


def test_interior_edges_are_not_antialiased():
    """Every pair of neighbouring pixels on two different faces of a closed convex mesh gets weight 0: no edge between
    front-facing neighbours is a silhouette edge.  The silhouette itself is antialiased."""
    from dgs_b200.cameras import get_turntable_cameras
    v, f = icosphere(3)
    H, W = 64, 96
    _, _, _, K, c2w = get_turntable_cameras(num_views=3, w=W, h=H, radius=2.4, elevation=30)
    opp = om.opposite_faces(f)
    for c, k in zip(c2w, K):
        clip = _opencv_clip(c, k, H, W)
        out = om.render(v, f, clip, H, W)
        fid, depth = out["face_id"][0], out["depth"][0]
        key = (om.fkey(depth).astype(np.uint64) << np.uint64(32)) | fid.astype(np.uint32).astype(np.uint64)
        X, Y, w = om.homogeneous(v, clip[0], H, W)
        facing = om.setup(X, Y, w, f, H, W, 0.01)["facing"]
        jj, ii = np.mgrid[0:H, 0:W]
        pairs = 0
        for horizontal, (a, b) in ((True, (np.s_[:, :-1], np.s_[:, 1:])), (False, (np.s_[:-1, :], np.s_[1:, :]))):
            sel = (fid[a] >= 0) & (fid[b] >= 0) & (fid[a] != fid[b])
            pairs += int(sel.sum())
            for p, q in ((a, b), (b, a)):
                wgt = om._aa_weight(key[p][sel], key[q][sel], ii[p][sel], jj[p][sel], ii[q][sel], jj[q][sel],
                                    horizontal, X, Y, w, f, opp, facing)
                assert (wgt == 0).all()
        assert pairs > 300
        assert ((out["alpha"][0] > 0) & (out["alpha"][0] < 1)).any()


def test_cameras_line_up_with_the_gaussian_rasterizer():
    from dgs_b200 import mesh_render as mr
    rng = np.random.default_rng(0)
    H, W = 90, 130
    c2w = look_at((2.0, -1.0, 0.8), (0.2, 0.1, 0.0))
    K = np.array([110.0, 105.0, 60.0, 47.0])
    _, proj, _, _, _ = orr.build_camera(torch.tensor(c2w, dtype=torch.float32), torch.tensor(K), H, W)
    M = mr.clip_from_opencv(c2w[None], K[None], H, W).numpy()[0]
    for p in rng.normal(0, 0.4, (20, 3)):
        ph = torch.tensor([*p, 1.0], dtype=torch.float32) @ proj  # the rasterizer's p_hom = p^T (P W2C)^T
        gx = ((ph[0] / ph[3] + 1) * W - 1) / 2  # ndc2Pix: pixel-centre coordinates
        gy = ((ph[1] / ph[3] + 1) * H - 1) / 2
        X, Y, w = om.homogeneous(p[None].astype(np.float32), M, H, W)
        assert abs(float(X[0] / w[0]) - 0.5 - float(gx)) < 1e-3 and abs(float(Y[0] / w[0]) - 0.5 - float(gy)) < 1e-3


def test_reference_drop_in_puts_up_at_the_top():
    from dgs_b200 import mesh_render as mr
    c2w, K = mr.get_camera("cpu", 64, 5, 12)
    clip = mr.clip_from_opengl(c2w, K).numpy()
    tri = np.array([[-0.1, 0.5, 0.0], [0.1, 0.5, 0.0], [0.0, 0.7, 0.0]], np.float32)  # above the optical axis (+y)
    fid = om.render(tri, np.array([[0, 1, 2]]), clip[:1], 64, 64)["face_id"][0]
    rows = np.nonzero((fid >= 0).any(1))[0]
    assert len(rows) and rows.max() < 32


def test_empty_zero_views_and_bad_input():
    v, f = icosphere(1)
    clip = _screen_clip(32, 24)
    out = om.render(v, f[:0], clip, 24, 32, normals=v, colors=v, normal_bg=(0, 0, 1), color_bg=(1, 1, 1))
    assert (out["face_id"] == -1).all() and (out["alpha"] == 0).all() and (out["rgb"] == 1).all()
    assert (out["normal"] == np.float32([0, 0, 1])).all()
    assert om.render(v, f, clip[:0], 24, 32)["face_id"].shape == (0, 24, 32)
    with pytest.raises(ValueError):
        om.render(v, np.array([[0, 1, len(v)]]), clip, 24, 32)


def test_python_argument_checks():
    from dgs_b200 import mesh_render as mr
    v, f = icosphere(1)
    with pytest.raises(ValueError, match="expected vertices"):
        mr.render_clip(v[:, :2], f, _screen_clip(8, 8), 8, 8)
    with pytest.raises(ValueError, match="clip matrices"):
        mr.render_clip(v, f, np.zeros((2, 3, 4), np.float32), 8, 8)
    with pytest.raises(TypeError):
        mr.render_clip(v, f.astype(np.float32), _screen_clip(8, 8), 8, 8)


def test_c_entry_rejects_bad_arguments_before_any_device_work():
    from dgs_b200 import _lib
    L = _lib.lib()
    fake = ctypes.c_void_p(256)
    alloc = _lib.ALLOC_FN(lambda n, u: None)

    def call(V=3, F=1, views=1, H=8, W=8, near=0.01, normals=None, colors=None, out_normal=None, out_rgb=None,
             clip=fake):
        return L.dgs_mesh_render(fake, V, fake, F, normals, colors, clip, views, H, W, near, None, None, 1 << 20,
                                 None, None, None, out_normal, out_rgb, alloc, None, None)
    for kw, msg in [(dict(F=-1), b"negative"), (dict(views=-1), b"n_views"), (dict(H=0), b"H and W"),
                    (dict(W=8193), b"H and W"), (dict(near=0.0), b"near"), (dict(clip=None), b"clip"),
                    (dict(out_normal=fake), b"normal map"), (dict(out_rgb=fake), b"colour map")]:
        assert call(**kw) == 1, kw
        assert msg in L.dgs_last_error(), (kw, L.dgs_last_error())
    assert call(views=0) == 0  # nothing to draw: no device work
