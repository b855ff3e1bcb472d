"""Vertex colours on the H100 (dgs_mesh_vertex_colors): normals bit for bit against the numpy oracle on marching-cubes,
cleaned, remeshed and decimated meshes; colours against the oracle over SH degrees, scaling modifiers and grids; the
convex-hull property; determinism and vertex-order independence; block boundaries; extract_mesh(vertex_colors=True) end
to end."""
import numpy as np
import pytest
import torch

from mesh_shapes import cuda_grid, mc, shell_model
from oracle import mesh_color as oc

pytestmark = pytest.mark.gpu

COLOR_TOL = 1e-4  # fp32 sums in list order against fp64


def _with_features(m, deg, seed, dc=None):
    """m with SH features of degree deg: random (or the given DC) coefficients, the rest random"""
    from dgs_b200.renderer import GaussianModel
    P = m._xyz.shape[0]
    g = torch.Generator().manual_seed(seed)
    f = torch.randn(P, (deg + 1) ** 2, 3, generator=g) * 0.6
    if dc is not None:
        f[:, 0] = torch.as_tensor(dc, dtype=torch.float32)
    out = GaussianModel(deg, m.scaling_modifier)
    out.set_data(m._xyz, f.cuda(), m._scaling, m._rotation, m._opacity)
    return out


def _colors(m, v, f, R, nb, stats=None):
    from dgs_b200 import mesh
    return mesh.vertex_colors(m._xyz, m.get_features, m._scaling, m._rotation, m._opacity, v, f, m.mesh_center,
                              m.mesh_scale, m.scaling_modifier, R, nb, stats=stats)


def _oracle(m, v, f, R, nb, subset=None):
    return oc.vertex_colors(*(t.cpu().numpy() for t in (m._xyz, m.get_features, m._scaling, m._rotation, m._opacity)),
                            v, f, R, nb, scaling_modifier=m.scaling_modifier, subset=subset, device="cuda")


def _no_gaussians():
    return (torch.zeros(0, 3, device="cuda"), torch.zeros(0, 1, 3, device="cuda"), torch.zeros(0, 3, device="cuda"),
            torch.zeros(0, 4, device="cuda"), torch.zeros(0, 1, device="cuda"))


def _normals(v, f):
    from dgs_b200 import mesh
    stats = {}
    rgb, n = mesh.vertex_colors(*_no_gaussians(), v, f, np.zeros(3, np.float32), 1.0, stats=stats)
    assert stats["unweighted"] == len(v) and (rgb == 1).all()
    return n


def test_normals_match_oracle_bitwise_and_point_out():
    from dgs_b200 import mesh
    n_grid, r = 96, 30.0
    X, Y, Z = cuda_grid(n_grid)
    v, f = mc((r - torch.sqrt(X * X + Y * Y + Z * Z)).contiguous())
    c = np.float32((n_grid - 1) / 2)
    passes = {"mc": (v, f)}
    passes["clean"] = mesh.clean(v, f)
    passes["remesh"] = mesh.remesh(*passes["clean"], 2.0)
    passes["decimate"] = mesh.decimate(*passes["clean"], len(passes["clean"][1]) // 4)
    for name, (pv, pf) in passes.items():
        n = _normals(pv, pf)
        ref = oc.normals(pv, pf)
        assert np.array_equal(n, ref), f"{name}: {(n != ref).any(1).sum()} normals differ"
        used = np.unique(pf)
        dots = np.einsum("ij,ij->i", n[used], pv[used] - c)
        print(f"sphere {name}: {len(pv)} vertices, {len(pf)} faces, min n.p {dots.min():.3f}")
        assert (dots > 0).all() and np.allclose(np.linalg.norm(n[used], axis=1), 1, atol=1e-6)
    # the shell's own surface, raw and after the reference's whole chain
    m = shell_model(60000, 3)
    raw = m.extract_mesh(resolution=128)
    chain = mesh.clean_remesh_then_decimate(raw.vertices, raw.faces, 20000)
    for name, (pv, pf) in {"shell mc": (raw.vertices, raw.faces), "shell chain": chain}.items():
        assert np.array_equal(_normals(pv, pf), oc.normals(pv, pf)), name


@pytest.mark.parametrize("grid", [(64, 16), (128, 32), (256, 64)], ids=lambda g: f"r{g[0]}_b{g[1]}")
@pytest.mark.parametrize("smod", [None, 0.8])
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_colors_match_oracle(deg, smod, grid):
    from dgs_b200 import mesh
    R, nb = grid
    m = _with_features(shell_model(40000, 5 + deg), deg, deg)
    m.scaling_modifier = smod
    occ = m.extract_fields(R, nb)
    raw = mesh.extract_mesh(occ, 0.005, R)
    v, f = raw.vertices, raw.faces
    assert len(f) > 1000
    stats = {}
    rgb, n = _colors(m, v, f, R, nb, stats)
    subset = None
    if len(v) > 20000:
        subset = np.sort(np.random.default_rng(deg).choice(len(v), 20000, replace=False))
    o = _oracle(m, v, f, R, nb, subset)
    idx = np.arange(len(v)) if subset is None else subset
    assert np.array_equal(n, o["normals"])
    # white is the colour of an unweighted vertex; a weighted one is white only where the oracle's colour is (err)
    assert (rgb[idx][o["unweighted"]] == 1).all()
    err = float(np.abs(rgb[idx] - o["rgb"]).max())
    print(f"degree {deg}, smod {smod}, {R} / {nb}: {len(v)} vertices ({len(idx)} checked), {stats['unweighted']} "
          f"white, max |rgb - oracle| {err:.2e}")
    assert err <= COLOR_TOL
    if subset is None:
        assert stats["unweighted"] == int(o["unweighted"].sum())


def test_convex_hull_of_the_gaussian_colours():
    m = _with_features(shell_model(30000, 8, floaters=False), 3, 9)
    m.extract_fields(128, 32)
    rng = np.random.default_rng(4)
    d = rng.normal(0, 1, (20000, 3))
    xyz_n = ((m._xyz.cpu().numpy() - m.mesh_center.cpu().numpy()) * np.float32(m.mesh_scale))
    radius = np.linalg.norm(xyz_n, axis=1).mean()
    v = (d / np.linalg.norm(d, axis=1, keepdims=True) * radius * rng.uniform(0.9, 1.1, (20000, 1))).astype(np.float32)
    f = rng.integers(0, len(v), (30000, 3))
    rgb, _ = _colors(m, v, f, 128, 32)
    o = _oracle(m, v, f, 128, 32)
    ok = ~o["unweighted"]
    lo, hi = np.minimum(o["cmin"][ok], 1.0), np.minimum(o["cmax"][ok], 1.0)
    below, above = float((lo - rgb[ok]).max()), float((rgb[ok] - hi).max())
    print(f"convex hull: {ok.sum()} weighted of {len(v)}, worst excess below {below:.2e}, above {above:.2e}")
    assert ok.sum() > 10000 and below <= 1e-6 and above <= 1e-6


def test_deterministic_and_independent_of_vertex_order():
    from dgs_b200 import mesh
    m = _with_features(shell_model(30000, 6), 2, 1)
    raw = m.extract_mesh(resolution=128)
    v, f = raw.vertices, raw.faces
    a = _colors(m, v, f, 128, 64)
    b = _colors(m, v, f, 128, 64)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    perm = np.random.default_rng(0).permutation(len(v))
    inv = np.empty_like(perm)
    inv[perm] = np.arange(len(v))
    rgb, n = _colors(m, v[perm], inv[f], 128, 64)
    assert np.array_equal(rgb, a[0][perm]) and np.array_equal(n, a[1][perm])
    # CUDA tensors in, CUDA tensors out, the same bits
    rt, nt = mesh.vertex_colors(m._xyz, m.get_features, m._scaling, m._rotation, m._opacity, torch.from_numpy(v).cuda(),
                                torch.from_numpy(f).cuda(), m.mesh_center, m.mesh_scale, None, 128, 64)
    assert rt.is_cuda and np.array_equal(rt.cpu().numpy(), a[0]) and np.array_equal(nt.cpu().numpy(), a[1])


def test_block_boundaries():
    """Vertices on the grid points that start and end blocks, one ulp below them, and outside [-1, 1]; two corner
    Gaussians make mesh_center 0 and mesh_scale 1, so the vertices sit where they are placed."""
    R, nb, split = 64, 16, 4
    m = _with_features(shell_model(20000, 1, floaters=False), 1, 2)
    xyz = m._xyz.clone()
    xyz[0], xyz[1] = -0.9, 0.9
    m._xyz = xyz
    m.extract_fields(R, nb)
    assert np.float32(m.mesh_scale) == 1.0 and not m.mesh_center.any()
    lin = torch.linspace(-1, 1, R).numpy()
    edges = np.concatenate([lin[0::split], lin[split - 1::split]])
    vals = np.concatenate([edges, np.nextafter(edges, np.float32(-2)), np.float32([-1.3, -1.0, 1.0, 1.3])])
    rng = np.random.default_rng(5)
    v = rng.choice(vals, (6000, 3)).astype(np.float32)
    f = rng.integers(0, len(v), (8000, 3))
    rgb, n = _colors(m, v, f, R, nb)
    o = _oracle(m, v, f, R, nb)
    err = float(np.abs(rgb - o["rgb"]).max())
    print(f"block boundaries: {int(o['unweighted'].sum())} white of {len(v)}, max |rgb - oracle| {err:.2e}")
    assert (rgb[o["unweighted"]] == 1).all() and err <= COLOR_TOL
    assert np.array_equal(n, o["normals"])


@pytest.fixture(scope="module")
def colored_shell():
    """A shell whose DC colour is 0.5 + 0.4 u (u the Gaussian's unit direction from the centre)"""
    m = shell_model(262146, 11, floaters=False)
    xyz = m._xyz
    u = (xyz - (xyz.amin(0) + xyz.amax(0)) / 2)
    u = u / u.norm(dim=1, keepdim=True)
    return _with_features(m, 0, 0, dc=(0.4 * u / oc.SH_C0).cpu())


@pytest.mark.parametrize("post", [None, "clean_then_decimate", "clean_remesh_then_decimate"])
def test_extract_mesh_with_vertex_colors(colored_shell, post):
    from dgs_b200 import mesh
    m = colored_shell
    pp = getattr(mesh, post) if post else None
    plain = m.extract_mesh(postprocess=pp)
    colored = m.extract_mesh(postprocess=pp, vertex_colors=True)
    assert plain.vertex_colors is None and plain.vertex_normals is None
    assert np.array_equal(plain.vertices, colored.vertices) and np.array_equal(plain.faces, colored.faces)
    rgb, n = colored.vertex_colors, colored.vertex_normals
    assert rgb.shape == colored.vertices.shape and (rgb >= 0).all() and (rgb <= 1).all()
    ln = np.linalg.norm(n, axis=1)
    assert ((np.abs(ln - 1) < 1e-6) | (ln == 0)).all()
    p = colored.vertices.astype(np.float64)
    want = 0.5 + 0.4 * p / np.linalg.norm(p, axis=1, keepdims=True)
    e = np.abs(rgb - want)
    print(f"extract_mesh({post}): {len(p)} vertices, |colour - (0.5 + 0.4 v)| mean {e.mean():.4f} max {e.max():.4f}")
    assert e.mean() < 0.05


def test_no_gaussians_no_faces_and_bad_faces():
    from dgs_b200 import _lib, mesh
    v = np.random.default_rng(0).normal(0, 0.3, (50, 3)).astype(np.float32)
    f = np.array([[0, 1, 2], [2, 1, 3]])
    stats = {}
    rgb, n = mesh.vertex_colors(*_no_gaussians(), v, f, np.zeros(3, np.float32), 1.0, stats=stats)
    assert stats["unweighted"] == 50 and (rgb == 1).all() and np.array_equal(n, oc.normals(v, f))
    m = _with_features(shell_model(5000, 2, floaters=False), 1, 3)
    m.extract_fields(64, 16)
    rgb, n = _colors(m, v, np.zeros((0, 3), np.int64), 64, 16)
    assert not n.any()
    o = _oracle(m, v, np.zeros((0, 3), np.int64), 64, 16)
    assert np.abs(rgb - o["rgb"]).max() <= COLOR_TOL
    e0, _ = _colors(m, np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64), 64, 16)
    assert e0.shape == (0, 3)
    for bad in ([[0, 1, 50]], [[-1, 0, 1]]):
        with pytest.raises(_lib.DgsError, match="outside"):
            _colors(m, v, np.array(bad), 64, 16)


def test_cli_writes_colours_and_normals(tmp_path):
    from dgs_b200 import mesh
    m = _with_features(shell_model(60000, 4, floaters=False), 0, 5)
    ply = m.save_ply(str(tmp_path / "model.ply"))  # zero-padded to degree 3 for the viewers
    out = str(tmp_path / "out.obj")
    mesh.main([ply, out, "--resolution", "128", "--clean", "--remesh", "--decimate-target", "20000", "--colors"])
    lines = open(out).read().splitlines()
    vl = np.float64([l.split()[1:] for l in lines if l.startswith("v ")])
    nl = [l for l in lines if l.startswith("vn ")]
    assert vl.shape[1] == 6 and len(nl) == len(vl) > 1000
    assert (vl[:, 3:] >= 0).all() and (vl[:, 3:] <= 1).all()
    # the file loads at degree 3, and its zero padding leaves the colours of the degree-0 model
    ref = m.extract_mesh(resolution=128, postprocess=lambda v, f, t: mesh._chain(v, f, True, 0.015, t),
                         decimate_target=20000, vertex_colors=True)
    assert np.array_equal(np.float32(vl[:, 3:]), ref.vertex_colors)
