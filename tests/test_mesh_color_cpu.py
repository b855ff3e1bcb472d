"""Vertex colours without a GPU: the numpy oracle (oracle/mesh_color.py) on hand-made cases, Mesh.export with and
without colours and normals, and the argument checks and CLI flags of dgs_b200.mesh."""
import os

import numpy as np
import pytest
import torch

from oracle import mesh_color as oc

SH0 = oc.SH_C0


def _gaussians(xyz, dc, rest=None, log_scale=-3.0, opacity=4.0):
    """Raw arrays of isotropic Gaussians at xyz with DC coefficients dc [P, 3] and optional rest [P, K, 3]"""
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    P = len(xyz)
    f = np.asarray(dc, np.float32).reshape(P, 1, 3)
    if rest is not None:
        f = np.concatenate([f, np.asarray(rest, np.float32)], 1)
    return dict(xyz=xyz, features=f, scaling=np.full((P, 3), log_scale, np.float32),
                rotation=np.tile(np.float32([1, 0, 0, 0]), (P, 1)), opacity=np.full((P, 1), opacity, np.float32))


def _run(g, vertices, faces, R=64, nb=16, **kw):
    return oc.vertex_colors(g["xyz"], g["features"], g["scaling"], g["rotation"], g["opacity"], vertices, faces, R, nb,
                            **kw)


def _cube():
    """The cube [-0.5, 0.5]^3: 8 corners, 12 triangles wound outwards"""
    v = np.array([[x, y, z] for x in (-0.5, 0.5) for y in (-0.5, 0.5) for z in (-0.5, 0.5)], np.float32)
    q = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    f = np.array([t for a, b, c, d in q for t in ((a, b, c), (a, c, d))], np.int64)
    return v, f


def test_cube_normals_point_out_and_follow_the_winding():
    v, f = _cube()
    n = oc.normals(v, f)
    assert np.allclose(np.linalg.norm(n, axis=1), 1, atol=1e-6)
    assert (np.einsum("ij,ij->i", n, v) > 0).all()
    assert np.array_equal(oc.normals(v, f[:, ::-1]), -n)
    # an extra vertex without faces, and one whose faces cancel, get 0
    v2 = np.concatenate([v, [[2, 2, 2], [3, 3, 3]]]).astype(np.float32)
    f2 = np.concatenate([f, [[9, 0, 1], [9, 1, 0]]])
    n2 = oc.normals(v2, f2)
    assert np.array_equal(n2[8], [0, 0, 0]) and np.array_equal(n2[9], [0, 0, 0])


def test_normals_add_faces_in_face_order_in_fp64():
    rng = np.random.default_rng(0)
    v = rng.normal(0, 1, (30, 3)).astype(np.float32)
    f = rng.integers(0, 30, (200, 3))
    n = oc.normals(v, f)
    v64 = v.astype(np.float64)
    for i in (0, 7, 29):
        s = np.zeros(3)
        for t in f:
            for c in t:
                if c == i:
                    a, b, cc = v64[t[0]], v64[t[1]], v64[t[2]]
                    s = s + np.cross(b - a, cc - a)
        ref = (s / np.sqrt(s[0] * s[0] + s[1] * s[1] + s[2] * s[2])).astype(np.float32)
        assert np.array_equal(n[i], ref)


def test_single_gaussian_gives_its_colour_or_white():
    # two faint grey Gaussians at the corners fix the frame (centre 0, scale 1.8 / 1.8 = 1) around one bright one at 0
    dc = np.float32([[0.8, -0.3, -3.0]])
    g = _gaussians([[-0.9, -0.9, -0.9], [0.9, 0.9, 0.9], [0.0, 0.0, 0.0]], np.concatenate([[[0, 0, 0]] * 2, dc]),
                   opacity=np.float32([[-30.0], [-30.0], [4.0]]))
    verts = np.float32([[0.01, 0.0, 0.0], [0.0, 0.02, -0.01], [0.97, 0.97, 0.97], [0.97, -0.97, 0.97]])
    out = _run(g, verts, np.zeros((0, 3), np.int64))
    want = np.maximum(0.5 + SH0 * dc[0].astype(np.float64), 0)
    assert np.allclose(out["rgb"][:2], want, atol=1e-9), out["rgb"]
    assert out["rgb"][0, 2] == 0.0  # the negative channel is clamped at 0
    # the corner block's list holds only the faint corner Gaussian: however small its weight, its colour is taken
    assert out["count"][2] == 1 and not out["unweighted"][2] and np.allclose(out["rgb"][2], 0.5, atol=1e-12)
    # no Gaussian lies near the block of (0.97, -0.97, 0.97): its list is empty and the vertex white
    assert out["count"][3] == 0 and out["unweighted"].tolist() == [False, False, False, True]
    assert np.array_equal(out["rgb"][3], [1, 1, 1])


def test_constant_colour_model():
    rng = np.random.default_rng(1)
    P = 300
    d = rng.normal(0, 1, (P, 3))
    xyz = (0.5 * d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    sh = rng.normal(0, 0.3, (1, 9, 3)).astype(np.float32)
    g = _gaussians(xyz, np.repeat(sh[:, 0], P, 0), np.repeat(sh[:, 1:], P, 0), log_scale=-2.5)
    v, f = _cube()
    v = v * np.float32(0.9)
    out = _run(g, v, f)
    n = oc.normals(v, f)
    want = np.maximum(0.5 + oc.sh_basis(-n, 2) @ sh[0].astype(np.float64), 0).clip(0, 1)
    ok = ~out["unweighted"]
    assert ok.sum() >= 6
    assert np.allclose(out["rgb"][ok], want[ok], atol=1e-12)


def test_vertex_chunks_on_boundaries():
    lin = torch.linspace(-1, 1, 64).numpy()
    split = 4
    p = np.concatenate([lin[[0, 3, 4, 7, 63]], np.nextafter(lin[[4, 8]], np.float32(-2)),
                        np.float32([-1.5, 1.5, np.nan])]).astype(np.float32)
    assert oc.vertex_chunks(p, lin, split).tolist() == [0, 0, 1, 1, 15, 0, 1, 0, 15, 0]


def _old_export(vertices, faces, path):
    """Mesh.export as it was before colours and normals"""
    ext = os.path.splitext(path)[1].lower()
    V, F = len(vertices), len(faces)
    if ext == ".ply":
        header = ("ply\nformat binary_little_endian 1.0\n"
                  f"element vertex {V}\nproperty float x\nproperty float y\nproperty float z\n"
                  f"element face {F}\nproperty list uchar int vertex_indices\nend_header\n")
        face = np.empty(F, dtype=[("n", "u1"), ("v", "<i4", (3,))])
        face["n"], face["v"] = 3, faces
        with open(path, "wb") as fh:
            fh.write(header.encode("ascii"))
            fh.write(vertices.astype("<f4").tobytes())
            fh.write(face.tobytes())
    else:
        with open(path, "w") as fh:
            np.savetxt(fh, vertices, fmt="v %.9g %.9g %.9g")
            np.savetxt(fh, faces + 1, fmt="f %d %d %d")


@pytest.mark.parametrize("ext", [".ply", ".obj"])
def test_export_without_colours_is_unchanged(tmp_path, ext):
    from dgs_b200.mesh import Mesh
    v, f = _cube()
    m = Mesh(v, f)
    a, b = str(tmp_path / ("new" + ext)), str(tmp_path / ("old" + ext))
    m.export(a)
    _old_export(m.vertices, m.faces, b)
    assert open(a, "rb").read() == open(b, "rb").read()


def _read_ply(path):
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    lines = data[:end].decode().splitlines()
    nv = int(next(l for l in lines if l.startswith("element vertex")).split()[-1])
    nf = int(next(l for l in lines if l.startswith("element face")).split()[-1])
    vprops = [l.split() for l in lines[lines.index(f"element vertex {nv}") + 1:] if l.startswith("property")]
    vprops = vprops[:next(i for i, p in enumerate(vprops) if p[1] == "list")]
    dt = np.dtype([(p[2], {"float": "<f4", "uchar": "u1"}[p[1]]) for p in vprops])
    vert = np.frombuffer(data, dt, nv, end)
    face = np.frombuffer(data, [("n", "u1"), ("v", "<i4", (3,))], nf, end + nv * dt.itemsize)
    assert end + nv * dt.itemsize + nf * 13 == len(data)
    return [p[2] for p in vprops], vert, face


def test_export_ply_with_colours_and_normals(tmp_path):
    from dgs_b200.mesh import Mesh
    v, f = _cube()
    rgb = np.linspace(0, 1, 24, dtype=np.float32).reshape(8, 3)
    rgb[0] = [1.0, 0.999, 0.0039]
    n = oc.normals(v, f)
    path = Mesh(v, f, rgb, n).export(str(tmp_path / "m.ply"))
    names, vert, face = _read_ply(path)
    assert names == ["x", "y", "z", "nx", "ny", "nz", "red", "green", "blue"]
    assert np.array_equal(np.stack([vert["x"], vert["y"], vert["z"]], 1), v)
    assert np.array_equal(np.stack([vert["nx"], vert["ny"], vert["nz"]], 1), n)
    q = np.stack([vert["red"], vert["green"], vert["blue"]], 1)
    assert np.array_equal(q, (rgb * 255.0).clip(0, 255).astype(np.uint8)) and q[0].tolist() == [255, 254, 0]
    assert np.array_equal(face["v"], f) and (face["n"] == 3).all()
    names, vert, _ = _read_ply(Mesh(v, f, vertex_colors=rgb).export(str(tmp_path / "c.ply")))
    assert names == ["x", "y", "z", "red", "green", "blue"]


def test_export_obj_with_colours_and_normals(tmp_path):
    from dgs_b200.mesh import Mesh
    v, f = _cube()
    rgb = np.random.default_rng(2).random((8, 3)).astype(np.float32)
    n = oc.normals(v, f)
    lines = open(Mesh(v, f, rgb, n).export(str(tmp_path / "m.obj"))).read().splitlines()
    vl = [l.split() for l in lines if l.startswith("v ")]
    nl = [l.split() for l in lines if l.startswith("vn ")]
    fl = [l.split() for l in lines if l.startswith("f ")]
    assert len(vl) == 8 and len(nl) == 8 and len(fl) == 12 and len(lines) == 28
    assert all(len(x) == 7 for x in vl)
    assert np.array_equal(np.float32([x[1:4] for x in vl]), v) and np.array_equal(np.float32([x[4:] for x in vl]), rgb)
    assert np.array_equal(np.float32([x[1:] for x in nl]), n)
    for x, t in zip(fl, f):
        assert x[1:] == [f"{c + 1}//{c + 1}" for c in t]
    lines = open(Mesh(v, f, rgb).export(str(tmp_path / "c.obj"))).read().splitlines()
    assert lines[8] == "f {} {} {}".format(*(f[0] + 1)) and len(lines[0].split()) == 7


def test_mesh_rejects_wrong_attribute_shapes():
    from dgs_b200.mesh import Mesh
    v, f = _cube()
    with pytest.raises(ValueError, match="vertex_colors"):
        Mesh(v, f, np.zeros((7, 3)))
    with pytest.raises(ValueError, match="vertex_normals"):
        Mesh(v, f, None, np.zeros((8, 2)))


def test_vertex_colors_argument_checks():
    from dgs_b200 import mesh
    v, f = _cube()
    g = _gaussians(np.zeros((5, 3)), np.zeros((5, 3)))
    args = (g["xyz"], g["features"], g["scaling"], g["rotation"], g["opacity"])
    with pytest.raises(TypeError, match="numpy arrays or CUDA tensors"):
        mesh.vertex_colors(*args, torch.from_numpy(v), f, np.zeros(3), 1.0)
    with pytest.raises(ValueError, match=r"vertices \[V, 3\]"):
        mesh.vertex_colors(*args, v[:, :2], f, np.zeros(3), 1.0)
    with pytest.raises(ValueError, match="features"):
        mesh.vertex_colors(g["xyz"], np.zeros((5, 2, 3), np.float32), *args[2:], v, f, np.zeros(3), 1.0)
    with pytest.raises(ValueError, match="features"):
        mesh.vertex_colors(g["xyz"], np.zeros((4, 1, 3), np.float32), *args[2:], v, f, np.zeros(3), 1.0)
    with pytest.raises(ValueError, match="mesh_center"):
        mesh.vertex_colors(*args, v, f, np.zeros(2), 1.0)
    with pytest.raises(ValueError, match="block size"):
        mesh.vertex_colors(*args, v, f, np.zeros(3), 1.0, resolution=100, num_blocks=3)


def test_cli_colors_flag_and_sh_degree_from_the_file(tmp_path):
    from dgs_b200 import mesh, synth
    from dgs_b200.renderer import GaussianModel
    a = mesh.parser().parse_args(["in.ply", "out.obj", "--clean", "--remesh", "--decimate-target", "100000",
                                  "--colors"])
    assert a.colors and a.clean and a.remesh == 0.015 and a.decimate_target == 100000
    assert not mesh.parser().parse_args(["in.ply", "out.obj"]).colors
    g = synth.make_gaussians(50, 0, "trained")
    for deg, viewer, want in [(0, True, 3), (0, False, 0), (2, False, 2), (1, True, 3)]:
        m = GaussianModel(deg)
        feats = np.zeros((50, (deg + 1) ** 2, 3), np.float32)
        feats[:, :1] = g["features"][:, :1]
        m.set_data(*(torch.tensor(x) for x in (g["xyz"], feats, g["scaling"], g["rotation"], g["opacity"])))
        path = m.save_ply(str(tmp_path / f"g{deg}{viewer}.ply"), enable_gs_viewer=viewer)
        assert mesh.ply_sh_degree(path) == want
        loaded = GaussianModel(want).load_ply(path)
        assert loaded.get_features.shape == (50, (want + 1) ** 2, 3)
