"""Mesh extraction without a GPU: the fp64 field oracle against the reference's own extract_fields (fixtures), the
generated marching-cubes table, the numpy marching cubes (closed, oriented, right topology), PLY / OBJ round trips."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from mesh_shapes import closed_and_oriented, euler, grid, volume
from oracle import mesh as om

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "mesh_fields_ref.npz")
GEN = os.path.join(ROOT, "open-diffusiongs_b200", "csrc", "gen_mc_tables.py")
NAMES = ("xyz", "scaling", "rotation", "opacity")
# fixture case -> (resolution, num_blocks, relax_ratio, scaling_modifier), as tests/golden/make_mesh_golden.py
CASES = {"r64_b16": (64, 16, 1.5, None), "r100_b16": (100, 16, 1.5, None), "r64_b16_smod": (64, 16, 1.5, 0.7),
         "r48_b8_relax1": (48, 8, 1.0, None)}


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_field_matches_reference(case):
    z = np.load(GOLDEN)
    R, nb, rr, smod = CASES[case]
    o = om.field(*[torch.from_numpy(z[f"{case}/in/{k}"]) for k in NAMES], resolution=R, num_blocks=nb, relax_ratio=rr,
                 scaling_modifier=smod)
    ref = z[f"{case}/occ"].astype(np.float64)
    rel = np.linalg.norm(o["occ"].numpy() - ref) / np.linalg.norm(ref)
    print(f"{case}: oracle vs reference rel_l2 = {rel:.2e}")
    assert rel <= 1e-6
    assert np.array_equal(o["center"].numpy(), z[f"{case}/mesh_center"])
    assert o["scale"] == float(z[f"{case}/mesh_scale"])


def test_generator_reproduces_committed_header():
    r = subprocess.run([sys.executable, GEN, "--check"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


def test_table_uses_exactly_the_sign_changing_edges():
    edges, ntri, tri = om.load_tables()
    for case in range(256):
        inside = [(case >> c) & 1 for c in range(8)]
        crossing = {e for e in range(12) if inside[edges[e, 0]] != inside[edges[e, 1]]}
        used = [e for e in tri[case, :3 * ntri[case]]]
        assert all(e >= 0 for e in used) and all(e == -1 for e in tri[case, 3 * ntri[case]:])
        assert set(used) == crossing, case
        # each case's triangles form closed oriented loops over the cube: every directed edge has its reverse
        directed = [(t[i], t[(i + 1) % 3]) for t in np.reshape(used, (-1, 3)) for i in range(3)]
        interior = [d for d in directed if (d[1], d[0]) in directed]
        boundary = sorted(set(directed) - set(interior))
        # the boundary (the part on the cube faces) is one cycle per loop: every crossing has in- and out-degree 1
        assert sorted(a for a, _ in boundary) == sorted(crossing) == sorted(b for _, b in boundary)
        # no interior chord lies in a cube face (the neighbouring cube could use the same one)
        faces = [{e for e in range(12) if all(((int(c) >> a) & 1) == s for c in edges[e])} for a in range(3) for s in (0, 1)]
        for a, b in {tuple(sorted(d)) for d in interior}:
            assert not any(a in f and b in f for f in faces), (case, a, b)


@pytest.mark.parametrize("seed", range(4))
def test_numpy_marching_cubes_random_fields_closed(seed):
    rng = np.random.default_rng(seed)
    f = rng.random((40, 33, 27))
    f[0], f[-1], f[:, 0], f[:, -1], f[:, :, 0], f[:, :, -1] = 0, 0, 0, 0, 0, 0  # surface stays inside the grid
    v, t = om.marching_cubes(f, 0.5)
    assert len(t) > 0
    closed_and_oriented(t)


def test_numpy_marching_cubes_sphere_and_torus():
    X, Y, Z = grid(40)
    r = 12.0
    v, t = om.marching_cubes(r - np.sqrt(X ** 2 + Y ** 2 + Z ** 2), 0.0)  # high inside
    closed_and_oriented(t)
    assert euler(t) == 2
    vol = volume(v, t, f64=False)
    assert abs(vol / (4 / 3 * np.pi * r ** 3) - 1) < 0.02  # positive: normals point outwards
    R0, r0 = 11.0, 4.5
    torus = r0 - np.sqrt((np.sqrt(X ** 2 + Y ** 2) - R0) ** 2 + Z ** 2)
    v, t = om.marching_cubes(torus, 0.0)
    closed_and_oriented(t)
    assert euler(t) == 0


def test_ply_roundtrip(tmp_path):
    from dgs_b200 import synth
    from dgs_b200.renderer import GaussianModel
    for deg in (0, 2):
        g = synth.make_gaussians(50, 3, "trained")
        feats = np.random.default_rng(1).normal(0, 1, (50, (deg + 1) ** 2, 3)).astype(np.float32)
        m = GaussianModel(deg).set_data(*[torch.from_numpy(a) for a in (g["xyz"], feats, g["scaling"], g["rotation"],
                                                                         g["opacity"])])
        # the viewer layout pads f_rest to degree 3, which load_ply (like the reference's) only reads back at degree 0 or 3
        path = m.save_ply(str(tmp_path / f"g{deg}.ply"), enable_gs_viewer=deg == 0)
        back = GaussianModel(deg).load_ply(path)
        for k in ("_xyz", "_features_dc", "_scaling", "_rotation", "_opacity"):
            assert torch.equal(getattr(back, k), getattr(m, k)), k
        if deg:
            assert torch.equal(back._features_rest, m._features_rest)
        else:
            assert back._features_rest is None


def test_get_covariance_matches_oracle():
    from dgs_b200 import synth
    from dgs_b200.renderer import GaussianModel
    g = synth.make_gaussians(200, 4, "trained")
    m = GaussianModel(0, scaling_modifier=0.8)
    m.set_data(*[torch.from_numpy(a) for a in (g["xyz"], g["features"], g["scaling"], g["rotation"] * 1.7, g["opacity"])])
    ref = torch.stack(om.covariance6(torch.exp(m._scaling) * 0.8 * 2.0, m._rotation), 1)
    assert torch.equal(m.get_covariance(2.0), ref)


def test_mesh_export_ply_and_obj(tmp_path):
    from dgs_b200.mesh import Mesh
    X, Y, Z = grid(12)
    v, t = om.marching_cubes(4.0 - np.sqrt(X ** 2 + Y ** 2 + Z ** 2), 0.0)
    m = Mesh(v, t)
    assert m.vertices.dtype == np.float32 and m.faces.dtype == np.int64
    p = m.export(str(tmp_path / "m.ply"))
    with open(p, "rb") as f:
        data = f.read()
    head, body = data.split(b"end_header\n", 1)
    assert f"element vertex {len(v)}".encode() in head and f"element face {len(t)}".encode() in head
    V = np.frombuffer(body[:12 * len(v)], "<f4").reshape(-1, 3)
    F = np.frombuffer(body[12 * len(v):], dtype=[("n", "u1"), ("v", "<i4", (3,))])
    assert np.array_equal(V, m.vertices) and (F["n"] == 3).all() and np.array_equal(F["v"], m.faces)
    p = m.export(str(tmp_path / "m.obj"))
    lines = open(p).read().split("\n")
    vs = np.array([[float(x) for x in ln.split()[1:]] for ln in lines if ln.startswith("v ")], np.float32)
    fs = np.array([[int(x) for x in ln.split()[1:]] for ln in lines if ln.startswith("f ")])
    assert np.array_equal(vs, m.vertices) and np.array_equal(fs - 1, m.faces)
    with pytest.raises(ValueError):
        m.export(str(tmp_path / "m.stl"))


def test_mesh_entry_points_validate_without_gpu():
    import ctypes
    from dgs_b200 import _lib
    L = _lib.lib()
    cb = _lib.ALLOC_FN(lambda n, u: None)
    fake = ctypes.c_void_p(256)
    pairs = ctypes.c_longlong(0)
    assert L.dgs_mesh_field(10, fake, fake, fake, fake, 1.0, fake, 1.0, 64, 128, 1.5, fake, fake, None,
                            ctypes.byref(pairs), cb, None, None) == 1
    assert b"num_blocks" in L.dgs_last_error()
    out = [ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_longlong(), ctypes.c_longlong()]
    assert L.dgs_marching_cubes(fake, 1, 4, 4, 0.5, cb, None, *[ctypes.byref(o) for o in out], None) == 1
    assert b"at least 2" in L.dgs_last_error()
    with pytest.raises(_lib.DgsError):
        from dgs_b200.renderer import GaussianModel
        g = GaussianModel(0)
        g._xyz = torch.zeros(4, 3)
        g.extract_fields(64, 16)
