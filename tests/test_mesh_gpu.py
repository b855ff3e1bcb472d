"""Mesh extraction on the H100: dgs_mesh_field against the reference's own extract_fields (committed fixtures) and the
fp64 oracle on the device (per-block Gaussian counts bit for bit), at the pipeline's full size; dgs_marching_cubes
against the numpy oracle; GaussianModel.extract_mesh end to end."""
import os

import numpy as np
import pytest
import torch

from oracle import mesh as om

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "mesh_fields_ref.npz")
NAMES = ("xyz", "scaling", "rotation", "opacity")
CASES = {"r64_b16": (64, 16, 1.5, None), "r100_b16": (100, 16, 1.5, None), "r64_b16_smod": (64, 16, 1.5, 0.7),
         "r48_b8_relax1": (48, 8, 1.0, None)}
# occupancy rel-L2 against the fp64 oracle (measured on an H100: at most 3.5e-7 over these cases) and against the
# reference's fp32 field (at most 5.5e-7)
FIELD_TOL, REF_TOL = 2e-6, 3e-6


def _field(t, R, nb, rr=1.5, smod=None):
    from dgs_b200 import mesh
    return mesh.opacity_field(*t, scaling_modifier=smod, resolution=R, num_blocks=nb, relax_ratio=rr, return_counts=True)


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def _shell(P, seed, dist="trained"):
    from dgs_b200 import synth
    g = synth.make_shell_gaussians(P, seed, dist)
    return [torch.tensor(g[k], device="cuda") for k in NAMES]


@pytest.mark.parametrize("case", list(CASES))
def test_field_matches_reference_fixture_and_oracle(case):
    z = np.load(GOLDEN)
    R, nb, rr, smod = CASES[case]
    t = [torch.from_numpy(z[f"{case}/in/{k}"]).cuda() for k in NAMES]
    occ, center, scale, counts, pairs = _field(t, R, nb, rr, smod)
    assert np.array_equal(center.cpu().numpy(), z[f"{case}/mesh_center"]) and scale == float(z[f"{case}/mesh_scale"])
    o = om.field(*t, resolution=R, num_blocks=nb, relax_ratio=rr, scaling_modifier=smod)
    e_ref = _rel(occ, torch.from_numpy(z[f"{case}/occ"]).cuda())
    e_orc = _rel(occ, o["occ"])
    print(f"{case}: rel_l2 vs reference {e_ref:.2e}, vs fp64 oracle {e_orc:.2e}, {pairs} pairs")
    assert torch.equal(counts.long(), o["counts"]) and pairs == int(o["counts"].sum())
    assert e_orc <= FIELD_TOL and e_ref <= REF_TOL


def test_field_20k_r128_b32():
    t = _shell(20000, 5)
    occ, _, _, counts, _ = _field(t, 128, 32)
    o = om.field(*t, resolution=128, num_blocks=32)
    e = _rel(occ, o["occ"])
    print(f"20k Gaussians at 128 / 32: rel_l2 vs fp64 oracle {e:.2e}")
    assert torch.equal(counts.long(), o["counts"]) and e <= FIELD_TOL


def test_membership_on_chunk_boundaries():
    """Centres exactly on the fp32 vmin / vmax values (and one ulp either side); two corner Gaussians make
    mesh_center 0 and mesh_scale 1, so the normalised centres are the placed values."""
    R, nb = 64, 16
    lin, bounds, vmin, vmax = om.chunks(R, nb, 1.5)
    edges = torch.cat([vmin, vmax])
    vals = torch.cat([edges, torch.nextafter(edges, torch.tensor(2.0)), torch.nextafter(edges, torch.tensor(-2.0))])
    vals = vals[(vals > -0.9) & (vals < 0.9)]
    rng = np.random.default_rng(0)
    n = 3000
    xyz = torch.from_numpy(rng.choice(vals.numpy(), size=(n, 3)))
    xyz = torch.cat([torch.full((1, 3), -0.9), torch.full((1, 3), 0.9), xyz]).float()
    g = _shell(n + 2, 1)
    t = [xyz.cuda()] + g[1:]
    occ, center, scale, counts, _ = _field(t, R, nb)
    assert np.float32(scale) == 1.0
    assert torch.equal(center.cpu(), torch.zeros(3))
    o = om.field(*t, resolution=R, num_blocks=nb)
    assert torch.equal(counts.long(), o["counts"])
    assert _rel(occ, o["occ"]) <= FIELD_TOL


@pytest.fixture(scope="module")
def full():
    t = _shell(262146, 11)
    occ, center, scale, counts, pairs = _field(t, 256, 64)
    return t, occ, counts, pairs


def test_full_size_counts_and_sampled_blocks(full):
    t, occ, counts, pairs = full
    center, scale, xyz_n, _, _ = om.normalise(*t)
    _, bounds, vmin, vmax = om.chunks(256, 64, 1.5, "cuda")
    ref_counts = om.block_counts(om.membership(xyz_n, vmin, vmax))
    assert torch.equal(counts.long(), ref_counts)
    nonempty = torch.nonzero(ref_counts).tolist()
    rng = np.random.default_rng(3)
    pick = [tuple(nonempty[i]) for i in rng.choice(len(nonempty), 64, replace=False)]
    o = om.field(*t, resolution=256, num_blocks=64, blocks=pick)
    sel = torch.zeros_like(occ, dtype=torch.bool)
    for bx, by, bz in pick:
        sel[bounds[bx][0]:bounds[bx][1], bounds[by][0]:bounds[by][1], bounds[bz][0]:bounds[bz][1]] = True
    e = _rel(occ[sel], o["occ"][sel])
    print(f"262,146 Gaussians at 256 / 64: {pairs} pairs, {len(nonempty)} non-empty blocks, rel_l2 on 64 blocks {e:.2e}")
    assert e <= FIELD_TOL


def test_field_is_deterministic(full):
    t, occ, counts, _ = full
    occ2, _, _, counts2, _ = _field(t, 256, 64)
    assert torch.equal(occ, occ2) and torch.equal(counts, counts2)


def _closed_and_oriented(faces):
    d = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    fwd = {tuple(e) for e in d.tolist()}
    assert len(fwd) == len(d), "a directed edge is used twice (inconsistent orientation)"
    assert all((b, a) in fwd for a, b in fwd), "an edge without its opposite (open surface)"


def _check_mc(field, iso):
    from dgs_b200 import mesh
    v, f = mesh.marching_cubes(field, iso)
    rv, rf = om.marching_cubes(field.cpu().numpy(), iso)
    assert v.shape == rv.shape and f.shape == rf.shape
    assert float(np.abs(v.cpu().numpy() - rv).max(initial=0.0)) <= 1e-5
    assert np.array_equal(f.cpu().numpy(), rf)
    return v.cpu().numpy().astype(np.float64), f.cpu().numpy().astype(np.int64)


def test_marching_cubes_matches_oracle_on_fields():
    z = np.load(GOLDEN)
    occ = torch.from_numpy(z["r100_b16/occ"]).cuda()
    for iso in (0.005, 0.5):
        _, f = _check_mc(occ, iso)
        assert len(f) > 0
    g = torch.Generator("cuda").manual_seed(0)
    rnd = torch.rand(40, 33, 27, device="cuda", generator=g)
    rnd[0], rnd[-1], rnd[:, 0], rnd[:, -1], rnd[:, :, 0], rnd[:, :, -1] = 0, 0, 0, 0, 0, 0
    _, f = _check_mc(rnd, 0.5)
    _closed_and_oriented(f)


def test_marching_cubes_sphere_volume():
    n, r = 128, 40.0
    x = torch.arange(n, device="cuda", dtype=torch.float32) - (n - 1) / 2
    X, Y, Z = torch.meshgrid(x, x, x, indexing="ij")
    v, f = _check_mc((r - torch.sqrt(X * X + Y * Y + Z * Z)).contiguous(), 0.0)
    _closed_and_oriented(f)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    vol = float(np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0)
    print(f"sphere r={r}: volume / analytic = {vol / (4 / 3 * np.pi * r ** 3):.5f}")
    assert abs(vol / (4 / 3 * np.pi * r ** 3) - 1) < 0.01


def _model(t):
    from dgs_b200.renderer import GaussianModel
    m = GaussianModel(0)
    m._xyz, m._scaling, m._rotation, m._opacity = t
    return m


def test_extract_mesh_end_to_end():
    m = _model(_shell(262146, 11, "fine"))
    mesh = m.extract_mesh()
    occ = m.extract_fields(256, 64)
    boundary = max(float(occ[[0, -1]].max()), float(occ[:, [0, -1]].max()), float(occ[:, :, [0, -1]].max()))
    print(f"extract_mesh: {len(mesh.vertices)} vertices, {len(mesh.faces)} faces, field max on the grid's faces "
          f"{boundary:.2e}")
    assert boundary <= 0.005
    assert len(mesh.faces) > 1000 and mesh.faces.dtype == np.int64 and mesh.vertices.dtype == np.float32
    assert (np.abs(mesh.vertices) <= 1).all()
    _closed_and_oriented(mesh.faces)
    calls = []
    m.extract_mesh(postprocess=lambda v, f, target: calls.append(target) or (v[:3], f[:1] * 0))
    assert calls == [1e5]


def test_extract_errors_and_empty():
    from dgs_b200 import _lib
    from dgs_b200.renderer import GaussianModel
    t = _shell(1000, 2)
    with pytest.raises(_lib.DgsError, match="CUDA"):
        _model([x.cpu() for x in t]).extract_fields()
    with pytest.raises(AssertionError):
        _model(t).extract_fields(resolution=128, num_blocks=3)
    empty = GaussianModel(0)
    empty._xyz, empty._scaling, empty._rotation, empty._opacity = (torch.zeros(0, k, device="cuda") for k in (3, 3, 4, 1))
    assert float(empty.extract_fields(64, 16).abs().sum()) == 0.0
    mesh = empty.extract_mesh(resolution=64)
    assert mesh.vertices.shape == (0, 3) and mesh.faces.shape == (0, 3)
