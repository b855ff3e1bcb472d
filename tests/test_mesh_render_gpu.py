"""dgs_mesh_render on the GPU: every output bit for bit against oracle/mesh_render.py (icosphere, a cleaned and
remeshed marching-cubes shell, an open patch; turntable, off-centre and near-plane-crossing cameras; non-square sizes;
a quad over the whole image), determinism, face-order independence, chunking, empty and culled calls, and the mesh chain
end to end against the Gaussians it came from."""
import numpy as np
import pytest
import torch

from mesh_shapes import cuda_grid, mc, patch, shell_model
from mesh_render_cases import icosphere, look_at
from oracle import mesh_render as om

pytestmark = pytest.mark.gpu

KEYS = ("face_id", "depth", "alpha", "normal", "rgb")


def _shell():
    from dgs_b200 import mesh
    X, Y, Z = cuda_grid(48)
    field = 16.0 - torch.sqrt(X * X + 1.3 * Y * Y + 0.8 * Z * Z) + 1.5 * torch.sin(0.4 * X) * torch.cos(0.3 * Z)
    v, f = mc(field, clean=True)
    v, f = mesh.remesh((v / 23.5 - 1.0).astype(np.float32), f, 0.08)
    return v, f


def _patch():
    v, f = patch(14)
    return ((v - np.array([6.5, 6.5, 0.0], np.float32)) / 7.0).astype(np.float32), f


MESHES = {"icosphere": lambda: icosphere(3), "shell": _shell, "patch": _patch}


def _cameras(kind, h, w):
    from dgs_b200.cameras import get_turntable_cameras
    if kind == "turntable":
        _, _, _, K, c2w = get_turntable_cameras(num_views=3, w=w, h=h, radius=2.4, elevation=20)
    elif kind == "offcentre":
        c2w = np.stack([look_at((1.9, -0.7, 0.9), (0.35, 0.2, -0.1)), look_at((-0.4, 2.2, -0.8), (-0.3, 0.0, 0.25))])
        K = np.array([[0.9 * w, 0.95 * w, 0.37 * w, 0.62 * h], [1.3 * w, 1.3 * w, 0.55 * w, 0.41 * h]])
    else:  # "near": cameras inside the bounding box, so faces cross the near plane
        c2w = np.stack([look_at((0.15, 0.05, 0.3), (1.0, 0.3, -0.2)), look_at((0.0, -0.2, 0.0), (0.0, 1.0, 0.3))])
        K = np.array([[0.5 * w, 0.5 * w, 0.5 * w, 0.5 * h]] * 2)
    return c2w, K


def _both(v, f, clip, h, w, n=None, c=None, **kw):
    from dgs_b200 import mesh_render as mr
    rng = np.random.default_rng(len(v))
    n = rng.normal(size=(len(v), 3)).astype(np.float32) if n is None else n
    c = rng.random((len(v), 3)).astype(np.float32) if c is None else c
    bg = dict(normal_bg=(0.0, 0.0, -1.0), color_bg=(1.0, 0.5, 0.25))
    gpu = mr.render_clip(v, f, clip, h, w, normals=n, colors=c, **bg, **kw)
    ref = om.render(v, f, clip.numpy(), h, w, normals=n, colors=c, **bg)
    return {k: t.cpu().numpy() for k, t in gpu.items()}, ref


def _assert_bitwise(gpu, ref):
    for k in KEYS:
        a, b = gpu[k], ref[k]
        assert a.shape == b.shape, k
        bad = a.view(np.uint32) != b.view(np.uint32) if a.dtype == np.float32 else a != b
        assert not bad.any(), f"{k}: {int(bad.sum())} of {bad.size} differ"


@pytest.mark.parametrize("size", [(64, 96), (131, 257)])
@pytest.mark.parametrize("cams", ["turntable", "offcentre", "near"])
@pytest.mark.parametrize("name", sorted(MESHES))
def test_bitwise_against_oracle(name, cams, size):
    from dgs_b200 import mesh_render as mr
    h, w = size
    v, f = MESHES[name]()
    c2w, K = _cameras(cams, h, w)
    clip = mr.clip_from_opencv(c2w, K, h, w)
    gpu, ref = _both(v, f, clip, h, w)
    _assert_bitwise(gpu, ref)
    fg = (ref["face_id"] >= 0).mean()
    edge = ((ref["alpha"] > 0) & (ref["alpha"] < 1)).sum()
    print(f"{name}/{cams} {w}x{h}: {len(f)} faces, coverage {fg:.3f}, {edge} antialiased alpha pixels, "
          f"{int((ref['tiles'] > 1).sum())} tiled (view, face) pairs")
    assert fg > 0.01
    if cams == "near":
        assert (ref["depth"][ref["face_id"] >= 0] > 0).all()


def test_quad_over_the_whole_image_takes_the_tile_path():
    from dgs_b200 import mesh_render as mr
    h, w = 131, 257
    v = np.array([[-3, -3, 0], [3, -3, 0], [3, 3, 0], [-3, 3, 0]], np.float32)
    f = np.array([[0, 1, 2], [0, 2, 3]])
    clip = mr.clip_from_opencv(look_at((0.1, -0.2, 2.0), (0.0, 0.0, 0.0))[None],
                               np.array([[0.8 * w, 0.8 * w, 0.5 * w, 0.5 * h]]), h, w)
    gpu, ref = _both(v, f, clip, h, w)
    _assert_bitwise(gpu, ref)
    assert (ref["face_id"] >= 0).all() and (ref["tiles"] > 100).all()
    assert (gpu["alpha"] == 1).all()


@pytest.fixture(scope="module")
def shell_case():
    from dgs_b200 import mesh_render as mr
    v, f = _shell()
    c2w, K = _cameras("turntable", 64, 96)
    return v, f, mr.clip_from_opencv(c2w, K, 64, 96)


def test_repeated_calls_and_chunks_give_the_same_bits(shell_case):
    from dgs_b200 import mesh_render as mr
    v, f, clip = shell_case
    n = np.random.default_rng(0).normal(size=(len(v), 3)).astype(np.float32)
    runs = [mr.render_clip(v, f, clip, 64, 96, normals=n, colors=np.abs(n), max_arena_bytes=b)
            for b in (1 << 30, 1 << 30, 1)]  # a budget of 1 byte renders one view at a time
    for r in runs[1:]:
        for k in KEYS:
            assert torch.equal(r[k], runs[0][k]), k


def test_face_permutation(shell_case):
    from dgs_b200 import mesh_render as mr
    v, f, clip = shell_case
    n = np.random.default_rng(1).normal(size=(len(v), 3)).astype(np.float32)
    a = mr.render_clip(v, f, clip, 64, 96, normals=n, colors=np.abs(n))
    perm = np.random.default_rng(2).permutation(len(f))
    b = mr.render_clip(v, f[perm], clip, 64, 96, normals=n, colors=np.abs(n))
    fa, fb = a["face_id"].cpu().numpy(), b["face_id"].cpu().numpy()
    mapped = np.where(fb >= 0, perm[np.maximum(fb, 0)], -1)
    assert np.array_equal(mapped, fa)
    for k in ("depth", "alpha", "normal", "rgb"):
        assert torch.equal(a[k], b[k]), k


def test_empty_zero_views_and_culled():
    from dgs_b200 import mesh_render as mr
    v, f = icosphere(2)
    clip = mr.clip_from_opencv(look_at((0, 0, 3.0), (0, 0, 0), up=(0, 1, 0))[None], np.array([[50.0, 50, 24, 16]]), 32, 48)
    out = mr.render_clip(v, f[:0], clip, 32, 48, normals=v, colors=v, color_bg=(0.5, 0.5, 0.5))
    assert (out["face_id"] == -1).all() and (out["depth"] == 0).all() and (out["alpha"] == 0).all()
    assert (out["rgb"] == 0.5).all() and (out["normal"] == 0).all()
    out = mr.render_clip(v, f, clip[:0], 32, 48, normals=v, colors=v)
    assert all(t.shape[0] == 0 for t in out.values())
    away = mr.clip_from_opencv(look_at((0, 0, 3.0), (0, 0, 6.0), up=(0, 1, 0))[None], np.array([[50.0, 50, 24, 16]]), 32, 48)
    gpu, ref = _both(v, f, away, 32, 48)
    _assert_bitwise(gpu, ref)
    assert (gpu["face_id"] == -1).all() and (ref["tiles"] == 0).all()


# Measured on an H100 80GB HBM3 at a 700 W power limit: IoU 0.9525, PSNR 26.85 dB (100,000 faces, 8 views at 256 x 256).  The floors sit
# 0.02 and 1.5 dB below, room for a change in the chain's post-processing but not for a misplaced or miscoloured mesh.
IOU_FLOOR, PSNR_FLOOR = 0.93, 25.3


def test_mesh_chain_matches_its_gaussians():
    """The obj-256 shell: extract_mesh(vertex_colors=True, clean_remesh_then_decimate), mapped back to world
    coordinates and drawn from the turntable cameras, against Renderer.forward_buffers of the same Gaussians."""
    from dgs_b200 import mesh, mesh_render as mr
    from dgs_b200.cameras import get_turntable_cameras
    from dgs_b200.renderer import Renderer
    from oracle import mesh_color as oc
    m = shell_model(262146, 11, floaters=False)
    xyz = m._xyz
    u = xyz - (xyz.amin(0) + xyz.amax(0)) / 2
    u = u / u.norm(dim=1, keepdim=True)
    m.set_data(xyz, (0.4 * u / oc.SH_C0)[:, None, :], m._scaling, m._rotation, m._opacity)
    got = m.extract_mesh(postprocess=mesh.clean_remesh_then_decimate, vertex_colors=True)
    h = w = 256
    _, _, nv, K, c2w = get_turntable_cameras(num_views=8, w=w, h=h)
    world = got.vertices / np.float32(m.mesh_scale) + m.mesh_center.cpu().numpy()
    r = mr.render(world, got.faces, c2w, K, h, w, vertex_colors=got.vertex_colors,
                  vertex_normals=got.vertex_normals)

    class Cfg:
        gaussians_sh_degree = 0
    ren = Renderer(Cfg()).cuda()
    C2W, FX = torch.tensor(c2w, dtype=torch.float32, device="cuda")[None], torch.tensor(K, dtype=torch.float32,
                                                                                      device="cuda")[None]
    with torch.no_grad():
        g = ren.forward_buffers(m._xyz[None], m.get_features[None], m._scaling[None], m._rotation[None],
                                m._opacity[None], h, w, C2W, FX)
    ga, ma = g["alpha"][0, :, 0] > 0.5, r["alpha"] > 0.5
    iou = float((ga & ma).sum() / (ga | ma).sum())
    mse = float(((g["render"][0].permute(0, 2, 3, 1).clamp(0, 1) - r["rgb"].clamp(0, 1)) ** 2).mean())
    psnr = -10.0 * np.log10(mse)
    print(f"mesh chain vs Gaussians: {len(got.faces)} faces, alpha IoU {iou:.4f}, colour PSNR {psnr:.2f} dB")
    assert iou > IOU_FLOOR and psnr > PSNR_FLOOR


def test_reference_drop_ins_and_turntable():
    from dgs_b200 import mesh as dm, mesh_render as mr
    v, f = icosphere(3)
    normal, depth = mr.get_render(v, f.astype(np.int32), "cuda", img_size=64)
    assert normal.shape == (64, 256, 3) and depth.shape == (64, 256, 1)
    assert float(depth.max()) == 1.0 and float(depth.min()) == 0.0
    assert (normal[0, 0] == -1).all()
    c2w, K = mr.get_camera("cuda", 64, 5, 12)
    out = mr.render_mesh(dm.Mesh(v, f), c2w, K, "cuda", 64, 64)
    assert {k: tuple(t.shape) for k, t in out.items()} == {"alpha": (4, 64, 64, 1), "depth": (4, 64, 64, 1),
                                                             "rgb": (4, 64, 64, 3), "normal": (4, 64, 64, 3)}
    a = torch.nn.functional.pad(out["alpha"][..., 0], (1, 1, 1, 1), value=0.5)
    near = torch.stack([a[:, 1:-1, :-2], a[:, 1:-1, 2:], a[:, :-2, 1:-1], a[:, 2:, 1:-1]]).amax(0)
    far = torch.stack([a[:, 1:-1, :-2], a[:, 1:-1, 2:], a[:, :-2, 1:-1], a[:, 2:, 1:-1]]).amin(0)
    inside, outside = far == 1, near == 0  # pixels whose 4 neighbours are all on the mesh / all off it
    assert inside.any() and outside.any()
    # the reference writes the constant; here it is interpolated, so within an ulp of it
    assert torch.allclose(out["rgb"][inside], torch.tensor(125.0, device="cuda"), rtol=1e-6, atol=0)
    assert (out["rgb"][outside] == 1).all()
    strip = mr.render_turntable(dm.Mesh(v, f), rendering_resolution=48, num_views=3)
    assert strip.shape == (48, 144, 3) and strip.dtype == np.uint8
    assert (strip[0, 0] == 255).all() and (strip != 255).any()
