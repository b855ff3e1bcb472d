"""TSDF fusion on the GPU (dgs_tsdf_integrate / dgs_tsdf_extract / dgs_tsdf_colors): the volume, the mesh and the
colours bit for bit against oracle/tsdf.py on soft analytic maps and on the shell model's own renders (sphere and
caller-given cameras, two image sizes), the same bits for any view chunking and on every call, the pixel each point
samples against the pixel the rasterizer draws a Gaussian at, the observed mask, an empty model, the command line, and
extract_mesh(method="tsdf") end to end against the Gaussians it came from."""
import math

import numpy as np
import pytest
import torch

from mesh_shapes import directed, shell_model
from oracle import tsdf as ot
from tsdf_cases import sphere_maps

pytestmark = pytest.mark.gpu

KEYS = ("tsdf_sum", "weight", "rgb_sum", "rgb_weight")
SH_C0 = 0.28209479177387814


def _coloured(m, seed=0):
    """m with degree-0 features: a colour that varies around the shell"""
    xyz = m._xyz
    u = xyz - (xyz.amin(0) + xyz.amax(0)) / 2
    u = u / u.norm(dim=1, keepdim=True)
    g = torch.Generator(device="cuda").manual_seed(seed)
    dc = 0.4 * u + 0.05 * torch.randn(u.shape, generator=g, device="cuda")
    return m.set_data(xyz, (dc / SH_C0)[:, None, :], m._scaling, m._rotation, m._opacity)


def _same_volume(vol, ref):
    for k in KEYS:
        got = vol[k].cpu().numpy()
        assert np.array_equal(got, ref[k]), f"{k}: {(got != ref[k]).sum()} of {got.size} differ"


def _same_mesh_and_colours(vol, ref):
    from dgs_b200 import mesh
    R = len(ref["lin"])
    v, f = mesh.tsdf_mesh(vol)
    rv, rf = ot.extract(ref)
    rv = ot.to_frame(rv, R)
    assert len(rf) > 100
    assert np.array_equal(v.cpu().numpy(), rv) and np.array_equal(f.cpu().numpy(), rf)
    assert np.array_equal(mesh.tsdf_colors(vol, v).cpu().numpy(), ot.colors(ref, rv))
    return v, f


def _soft_maps(c2w, K, H, W, seed):
    """Sphere maps with partial alpha in the foreground and faint alpha in the background, and random colours"""
    image, depth, alpha = sphere_maps(c2w, K, H, W, 0.62)
    rng = np.random.default_rng(seed)
    a = np.where(alpha > 0, rng.uniform(0.45, 1.0, alpha.shape), rng.uniform(0.0, 0.2, alpha.shape)).astype(np.float32)
    depth = (depth * a).astype(np.float32)
    image = rng.uniform(0, 1, image.shape).astype(np.float32)
    return image, depth, a


@pytest.mark.parametrize("R,H,W", [(64, 96, 96), (72, 80, 112)])
def test_integrate_extract_colors_match_the_oracle_on_analytic_maps(R, H, W):
    from dgs_b200 import mesh
    from dgs_b200.cameras import sphere_cameras
    K, c2w = sphere_cameras(30, 96)
    K[:, 2], K[:, 3] = W / 2.0, H / 2.0
    K, c2w = K.astype(np.float32), c2w.astype(np.float32)
    maps = _soft_maps(c2w, K, H, W, R)
    ref = ot.integrate(ot.volume(R), c2w, K, *maps, trunc=16.0 / (R - 1))
    vol = mesh.tsdf_volume(R, "cuda")
    cu = [torch.from_numpy(a).cuda() for a in (c2w, K, *maps)]
    mesh.tsdf_integrate(vol, *cu)
    _same_volume(vol, ref)
    _same_mesh_and_colours(vol, ref)
    # one view per call: the same bits
    one = mesh.tsdf_volume(R, "cuda")
    for k in range(len(K)):
        mesh.tsdf_integrate(one, *(t[k:k + 1] for t in cu))
    for key in KEYS:
        assert torch.equal(one[key], vol[key])


def _world_cameras(m, n, size):
    """sphere_cameras placed around the model in world coordinates, as a caller's own views would be"""
    from dgs_b200 import mesh
    from dgs_b200.cameras import sphere_cameras
    c, s = mesh.mesh_frame(m._xyz)
    K, c2w = sphere_cameras(n, size)
    c2w[:, :3, 3] = c2w[:, :3, 3] / s + c.double().cpu().numpy()
    return K, c2w


def _oracle_of_renders(m, R, size, K=None, c2w=None, n=24):
    """The oracle volume of the maps the rasterizer renders of m in the normalised frame, as tsdf_fusion renders them"""
    from dgs_b200 import mesh, raster
    from dgs_b200.cameras import sphere_cameras
    c, s = mesh.mesh_frame(m._xyz)
    if K is None:
        K, c2w = sphere_cameras(n, size)
    else:
        c2w = c2w.copy()
        c2w[:, :3, 3] = (c2w[:, :3, 3] - c.double().cpu().numpy()) * s
    C2W, FX = (torch.tensor(a, dtype=torch.float32, device="cuda") for a in (c2w, K))
    gs = ((m._xyz - c) * s, m.get_features, m._scaling + math.log(s), m._rotation, m._opacity)
    with torch.no_grad():
        image, depth, alpha, _ = raster.render_batch_forward(*(t[None] for t in gs), size, size, C2W[None], FX[None],
                                                             aux=True)
    maps = (image[0].cpu().numpy(), depth[0, :, 0].cpu().numpy(), alpha[0, :, 0].cpu().numpy())
    return ot.integrate(ot.volume(R), C2W.cpu().numpy(), FX.cpu().numpy(), *maps, trunc=16.0 / (R - 1))


@pytest.fixture(scope="module")
def small_shell():
    return _coloured(shell_model(20000, 5, floaters=False))


@pytest.mark.parametrize("R,size,cameras", [(64, 64, "sphere"), (96, 96, "sphere"), (80, 64, "caller")])
def test_fused_renders_match_the_oracle(small_shell, R, size, cameras):
    from dgs_b200 import mesh
    m = small_shell
    K = c2w = None
    if cameras == "caller":
        K, c2w = _world_cameras(m, 24, size)
    vol = mesh.tsdf_fusion(m._xyz, m.get_features, m._scaling, m._rotation, m._opacity, resolution=R, num_views=24,
                           image_size=size, c2ws=c2w, fxfycxcy=K, max_arena_bytes=1 << 40)
    ref = _oracle_of_renders(m, R, size, K, c2w)
    _same_volume(vol, ref)
    _same_mesh_and_colours(vol, ref)


def test_chunking_and_repeats_give_the_same_bits(small_shell):
    from dgs_b200 import mesh
    m = small_shell
    args = (m._xyz, m.get_features, m._scaling, m._rotation, m._opacity)
    vols = [mesh.tsdf_fusion(*args, resolution=64, num_views=20, image_size=64, max_arena_bytes=b)
            for b in (1, 1 << 40, 1 << 40)]
    meshes = [mesh.tsdf_mesh(v) for v in vols]
    for v, (mv, mf) in zip(vols[1:], meshes[1:]):
        for k in KEYS:
            assert torch.equal(v[k], vols[0][k])
        assert torch.equal(mv, meshes[0][0]) and torch.equal(mf, meshes[0][1])
        assert torch.equal(mesh.tsdf_colors(v, mv), mesh.tsdf_colors(vols[0], meshes[0][0]))


def test_a_point_samples_the_pixel_the_rasterizer_draws_it_at():
    """A small opaque Gaussian on a grid point, placed 0.3 and 0.2 pixel past a pixel corner in pinhole coordinates:
    floor(u) and floor(u - 1/2) (pixel centres at integer coordinates) name different pixels."""
    from dgs_b200 import mesh, raster
    from dgs_b200.cameras import sphere_cameras
    R, H, W = 33, 64, 64
    lin = torch.linspace(-1, 1, R).numpy().astype(np.float64)
    ijk = (20, 14, 17)
    p = lin[list(ijk)]
    K, c2w = sphere_cameras(5, 64)
    K, c2w = K[2:3].copy(), c2w[2:3]
    pc = (p - c2w[0, :3, 3]) @ c2w[0, :3, :3]
    u, v = K[0, 0] * pc[0] / pc[2] + K[0, 2], K[0, 1] * pc[1] / pc[2] + K[0, 3]
    iu, iv = int(np.floor(u)), int(np.floor(v))
    K[0, 2] += iu + 0.3 - u
    K[0, 3] += iv + 0.2 - v
    C2W, FX = (torch.tensor(a, dtype=torch.float32, device="cuda") for a in (c2w, K))
    xyz = torch.tensor(p[None], dtype=torch.float32, device="cuda")
    feats = torch.tensor([[[0.3 / SH_C0, -0.3 / SH_C0, 0.1 / SH_C0]]], device="cuda")
    gs = (xyz, feats, torch.full((1, 3), math.log(1e-3), device="cuda"),
          torch.tensor([[1.0, 0, 0, 0]], device="cuda"), torch.full((1, 1), 6.0, device="cuda"))
    image, depth, alpha, _ = raster.render_batch_forward(*(t[None] for t in gs), H, W, C2W[None], FX[None], aux=True)
    a = alpha[0, 0, 0]
    assert float(a[iv, iu]) > 0.5 and int((a > 0.5).sum()) == 1, "the Gaussian covers one pixel past alpha 0.5"
    vol = mesh.tsdf_volume(R, "cuda")
    mesh.tsdf_integrate(vol, C2W, FX, image[0], depth[0, :, 0], alpha[0, :, 0])
    assert int(vol["weight"][ijk]) == 1 and int(vol["rgb_weight"][ijk]) == 1, "the point sampled another pixel"
    assert abs(float(vol["tsdf_sum"][ijk])) < 0.05
    ref = ot.integrate(ot.volume(R), C2W.cpu().numpy(), FX.cpu().numpy(), image[0].cpu().numpy(),
                       depth[0, :, 0].cpu().numpy(), alpha[0, :, 0].cpu().numpy(), trunc=16.0 / (R - 1))
    _same_volume(vol, ref)


def test_observed_mask_matches_the_oracle():
    from dgs_b200 import mesh
    rng = np.random.default_rng(3)
    R = 40
    ref = ot.volume(R)
    ref["weight"][:] = rng.integers(1, 4, (R, R, R)) * (rng.random((R, R, R)) > 0.06)
    ref["tsdf_sum"][:] = rng.uniform(0.05, 1.0, (R, R, R)).astype(np.float32) * rng.choice([-1, 1], (R, R, R))
    ref["rgb_weight"][:] = rng.integers(0, 3, (R, R, R))
    ref["rgb_sum"][:] = rng.uniform(-0.2, 2.5, (R, R, R, 3)).astype(np.float32)
    vol = mesh.tsdf_volume(R, "cuda")
    for k in KEYS:
        vol[k].copy_(torch.from_numpy(ref[k]))
    v, f = _same_mesh_and_colours(vol, ref)
    assert torch.equal(torch.unique(f), torch.arange(len(v), device="cuda"))


def test_empty_model_gives_an_empty_mesh():
    from dgs_b200 import mesh
    z = torch.zeros(0, 3, device="cuda")
    vol = mesh.tsdf_fusion(z, torch.zeros(0, 1, 3, device="cuda"), z, torch.zeros(0, 4, device="cuda"),
                           torch.zeros(0, 1, device="cuda"), resolution=32, num_views=6, image_size=32)
    assert int(vol["weight"].min()) > 0 and torch.equal(vol["tsdf_sum"], vol["weight"].float())
    v, f = mesh.tsdf_mesh(vol)
    assert v.shape == (0, 3) and f.shape == (0, 3)
    assert mesh.tsdf_colors(vol, v).shape == (0, 3)


def test_cli_writes_a_coloured_tsdf_mesh(tmp_path):
    from dgs_b200 import mesh
    m = _coloured(shell_model(60000, 4, floaters=False))
    ply = m.save_ply(str(tmp_path / "model.ply"))
    out = str(tmp_path / "out.ply")
    mesh.main([ply, out, "--resolution", "128", "--tsdf", "--clean", "--colors"])
    head = open(out, "rb").read(400).split(b"end_header")[0].decode()
    assert "property uchar red" in head and "property float nx" in head
    assert int(head.split("element face ")[1].split()[0]) > 1000


def test_tsdf_mesh_matches_its_gaussians():
    """The obj-256 shell, set up as test_mesh_render_gpu.py's field-chain test: extract_mesh(method="tsdf",
    vertex_colors=True, clean_remesh_then_decimate), mapped back to world coordinates and drawn from the turntable
    cameras (not among the fusion views), against Renderer.forward_buffers of the same Gaussians."""
    from dgs_b200 import mesh, mesh_render as mr
    from dgs_b200.cameras import get_turntable_cameras
    from dgs_b200.renderer import Renderer
    m = shell_model(262146, 11, floaters=False)
    u = m._xyz - (m._xyz.amin(0) + m._xyz.amax(0)) / 2
    m.set_data(m._xyz, (0.4 * u / u.norm(dim=1, keepdim=True) / SH_C0)[:, None, :], m._scaling, m._rotation,
               m._opacity)
    raw = {}

    def post(v, f, target):
        raw["v"], raw["f"] = v, f
        return mesh.clean_remesh_then_decimate(v, f, target)
    got = m.extract_mesh(method="tsdf", postprocess=post, vertex_colors=True)
    d = directed(raw["f"])
    assert len(np.unique(d, axis=0)) == len(d), "the raw TSDF mesh is consistently oriented"
    _, cnt = np.unique(np.sort(d, 1), axis=0, return_counts=True)
    assert cnt.max() <= 2, "the raw TSDF mesh is edge-manifold"
    h = w = 256
    _, _, _, K, c2w = get_turntable_cameras(num_views=8, w=w, h=h)
    world = got.vertices / np.float32(m.mesh_scale) + m.mesh_center.cpu().numpy()
    r = mr.render(world, got.faces, c2w, K, h, w, vertex_colors=got.vertex_colors, vertex_normals=got.vertex_normals)

    class Cfg:
        gaussians_sh_degree = 0
    ren = Renderer(Cfg()).cuda()
    C2W, FX = (torch.tensor(a, dtype=torch.float32, device="cuda")[None] for a in (c2w, K))
    with torch.no_grad():
        g = ren.forward_buffers(m._xyz[None], m.get_features[None], m._scaling[None], m._rotation[None],
                                m._opacity[None], h, w, C2W, FX)
    ga, ma = g["alpha"][0, :, 0] > 0.5, r["alpha"] > 0.5
    iou = float((ga & ma).sum() / (ga | ma).sum())
    mse = float(((g["render"][0].permute(0, 2, 3, 1).clamp(0, 1) - r["rgb"].clamp(0, 1)) ** 2).mean())
    psnr = -10.0 * np.log10(mse)
    print(f"tsdf chain vs Gaussians: {len(raw['f'])} raw faces, {len(got.faces)} faces, alpha IoU {iou:.4f}, colour "
          f"PSNR {psnr:.2f} dB (field chain: 0.95, 26.9 dB)")
    assert iou > 0.93 and psnr > 25.3
