"""Mesh rendering on libdgs_b200.so (dgs_mesh_render): depth-tested triangle rasterization with silhouette
antialiasing into alpha, depth, normal, face-id and colour maps, forward only.

* `render` draws a mesh from the Gaussian rasterizer's OpenCV cameras (c2w, fx fy cx cy), with the clip matrix
  oracle/renderer.py's build_camera builds (gs_core.py:277-316), so a mesh and the Gaussians land on the same pixels.
* `render_turntable` draws an extracted mesh from `renderer.render_turntable`'s cameras, background and quantisation.
* `render_mesh` and `get_render` are drop-ins for the reference's nvdiffrast helpers (diffusionGS/systems/utils.py:
  397-444 and 532-545), with their signatures, output keys, shapes [B, H, W, C] and conventions.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import Alloc, check, stream
from . import mesh as _mesh

ZNEAR, ZFAR = 0.01, 100.0  # gs_core.py:286-287, and render_mesh's near / far
# Scratch budget per call: the views are rendered in chunks that fit it (32 B per pixel and 9 B per face of each view,
# so 1 GiB holds about 60 views of a 680 k-face mesh at 512 x 512).
ARENA_BYTES = 1 << 30
_SCRATCH = {}


def clip_from_opencv(c2ws, fxfycxcy, h, w, znear=ZNEAR, zfar=ZFAR):
    """OpenCV cameras c2ws [v, 4, 4], fxfycxcy [v, 4] -> row-major world -> clip matrices fp32 [v, 4, 4]: the
    projection of gs_core.py:296-316 times the inverse of c2w, formed in fp64."""
    c2ws = torch.as_tensor(c2ws).detach().double().cpu().reshape(-1, 4, 4)
    K = torch.as_tensor(fxfycxcy).detach().double().cpu().reshape(-1, 4)
    P = torch.zeros(len(c2ws), 4, 4, dtype=torch.float64)
    P[:, 0, 0] = 2 * K[:, 0] / w
    P[:, 1, 1] = 2 * K[:, 1] / h
    P[:, 0, 2] = 2 * (K[:, 2] / w) - 1
    P[:, 1, 2] = 2 * (K[:, 3] / h) - 1
    P[:, 2, 2] = -(zfar + znear) / (zfar - znear)
    P[:, 3, 2] = 1.0
    P[:, 2, 3] = -(2 * zfar * znear) / (zfar - znear)
    return (P @ torch.linalg.inv(c2ws)).float()


def clip_from_opengl(c2ws, intrinsics, znear=ZNEAR, zfar=ZFAR):
    """The reference's get_mvp_matrix(c2w, get_projection_matrix_perspective(intrinsics)) (systems/utils.py:364-395):
    OpenGL c2ws [b, 4, 4] (camera looking down -z), normalised intrinsics [b, 3, 3] (the principal point is not used),
    y flipped so that row 0 is the top of the image -> fp32 [b, 4, 4], formed in fp64."""
    c2ws = torch.as_tensor(c2ws).detach().double().cpu().reshape(-1, 4, 4)
    K = torch.as_tensor(intrinsics).detach().double().cpu().reshape(-1, 3, 3)
    P = torch.zeros(len(c2ws), 4, 4, dtype=torch.float64)
    P[:, 0, 0] = 2 * K[:, 0, 0]
    P[:, 1, 1] = -2 * K[:, 1, 1]
    P[:, 2, 2] = -(zfar + znear) / (zfar - znear)
    P[:, 2, 3] = -2.0 * zfar * znear / (zfar - znear)
    P[:, 3, 2] = -1.0
    R, t = c2ws[:, :3, :3], c2ws[:, :3, 3:]
    w2c = torch.zeros_like(c2ws)
    w2c[:, :3, :3] = R.transpose(1, 2)
    w2c[:, :3, 3:] = -R.transpose(1, 2) @ t
    w2c[:, 3, 3] = 1.0
    return (P @ w2c).float()


def _attr(name, a, V, dev):
    if a is None:
        return None
    a = torch.as_tensor(a).detach().to(device=dev, dtype=torch.float32).contiguous()
    if tuple(a.shape) != (V, 3):
        raise ValueError(f"mesh_render: {name} must be [{V}, 3], got {tuple(a.shape)}")
    return a


def render_clip(vertices, faces, clip, h, w, normals=None, colors=None, normal_bg=(0.0, 0.0, 0.0),
                color_bg=(0.0, 0.0, 0.0), near=ZNEAR, outputs=("face_id", "depth", "alpha", "normal", "rgb"),
                max_arena_bytes=ARENA_BYTES):
    """dgs_mesh_render with explicit clip matrices [v, 4, 4] -> dict of CUDA tensors, views first: face_id int32 [v, h,
    w], depth and alpha fp32 [v, h, w], normal and rgb fp32 [v, h, w, 3] (each of `outputs`; normal only with normals,
    rgb only with colors).  vertices / faces are numpy arrays or CUDA tensors (numpy runs on the current device)."""
    is_numpy = _mesh._mesh_check("mesh_render", vertices, faces)
    h, w = int(h), int(w)
    clip = torch.as_tensor(clip)
    if clip.dim() != 3 or tuple(clip.shape[1:]) != (4, 4):
        raise ValueError(f"mesh_render: expected clip matrices [v, 4, 4], got {tuple(clip.shape)}")
    dev, v, f = _mesh._mesh_in("mesh_render", is_numpy, vertices, faces)
    V, n = len(v), len(clip)
    normals, colors = _attr("normals", normals, V, dev), _attr("colors", colors, V, dev)
    clip = clip.detach().to(device=dev, dtype=torch.float32).contiguous()
    want = set(outputs) - ({"normal"} if normals is None else set()) - ({"rgb"} if colors is None else set())
    out = {}
    for k in ("face_id", "depth", "alpha", "normal", "rgb"):
        if k in want:
            shape = (n, h, w, 3) if k in ("normal", "rgb") else (n, h, w)
            out[k] = torch.empty(shape, dtype=torch.int32 if k == "face_id" else torch.float32, device=dev)
    nbg = (C.c_float * 3)(*[float(x) for x in normal_bg])
    cbg = (C.c_float * 3)(*[float(x) for x in color_bg])
    alloc = Alloc(dev, _SCRATCH, (str(dev), "render"), cached=1)
    with torch.cuda.device(dev):
        check(_lib.lib().dgs_mesh_render(
            v.data_ptr(), V, f.data_ptr(), len(f), _lib.ptr(normals), _lib.ptr(colors), _lib.ptr(clip), n, h, w,
            float(near), nbg, cbg, int(max_arena_bytes), *[_lib.ptr(out.get(k)) for k in
                                                            ("face_id", "depth", "alpha", "normal", "rgb")],
            alloc.cb, None, stream(dev)))
    return out


def unit_vertex_normals(vertices, faces):
    """Unit vertex normals of a mesh (the fp64 face-normal sums of dgs_mesh_vertex_colors' normals pass; 0 for a zero
    sum) -> fp32 [V, 3] CUDA tensor."""
    is_numpy = _mesh._mesh_check("vertex_normals", vertices, faces)
    dev, v, f = _mesh._mesh_in("vertex_normals", is_numpy, vertices, faces)
    z = torch.zeros(0, 3, device=dev)
    _, n = _mesh.vertex_colors(z, torch.zeros(0, 1, 3, device=dev), z, torch.zeros(0, 4, device=dev),
                               torch.zeros(0, 1, device=dev), v, f, torch.zeros(3), 1.0, resolution=2, num_blocks=1)
    return n


def render(vertices, faces, c2ws, fxfycxcy, h, w, vertex_colors=None, vertex_normals=None,
           max_arena_bytes=ARENA_BYTES):
    """The mesh seen from OpenCV cameras c2ws [v, 4, 4], fxfycxcy [v, 4] (the Gaussian rasterizer's) at h x w ->
    dict(alpha [v, h, w], depth [v, h, w] (clip w = view-space z, 0 on background), normal [v, h, w, 3] (background 0),
    face_id [v, h, w] (-1 on background), and rgb [v, h, w, 3] (background 1, white, as the Gaussian renders) when
    vertex_colors [V, 3] are given), CUDA tensors.  Without vertex_normals they are computed (`unit_vertex_normals`)."""
    n = unit_vertex_normals(vertices, faces) if vertex_normals is None else vertex_normals
    clip = clip_from_opencv(c2ws, fxfycxcy, h, w)
    return render_clip(vertices, faces, clip, h, w, normals=n, colors=vertex_colors, color_bg=(1.0, 1.0, 1.0),
                       max_arena_bytes=max_arena_bytes)


def _world(mesh, mesh_center, mesh_scale):
    v = np.asarray(mesh.vertices, np.float32)
    if mesh_scale is not None:
        v = v / np.float32(mesh_scale)
    if mesh_center is not None:
        v = v + torch.as_tensor(mesh_center).detach().float().cpu().numpy()
    return v


def render_turntable(mesh, rendering_resolution=384, num_views=8, mesh_center=None, mesh_scale=None):
    """A `dgs_b200.mesh.Mesh` from `renderer.render_turntable`'s cameras -> uint8 numpy [h, num_views * w, 3], the views
    side by side on white, quantised as that strip is ((c * 255) clipped, truncated).  The vertices are mapped back to
    world coordinates by v / mesh_scale + mesh_center when these are given (extract_mesh leaves the mesh in the field's
    normalised frame).  The colour is the mesh's vertex_colors, or n * 0.5 + 0.5 of its vertex normals without them."""
    from .cameras import get_turntable_cameras
    w, h, v, fxfycxcy, c2ws = get_turntable_cameras(h=rendering_resolution, w=rendering_resolution,
                                                    num_views=num_views)
    verts, faces = _world(mesh, mesh_center, mesh_scale), np.asarray(mesh.faces)
    colors = mesh.vertex_colors
    if colors is None:
        nrm = mesh.vertex_normals
        nrm = unit_vertex_normals(verts, faces) if nrm is None else torch.as_tensor(nrm).cuda()
        colors = nrm * 0.5 + 0.5
    out = render_clip(verts, faces, clip_from_opencv(c2ws, fxfycxcy, h, w), h, w, colors=colors,
                      color_bg=(1.0, 1.0, 1.0), outputs=("rgb",))
    frames = out["rgb"].mul_(255.0).clamp_(0.0, 255.0).to(torch.uint8).cpu().numpy()  # in place: no fp32 copies
    return frames.transpose(1, 0, 2, 3).reshape(h, v * w, 3)


def reference_vertex_normals(vertices, faces):
    """The reference Mesh.v_nrm (utils/structure.py:163-189) from the fp64 normals pass: the normalised sum of the face
    normals, (0, 0, 1) where the sum is 0 -> fp32 [V, 3] CUDA tensor.  (The reference also replaces sums of squared
    length up to 1e-20; the pass returns those normalised.)"""
    n = unit_vertex_normals(vertices, faces)
    zero = (n == 0).all(1)
    n[zero] = torch.tensor([0.0, 0.0, 1.0], device=n.device)
    return n


def render_mesh(mesh, cam2world_matrices, intrinsics, device, height=224, width=224, radius=1):
    """Drop-in for the reference's render_mesh (systems/utils.py:397-444): `mesh` with v_pos / t_pos_idx (the
    reference's Mesh) or vertices / faces, OpenGL cam2world_matrices [B, 4, 4], normalised intrinsics [B, 3, 3] ->
    dict(alpha [B, H, W, 1], depth [B, H, W, 1] (clip w, 0 on background), rgb [B, H, W, 3] (125 on the mesh over 1),
    normal [B, H, W, 3] (background -1)), antialiased but for depth, on `device`.  `radius` is unused, as there."""
    verts = getattr(mesh, "v_pos", None)
    faces = getattr(mesh, "t_pos_idx", None)
    if verts is None:
        verts, faces = mesh.vertices, mesh.faces
    dev = torch.device(device)
    verts = torch.as_tensor(verts).detach().to(dev, torch.float32).contiguous()
    faces = torch.as_tensor(faces).detach().to(dev, torch.int32).contiguous()
    nrm = reference_vertex_normals(verts, faces)
    colors = torch.full_like(verts, 125.0)
    clip = clip_from_opengl(cam2world_matrices, intrinsics)
    with torch.cuda.device(dev):
        out = render_clip(verts, faces, clip, height, width, normals=nrm, colors=colors, normal_bg=(-1.0, -1.0, -1.0),
                          color_bg=(1.0, 1.0, 1.0), outputs=("depth", "alpha", "normal", "rgb"))
    return {"alpha": out["alpha"][..., None], "depth": out["depth"][..., None], "rgb": out["rgb"],
            "normal": out["normal"]}


def get_camera(device, img_size=224, focal=5, distance=10):
    """The reference's get_camera (systems/utils.py:446-478): four fixed OpenGL cameras around the origin and their
    intrinsics -> (cam2world_matrices [4, 4, 4], intrinsics [4, 3, 3])."""
    d = distance
    c2w = torch.as_tensor([[[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, d], [0, 0, 0, 1]],
                           [[0, 0, 1, d], [0, 1, 0, 0], [1, 0, 0, 0], [0, 0, 0, 1]],
                           [[-1, 0, 0, 0], [0, 1, 0, 0], [0, 0, -1, -d], [0, 0, 0, 1]],
                           [[0, 0, -1, -d], [0, 1, 0, 0], [-1, 0, 0, 0], [0, 0, 0, 1]]],
                          dtype=torch.float32).to(device)
    K = torch.zeros([3, 3])
    K[0, 0] = focal
    K[1, 1] = focal
    K[1, 2] = img_size // 2
    K[0, 2] = img_size // 2
    return c2w, K.unsqueeze(0).repeat(4, 1, 1).to(device)


def get_render(vertices, faces, device, img_size=224, focal=5, distance=12):
    """Drop-in for the reference's get_render (systems/utils.py:532-545): numpy vertices / faces -> (normal
    [img_size, 4 img_size, 3], depth [img_size, 4 img_size, 1]), the four views of get_camera side by side, the depth's
    non-zero values normalised to [0, 1] over the strip."""
    c2w, K = get_camera(device, img_size, focal, distance)
    out = render_mesh(_RefMesh(torch.from_numpy(np.asarray(vertices)), torch.from_numpy(np.asarray(faces))), c2w, K,
                      device, img_size, img_size)
    v, h, w, _ = out["normal"].shape
    normal = out["normal"].transpose(1, 0).contiguous().view(h, w * v, 3)
    depth = out["depth"].transpose(1, 0).contiguous().view(h, w * v, 1)
    nz = depth != 0
    if nz.any():
        d = depth[nz]
        depth[nz] = (d - d.min()) / (d.max() - d.min())
    return normal, depth


class _RefMesh:
    def __init__(self, v_pos, t_pos_idx):
        self.v_pos, self.t_pos_idx = v_pos, t_pos_idx
