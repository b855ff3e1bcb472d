"""Host-side mirror of the reference's `Renderer` (diffusionGS/models/gsrenderer/renderer.py:21-92)
on top of the batched sm_90a rasterizer.

`Renderer.forward(xyz, features, scaling, rotation, opacity, height, width, C2W, fxfycxcy, deferred=True)`
keeps the reference signature and returns [b, v, 3, H, W] fp32.  Where the reference loops over
(sample, view) in Python and RE-RENDERS every view in the backward (gs_core.py:990-1001, 1041-1056),
this issues one batched launch set and keeps the sorted tile lists for the backward.
"""
import copy

import torch
import torch.nn as nn

from . import raster as _raster


class BatchedGaussianRender(torch.autograd.Function):
    """Replaces DeferredGaussianRender (gs_core.py:949-1060); same inputs, same gradient outputs
    (sum over views of d/d{xyz, features, scaling, rotation, opacity}, all w.r.t. the RAW tensors)."""

    @staticmethod
    def forward(ctx, xyz, features, scaling, rotation, opacity, height, width, C2W, fxfycxcy,
                scaling_modifier=None, use_gssplat=False, arena_cache=None):
        needs_bwd = any(ctx.needs_input_grad[:5])
        # Arenas: the inference path re-uses ONE grow-only set (arena_cache["infer"]); a forward that will be
        # differentiated checks a set out of a pool and its backward returns it, so steady-state training does no
        # allocator traffic either (cudaMalloc / cudaFree of multi-GB arenas showed up as 40-70 ms step outliers)
        # while two live forwards (e.g. two renders feeding one loss) never share buffers.
        cache = None
        if arena_cache is not None:
            if needs_bwd:
                pool = arena_cache.setdefault("pool", [])
                cache = pool.pop() if pool else {}
            else:
                cache = arena_cache.setdefault("infer", {})
        with torch.no_grad():
            images, state = _raster.render_batch_forward(xyz, features, scaling, rotation, opacity, height, width,
                                                         C2W, fxfycxcy, scaling_modifier, arena_cache=cache)
        ctx.state = state
        ctx.pool = (arena_cache, cache) if needs_bwd and arena_cache is not None else None
        ctx.in_dtypes = (xyz.dtype, features.dtype, scaling.dtype, rotation.dtype, opacity.dtype)
        ctx.num_rendered = state["R"]
        return images

    @staticmethod
    def backward(ctx, grad_output):
        cache = ctx.pool[1] if ctx.pool else None
        grads = _raster.render_batch_backward(ctx.state, grad_output, arena_cache=cache)
        ctx.state = None  # release the arenas ...
        if ctx.pool:      # ... back into the pool for the next step
            ctx.pool[0]["pool"].append(cache)
            ctx.pool = None
        grads = tuple(g.to(dt) for g, dt in zip(grads, ctx.in_dtypes))
        return (*grads, None, None, None, None, None, None, None)


class BatchedGaussianRenderMSE(torch.autograd.Function):
    """Render + the l2 term of LossComputer.forward (diffusionGS/utils/losses.py:261-284) as ONE node:
    -> (images [b,v,3,H,W], l2_loss [b] = mean over (v,3,h,w) of (images - target[:, :, :3])^2).
    The per-sample sums come out of the blend-forward kernel and the backward forms the MSE part of dL/dpix inside the
    blend-backward kernel from (images, target, dL/dl2_loss) -- no per-element loss or gradient image."""

    @staticmethod
    def forward(ctx, xyz, features, scaling, rotation, opacity, height, width, C2W, fxfycxcy, target,
                scaling_modifier=None, arena_cache=None):
        ctx.set_materialize_grads(False)
        needs_bwd = any(ctx.needs_input_grad[:5])
        cache = None
        if arena_cache is not None:
            if needs_bwd:
                pool = arena_cache.setdefault("pool", [])
                cache = pool.pop() if pool else {}
            else:
                cache = arena_cache.setdefault("infer", {})
        b, v = C2W.shape[0], C2W.shape[1]
        with torch.no_grad():
            loss_sum = torch.zeros(b, dtype=torch.float64, device=xyz.device)
            images, state = _raster.render_batch_forward(xyz, features, scaling, rotation, opacity, height, width, C2W,
                                                         fxfycxcy, scaling_modifier, arena_cache=cache,
                                                         mse_target=target, mse_loss_sum=loss_sum)
            n = v * 3 * int(height) * int(width)
            l2 = (loss_sum / n).float()
        ctx.state, ctx.n = state, n
        ctx.pool = (arena_cache, cache) if needs_bwd and arena_cache is not None else None
        ctx.in_dtypes = (xyz.dtype, features.dtype, scaling.dtype, rotation.dtype, opacity.dtype)
        return images, l2

    @staticmethod
    def backward(ctx, g_images, g_l2):
        cache = ctx.pool[1] if ctx.pool else None
        if g_images is None and g_l2 is None:
            raise RuntimeError("BatchedGaussianRenderMSE.backward without any upstream gradient")
        coef = None if g_l2 is None else (g_l2.float() * (2.0 / ctx.n)).contiguous()
        grads = _raster.render_batch_backward(ctx.state, g_images, arena_cache=cache, mse_coef=coef)
        ctx.state = None
        if ctx.pool:
            ctx.pool[0]["pool"].append(cache)
            ctx.pool = None
        grads = tuple(g.to(dt) for g, dt in zip(grads, ctx.in_dtypes))
        return (*grads, None, None, None, None, None, None, None)


batched_gaussian_render = BatchedGaussianRender.apply
deferred_gaussian_render = batched_gaussian_render  # reference name (gs_core.py:1064)


class GaussianModel:
    """Parameter holder with the reference's activations (gs_core.py:323-373, 545-575), its post-sampler filters
    (386-475), PLY export and import (577-785) and mesh extraction (786-869): `extract_fields` and `extract_mesh` run
    on the sm_90a kernels of dgs_b200.mesh and need CUDA tensors."""

    def __init__(self, sh_degree: int, scaling_modifier=None):
        self.sh_degree = sh_degree
        self.scaling_modifier = scaling_modifier
        self._xyz = self._features_dc = self._scaling = self._rotation = self._opacity = torch.empty(0)
        self._features_rest = torch.empty(0) if sh_degree > 0 else None

    def empty(self):
        self.__init__(self.sh_degree, self.scaling_modifier)

    def set_data(self, xyz, features, scaling, rotation, opacity):
        self._xyz = xyz
        self._features_dc = features[:, :1, :].contiguous()
        self._features_rest = features[:, 1:, :].contiguous() if self.sh_degree > 0 else None
        self._scaling, self._rotation, self._opacity = scaling, rotation, opacity
        return self

    @property
    def get_xyz(self):
        return self._xyz

    @property
    def get_scaling(self):
        s = torch.exp(self._scaling)
        return s * self.scaling_modifier if self.scaling_modifier is not None else s

    @property
    def get_rotation(self):
        return torch.nn.functional.normalize(self._rotation)

    @property
    def get_opacity(self):
        return torch.sigmoid(self._opacity)

    @property
    def get_features(self):
        if self.sh_degree > 0:
            return torch.cat((self._features_dc, self._features_rest), dim=1)
        return self._features_dc


    def get_covariance(self, scaling_modifier=1):
        """gs_core.py:572-575: (R S)(R S)^T of the scales times scaling_modifier and the raw rotation over its Euclidean
        norm, as [P, 6] = (xx, xy, xz, yy, yz, zz)."""
        return _covariance6(scaling_modifier * self.get_scaling, self._rotation)

    # ---- post-processing after the sampler loop: gs_core.py:386-475 filters, 577-785 PLY, 786-869 mesh ----
    def to(self, device):
        for k in ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity"):
            v = getattr(self, k)
            if v is not None:
                setattr(self, k, v.to(device))
        return self

    def filter(self, valid_mask):  # gs_core.py:394-403
        for k in ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity"):
            v = getattr(self, k)
            if v is not None and (k != "_features_rest" or self.sh_degree > 0):
                setattr(self, k, v[valid_mask])
        return self

    def crop(self, crop_bbx=(-1, 1, -1, 1, -1, 1)):  # gs_core.py:406-419
        x0, x1, y0, y1, z0, z1 = crop_bbx
        p = self._xyz
        bad = (p[:, 0] < x0) | (p[:, 0] > x1) | (p[:, 1] < y0) | (p[:, 1] > y1) | (p[:, 2] < z0) | (p[:, 2] > z1)
        return self.filter(~bad)

    def prune(self, opacity_thres=0.05):  # gs_core.py:421-425
        return self.filter(self.get_opacity.squeeze(1) > opacity_thres)

    def prune_by_nearfar(self, cam_origins, nearfar_percent=(0.01, 0.99)):  # gs_core.py:427-461
        assert len(nearfar_percent) == 2 and 0 <= nearfar_percent[0] < nearfar_percent[1] <= 1
        dev = self._xyz.device
        dists = torch.cdist(self._xyz[None], cam_origins[None].to(dev))[0]               # [points, cams]
        pct = torch.quantile(dists, torch.tensor(nearfar_percent).to(dev), dim=0)        # [2, cams]
        reject = ((dists < pct[0:1, :]) | (dists > pct[1:2, :])).any(dim=1)
        return self.filter(~reject)

    def apply_all_filters(self, opacity_thres=0.05, crop_bbx=(-1, 1, -1, 1, -1, 1), cam_origins=None,
                          nearfar_percent=(0.005, 1.0)):  # gs_core.py:463-475
        self.prune(opacity_thres)
        if crop_bbx is not None:
            self.crop(crop_bbx)
        if cam_origins is not None:
            self.prune_by_nearfar(cam_origins, nearfar_percent)
        return self

    def construct_dtypes(self, use_fp16=False, enable_gs_viewer=True):  # gs_core.py:578-633
        if use_fp16:
            raise NotImplementedError("fp16 PLY: the reference builds 'f2' properties, which plyfile (and the PLY format) cannot write")
        names = ["x", "y", "z"]
        l = [(n, "f4") for n in names] + [(n, "u1") for n in ("red", "green", "blue")]
        l += [(f"f_dc_{i}", "f4") for i in range(self._features_dc.shape[1] * self._features_dc.shape[2])]
        if enable_gs_viewer:
            assert self.sh_degree <= 3, "GS viewer only supports SH up to degree 3"
            l += [(f"f_rest_{i}", "f4") for i in range(((3 + 1) ** 2 - 1) * 3)]
        elif self.sh_degree > 0:
            l += [(f"f_rest_{i}", "f4") for i in range(self._features_rest.shape[1] * self._features_rest.shape[2])]
        l.append(("opacity", "f4"))
        l += [(f"scale_{i}", "f4") for i in range(self._scaling.shape[1])]
        l += [(f"rot_{i}", "f4") for i in range(self._rotation.shape[1])]
        return l

    def save_ply(self, path, use_fp16=False, enable_gs_viewer=True, color_code=False, filter_mask=None):
        """gs_core.py:637-713: xyz, 8-bit RGB (from the SH DC term), f_dc, f_rest (padded to degree 3 for the viewers),
        raw opacity / log-scale / rotation, one binary little-endian `vertex` element -- the file plyfile's
        PlyData([PlyElement.describe(elements, "vertex")]).write(path) produces; written with numpy (plyfile is not
        installed here)."""
        import os

        import numpy as np
        if color_code:
            raise NotImplementedError("color_code=True needs matplotlib's viridis colour map (visualisation, out of scope)")
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        xyz = self._xyz.detach().cpu().numpy()
        f_dc = self._features_dc.detach().transpose(1, 2).flatten(start_dim=1).contiguous().cpu().numpy()
        rgb = ((f_dc * 0.28209479177387814 + 0.5) * 255.0).clip(0.0, 255.0).astype(np.uint8)  # SH2RGB, gs_core.py:252
        opac = self._opacity.detach().cpu().numpy()
        scale = (torch.log(self.get_scaling) if self.scaling_modifier is not None else self._scaling).detach().cpu().numpy()
        rot = self._rotation.detach().cpu().numpy()
        f_rest = None
        if self.sh_degree > 0:
            f_rest = self._features_rest.detach().transpose(1, 2).flatten(start_dim=1).contiguous().cpu().numpy()
        if enable_gs_viewer:
            full = 3 * ((3 + 1) ** 2 - 1)
            pad = np.zeros((xyz.shape[0], full), np.float32)
            if f_rest is not None:
                pad[:, :f_rest.shape[1]] = f_rest
            f_rest = pad
        dtype = self.construct_dtypes(use_fp16, enable_gs_viewer)
        cols = [xyz, rgb, f_dc] + ([f_rest] if f_rest is not None else []) + [opac, scale, rot]
        attributes = np.concatenate([c.astype(np.float32) for c in cols], axis=1)
        if filter_mask is not None:
            attributes = attributes[np.asarray(filter_mask)]
        elements = np.empty(attributes.shape[0], dtype=dtype)
        for i, (name, _) in enumerate(dtype):
            elements[name] = attributes[:, i]
        ply_type = {"f4": "float", "u1": "uchar"}
        header = ["ply", "format binary_little_endian 1.0", f"element vertex {elements.shape[0]}"]
        header += [f"property {ply_type[t]} {n}" for n, t in dtype] + ["end_header"]
        with open(path, "wb") as f:
            f.write(("\n".join(header) + "\n").encode("ascii"))
            f.write(elements.astype(elements.dtype.newbyteorder("<")).tobytes())
        return path


    def load_ply(self, path):
        """gs_core.py:716-785: the inverse of save_ply (xyz, f_dc, f_rest when sh_degree > 0, raw opacity / log-scale /
        rotation) into CPU fp32 tensors; read with numpy from binary PLY (plyfile is not installed here)."""
        import numpy as np
        v = _read_ply_vertices(path)
        n = len(v)
        xyz = np.stack([v["x"], v["y"], v["z"]], axis=1)
        opacities = np.asarray(v["opacity"])[..., np.newaxis]
        features_dc = np.stack([v["f_dc_0"], v["f_dc_1"], v["f_dc_2"]], axis=1)[..., np.newaxis]  # [P, 3, 1]

        def group(prefix):
            names = sorted((k for k in v.dtype.names if k.startswith(prefix)), key=lambda k: int(k.split("_")[-1]))
            return np.stack([v[k] for k in names], axis=1) if names else np.zeros((n, 0))
        if self.sh_degree > 0:
            extra = group("f_rest_")
            assert extra.shape[1] == 3 * (self.sh_degree + 1) ** 2 - 3
            extra = extra.reshape(n, 3, (self.sh_degree + 1) ** 2 - 1)
            self._features_rest = torch.from_numpy(extra.astype(np.float32)).transpose(1, 2).contiguous()
        else:
            self._features_rest = None
        self._xyz = torch.from_numpy(xyz.astype(np.float32))
        self._features_dc = torch.from_numpy(features_dc.astype(np.float32)).transpose(1, 2).contiguous()
        self._opacity = torch.from_numpy(opacities.astype(np.float32)).contiguous()
        self._scaling = torch.from_numpy(group("scale_").astype(np.float32)).contiguous()
        self._rotation = torch.from_numpy(group("rot").astype(np.float32)).contiguous()
        return self

    def extract_fields(self, resolution=128, num_blocks=16, relax_ratio=1.5):
        """gs_core.py:786-852: the opacity field [resolution]^3 (fp32, on the model's CUDA device, indexed [x][y][z]) on
        the grid linspace(-1, 1, resolution) after normalising the centres to about [-0.9, 0.9]^3; sets mesh_center and
        mesh_scale.  Each point sums only the Gaussians whose centre lies within relax_ratio block sizes of its block, as
        the reference does.  With no Gaussians the field is 0 (mesh_center 0, mesh_scale 1)."""
        from . import mesh as _mesh
        occ, self.mesh_center, self.mesh_scale = _mesh.opacity_field(
            self._xyz, self._scaling, self._rotation, self._opacity, self.scaling_modifier, resolution, num_blocks,
            relax_ratio)
        return occ

    def extract_mesh(self, density_thresh=0.005, resolution=256, decimate_target=1e5, postprocess=None):
        """gs_core.py:855-869: extract_fields(resolution, num_blocks=64), marching cubes at density_thresh on the GPU,
        vertices mapped by v / (resolution - 1) * 2 - 1 (in the normalised frame: not mapped back by mesh_center /
        mesh_scale, as in the reference) -> dgs_b200.mesh.Mesh (vertices float32 [V, 3], faces int64 [F, 3]).
        The reference then cleans, remeshes and decimates with pymeshlab; that is not done here: without `postprocess`
        the raw marching-cubes mesh is returned and `decimate_target` is unused.  `postprocess(vertices, faces,
        decimate_target) -> (vertices, faces)` runs on the numpy arrays, e.g. a wrapper of the reference's clean_mesh /
        decimate_mesh."""
        from . import mesh as _mesh
        occ = self.extract_fields(resolution, num_blocks=64)
        return _mesh.extract_mesh(occ, density_thresh, resolution, postprocess, decimate_target)


def _covariance6(stds, r):
    """build_covariance_from_scaling_rotation (gs_core.py:112-147, 324-328) in elementwise fp32 ops."""
    norm = torch.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = [[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
         [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
         [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]]
    L = [[R[i][j] * stds[:, j] for j in range(3)] for i in range(3)]
    dot = lambda i, k: (L[i][0] * L[k][0] + L[i][1] * L[k][1]) + L[i][2] * L[k][2]  # noqa: E731
    return torch.stack([dot(0, 0), dot(0, 1), dot(0, 2), dot(1, 1), dot(1, 2), dot(2, 2)], dim=1)


_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2",
              "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4",
              "double": "f8", "float64": "f8"}


def _read_ply_vertices(path):
    """The `vertex` element of a binary PLY whose first element it is, as a numpy structured array."""
    import numpy as np
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        fmt, n, props, in_vertex = None, None, [], False
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f"{path}: PLY header without end_header")
            tok = line.decode("ascii").split()
            if not tok:
                continue
            if tok[0] == "end_header":
                break
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                in_vertex = tok[1] == "vertex" and n is None
                if in_vertex:
                    n = int(tok[2])
                elif n is None:
                    raise ValueError(f"{path}: the vertex element must come first")
            elif tok[0] == "property" and in_vertex:
                if tok[1] == "list":
                    raise ValueError(f"{path}: list properties in the vertex element are not supported")
                props.append((tok[2], _PLY_TYPES[tok[1]]))
        if fmt not in ("binary_little_endian", "binary_big_endian") or n is None:
            raise ValueError(f"{path}: need a binary PLY with a vertex element (format {fmt})")
        order = "<" if fmt == "binary_little_endian" else ">"
        dtype = np.dtype([(name, order + t) for name, t in props])
        data = np.frombuffer(f.read(dtype.itemsize * n), dtype=dtype, count=n)
    return data


class Renderer(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.scaling_modifier = None
        sh_degree = getattr(config, "gaussians_sh_degree", 0)
        self.gaussians_model = GaussianModel(sh_degree, self.scaling_modifier)
        self._arena_cache = {}  # inference-path arenas, grown on demand, re-used step after step

    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(self, xyz, features, scaling, rotation, opacity, height, width, C2W, fxfycxcy, deferred=True):
        """xyz [b,n,3], features [b,n,(deg+1)^2,3], scaling [b,n,3], rotation [b,n,4], opacity [b,n,1],
        C2W [b,v,4,4], fxfycxcy [b,v,4] -> [b,v,3,height,width] fp32.  `deferred` is accepted for
        signature parity: both reference branches compute the same images; here both map to the
        batched kernel set."""
        out = batched_gaussian_render(xyz, features, scaling, rotation, opacity, height, width, C2W, fxfycxcy,
                                      self.scaling_modifier, getattr(self.config, "use_gssplat", False),
                                      self._arena_cache)
        self.last_num_rendered = _raster.LAST_NUM_RENDERED
        return out

    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward_mse(self, xyz, features, scaling, rotation, opacity, height, width, C2W, fxfycxcy, target):
        """forward() + the image-space MSE of the training loss in the same launch set:
        -> (renderings [b,v,3,H,W], l2_loss [b]) with l2_loss exactly LossComputer.forward's first output
        (losses.py:261-284; target [b,v,3|4,H,W], a 4th mask channel is ignored as there)."""
        out = BatchedGaussianRenderMSE.apply(xyz, features, scaling, rotation, opacity, height, width, C2W, fxfycxcy, target,
                                             self.scaling_modifier, self._arena_cache)
        self.last_num_rendered = _raster.LAST_NUM_RENDERED
        return out

    def new_gaussians_model(self):
        return copy.deepcopy(self.gaussians_model)
