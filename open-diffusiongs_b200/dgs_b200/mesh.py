"""Mesh extraction on libdgs_b200.so (dgs_mesh_field / dgs_marching_cubes): the layer under
`GaussianModel.extract_fields` / `extract_mesh`, and a command line that meshes a saved Gaussian PLY.

    python -m dgs_b200.mesh in.ply out.obj [--resolution 256] [--density-thresh 0.005]

reads a PLY written by `GaussianModel.save_ply` (or the reference's), extracts the mesh exactly as
`extract_mesh(density_thresh, resolution)` does and writes it as OBJ or binary PLY, chosen by the suffix.

Marching cubes produces the same vertex set as PyMCubes (one vertex per sign-changing grid edge, at the linear
interpolation of the iso value); on the ambiguous cases the triangulation may differ (a face with two diagonally
opposite inside corners always keeps them apart).  The mesh is closed wherever the surface does not reach the edge of
the grid.
"""
import argparse
import ctypes as C
import os

import numpy as np
import torch

from . import _lib
from ._lib import ALLOC_FN, check

_SCRATCH = {}  # grow-only scratch buffers, re-used across calls: {(device, slot): uint8 tensor}


class _Alloc:
    """dgs_alloc_fn: the first `cached` requests come from the grow-only scratch cache, later ones (outputs the caller
    keeps) are fresh tensors."""

    def __init__(self, device, name, cached):
        self.device, self.name, self.cached = device, name, cached
        self.tensors = []
        self.cb = ALLOC_FN(self._alloc)

    def _alloc(self, nbytes, _user):
        try:
            i = len(self.tensors)
            if i < self.cached:
                key = (str(self.device), self.name, i)
                t = _SCRATCH.get(key)
                if t is None or t.numel() < nbytes:
                    _SCRATCH.pop(key, None)
                    t = torch.empty(int(nbytes * 1.25) + 256, dtype=torch.uint8, device=self.device)
                    _SCRATCH[key] = t
            else:
                t = torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=self.device)
            self.tensors.append(t)
            return t.data_ptr()
        except Exception as e:  # noqa: BLE001  (reported as DGS_ERR_ALLOC by the C side)
            import sys
            print(f"[dgs_b200] mesh allocation of {nbytes} bytes failed: {e!r}"[:600], file=sys.stderr)
            return None


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _f32(t):
    return t.detach().to(torch.float32).contiguous()


def opacity_field(xyz, scaling, rotation, opacity, scaling_modifier=None, resolution=128, num_blocks=16, relax_ratio=1.5,
                  return_counts=False):
    """GaussianModel.extract_fields on raw CUDA tensors -> (occ [R, R, R] fp32, mesh_center fp32 [3], mesh_scale float),
    plus (block_counts int32 [nc, nc, nc], pair count) with return_counts.  No Gaussians: a zero field, centre 0 and
    scale 1."""
    block_size = 2 / num_blocks
    assert resolution % block_size == 0
    if not xyz.is_cuda:
        raise _lib.DgsError("extract_fields needs CUDA tensors (no CPU path)")
    dev = xyz.device
    xyz, scaling, rotation, opacity = (_f32(t) for t in (xyz, scaling, rotation, opacity))
    P = xyz.shape[0]
    with torch.cuda.device(dev):
        if P > 0:
            mn, mx = xyz.amin(0), xyz.amax(0)
            center = (mn + mx) / 2
            scale = 1.8 / (mx - mn).amax().item()
        else:
            center, scale = torch.zeros(3, dtype=torch.float32, device=dev), 1.0
        lin = torch.linspace(-1, 1, resolution).to(dev)
        nc = -(-resolution // (resolution // num_blocks))
        occ = torch.empty([resolution] * 3, dtype=torch.float32, device=dev)
        counts = torch.empty([nc] * 3, dtype=torch.int32, device=dev) if return_counts else None
        pairs = C.c_longlong(0)
        alloc = _Alloc(dev, "field", 2)
        smod = 1.0 if scaling_modifier is None else float(scaling_modifier)
        # the reference multiplies fp32 tensors by these Python floats, i.e. by their fp32 roundings
        check(_lib.lib().dgs_mesh_field(P, xyz.data_ptr(), scaling.data_ptr(), rotation.data_ptr(), opacity.data_ptr(),
                                        float(np.float32(smod)), center.data_ptr(), float(np.float32(scale)), resolution,
                                        num_blocks, float(relax_ratio), lin.data_ptr(), occ.data_ptr(),
                                        counts.data_ptr() if return_counts else None, C.byref(pairs), alloc.cb, None,
                                        _stream(dev)))
    if return_counts:
        return occ, center, scale, counts, pairs.value
    return occ, center, scale


def marching_cubes(field, iso):
    """field [nx, ny, nz] fp32 CUDA tensor -> (vertices fp32 [V, 3] in index coordinates, faces int32 [F, 3]) on the
    field's device.  A point is inside iff value > iso; faces are oriented with normals from inside to outside."""
    if not field.is_cuda:
        raise _lib.DgsError("marching_cubes needs a CUDA tensor (no CPU path)")
    if field.dim() != 3:
        raise ValueError(f"marching_cubes: expected a 3-d field, got shape {tuple(field.shape)}")
    dev = field.device
    f = _f32(field)
    alloc = _Alloc(dev, "mc", 1)
    vp, tp = C.c_void_p(), C.c_void_p()
    nv, nt = C.c_longlong(0), C.c_longlong(0)
    with torch.cuda.device(dev):
        check(_lib.lib().dgs_marching_cubes(f.data_ptr(), *f.shape, float(iso), alloc.cb, None, C.byref(vp), C.byref(tp),
                                            C.byref(nv), C.byref(nt), _stream(dev)))
    V, F = nv.value, nt.value
    verts = alloc.tensors[1][:V * 12].view(torch.float32).view(V, 3) if V else torch.zeros(0, 3, device=dev)
    faces = alloc.tensors[2][:F * 12].view(torch.int32).view(F, 3) if F else torch.zeros(0, 3, dtype=torch.int32,
                                                                                          device=dev)
    return verts, faces


class Mesh:
    """The triangle mesh extract_mesh returns: `vertices` float32 [V, 3] and `faces` int64 [F, 3] numpy arrays (the
    attribute names of trimesh.Trimesh)."""

    def __init__(self, vertices, faces):
        self.vertices = np.ascontiguousarray(vertices, dtype=np.float32).reshape(-1, 3)
        self.faces = np.ascontiguousarray(faces, dtype=np.int64).reshape(-1, 3)

    def export(self, path):
        """Writes binary little-endian PLY (.ply) or Wavefront OBJ (.obj), by suffix.  -> path"""
        ext = os.path.splitext(path)[1].lower()
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        V, F = len(self.vertices), len(self.faces)
        if ext == ".ply":
            header = ("ply\nformat binary_little_endian 1.0\n"
                      f"element vertex {V}\nproperty float x\nproperty float y\nproperty float z\n"
                      f"element face {F}\nproperty list uchar int vertex_indices\nend_header\n")
            face = np.empty(F, dtype=[("n", "u1"), ("v", "<i4", (3,))])
            face["n"], face["v"] = 3, self.faces
            with open(path, "wb") as fh:
                fh.write(header.encode("ascii"))
                fh.write(self.vertices.astype("<f4").tobytes())
                fh.write(face.tobytes())
        elif ext == ".obj":
            with open(path, "w") as fh:
                np.savetxt(fh, self.vertices, fmt="v %.9g %.9g %.9g")
                np.savetxt(fh, self.faces + 1, fmt="f %d %d %d")
        else:
            raise ValueError(f"Mesh.export: unsupported suffix {ext!r} (use .ply or .obj)")
        return path


def extract_mesh(field, density_thresh, resolution, postprocess=None, decimate_target=1e5):
    """Marching cubes of `field` at density_thresh, vertices mapped by v / (resolution - 1) * 2 - 1 (not back by
    mesh_center / mesh_scale, as the reference), then `postprocess(vertices, faces, decimate_target)` if given."""
    v, f = marching_cubes(field, density_thresh)
    vertices = (v.cpu().numpy().astype(np.float64) / (resolution - 1.0) * 2 - 1).astype(np.float32)
    faces = f.cpu().numpy().astype(np.int64)
    if postprocess is not None:
        vertices, faces = postprocess(vertices, faces, decimate_target)
    return Mesh(vertices, faces)


def main(argv=None):
    ap = argparse.ArgumentParser(description="Extract a mesh from a Gaussian PLY (GaussianModel.extract_mesh)")
    ap.add_argument("ply", help="Gaussians, as written by GaussianModel.save_ply")
    ap.add_argument("out", help="output mesh, .obj or .ply")
    ap.add_argument("--resolution", type=int, default=256, help="grid points per axis (default 256)")
    ap.add_argument("--density-thresh", type=float, default=0.005, help="iso value of the opacity field (default 0.005)")
    args = ap.parse_args(argv)
    from .renderer import GaussianModel
    gm = GaussianModel(0)
    gm.load_ply(args.ply)
    mesh = gm.to("cuda").extract_mesh(density_thresh=args.density_thresh, resolution=args.resolution)
    mesh.export(args.out)
    print(f"{args.out}: {len(mesh.vertices)} vertices, {len(mesh.faces)} faces")


if __name__ == "__main__":
    main()
