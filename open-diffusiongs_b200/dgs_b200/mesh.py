"""Mesh extraction on libdgs_b200.so (dgs_mesh_field / dgs_marching_cubes / dgs_mesh_clean / dgs_mesh_remesh /
dgs_mesh_decimate / dgs_mesh_vertex_colors / dgs_tsdf_*): the layer under `GaussianModel.extract_fields` /
`extract_mesh`, and a command line that meshes a saved Gaussian PLY.

    python -m dgs_b200.mesh in.ply out.obj [--resolution 256] [--density-thresh 0.005] [--clean] [--remesh [LEN]]
                                           [--decimate-target N] [--colors] [--poisson [DEPTH] | --tsdf]

reads a PLY written by `GaussianModel.save_ply` (or the reference's), extracts the mesh exactly as
`extract_mesh(density_thresh, resolution)` does and writes it as OBJ or binary PLY, chosen by the suffix; with `--clean`
the mesh is first cleaned (`clean`, dgs_mesh_clean), with `--remesh [LEN]` then remeshed to edges of about LEN (default
0.015; `remesh`, dgs_mesh_remesh), and with `--decimate-target N` then decimated to at most N faces (`decimate`,
dgs_mesh_decimate).  With `--colors` the final vertices get colours and normals from the Gaussians (`vertex_colors`,
dgs_mesh_vertex_colors), written as PLY vertex properties or OBJ `v x y z r g b` / `vn` lines; the model is then loaded at
the SH degree its `f_rest_*` properties give.  With `--poisson [DEPTH]` the surface is reconstructed instead by screened
Poisson (`poisson_reconstruction`, dgs_poisson_reconstruct) from the Gaussians' centres and shortest axes, as
`extract_mesh(method="poisson", depth=DEPTH)` does; the flags above apply to it unchanged.  With `--tsdf` the
Gaussians' own depth renders from 100 views are fused into a truncated signed distance volume at `--resolution` and its
zero crossing is marched where it was observed (`tsdf_fusion`, `tsdf_mesh`; dgs_tsdf_integrate / dgs_tsdf_extract), as
`extract_mesh(method="tsdf")` does; `--colors` then takes the colours the views show (`tsdf_colors`).

Marching cubes produces the same vertex set as PyMCubes (one vertex per sign-changing grid edge, at the linear
interpolation of the iso value); on the ambiguous cases the triangulation may differ (a face with two diagonally
opposite inside corners always keeps them apart).  The mesh is closed wherever the surface does not reach the edge of
the grid.
"""
import argparse
import ctypes as C
import math
import os

import numpy as np
import torch

from . import _lib
from ._lib import Alloc, check, f32, stream

_SCRATCH = {}  # grow-only scratch buffers, re-used across calls: {((device, name), i): uint8 tensor}


def mesh_frame(xyz):
    """The normalisation of extract_fields: (mesh_center fp32 [3], mesh_scale float) that map the centres xyz (fp32
    [P, 3]) to about [-0.9, 0.9]^3 by (xyz - mesh_center) * mesh_scale; centre 0 and scale 1 without centres"""
    if xyz.shape[0] == 0:
        return torch.zeros(3, dtype=torch.float32, device=xyz.device), 1.0
    mn, mx = xyz.amin(0), xyz.amax(0)
    return (mn + mx) / 2, 1.8 / (mx - mn).amax().item()


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
    xyz, scaling, rotation, opacity = (f32(t) for t in (xyz, scaling, rotation, opacity))
    P = xyz.shape[0]
    with torch.cuda.device(dev):
        center, scale = mesh_frame(xyz)
        lin = torch.linspace(-1, 1, resolution).to(dev)
        nc = -(-resolution // (resolution // num_blocks))
        occ = torch.empty([resolution] * 3, dtype=torch.float32, device=dev)
        counts = torch.empty([nc] * 3, dtype=torch.int32, device=dev) if return_counts else None
        pairs = C.c_longlong(0)
        alloc = Alloc(dev, _SCRATCH, (str(dev), "field"), cached=2)
        smod = 1.0 if scaling_modifier is None else float(scaling_modifier)
        # the reference multiplies fp32 tensors by these Python floats, i.e. by their fp32 roundings
        check(_lib.lib().dgs_mesh_field(P, xyz.data_ptr(), scaling.data_ptr(), rotation.data_ptr(), opacity.data_ptr(),
                                        float(np.float32(smod)), center.data_ptr(), float(np.float32(scale)), resolution,
                                        num_blocks, float(relax_ratio), lin.data_ptr(), occ.data_ptr(),
                                        counts.data_ptr() if return_counts else None, C.byref(pairs), alloc.cb, None,
                                        stream(dev)))
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
    f = f32(field)
    alloc = Alloc(dev, _SCRATCH, (str(dev), "mc"), cached=1)
    vp, tp = C.c_void_p(), C.c_void_p()
    nv, nt = C.c_longlong(0), C.c_longlong(0)
    with torch.cuda.device(dev):
        check(_lib.lib().dgs_marching_cubes(f.data_ptr(), *f.shape, float(iso), alloc.cb, None, C.byref(vp), C.byref(tp),
                                            C.byref(nv), C.byref(nt), stream(dev)))
    V, F = nv.value, nt.value
    verts = alloc.tensors[1][:V * 12].view(torch.float32).view(V, 3) if V else torch.zeros(0, 3, device=dev)
    faces = alloc.tensors[2][:F * 12].view(torch.int32).view(F, 3) if F else torch.zeros(0, 3, dtype=torch.int32,
                                                                                          device=dev)
    return verts, faces


def _mesh_check(name, vertices, faces):
    """Checks the types, shapes and dtypes of a mesh argument pair -> whether it is numpy (else CUDA tensors)"""
    is_numpy = isinstance(vertices, np.ndarray) and isinstance(faces, np.ndarray)
    if not is_numpy and not (isinstance(vertices, torch.Tensor) and isinstance(faces, torch.Tensor)
                             and vertices.is_cuda and faces.is_cuda and vertices.device == faces.device):
        raise TypeError(f"{name}: vertices and faces must both be numpy arrays or CUDA tensors on one device")
    if vertices.ndim != 2 or vertices.shape[1] != 3 or faces.ndim != 2 or faces.shape[1] != 3:
        raise ValueError(f"{name}: expected vertices [V, 3] and faces [F, 3], got {tuple(vertices.shape)} and "
                         f"{tuple(faces.shape)}")
    float_v = vertices.dtype.kind == "f" if is_numpy else vertices.dtype.is_floating_point
    int_f = faces.dtype.kind in "iu" if is_numpy else not (faces.dtype.is_floating_point or faces.dtype.is_complex
                                                             or faces.dtype == torch.bool)
    if not float_v or not int_f:
        raise TypeError(f"{name}: vertices must be floating point and faces integer (got {vertices.dtype}, "
                        f"{faces.dtype})")
    return is_numpy


def _mesh_in(name, is_numpy, vertices, faces):
    """A checked mesh argument pair -> (device, vertices fp32 [V, 3], faces int32 [F, 3]) as contiguous CUDA tensors;
    numpy input goes to the current CUDA device."""
    i32 = np.iinfo(np.int32)
    if len(faces) and (int(faces.min()) < i32.min or int(faces.max()) > i32.max):
        raise ValueError(f"{name}: face indices do not fit int32")
    if is_numpy:
        dev = torch.device("cuda", torch.cuda.current_device())
        v = torch.from_numpy(np.ascontiguousarray(vertices, np.float32)).to(dev)
        f = torch.from_numpy(np.ascontiguousarray(faces, np.int32)).to(dev)
    else:
        dev = vertices.device
        v = vertices.detach().to(torch.float32).contiguous()
        f = faces.detach().to(torch.int32).contiguous()
    return dev, v, f


def _mesh_out(is_numpy, dev, alloc, V, F):
    """The output buffers a mesh call allocated last, after its scratch -> (vertices fp32 [V, 3], faces int64 [F, 3])"""
    out = alloc.tensors[len(alloc.tensors) - bool(V) - bool(F):]  # an empty output is not allocated
    ov = out[0][:V * 12].view(torch.float32).view(V, 3) if V else torch.zeros(0, 3, device=dev)
    of = out[-1][:F * 12].view(torch.int32).view(F, 3).long() if F else torch.zeros(0, 3, dtype=torch.int64,
                                                                                              device=dev)
    if is_numpy:
        return ov.cpu().numpy(), of.cpu().numpy()
    return ov, of


def _run_mesh(name, is_numpy, vertices, faces, args, stats=()):
    """Runs dgs_mesh_<name>(vertices, V, faces, F, *args, alloc, NULL, the four outputs, *stats, stream) on a checked
    mesh argument pair -> (vertices, faces) as `_mesh_out`"""
    dev, v, f = _mesh_in(name, is_numpy, vertices, faces)
    alloc = Alloc(dev, _SCRATCH, (str(dev), name), cached=1)  # only the first scratch: remesh's later requests differ
    vp, fp = C.c_void_p(), C.c_void_p()
    nv, nf = C.c_longlong(0), C.c_longlong(0)
    with torch.cuda.device(dev):
        check(getattr(_lib.lib(), f"dgs_mesh_{name}")(v.data_ptr(), len(v), f.data_ptr(), len(f), *args, alloc.cb, None,
                                                       C.byref(vp), C.byref(fp), C.byref(nv), C.byref(nf), *stats,
                                                       stream(dev)))
    return _mesh_out(is_numpy, dev, alloc, nv.value, nf.value)


def _chain(vertices, faces, clean_first, remesh_len, decimate_target):
    """`clean` with its defaults when clean_first, `remesh` to edges of remesh_len when it is given, then `decimate` to
    decimate_target faces when it is given and more are left"""
    if clean_first:
        vertices, faces = clean(vertices, faces)
    if remesh_len is not None:
        vertices, faces = remesh(vertices, faces, remesh_len)
    if decimate_target is not None and len(faces) > decimate_target:
        vertices, faces = decimate(vertices, faces, decimate_target)
    return vertices, faces


def decimate(vertices, faces, target_faces):
    """Quadric edge-collapse decimation to at most `target_faces` faces (dgs_mesh_decimate; the reference's
    decimate_mesh with optimalplacement=True, boundary loops kept) -> (vertices, faces).  The signature of
    extract_mesh's `postprocess`, so `extract_mesh(postprocess=decimate)` returns the reference's <= decimate_target
    (1e5) face mesh.  numpy input (vertices float [V, 3], faces integer [F, 3]) runs on the current CUDA device and returns
    numpy float32 [V', 3] / int64 [F', 3]; CUDA tensors return CUDA tensors of those dtypes on their device.  The
    result has target_faces or target_faces - 1 faces unless no further edge can be collapsed; a mesh within the target
    comes back unchanged."""
    is_numpy = _mesh_check("decimate", vertices, faces)
    target = float(target_faces)
    if not np.isfinite(target) or target < 0:
        raise ValueError(f"decimate: target_faces must be a finite number >= 0 (got {target_faces!r})")
    return _run_mesh("decimate", is_numpy, vertices, faces, (int(target),), (C.byref(C.c_int(0)),))


def clean(vertices, faces, v_pct=1, min_f=64, min_d=20, repair=True, stats=None):
    """The reference's clean_mesh with remesh=False (dgs_mesh_clean) -> (vertices, faces): drop unreferenced
    vertices, merge vertices closer than v_pct % of the bounding-box diagonal (v_pct <= 0: no merge), drop duplicate
    and zero-area faces, edge-connected components with a diagonal under min_d % of the mesh's (min_d <= 0: kept) or
    fewer than min_f faces (min_f <= 0: kept), and with `repair` the non-manifold edges' smallest faces and the
    non-manifold vertices (split: one copy per extra fan).  Input and output types as `decimate`; the output positions
    are copies of input positions, and the result is the same bits on every run.  `stats`, a dict, receives
    "merge_rounds" and "stage_faces" (the face count after each of the nine stages of include/dgs_b200.h)."""
    is_numpy = _mesh_check("clean", vertices, faces)
    v_pct, min_d = float(v_pct), float(min_d)
    if not (np.isfinite(v_pct) and np.isfinite(min_d)):
        raise ValueError(f"clean: v_pct and min_d must be finite (got {v_pct!r}, {min_d!r})")
    rounds, counts = C.c_int(0), (C.c_longlong * 9)()
    out = _run_mesh("clean", is_numpy, vertices, faces, (v_pct, int(min_f), min_d, int(bool(repair))),
                    (C.byref(rounds), counts))
    if stats is not None:
        stats["merge_rounds"] = rounds.value
        stats["stage_faces"] = list(counts)
    return out


def clean_then_decimate(vertices, faces, decimate_target):
    """The reference's extract_mesh post-processing without its remeshing (gs_core.py:862-863): `clean` with its
    defaults, then `decimate` to decimate_target faces when more are left.  The signature of extract_mesh's
    `postprocess`: `extract_mesh(postprocess=clean_then_decimate)`."""
    return _chain(vertices, faces, True, None, decimate_target)


def remesh(vertices, faces, target_len=0.015, iterations=3, feature_deg=30, max_surf_dist=None, stats=None):
    """Isotropic remeshing towards edges of target_len (dgs_mesh_remesh; the reference's clean_mesh remeshing step,
    pymeshlab's meshing_isotropic_explicit_remeshing) -> (vertices, faces): per iteration, split edges longer than
    4/3 target_len, collapse edges shorter than 4/5 target_len, flip edges towards valence 6, smooth tangentially and
    project back onto the input surface.  Boundary, non-manifold and feature edges (dihedral angle above feature_deg)
    are kept; no vertex moves farther than max_surf_dist (default: 1 % of the bounding-box diagonal) from the input by a
    collapse or flip.  Input and output types as `decimate`; iterations=0 returns the input unchanged, and the result
    is the same bits on every run.  `stats`, a dict, receives "iterations": per iteration [faces after the split,
    collapse rounds, flip rounds, 1 if a stage stopped at its 256-round cap]."""
    is_numpy = _mesh_check("remesh", vertices, faces)
    L, deg = float(target_len), float(feature_deg)
    if not (np.isfinite(L) and L > 0):
        raise ValueError(f"remesh: target_len must be a finite number > 0 (got {target_len!r})")
    if int(iterations) != iterations or iterations < 0:
        raise ValueError(f"remesh: iterations must be an integer >= 0 (got {iterations!r})")
    msd = -1.0 if max_surf_dist is None else float(max_surf_dist)
    if not (np.isfinite(deg) and np.isfinite(msd)) or (max_surf_dist is not None and msd < 0):
        raise ValueError(f"remesh: feature_deg and max_surf_dist must be finite, max_surf_dist >= 0 (got "
                         f"{feature_deg!r}, {max_surf_dist!r})")
    it = int(iterations)
    st = (C.c_longlong * max(4 * it, 1))()
    out = _run_mesh("remesh", is_numpy, vertices, faces, (L, it, deg, msd), (st,))
    if stats is not None:
        stats["iterations"] = [list(st[4 * i:4 * i + 4]) for i in range(it)]
    return out


def closest_points(vertices, faces, queries):
    """The closest point of the surface (vertices, faces) to each query (dgs_mesh_closest_points, the query `remesh`
    reprojects with) -> (points float64 [Q, 3], squared distances float64 [Q], faces int64 [Q]): the smallest (squared
    distance, face index) over all faces, in fp64.  numpy input (queries float [Q, 3]) returns numpy; CUDA tensors
    return CUDA tensors on their device."""
    is_numpy = _mesh_check("closest_points", vertices, faces)
    if len(faces) == 0:
        raise ValueError("closest_points: the surface has no faces")
    if queries.ndim != 2 or queries.shape[1] != 3:
        raise ValueError(f"closest_points: expected queries [Q, 3], got {tuple(queries.shape)}")
    dev, v, f = _mesh_in("closest_points", is_numpy, vertices, faces)
    if is_numpy:
        q = torch.from_numpy(np.ascontiguousarray(queries, np.float64)).to(dev)
    else:
        q = queries.detach().to(device=dev, dtype=torch.float64).contiguous()
    Q = len(q)
    pts = torch.empty(Q, 3, dtype=torch.float64, device=dev)
    d2 = torch.empty(Q, dtype=torch.float64, device=dev)
    fi = torch.empty(Q, dtype=torch.int32, device=dev)
    alloc = Alloc(dev, _SCRATCH, (str(dev), "closest"), cached=2)  # scratch and grid; the outputs are the caller's
    with torch.cuda.device(dev):
        check(_lib.lib().dgs_mesh_closest_points(v.data_ptr(), len(v), f.data_ptr(), len(f), q.data_ptr(), Q,
                                                 pts.data_ptr(), d2.data_ptr(), fi.data_ptr(), alloc.cb, None,
                                                 stream(dev)))
    if is_numpy:
        return pts.cpu().numpy(), d2.cpu().numpy(), fi.long().cpu().numpy()
    return pts, d2, fi.long()


def _points_check(name, points, normals=None):
    """Checks a point cloud argument (and its normals) -> whether it is numpy (else CUDA tensors)"""
    is_numpy = isinstance(points, np.ndarray)
    if not is_numpy and not (isinstance(points, torch.Tensor) and points.is_cuda):
        raise TypeError(f"{name}: points must be a numpy array or a CUDA tensor")
    if points.ndim != 2 or points.shape[1] != 3:
        raise ValueError(f"{name}: expected points [P, 3], got {tuple(points.shape)}")
    if normals is not None:
        if is_numpy != isinstance(normals, np.ndarray) or (not is_numpy and not (
                isinstance(normals, torch.Tensor) and normals.device == points.device)):
            raise TypeError(f"{name}: points and normals must both be numpy arrays or CUDA tensors on one device")
        if tuple(normals.shape) != tuple(points.shape):
            raise ValueError(f"{name}: normals {tuple(normals.shape)} do not match points {tuple(points.shape)}")
    if is_numpy:
        for a, what in ((points, "points"), (normals, "normals")):
            if a is not None and not np.isfinite(a).all():
                raise ValueError(f"{name}: {what} have a non-finite coordinate")
    return is_numpy


def _points_in(is_numpy, a):
    """A checked point array -> a contiguous fp32 CUDA tensor (numpy goes to the current CUDA device)"""
    if is_numpy:
        return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(torch.device("cuda", torch.cuda.current_device()))
    return a.detach().to(torch.float32).contiguous()


def knn(points, k):
    """Exact k nearest neighbours of every point (dgs_knn) -> (idx int32 [P, k], d2 float32 [P, k]): in (squared
    distance, index) order, the point itself included at distance 0, duplicates included; d2 is the fp32
    (dx*dx + dy*dy) + dz*dz, ties go to the smaller index, and slots beyond P get index -1 and distance inf.  numpy
    input (float [P, 3]) runs on the current CUDA device and returns numpy; CUDA tensors return CUDA tensors.  The result
    is the same bits on every run."""
    is_numpy = _points_check("knn", points)
    if int(k) != k or not 1 <= k <= 32:
        raise ValueError(f"knn: k must be an integer in [1, 32] (got {k!r})")
    p = _points_in(is_numpy, points)
    dev, P, k = p.device, len(p), int(k)
    idx = torch.empty(P, k, dtype=torch.int32, device=dev)
    d2 = torch.empty(P, k, dtype=torch.float32, device=dev)
    alloc = Alloc(dev)
    with torch.cuda.device(dev):
        check(_lib.lib().dgs_knn(p.data_ptr(), P, k, idx.data_ptr(), d2.data_ptr(), alloc.cb, None, stream(dev)))
    alloc.tensors.clear()  # the callback keeps the Alloc in a reference cycle: free the scratch now, not at collection
    alloc.tensor = None
    if is_numpy:
        return idx.cpu().numpy(), d2.cpu().numpy()
    return idx, d2


POISSON_STAGES = ("knn", "outliers_normals", "splat", "solve", "marching_cubes", "trim")


def poisson_reconstruction(points, normals=None, depth=9, nb_neighbors=20, std_ratio=10.0, scale=1.1, point_weight=4.0,
                           density_quantile=0.1, tol=1e-6, max_iters=100, stats=None, trace=None):
    """The reference's poisson_mesh_reconstruction (dgs_poisson_reconstruct; the exact contract is csrc/poisson.cu's
    header) -> (vertices, faces): statistical outlier removal over nb_neighbors nearest points, the given normals or PCA
    normals oriented away from the centroid, screened Poisson on 2^depth + 1 nodes per axis over the points' bounding
    cube scaled by `scale`, marching cubes at the mean indicator value of the points, then the removal of the vertices
    whose sample density is below the density_quantile (0: none) and of the faces that touch them.  The defaults are
    the reference call's (depth 9, 20 neighbours, std_ratio 10, the 10 % quantile).  Faces are oriented outwards for
    outward normals; the vertices are in the input's frame.  numpy input (points float [P, 3], normals None or float
    [P, 3]) runs on the current CUDA device and returns numpy float32 [V, 3] / int64 [F, 3]; CUDA tensors return CUDA
    tensors.  The result is the same bits on every run.  `stats`, a dict, receives "iterations", "residual" (the final
    ||r|| / ||b||), "iso", "inliers", "vertices_before" / "faces_before" (before the trim), "vertices", "faces" and
    "stage_ms" (device ms per stage of POISSON_STAGES); `trace`, a dict, receives the CUDA tensors "inliers" (bool [P]),
    "normals" (float32 [inliers, 3]), "chi" (float32 [R, R, R]) and "density" (float32 [vertices_before])."""
    name = "poisson_reconstruction"
    is_numpy = _points_check(name, points, normals)
    P = len(points)
    if int(nb_neighbors) != nb_neighbors or not 1 <= nb_neighbors <= 32:
        raise ValueError(f"{name}: nb_neighbors must be an integer in [1, 32] (got {nb_neighbors!r})")
    if P < nb_neighbors:
        raise ValueError(f"{name}: {P} points is fewer than nb_neighbors = {nb_neighbors}")
    if int(depth) != depth or not 4 <= depth <= 9:
        raise ValueError(f"{name}: depth must be an integer in [4, 9] (got {depth!r})")
    if not (np.isfinite(scale) and scale >= 1):
        raise ValueError(f"{name}: scale must be finite and >= 1 (got {scale!r})")
    if not 0 <= density_quantile <= 1:
        raise ValueError(f"{name}: density_quantile must be in [0, 1] (got {density_quantile!r})")
    p = _points_in(is_numpy, points)
    n = None if normals is None else _points_in(is_numpy, normals)
    dev, R = p.device, 2 ** int(depth) + 1
    st = _lib.PoissonStats()
    tr, cap = None, 0
    if trace is not None:
        cap = 8 * R * R + 1024
        tensors = dict(inliers=torch.empty(P, dtype=torch.uint8, device=dev),
                       normals=torch.empty(P, 3, dtype=torch.float32, device=dev),
                       chi=torch.empty(R, R, R, dtype=torch.float32, device=dev))
    while True:
        if trace is not None:
            tensors["density"] = torch.empty(cap, dtype=torch.float32, device=dev)
            tr = _lib.PoissonTrace(*(tensors[k].data_ptr() for k in ("inliers", "normals", "chi", "density")), cap)
        alloc = Alloc(dev)  # no cache: the last two buffers are the caller's output
        vp, fp = C.c_void_p(), C.c_void_p()
        nv, nf = C.c_longlong(0), C.c_longlong(0)
        with torch.cuda.device(dev):
            check(_lib.lib().dgs_poisson_reconstruct(
                p.data_ptr(), P, None if n is None else n.data_ptr(), int(depth), int(nb_neighbors), float(std_ratio),
                float(scale), float(point_weight), float(density_quantile), float(tol), int(max_iters), alloc.cb, None,
                C.byref(vp), C.byref(fp), C.byref(nv), C.byref(nf), C.byref(st), C.byref(tr) if tr is not None else None,
                stream(dev)))
        if trace is None or st.vertices_before <= cap:
            break
        alloc.tensors.clear()
        alloc.tensor = None
        cap = st.vertices_before  # the densities did not fit: once more, with room for all of them
    if stats is not None:
        stats.update({k: getattr(st, k) for k in ("iterations", "residual", "iso", "inliers", "vertices_before",
                                                  "faces_before", "vertices", "faces")})
        stats["stage_ms"] = dict(zip(POISSON_STAGES, st.stage_ms))
    if trace is not None:
        trace.update(inliers=tensors["inliers"].bool(), normals=tensors["normals"][:st.inliers], chi=tensors["chi"],
                     density=tensors["density"][:st.vertices_before])
    out = _mesh_out(is_numpy, dev, alloc, nv.value, nf.value)
    alloc.tensors.clear()  # the scratch (GBs at depth 9) goes now; the outputs are views that keep their own buffers
    alloc.tensor = None
    return out


def gaussian_points(xyz, scaling, rotation, mesh_center, mesh_scale):
    """The oriented points extract_mesh(method="poisson") reconstructs from: the centres normalised by
    (xyz - mesh_center) * mesh_scale (fp32), and each Gaussian's shortest axis (the rotation's column of the smallest
    scaling; rotation [P, 4] as w, x, y, z, not normalised) turned to point away from the normalised origin."""
    p = (f32(xyz) - mesh_center) * mesh_scale
    q = torch.nn.functional.normalize(f32(rotation).double(), dim=1)
    w, x, y, z = q.unbind(1)
    cols = torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y + w * z), 2 * (x * z - w * y)], 1),
                        torch.stack([2 * (x * y - w * z), 1 - 2 * (x * x + z * z), 2 * (y * z + w * x)], 1),
                        torch.stack([2 * (x * z + w * y), 2 * (y * z - w * x), 1 - 2 * (x * x + y * y)], 1)], 1)
    n = cols[torch.arange(len(p), device=p.device), f32(scaling).argmin(1)]
    n = torch.where(((n * p.double()).sum(1) < 0)[:, None], -n, n)
    return p.contiguous(), n.float().contiguous()


def clean_remesh_then_decimate(vertices, faces, decimate_target):
    """The reference's whole extract_mesh post-processing (gs_core.py:862-863): `clean` with its defaults, `remesh` to
    edges of 0.015 in 3 iterations, then `decimate` to decimate_target faces when more are left.  The signature of
    extract_mesh's `postprocess`: `extract_mesh(postprocess=clean_remesh_then_decimate)`."""
    return _chain(vertices, faces, True, 0.015, decimate_target)


def vertex_colors(xyz, features, scaling, rotation, opacity, vertices, faces, mesh_center, mesh_scale,
                  scaling_modifier=None, resolution=256, num_blocks=64, relax_ratio=1.5, stats=None):
    """Per-vertex colours and normals of a mesh extract_mesh returned, from the Gaussians of its field
    (dgs_mesh_vertex_colors; the semantics are include/dgs_b200.h's) -> (rgb float32 [V, 3] in [0, 1], normals float32
    [V, 3], unit or 0).  The Gaussians are the raw xyz [P, 3], features [P, (d + 1)^2, 3] (SH degree d in 0..3),
    scaling [P, 3], rotation [P, 4] and opacity [P, 1]; mesh_center / mesh_scale, scaling_modifier, resolution,
    num_blocks and relax_ratio are the field's (what extract_fields used and set).  Each vertex gets the weighted mean,
    by the field's own weights over its block's Gaussians, of their colours seen from its outward normal; a vertex that
    no Gaussian weighs is white.  Input and output types as `decimate` (the Gaussians may be numpy arrays or tensors on
    any device); the result is the same bits on every run and does not depend on the vertex order.  `stats`, a dict,
    receives "unweighted", the number of white vertices."""
    is_numpy = _mesh_check("vertex_colors", vertices, faces)
    if resolution % (2 / num_blocks) != 0:
        raise ValueError(f"vertex_colors: resolution {resolution} is not a multiple of the block size 2 / {num_blocks}")
    P = len(xyz)
    # a model without Gaussians may hold features of no particular shape
    fshape = tuple(features.shape) if P or len(features.shape) == 3 else (0, 1, 3)
    if len(fshape) != 3 or fshape[0] != P or fshape[2] != 3 or fshape[1] not in (1, 4, 9, 16):
        raise ValueError(f"vertex_colors: expected features [P, (d + 1)^2, 3] with d in 0..3 and P = {P}, got "
                         f"{tuple(features.shape)}")
    if torch.as_tensor(mesh_center).numel() != 3:
        raise ValueError(f"vertex_colors: mesh_center must have 3 values (got {mesh_center!r})")
    dev, v, f = _mesh_in("vertex_colors", is_numpy, vertices, faces)
    xyz, features, scaling, rotation, opacity, center = (
        f32(torch.as_tensor(t).to(dev)) for t in (xyz, features, scaling, rotation, opacity, mesh_center))
    features = features.reshape(fshape)
    sh_degree = int(round(fshape[1] ** 0.5)) - 1
    V = len(v)
    rgb = torch.empty(V, 3, dtype=torch.float32, device=dev)
    normals = torch.empty(V, 3, dtype=torch.float32, device=dev)
    unweighted = C.c_longlong(0)
    smod = 1.0 if scaling_modifier is None else float(scaling_modifier)
    alloc = Alloc(dev, _SCRATCH, (str(dev), "colors"), cached=3)  # the mesh scratch and the field's two lists
    with torch.cuda.device(dev):
        lin = torch.linspace(-1, 1, resolution).to(dev)
        # the field's fp32 roundings of the Python floats (opacity_field)
        check(_lib.lib().dgs_mesh_vertex_colors(P, xyz.data_ptr(), features.data_ptr(), sh_degree, scaling.data_ptr(),
                                                rotation.data_ptr(), opacity.data_ptr(), float(np.float32(smod)),
                                                center.data_ptr(), float(np.float32(mesh_scale)), int(resolution),
                                                int(num_blocks), float(relax_ratio), lin.data_ptr(), v.data_ptr(), V,
                                                f.data_ptr(), len(f), rgb.data_ptr(), normals.data_ptr(),
                                                C.byref(unweighted), alloc.cb, None, stream(dev)))
    if stats is not None:
        stats["unweighted"] = unweighted.value
    if is_numpy:
        return rgb.cpu().numpy(), normals.cpu().numpy()
    return rgb, normals


def _tsdf_resolution(resolution):
    if int(resolution) != resolution or not 2 <= resolution <= 512:
        raise ValueError(f"tsdf: resolution must be an integer in [2, 512] (got {resolution!r})")
    return int(resolution)


def tsdf_volume(resolution, device, mesh_center=None, mesh_scale=1.0):
    """An empty TSDF volume over linspace(-1, 1, resolution)^3 (include/dgs_b200.h's dgs_tsdf_integrate): a dict of the
    zeroed CUDA tensors tsdf_sum fp32 [R, R, R], weight int32 [R, R, R], rgb_sum fp32 [R, R, R, 3], rgb_weight int32
    [R, R, R], the grid lin fp32 [R], and the frame mesh_center / mesh_scale its points are in."""
    R = _tsdf_resolution(resolution)
    dev = torch.device(device)
    z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=dev)  # noqa: E731
    with torch.cuda.device(dev):
        lin = torch.linspace(-1, 1, R).to(dev)
    return dict(tsdf_sum=z(R, R, R), weight=z(R, R, R, dt=torch.int32), rgb_sum=z(R, R, R, 3),
                rgb_weight=z(R, R, R, dt=torch.int32), lin=lin,
                mesh_center=z(3) if mesh_center is None else mesh_center, mesh_scale=float(mesh_scale))


def tsdf_integrate(volume, c2ws, fxfycxcy, image, depth, alpha, sdf_trunc=None, alpha_thresh=0.5):
    """Fuses views into `volume` in place (dgs_tsdf_integrate; the exact contract is csrc/tsdf.cu's header): c2ws
    [n, 4, 4] and fxfycxcy [n, 4] are OpenCV cameras in the volume's grid frame, image [n, 3, H, W] the rendered colour
    on a white background, depth [n, H, W] the accumulated depth and alpha [n, H, W], all on the volume's device.
    sdf_trunc defaults to 8 grid spacings, 16 / (R - 1): the rendered depth is the blend-weighted depth of the
    Gaussians' centres, which lies inside the silhouette their extent draws, and a wider band of negative updates from
    the views that graze the surface moves the zero crossing out towards it (on the obj-256 shell, 4 spacings give an
    alpha IoU of 0.922 against the Gaussians, 8 give 0.933 and 16 give 0.946).  Pixels of alpha below alpha_thresh are
    background and carve free space."""
    R = volume["lin"].numel()
    n = c2ws.shape[0] if c2ws.dim() == 3 else -1
    if tuple(c2ws.shape[1:]) != (4, 4) or tuple(fxfycxcy.shape) != (n, 4) or image.dim() != 4 or \
            tuple(image.shape[:2]) != (n, 3):
        raise ValueError(f"tsdf_integrate: expected c2ws [n, 4, 4], fxfycxcy [n, 4] and image [n, 3, H, W], got "
                         f"{tuple(c2ws.shape)}, {tuple(fxfycxcy.shape)} and {tuple(image.shape)}")
    H, W = image.shape[2], image.shape[3]
    if tuple(depth.shape) != (n, H, W) or tuple(alpha.shape) != (n, H, W):
        raise ValueError(f"tsdf_integrate: depth {tuple(depth.shape)} and alpha {tuple(alpha.shape)} must be "
                         f"[{n}, {H}, {W}]")
    trunc = 16.0 / (R - 1) if sdf_trunc is None else float(sdf_trunc)
    if not (np.isfinite(trunc) and trunc > 0) or not 0 < alpha_thresh <= 1:
        raise ValueError(f"tsdf_integrate: sdf_trunc must be finite and > 0 and alpha_thresh in (0, 1] (got "
                         f"{sdf_trunc!r}, {alpha_thresh!r})")
    dev = volume["tsdf_sum"].device
    cams = [f32(t.to(dev)) for t in (c2ws, fxfycxcy, image, depth, alpha)]
    alloc = Alloc(dev, _SCRATCH, (str(dev), "tsdf_cams"), cached=1)
    with torch.cuda.device(dev):
        check(_lib.lib().dgs_tsdf_integrate(n, *(t.data_ptr() for t in cams[:2]), H, W,
                                            *(t.data_ptr() for t in cams[2:]), volume["lin"].data_ptr(), R, trunc,
                                            float(alpha_thresh), *(volume[k].data_ptr() for k in
                                                                   ("tsdf_sum", "weight", "rgb_sum", "rgb_weight")),
                                            alloc.cb, None, stream(dev)))
    return volume


def tsdf_fusion(xyz, features, scaling, rotation, opacity, scaling_modifier=None, resolution=256, num_views=100,
                image_size=512, c2ws=None, fxfycxcy=None, sdf_trunc=None, alpha_thresh=0.5, max_arena_bytes=None,
                stats=None):
    """TSDF fusion of the Gaussians' own renders -> the volume (`tsdf_volume`'s dict, CUDA tensors, with the frame
    mesh_center / mesh_scale of `mesh_frame`).  The Gaussians (raw xyz [P, 3], features [P, (d + 1)^2, 3], scaling,
    rotation, opacity, CUDA tensors) are rendered in the normalised frame, centres (xyz - mesh_center) * mesh_scale and
    log-scales + log(mesh_scale), by the batched rasterizer (depth and alpha maps included) from the `sphere_cameras`
    (num_views, image_size), or from the caller's world-space c2ws [n, 4, 4] / fxfycxcy [n, 4] at image_size (an int or
    (H, W)), mapped into that frame on the host in fp64.  The views go in chunks sized as render_frames sizes them
    (max_arena_bytes, default raster.FRAMES_ARENA_BYTES), each fused (`tsdf_integrate` with sdf_trunc and alpha_thresh)
    and dropped.  `stats`, a dict, receives "render_ms" and "integrate_ms" (device time, summed over the chunks)."""
    from . import raster
    from .cameras import sphere_cameras
    _tsdf_resolution(resolution)
    if (c2ws is None) != (fxfycxcy is None):
        raise ValueError("tsdf_fusion: give both c2ws and fxfycxcy, or neither")
    H, W = (image_size, image_size) if np.ndim(image_size) == 0 else tuple(image_size)
    if int(H) != H or int(W) != W or H < 1 or W < 1:
        raise ValueError(f"tsdf_fusion: image_size must be a positive int or (H, W) (got {image_size!r})")
    H, W = int(H), int(W)
    if c2ws is None:
        if H != W or int(num_views) != num_views or num_views < 1:
            raise ValueError(f"tsdf_fusion: the sphere cameras need num_views >= 1 and a square image (got "
                             f"{num_views!r}, {image_size!r})")
        K, c2w = sphere_cameras(int(num_views), H)
    else:
        as64 = lambda a: np.array(a.detach().cpu().numpy() if torch.is_tensor(a) else a, np.float64)  # noqa: E731
        c2w, K = as64(c2ws), as64(fxfycxcy)
        if c2w.ndim != 3 or c2w.shape[1:] != (4, 4) or K.shape != (len(c2w), 4) or len(c2w) == 0:
            raise ValueError(f"tsdf_fusion: expected c2ws [n, 4, 4] and fxfycxcy [n, 4] with n >= 1, got {c2w.shape} "
                             f"and {K.shape}")
    if sdf_trunc is not None and not (np.isfinite(sdf_trunc) and sdf_trunc > 0) or not 0 < alpha_thresh <= 1:
        raise ValueError(f"tsdf_fusion: sdf_trunc must be finite and > 0 and alpha_thresh in (0, 1] (got "
                         f"{sdf_trunc!r}, {alpha_thresh!r})")
    if not xyz.is_cuda:
        raise _lib.DgsError("tsdf_fusion needs CUDA tensors (no CPU path)")
    dev = xyz.device
    xyz, features, scaling, rotation, opacity = (f32(t) for t in (xyz, features, scaling, rotation, opacity))
    P = xyz.shape[0]
    center, scale = mesh_frame(xyz)
    volume = tsdf_volume(resolution, dev, center, scale)
    if c2ws is not None:  # world -> normalised: the rotation stays, the centre moves; pixels are scale-invariant
        c2w[:, :3, 3] = (c2w[:, :3, 3] - center.double().cpu().numpy()) * scale
    V = len(c2w)
    C2W = torch.tensor(c2w, dtype=torch.float32, device=dev)
    FX = torch.tensor(K, dtype=torch.float32, device=dev)
    budget = raster.FRAMES_ARENA_BYTES if max_arena_bytes is None else max_arena_bytes
    n = raster.frames_chunk_views(V, max(P, 1), H, W, budget)
    gs = ((xyz - center) * scale, features, scaling + math.log(scale), rotation, opacity)
    cache, ev = {}, []
    with torch.cuda.device(dev):
        for v0 in range(0, V, n):
            v1 = min(V, v0 + n)
            ev.append([torch.cuda.Event(enable_timing=True) for _ in range(3)] if stats is not None else None)
            if ev[-1]:
                ev[-1][0].record()
            if P:
                image, depth, alpha, state = raster.render_batch_forward(
                    *(t[None] for t in gs), H, W, C2W[None, v0:v1], FX[None, v0:v1], scaling_modifier,
                    arena_cache=cache, aux=True)
                del state  # inference only: nothing is kept for a backward
                image, depth, alpha = image[0], depth[0, :, 0], alpha[0, :, 0]
            else:  # no Gaussians: every pixel is background
                image = torch.ones(v1 - v0, 3, H, W, device=dev)
                depth = alpha = torch.zeros(v1 - v0, H, W, device=dev)
            if ev[-1]:
                ev[-1][1].record()
            tsdf_integrate(volume, C2W[v0:v1], FX[v0:v1], image, depth, alpha, sdf_trunc, alpha_thresh)
            if ev[-1]:
                ev[-1][2].record()
            del image, depth, alpha
    if stats is not None:
        torch.cuda.synchronize(dev)
        stats["render_ms"] = sum(a.elapsed_time(b) for a, b, _ in ev)
        stats["integrate_ms"] = sum(b.elapsed_time(c) for _, b, c in ev)
    return volume


def _timed(stats, key, dev, fn):
    """fn() with its device time in stats[key] when stats is a dict"""
    if stats is None:
        return fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.device(dev):
        a.record()
        out = fn()
        b.record()
    b.synchronize()
    stats[key] = a.elapsed_time(b)
    return out


def tsdf_mesh(volume, stats=None):
    """The surface of a TSDF volume (dgs_tsdf_extract): marching cubes of the mean tsdf_sum / weight at 0 over its
    observed points -> (vertices fp32 [V, 3] in the volume's grid frame, mapped by v / (R - 1) * 2 - 1 as
    extract_mesh maps them, faces int64 [F, 3] oriented outwards), CUDA tensors.  Every vertex is referenced and no face
    touches an unobserved point.  `stats`, a dict, receives "extract_ms"."""
    dev, R = volume["tsdf_sum"].device, volume["lin"].numel()
    alloc = Alloc(dev)  # no cache: the last two buffers are the caller's output
    vp, fp = C.c_void_p(), C.c_void_p()
    nv, nf = C.c_longlong(0), C.c_longlong(0)

    def run():
        check(_lib.lib().dgs_tsdf_extract(volume["tsdf_sum"].data_ptr(), volume["weight"].data_ptr(), R, alloc.cb, None,
                                          C.byref(vp), C.byref(fp), C.byref(nv), C.byref(nf), stream(dev)))
    _timed(stats, "extract_ms", dev, run)
    v, f = _mesh_out(False, dev, alloc, nv.value, nf.value)
    alloc.tensors.clear()  # the scratch goes now; the outputs are views that keep their own buffers
    alloc.tensor = None
    return (v.double() / (R - 1.0) * 2 - 1).float(), f


def tsdf_colors(volume, vertices, stats=None):
    """Colours of vertices (float [V, 3], in the volume's grid frame) from a TSDF volume (dgs_tsdf_colors): the
    trilinear blend over the containing cell's coloured corners of their mean colour -> rgb float32 [V, 3] in [0, 1],
    white where no corner is coloured.  numpy input returns numpy, CUDA tensors return CUDA tensors.  `stats`, a dict,
    receives "colors_ms"."""
    is_numpy = isinstance(vertices, np.ndarray)
    if vertices.ndim != 2 or vertices.shape[1] != 3:
        raise ValueError(f"tsdf_colors: expected vertices [V, 3], got {tuple(vertices.shape)}")
    dev, R = volume["rgb_sum"].device, volume["lin"].numel()
    v = torch.as_tensor(np.ascontiguousarray(vertices, np.float32) if is_numpy else vertices).to(dev)
    v = f32(v)
    rgb = torch.empty(len(v), 3, dtype=torch.float32, device=dev)

    def run():
        check(_lib.lib().dgs_tsdf_colors(volume["rgb_sum"].data_ptr(), volume["rgb_weight"].data_ptr(), R, v.data_ptr(),
                                         len(v), rgb.data_ptr(), stream(dev)))
    _timed(stats, "colors_ms", dev, run)
    return rgb.cpu().numpy() if is_numpy else rgb


class Mesh:
    """The triangle mesh extract_mesh returns: `vertices` float32 [V, 3] and `faces` int64 [F, 3] numpy arrays (the
    attribute names of trimesh.Trimesh), and optionally `vertex_colors` (float32 [V, 3] in [0, 1]) and
    `vertex_normals` (float32 [V, 3]), as `vertex_colors` computes them."""

    def __init__(self, vertices, faces, vertex_colors=None, vertex_normals=None):
        self.vertices = np.ascontiguousarray(vertices, dtype=np.float32).reshape(-1, 3)
        self.faces = np.ascontiguousarray(faces, dtype=np.int64).reshape(-1, 3)
        self.vertex_colors = self._per_vertex("vertex_colors", vertex_colors)
        self.vertex_normals = self._per_vertex("vertex_normals", vertex_normals)

    def _per_vertex(self, name, a):
        if a is None:
            return None
        a = np.ascontiguousarray(a, dtype=np.float32)
        if a.shape != self.vertices.shape:
            raise ValueError(f"Mesh: {name} must be [{len(self.vertices)}, 3], got {a.shape}")
        return a

    def export(self, path):
        """Writes binary little-endian PLY (.ply) or Wavefront OBJ (.obj), by suffix, with the colours and normals when
        the mesh has them: PLY vertex properties `nx ny nz` (float) and `red green blue` (uchar, (c * 255) clipped to
        [0, 255] and truncated, as GaussianModel.save_ply quantises), OBJ `v x y z r g b` lines (float colours), `vn`
        lines and `f a//a b//b c//c` faces.  -> path"""
        ext = os.path.splitext(path)[1].lower()
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        V, F = len(self.vertices), len(self.faces)
        rgb, nrm = self.vertex_colors, self.vertex_normals
        if ext == ".ply":
            props = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
            if nrm is not None:
                props += [("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4")]
            if rgb is not None:
                props += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
            ply_type = {"<f4": "float", "u1": "uchar"}
            header = ("ply\nformat binary_little_endian 1.0\n"
                      f"element vertex {V}\n" + "".join(f"property {ply_type[t]} {n}\n" for n, t in props) +
                      f"element face {F}\nproperty list uchar int vertex_indices\nend_header\n")
            vert = np.empty(V, dtype=props)
            for k, n in enumerate("xyz"):
                vert[n] = self.vertices[:, k]
            if nrm is not None:
                for k, n in enumerate(("nx", "ny", "nz")):
                    vert[n] = nrm[:, k]
            if rgb is not None:
                q = (rgb * 255.0).clip(0.0, 255.0).astype(np.uint8)
                for k, n in enumerate(("red", "green", "blue")):
                    vert[n] = q[:, k]
            face = np.empty(F, dtype=[("n", "u1"), ("v", "<i4", (3,))])
            face["n"], face["v"] = 3, self.faces
            with open(path, "wb") as fh:
                fh.write(header.encode("ascii"))
                fh.write(vert.tobytes())
                fh.write(face.tobytes())
        elif ext == ".obj":
            with open(path, "w") as fh:
                if rgb is None:
                    np.savetxt(fh, self.vertices, fmt="v %.9g %.9g %.9g")
                else:
                    np.savetxt(fh, np.concatenate([self.vertices, rgb], 1), fmt="v %.9g %.9g %.9g %.9g %.9g %.9g")
                if nrm is None:
                    np.savetxt(fh, self.faces + 1, fmt="f %d %d %d")
                else:
                    np.savetxt(fh, nrm, fmt="vn %.9g %.9g %.9g")
                    np.savetxt(fh, np.repeat(self.faces + 1, 2, axis=1), fmt="f %d//%d %d//%d %d//%d")
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


def parser():
    ap = argparse.ArgumentParser(description="Extract a mesh from a Gaussian PLY (GaussianModel.extract_mesh)")
    ap.add_argument("ply", help="Gaussians, as written by GaussianModel.save_ply")
    ap.add_argument("out", help="output mesh, .obj or .ply")
    ap.add_argument("--resolution", type=int, default=256, help="grid points per axis (default 256)")
    ap.add_argument("--density-thresh", type=float, default=0.005, help="iso value of the opacity field (default 0.005)")
    ap.add_argument("--decimate-target", type=int, default=None, metavar="N",
                    help="decimate to at most N faces (quadric edge collapse; default: the raw marching-cubes mesh)")
    ap.add_argument("--clean", action="store_true",
                    help="clean first (merge close vertices, drop duplicate / null faces and small components, repair "
                         "non-manifold parts), as the reference's clean_mesh without remeshing")
    ap.add_argument("--remesh", type=float, nargs="?", const=0.015, default=None, metavar="LEN",
                    help="remesh isotropically to edges of about LEN (default 0.015), after --clean when both are given")
    surface = ap.add_mutually_exclusive_group()
    surface.add_argument("--poisson", type=int, nargs="?", const=9, default=None, metavar="DEPTH",
                         help="reconstruct by screened Poisson from the Gaussians' centres and shortest axes at DEPTH "
                              "(default 9) instead of marching the opacity field (--resolution and --density-thresh are "
                              "then unused)")
    surface.add_argument("--tsdf", action="store_true",
                         help="fuse the Gaussians' depth renders from 100 views around them into a TSDF at --resolution "
                              "points per axis and march its zero crossing, instead of the opacity field "
                              "(--density-thresh is then unused; --colors then colours from the renders)")
    ap.add_argument("--colors", action="store_true",
                    help="colour the final vertices from the Gaussians (at the SH degree of the file's f_rest_* "
                         "properties) and write the colours and vertex normals")
    return ap


def ply_sh_degree(path):
    """The SH degree of a Gaussian PLY from its number of f_rest_* properties (0, 9, 24 or 45)"""
    from .renderer import _read_ply_vertices
    n = sum(k.startswith("f_rest_") for k in _read_ply_vertices(path).dtype.names)
    degrees = {0: 0, 9: 1, 24: 2, 45: 3}
    if n not in degrees:
        raise ValueError(f"{path}: {n} f_rest_* properties is no SH degree of 0 to 3 (expected 0, 9, 24 or 45)")
    return degrees[n]


def _postprocess(args):
    """-> extract_mesh keyword arguments for the --clean / --remesh / --decimate-target flags"""
    if args.remesh is not None:
        return dict(postprocess=lambda v, f, target: _chain(v, f, args.clean, args.remesh, target),
                    decimate_target=args.decimate_target)
    if args.clean and args.decimate_target is not None:
        return dict(postprocess=clean_then_decimate, decimate_target=args.decimate_target)
    if args.clean:
        return dict(postprocess=lambda v, f, _target: clean(v, f))
    if args.decimate_target is not None:
        return dict(postprocess=decimate, decimate_target=args.decimate_target)
    return {}


def main(argv=None):
    args = parser().parse_args(argv)
    from .renderer import GaussianModel
    gm = GaussianModel(ply_sh_degree(args.ply) if args.colors else 0)
    gm.load_ply(args.ply)
    method = dict(method="field")
    if args.poisson is not None:
        method = dict(method="poisson", depth=args.poisson)
    elif args.tsdf:
        method = dict(method="tsdf")
    mesh = gm.to("cuda").extract_mesh(density_thresh=args.density_thresh, resolution=args.resolution,
                                      vertex_colors=args.colors, **method, **_postprocess(args))
    mesh.export(args.out)
    print(f"{args.out}: {len(mesh.vertices)} vertices, {len(mesh.faces)} faces")


if __name__ == "__main__":
    main()
