"""Torch-facing host side of the rasterizer C ABI.

`rasterize_gaussians`, `rasterize_gaussians_backward`, `mark_visible` have the exact signatures and
return tuples of the reference's pybind module `_C` (DGR/ext.cpp:15-19, DGR/rasterize_points.cu:35-217);
torch only supplies device memory (the arena allocator callbacks) and the current stream.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import Alloc, DgsError, RasterArgs, RenderAux, RenderBatchArgs, RenderMse, check, f32, ptr, stream


LAST_NUM_RENDERED = None  # instance count R of the most recent batched forward (bench/roofline bookkeeping)


def _require_cuda(t, name):
    if not t.is_cuda:
        raise _lib.DgsError(f"{name} must be a CUDA tensor: libdgs_b200 has no CPU path")


def rasterize_gaussians(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                        viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree,
                        campos, prefiltered, debug):
    """-> (num_rendered, out_color[3,H,W], radii[P] int32, geomBuffer, binningBuffer, imgBuffer)
    (RasterizeGaussiansCUDA, rasterize_points.cu:35-115)."""
    if means3D.ndimension() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")  # rasterize_points.cu:57-59
    _require_cuda(means3D, "means3D")
    dev = means3D.device
    P, H, W = means3D.size(0), int(image_height), int(image_width)
    with torch.cuda.device(dev):
        out_color = torch.zeros(3, H, W, dtype=torch.float32, device=dev)
        radii = torch.zeros(P, dtype=torch.int32, device=dev)
        geom, binning, img = Alloc(dev), Alloc(dev), Alloc(dev)
        if P == 0:
            return 0, out_color, radii, geom.tensor, binning.tensor, img.tensor
        keep = [f32(t) for t in (background, means3D, sh, colors, opacity, scales, rotations, cov3D_precomp,
                                 viewmatrix, projmatrix, campos)]
        bg, m3, sh_, col, op, sc, ro, cov, vm, pm, cp = keep
        M = sh_.size(1) if (sh_ is not None and sh_.numel()) else 0
        a = RasterArgs(P=P, D=int(degree), M=M, W=W, H=H, background=ptr(bg), means3D=ptr(m3), shs=ptr(sh_),
                       colors_precomp=ptr(col), opacities=ptr(op), scales=ptr(sc), rotations=ptr(ro),
                       cov3D_precomp=ptr(cov), viewmatrix=ptr(vm), projmatrix=ptr(pm), campos=ptr(cp),
                       scale_modifier=float(scale_modifier), tan_fovx=float(tan_fovx), tan_fovy=float(tan_fovy),
                       prefiltered=int(bool(prefiltered)), debug=int(bool(debug)))
        R = C.c_int(0)
        check(_lib.lib().dgs_raster_forward(C.byref(a), geom.cb, None, binning.cb, None, img.cb, None,
                                            out_color.data_ptr(), radii.data_ptr(), C.byref(R), stream(dev)))
    return R.value, out_color, radii, geom.tensor, binning.tensor, img.tensor


def rasterize_gaussians_backward(background, means3D, radii, colors, scales, rotations, scale_modifier,
                                 cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color, sh,
                                 degree, campos, geomBuffer, R, binningBuffer, imageBuffer, debug,
                                 opacities=None):
    """-> (dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations)
    (RasterizeGaussiansBackwardCUDA, rasterize_points.cu:117-196).  `opacities` is unused (the forward
    state already holds them), kept only so callers may pass it."""
    _require_cuda(means3D, "means3D")
    dev = means3D.device
    P = means3D.size(0)
    H, W = dL_dout_color.size(1), dL_dout_color.size(2)
    M = sh.size(1) if (sh is not None and sh.numel()) else 0
    with torch.cuda.device(dev):
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)  # noqa: E731
        dm3, dm2, dcol, dcon = z(P, 3), z(P, 3), z(P, 3), z(P, 2, 2)
        dop, dcov, dsh, dsc, dro = z(P, 1), z(P, 6), z(P, M, 3), z(P, 3), z(P, 4)
        if P != 0:
            keep = [f32(t) for t in (background, means3D, sh, colors, scales, rotations, cov3D_precomp, viewmatrix,
                                     projmatrix, campos, dL_dout_color)]
            bg, m3, sh_, col, sc, ro, cov, vm, pm, cp, dpix = keep
            a = RasterArgs(P=P, D=int(degree), M=M, W=W, H=H, background=ptr(bg), means3D=ptr(m3), shs=ptr(sh_),
                           colors_precomp=ptr(col), opacities=None, scales=ptr(sc), rotations=ptr(ro),
                           cov3D_precomp=ptr(cov), viewmatrix=ptr(vm), projmatrix=ptr(pm), campos=ptr(cp),
                           scale_modifier=float(scale_modifier), tan_fovx=float(tan_fovx),
                           tan_fovy=float(tan_fovy), prefiltered=0, debug=int(bool(debug)))
            check(_lib.lib().dgs_raster_backward(
                C.byref(a), int(R), ptr(radii), ptr(geomBuffer), ptr(binningBuffer), ptr(imageBuffer),
                dpix.data_ptr(), dm2.data_ptr(), dcon.data_ptr(), dop.data_ptr(), dcol.data_ptr(), dm3.data_ptr(),
                dcov.data_ptr(), ptr(dsh), dsc.data_ptr(), dro.data_ptr(), stream(dev)))
    return dm2, dcol, dop, dm3, dcov, dsh, dsc, dro


def mark_visible(means3D, viewmatrix, projmatrix):
    """-> bool[P] (markVisible, rasterize_points.cu:198-217)."""
    _require_cuda(means3D, "means3D")
    dev = means3D.device
    P = means3D.size(0)
    present = torch.zeros(P, dtype=torch.bool, device=dev)
    if P:
        with torch.cuda.device(dev):
            m3, vm, pm = f32(means3D), f32(viewmatrix), f32(projmatrix)
            check(_lib.lib().dgs_mark_visible(P, m3.data_ptr(), vm.data_ptr(), pm.data_ptr(), present.data_ptr(),
                                              stream(dev)))
    return present


# ------------------------------------------------------------------------------------------------
# batched renderer
# ------------------------------------------------------------------------------------------------
def _batch_args(xyz, features, scaling, rotation, opacity, C2W, fxfycxcy, H, W, scale_modifier, debug=False,
                near_log2=0):
    B, P = xyz.shape[0], xyz.shape[1]
    V = C2W.shape[1]
    M = features.shape[2]
    D = int(round(M ** 0.5)) - 1  # gs_core.py:978
    a = RenderBatchArgs(B=B, V=V, P=P, M=M, D=D, W=int(W), H=int(H), xyz=xyz.data_ptr(), features=features.data_ptr(),
                        scaling=scaling.data_ptr(), rotation=rotation.data_ptr(), opacity=opacity.data_ptr(),
                        c2w=C2W.data_ptr(), fxfycxcy=fxfycxcy.data_ptr(),
                        scale_modifier=1.0 if scale_modifier is None else float(scale_modifier), debug=int(debug),
                        near_log2=int(near_log2))
    a.bg[0] = a.bg[1] = a.bg[2] = 1.0  # render_opencv_cam's default bg_color, gs_core.py:880
    return a


def render_batch_forward(xyz, features, scaling, rotation, opacity, H, W, C2W, fxfycxcy, scale_modifier=None,
                         arena_cache=None, near_log2=None, mse_target=None, mse_loss_sum=None, aux=False):
    """All (sample, view) pairs in one launch set -> (images [B,V,3,H,W] fp32, state).
    mse_target [B,V,3|4,H,W] + mse_loss_sum (fp64 [B], zeroed by the caller): the blend kernel also adds
    sum (render - target)^2 of every sample into mse_loss_sum (dgs_render_mse).
    aux=True: also the depth and alpha maps of the same blend -> (images, depth [B,V,1,H,W], alpha [B,V,1,H,W], state),
    depth = sum_i w_i z_i (accumulated view-space depth; expected depth = depth / alpha), alpha = 1 - final T
    (dgs_render_aux).  When the batch holds more than
    2^31-1 instances (e.g. a random-init denoiser at 512x512: ~6e8 per view) the views are rendered in halves,
    recursively -- the reference renders one view per call anyway (gs_core.py:990-1001); `state` then carries one
    sub-state per chunk and render_batch_backward sums the chunks' gradients."""
    try:
        return _render_batch_forward_one(xyz, features, scaling, rotation, opacity, H, W, C2W, fxfycxcy, scale_modifier,
                                         arena_cache, near_log2, mse_target, mse_loss_sum, aux)
    except DgsError as e:
        V = C2W.shape[1]
        if "exceeds 2^31-1" not in str(e) or V < 2:
            raise
    global LAST_NUM_RENDERED
    outs, subs, total = [], [], 0
    for ci, (v0, v1) in enumerate(((0, V // 2), (V // 2, V))):
        sub_cache = None if arena_cache is None else arena_cache.setdefault(("views", ci), {})
        if mse_loss_sum is not None and ci == 0:
            mse_loss_sum.zero_()  # the failed whole-batch attempt may have counted some tiles already
        *o, st = render_batch_forward(xyz, features, scaling, rotation, opacity, H, W, C2W[:, v0:v1].contiguous(),
                                      fxfycxcy[:, v0:v1].contiguous(), scale_modifier, sub_cache, near_log2,
                                      None if mse_target is None else mse_target[:, v0:v1].contiguous(), mse_loss_sum,
                                      aux)
        outs.append(o)
        subs.append((v0, v1, st))
        total += st["R"]
    LAST_NUM_RENDERED = total
    return (*(torch.cat(maps, dim=1) for maps in zip(*outs)), dict(sub=subs, R=total, tensors=subs[0][2]["tensors"]))


def _render_batch_forward_one(xyz, features, scaling, rotation, opacity, H, W, C2W, fxfycxcy, scale_modifier=None,
                              arena_cache=None, near_log2=None, mse_target=None, mse_loss_sum=None, aux=False):
    """One launch set over every (sample, view) pair.  `arena_cache` (a dict): re-use grow-only arenas across calls; the caller must not hand the same dict to another
    forward while this call's state is still needed (renderer.py keeps one dict for inference and a pool of dicts for
    differentiated forwards); stream order makes the re-use safe."""
    _require_cuda(xyz, "xyz")
    dev = xyz.device
    tens = [f32(t) for t in (xyz, features, scaling, rotation, opacity, C2W, fxfycxcy)]
    B, V = tens[5].shape[0], tens[5].shape[1]
    with torch.cuda.device(dev):
        out = torch.empty(B, V, 3, int(H), int(W), dtype=torch.float32, device=dev)
        geom, binning, img = (Alloc(dev, arena_cache, k) for k in ("geom", "binning", "img"))
        # two-phase binning: phase A = the nearest 1/2^k of every view's Gaussians (0 = single pass, -1 = adaptive)
        near_log2 = -1 if near_log2 is None else near_log2
        a = _batch_args(*tens, H, W, scale_modifier, near_log2=near_log2)
        R = C.c_longlong(0)
        chunks = (C.c_longlong * 2)(0, 0)
        mse = None
        if mse_target is not None:
            mse_target = f32(mse_target)
            if tuple(mse_target.shape) not in ((B, V, 3, int(H), int(W)), (B, V, 4, int(H), int(W))):
                raise ValueError(f"mse target shape {tuple(mse_target.shape)} != [{B},{V},3|4,{H},{W}]")
            if mse_loss_sum.dtype != torch.float64 or mse_loss_sum.numel() != B:
                raise ValueError("mse_loss_sum must be a float64 tensor with one entry per sample")
            mse = RenderMse(target=mse_target.data_ptr(), target_channels=mse_target.shape[2],
                            loss_sum=mse_loss_sum.data_ptr(), coef=None, images=None)
        maps, aux_args = (), None
        if aux:
            maps = tuple(torch.empty(B, V, 1, int(H), int(W), dtype=torch.float32, device=dev) for _ in range(2))
            aux_args = RenderAux(depth=maps[0].data_ptr(), alpha=maps[1].data_ptr(), dL_ddepth=None, dL_dalpha=None)
        check(_lib.lib().dgs_render_batch_forward(C.byref(a), geom.cb, None, binning.cb, None, img.cb, None, out.data_ptr(),
                                                  C.byref(R), chunks, None if mse is None else C.byref(mse),
                                                  None if aux_args is None else C.byref(aux_args), stream(dev)))
    global LAST_NUM_RENDERED
    LAST_NUM_RENDERED = R.value
    state = dict(mse_target=mse_target, images=out if mse_target is not None else None, tensors=tens, geom=geom.tensor, binning=binning.tensors[0],
                 binning_b=binning.tensors[1] if len(binning.tensors) > 1 else None, img=img.tensor, R=R.value,
                 chunks=(int(chunks[0]), int(chunks[1])), H=int(H), W=int(W), scale_modifier=scale_modifier,
                 near_log2=near_log2)
    return (out, *maps, state)


# Default budget of render_frames' geometry and image arenas, per chunk of views.  The geometry state is about 100 B per
# (view, Gaussian): 2 GiB holds about 20 views of a million Gaussians, plenty to fill the GPU, where a whole 150-view
# turntable would take 15 GB of a card that other work may share.  (The binning arena, which grows with the chunk's
# instance count, comes on top.)
FRAMES_ARENA_BYTES = 2 << 30


def frames_chunk_views(V, P, H, W, max_arena_bytes=FRAMES_ARENA_BYTES):
    """Views per render_frames call: the largest n <= V whose geometry and image arenas for n views of P Gaussians at
    H x W fit in max_arena_bytes; at least 1.  The binning arena depends on the instance count and is not part of it."""
    L = _lib.lib()
    fits = lambda n: L.dgs_raster_geom_bytes(n, P) + L.dgs_raster_image_bytes(n, W, H) <= max_arena_bytes  # noqa: E731
    lo, hi = 1, V
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if fits(mid) else (lo, mid - 1)
    return lo


def render_frames(xyz, features, scaling, rotation, opacity, H, W, C2W, fxfycxcy, scale_modifier=None,
                  max_arena_bytes=FRAMES_ARENA_BYTES, arena_cache=None, near_log2=None):
    """Video frames of every (sample, view) pair -> uint8 [B,V,H,W,3] on xyz's device: each value is the reference's
    (image * 255).clip(0, 255).astype(uint8) of render_batch_forward's image for the same inputs (gs_core.py:1215-1216),
    written by the blend kernel itself (dgs_render_frames), with no fp32 image in between.  Inference only: nothing is
    kept for a backward.

    The views of each sample are rendered frames_chunk_views(V, P, H, W, max_arena_bytes) at a time, into their slice of
    the one output, so the arenas do not grow with the frame count; every chunk re-uses one grow-only arena set
    (`arena_cache`, a dict; a fresh one when None).  A chunk of more than 2^31-1 instances is rendered in halves, as
    render_batch_forward does.  With no Gaussians (P = 0) the frames are black: the reference's rasterizer returns its
    zero-filled image for an empty model, not the background."""
    _require_cuda(xyz, "xyz")
    dev = xyz.device
    tens = [f32(t) for t in (xyz, features, scaling, rotation, opacity, C2W, fxfycxcy)]
    B, V, P = tens[5].shape[0], tens[5].shape[1], tens[0].shape[1]
    H, W = int(H), int(W)
    near_log2 = -1 if near_log2 is None else near_log2
    cache = {} if arena_cache is None else arena_cache
    n = frames_chunk_views(V, P, H, W, max_arena_bytes)
    total = 0
    with torch.cuda.device(dev):
        frames = torch.zeros(B, V, H, W, 3, dtype=torch.uint8, device=dev)
        b, v0 = 0, 0
        while b < B:
            v1 = min(V, v0 + n)
            cams = (t[b:b + 1, v0:v1] for t in tens[5:])
            a = _batch_args(*(t[b:b + 1] for t in tens[:5]), *cams, H, W, scale_modifier, near_log2=near_log2)
            geom, binning, img = (Alloc(dev, cache, k) for k in ("geom", "binning", "img"))
            R = C.c_longlong(0)
            try:
                check(_lib.lib().dgs_render_frames(C.byref(a), geom.cb, None, binning.cb, None, img.cb, None,
                                                   frames[b, v0:v1].data_ptr(), C.byref(R), stream(dev)))
            except DgsError as e:
                if "exceeds 2^31-1" not in str(e) or v1 - v0 < 2:
                    raise
                n = (v1 - v0) // 2  # this chunk again, and the ones after it, in halves
                continue
            total += R.value
            b, v0 = (b + 1, 0) if v1 == V else (b, v1)
    global LAST_NUM_RENDERED
    LAST_NUM_RENDERED = total
    return frames


def _view_slice(t, v0, v1):
    return None if t is None else t[:, v0:v1]


def render_batch_backward(state, grad_images, arena_cache=None, mse_coef=None, grad_depth=None, grad_alpha=None):
    """-> (d_xyz, d_features, d_scaling, d_rotation, d_opacity), re-using the forward's sorted lists.
    mse_coef (fp32 [B], device): dL/dpix += mse_coef[b] * (render - target) is formed inside the blend-backward kernel
    (the forward must have been given mse_target); grad_images may then be None.
    grad_depth / grad_alpha ([B,V,1,H,W], either may be None): upstream gradients of the aux=True forward's depth and alpha
    maps (dgs_render_aux); without them the plain kernels run."""
    if "sub" in state:  # view-chunked forward: the per-Gaussian gradients are sums over views
        total = None
        for ci, (v0, v1, st) in enumerate(state["sub"]):
            sub_cache = None if arena_cache is None else arena_cache.setdefault(("views", ci), {})
            g = render_batch_backward(st, _view_slice(grad_images, v0, v1), sub_cache, mse_coef,
                                      _view_slice(grad_depth, v0, v1), _view_slice(grad_alpha, v0, v1))
            total = g if total is None else tuple(a + b for a, b in zip(total, g))
        return total
    tens = state["tensors"]
    dev = tens[0].device
    g = f32(grad_images)
    gd, ga = f32(grad_depth), f32(grad_alpha)
    if g is None and mse_coef is None and gd is None and ga is None:
        raise ValueError("render_batch_backward needs grad_images, mse_coef, grad_depth or grad_alpha")
    aux = None
    if gd is not None or ga is not None:
        shape = (tens[0].shape[0], tens[5].shape[1], 1, state["H"], state["W"])
        for name, t in (("grad_depth", gd), ("grad_alpha", ga)):
            if t is not None and tuple(t.shape) != shape:
                raise ValueError(f"{name} shape {tuple(t.shape)} != {list(shape)}")
        aux = RenderAux(depth=None, alpha=None, dL_ddepth=ptr(gd), dL_dalpha=ptr(ga))
    mse = None
    if mse_coef is not None:
        if state.get("mse_target") is None:
            raise ValueError("mse_coef given but the forward ran without mse_target")
        mse_coef = f32(mse_coef)
        mse = RenderMse(target=state["mse_target"].data_ptr(), target_channels=state["mse_target"].shape[2], loss_sum=None,
                        coef=mse_coef.data_ptr(), images=state["images"].data_ptr())
    with torch.cuda.device(dev):
        outs = [torch.empty_like(t) for t in tens[:5]]
        scratch = Alloc(dev, arena_cache, "bwd_scratch")
        a = _batch_args(*tens, state["H"], state["W"], state["scale_modifier"], near_log2=state["near_log2"])
        chunks = (C.c_longlong * 2)(*state["chunks"])
        check(_lib.lib().dgs_render_batch_backward(
            C.byref(a), state["R"], chunks, ptr(state["geom"]), ptr(state["binning"]), ptr(state["binning_b"]),
            ptr(state["img"]), None if g is None else g.data_ptr(), None if mse is None else C.byref(mse),
            None if aux is None else C.byref(aux), outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(),
            outs[3].data_ptr(), outs[4].data_ptr(), scratch.cb, None, stream(dev)))
    return tuple(outs)


def export_state(n_views, P, W, H, R, geom, binning, img):
    """Debug/test introspection of the opaque arenas -> dict of torch tensors."""
    dev = geom.device
    N = n_views * P
    tiles = n_views * ((W + 15) // 16) * ((H + 15) // 16)
    o = dict(xy=torch.zeros(N, 2, device=dev), depth=torch.zeros(N, device=dev),
             conic_opacity=torch.zeros(N, 4, device=dev), rgb=torch.zeros(N, 3, device=dev),
             tiles_touched=torch.zeros(N, dtype=torch.int32, device=dev),
             point_list=torch.zeros(max(R, 1), dtype=torch.int32, device=dev),
             ranges=torch.zeros(tiles, 2, dtype=torch.int32, device=dev),
             final_T=torch.zeros(n_views * H * W, device=dev),
             n_contrib=torch.zeros(n_views * H * W, dtype=torch.int32, device=dev))
    with torch.cuda.device(dev):
        check(_lib.lib().dgs_raster_export_state(
            n_views, P, W, H, R, ptr(geom), ptr(binning), ptr(img), o["xy"].data_ptr(), o["depth"].data_ptr(),
            o["conic_opacity"].data_ptr(), o["rgb"].data_ptr(), o["tiles_touched"].data_ptr(),
            o["point_list"].data_ptr(), o["ranges"].data_ptr(), o["final_T"].data_ptr(), o["n_contrib"].data_ptr(),
            stream(dev)))
    o["point_list"] = o["point_list"][:R]
    return o
