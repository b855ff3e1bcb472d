"""ctypes binding of libdgs_b200.so (include/dgs_b200.h).  There is NO fallback: if the CUDA
library is missing, importing any compute entry point raises."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libdgs_b200.so")

ALLOC_FN = C.CFUNCTYPE(C.c_void_p, C.c_size_t, C.c_void_p)


class RasterArgs(C.Structure):
    _fields_ = [("P", C.c_int), ("D", C.c_int), ("M", C.c_int), ("W", C.c_int), ("H", C.c_int),
                ("background", C.c_void_p), ("means3D", C.c_void_p), ("shs", C.c_void_p),
                ("colors_precomp", C.c_void_p), ("opacities", C.c_void_p), ("scales", C.c_void_p),
                ("rotations", C.c_void_p), ("cov3D_precomp", C.c_void_p), ("viewmatrix", C.c_void_p),
                ("projmatrix", C.c_void_p), ("campos", C.c_void_p), ("scale_modifier", C.c_float),
                ("tan_fovx", C.c_float), ("tan_fovy", C.c_float), ("prefiltered", C.c_int),
                ("debug", C.c_int)]


class RenderBatchArgs(C.Structure):
    _fields_ = [("B", C.c_int), ("V", C.c_int), ("P", C.c_int), ("M", C.c_int), ("D", C.c_int),
                ("W", C.c_int), ("H", C.c_int), ("xyz", C.c_void_p), ("features", C.c_void_p),
                ("scaling", C.c_void_p), ("rotation", C.c_void_p), ("opacity", C.c_void_p),
                ("c2w", C.c_void_p), ("fxfycxcy", C.c_void_p), ("scale_modifier", C.c_float),
                ("bg", C.c_float * 3), ("debug", C.c_int), ("near_log2", C.c_int)]


class DitWeights(C.Structure):
    _fields_ = [("width", C.c_int), ("heads", C.c_int), ("layers", C.c_int), ("patch", C.c_int),
                ("n_gaussians", C.c_int), ("mlp_hidden", C.c_int)] + [
        (n, C.c_void_p) for n in (
            "tokenizer_w", "pos_embed", "in_ln_w", "t0_w", "t0_b", "t2_w", "t2_b", "adaln_w", "adaln_b", "qkv_w",
            "qkv_b", "proj_w", "proj_b", "fc1_w", "fc1_b", "fc2_w", "fc2_b", "ups_ln_w", "ups_w", "dec_ln_w", "dec_w")]


class DitIO(C.Structure):
    _fields_ = [("B", C.c_int), ("V", C.c_int), ("H", C.c_int), ("W", C.c_int), ("plucker_mode", C.c_int),
                ("scene_depth", C.c_int), ("range_near", C.c_float), ("range_far", C.c_float)] + [
        (n, C.c_void_p) for n in ("images", "ray_o", "ray_d", "t", "xyz", "features", "scaling", "rotation",
                                  "opacity", "img_aligned_xyz", "tokens_out", "train_state")] + [("train_mode", C.c_int)]


TRAIN_STORE, TRAIN_RECOMPUTE = 0, 1  # dgs_dit_io.train_mode


class DitWeightsFp8(C.Structure):  # dgs_dit_weights_fp8
    _fields_ = [(n, C.c_void_p) for n in ("qkv_w", "qkv_s", "fc1_w", "fc1_s", "fc2_w", "fc2_s")]


FP8_EPI_BIAS_BF16, FP8_EPI_GATE_RESID_F32, FP8_EPI_F32, FP8_EPI_BIAS_GELU_E4M3 = 0, 2, 3, 6  # dgs_gemm_fp8 epi


BWD_TRACE_FIELDS = ("dx", "dx_mid", "d_fc2_out", "du_pre", "dh2", "d_proj_out", "d_attn", "dsum", "dqkv", "dh1")


class DitBwdTrace(C.Structure):  # dgs_dit_bwd_trace
    _fields_ = [(n, C.c_void_p) for n in BWD_TRACE_FIELDS]


class DitBwdOpts(C.Structure):  # dgs_dit_bwd_opts
    _fields_ = [("block_done", C.POINTER(C.c_void_p)), ("trace", C.POINTER(DitBwdTrace))]


class RenderMse(C.Structure):  # dgs_render_mse
    _fields_ = [("target", C.c_void_p), ("target_channels", C.c_int), ("loss_sum", C.c_void_p), ("coef", C.c_void_p),
                ("images", C.c_void_p)]


class LpipsWeights(C.Structure):  # dgs_lpips_weights
    _fields_ = [("conv_w", C.c_void_p * 13), ("conv_wt", C.c_void_p * 13), ("conv_b", C.c_void_p * 13),
                ("lin", C.c_void_p * 5), ("shift", C.c_void_p), ("scale", C.c_void_p)]


GRAD_FIELDS_A = ("tokenizer_w", "pos_embed", "in_ln_w", "t0_w", "t0_b", "t2_w", "t2_b")
GRAD_FIELDS_B = ("qkv_w", "qkv_b", "proj_w", "proj_b", "fc1_w", "fc1_b", "fc2_w", "fc2_b", "adaln_w", "adaln_b", "ups_ln_w",
                 "ups_w", "ups_adaln_w", "ups_adaln_b", "dec_ln_w", "dec_w", "dec_adaln_w", "dec_adaln_b")


class DitWeightsT(C.Structure):  # dgs_dit_weights_t
    _fields_ = [(n, C.c_void_p) for n in ("qkv_wT", "proj_wT", "fc1_wT", "fc2_wT", "dec_wT", "ups_w")]


class DitGrads(C.Structure):  # dgs_dit_grads
    _fields_ = [(n, C.c_void_p) for n in GRAD_FIELDS_A] + [("layer_stride", C.c_longlong)] + \
        [(n, C.c_void_p) for n in GRAD_FIELDS_B]


class DitOutGrads(C.Structure):  # dgs_dit_out_grads
    _fields_ = [(n, C.c_void_p) for n in ("d_xyz", "d_features", "d_scaling", "d_rotation", "d_opacity")]


_lib = None


class DgsError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise DgsError(
                f"libdgs_b200.so not found at {LIB_PATH}: build it with "
                "`python open-diffusiongs_b200/csrc/build.py` (there is no CPU/PyTorch fallback)")
        L = C.CDLL(LIB_PATH)
        L.dgs_last_error.restype = C.c_char_p
        L.dgs_version.restype = C.c_int
        L.dgs_kernel_launch_count.restype = C.c_ulonglong
        L.dgs_profile_read.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        for name in ("dgs_raster_geom_bytes", "dgs_raster_binning_bytes", "dgs_raster_image_bytes"):
            getattr(L, name).restype = C.c_size_t
        L.dgs_raster_geom_bytes.argtypes = [C.c_int, C.c_int]
        L.dgs_raster_binning_bytes.argtypes = [C.c_longlong]
        L.dgs_raster_image_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
        vp = C.c_void_p
        L.dgs_raster_forward.argtypes = [C.POINTER(RasterArgs), ALLOC_FN, vp, ALLOC_FN, vp, ALLOC_FN, vp,
                                         vp, vp, C.POINTER(C.c_int), vp]
        L.dgs_raster_backward.argtypes = [C.POINTER(RasterArgs), C.c_int] + [vp] * 15
        L.dgs_mark_visible.argtypes = [C.c_int, vp, vp, vp, vp, vp]
        L.dgs_render_batch_forward.argtypes = [C.POINTER(RenderBatchArgs), ALLOC_FN, vp, ALLOC_FN, vp,
                                               ALLOC_FN, vp, vp, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong), vp]
        L.dgs_render_batch_backward.argtypes = [C.POINTER(RenderBatchArgs), C.c_longlong, C.POINTER(C.c_longlong)] + \
            [vp] * 10 + [ALLOC_FN, vp, vp]
        L.dgs_raster_export_state.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_longlong] + [vp] * 13
        L.dgs_dit_workspace_bytes.restype = C.c_size_t
        L.dgs_dit_workspace_bytes.argtypes = [C.POINTER(DitWeights), C.c_int, C.c_int, C.c_int, C.c_int]
        L.dgs_dit_forward.argtypes = [C.POINTER(DitWeights), C.POINTER(DitIO), vp, C.c_size_t, vp]
        L.dgs_gemm_bf16.argtypes = [vp, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                    C.c_int, vp]
        L.dgs_attention_fwd.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp]
        L.dgs_ln_modulate.argtypes = [vp, vp, vp, vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.c_float, vp]
        L.dgs_dit_train_state_bytes.restype = C.c_size_t
        L.dgs_dit_train_state_bytes.argtypes = [C.POINTER(DitWeights), C.c_int, C.c_int, C.c_int, C.c_int]
        L.dgs_dit_backward.argtypes = [C.POINTER(DitWeights), C.POINTER(DitWeightsT), C.POINTER(DitIO),
                                       C.POINTER(DitOutGrads), C.POINTER(DitGrads), vp, C.c_size_t, vp]
        L.dgs_dit_train_state_bytes_ex.restype = C.c_size_t
        L.dgs_dit_train_state_bytes_ex.argtypes = [C.POINTER(DitWeights), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        L.dgs_dit_backward_ex.argtypes = [C.POINTER(DitWeights), C.POINTER(DitWeightsT), C.POINTER(DitIO),
                                          C.POINTER(DitOutGrads), C.POINTER(DitGrads), C.POINTER(DitBwdOpts), vp,
                                          C.c_size_t, vp]
        L.dgs_dit_export_state.argtypes = [C.POINTER(DitWeights)] + [C.c_int] * 5 + [vp, C.c_int] + [vp] * 12
        L.dgs_dit_export_ends.argtypes = [C.POINTER(DitWeights)] + [C.c_int] * 5 + [vp, vp, C.c_size_t] + [vp] * 11
        L.dgs_event_create.argtypes = [C.POINTER(C.c_void_p)]
        L.dgs_event_destroy.argtypes = [vp]
        L.dgs_stream_wait_event.argtypes = [vp, vp]
        L.dgs_adamw_ema_step.argtypes = [vp, vp, vp, vp, vp, C.c_size_t] + [C.c_float] * 5 + [C.c_int, C.c_float, vp,
                                                                                               C.c_float, vp]
        L.dgs_render_batch_forward_mse.argtypes = [C.POINTER(RenderBatchArgs), ALLOC_FN, vp, ALLOC_FN, vp, ALLOC_FN, vp, vp,
                                                   C.POINTER(C.c_longlong), C.POINTER(C.c_longlong),
                                                   C.POINTER(RenderMse), vp]
        L.dgs_render_batch_backward_mse.argtypes = [C.POINTER(RenderBatchArgs), C.c_longlong, C.POINTER(C.c_longlong)] + \
            [vp] * 5 + [C.POINTER(RenderMse)] + [vp] * 5 + [ALLOC_FN, vp, vp]
        L.dgs_transpose_bf16.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, vp, vp]
        L.dgs_adamw_step.argtypes = [vp, vp, vp, vp, C.c_size_t] + [C.c_float] * 5 + [C.c_int, C.c_float, vp, vp]
        L.dgs_cast_transpose_f32.argtypes = [vp, C.c_longlong, C.c_int, C.c_int, C.c_int, vp, vp, vp]
        L.dgs_attention_fwd_train.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, vp]
        L.dgs_attention_bwd.argtypes = [vp, vp, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, vp]
        L.dgs_gemm_bf16_ex.argtypes = [vp] * 7 + [C.c_int] * 9 + [vp]
        L.dgs_gemm_bf16_tn.argtypes = [vp, vp, vp] + [C.c_int] * 6 + [vp]
        L.dgs_ln_modulate_bwd.argtypes = [vp, vp, C.c_int, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, vp,
                                          C.c_int, vp, vp, vp, vp, vp]
        L.dgs_gate_bwd.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, vp]
        L.dgs_rays_from_cameras.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp]
        L.dgs_q_sample.argtypes = [vp, vp, vp, vp, vp, C.c_int, C.c_longlong, vp, vp]
        L.dgs_p_sample_step.argtypes = [vp, vp, vp, vp, vp, vp, vp, C.c_int, C.c_longlong, vp, vp]
        L.dgs_lpips_workspace_bytes.restype = C.c_size_t
        L.dgs_lpips_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
        L.dgs_lpips_state_bytes.restype = C.c_size_t
        L.dgs_lpips_state_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
        L.dgs_lpips_forward.argtypes = [C.POINTER(LpipsWeights), C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, vp, C.c_size_t,
                                        vp]
        L.dgs_lpips_backward.argtypes = [C.POINTER(LpipsWeights), C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, C.c_size_t, vp]
        L.dgs_ssim_workspace_bytes.restype = C.c_size_t
        L.dgs_ssim_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
        L.dgs_ssim_state_bytes.restype = C.c_size_t
        L.dgs_ssim_state_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
        L.dgs_ssim_forward.argtypes = [C.c_int, C.c_int, C.c_int, vp, vp, C.c_float, C.c_int, vp, vp, vp, vp, C.c_size_t,
                                       vp]
        L.dgs_ssim_backward.argtypes = [C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp]
        L.dgs_dit_workspace_bytes_fp8.restype = C.c_size_t
        L.dgs_dit_workspace_bytes_fp8.argtypes = [C.POINTER(DitWeights), C.c_int, C.c_int, C.c_int, C.c_int]
        L.dgs_dit_forward_fp8.argtypes = [C.POINTER(DitWeights), C.POINTER(DitWeightsFp8), C.POINTER(DitIO), vp, C.c_size_t,
                                          vp]
        L.dgs_quantize_rows_e4m3.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp]
        L.dgs_ln_modulate_fp8.argtypes = [vp, vp, vp, C.c_int, vp, vp, C.c_int, C.c_int, C.c_int, C.c_float, vp]
        L.dgs_gemm_fp8.argtypes = [vp] * 8 + [C.c_int] * 7 + [vp]
        L.dgs_mesh_field.argtypes = [C.c_int, vp, vp, vp, vp, C.c_float, vp, C.c_float, C.c_int, C.c_int, C.c_double,
                                     vp, vp, vp, C.POINTER(C.c_longlong), ALLOC_FN, vp, vp]
        L.dgs_marching_cubes.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_float, ALLOC_FN, vp, C.POINTER(C.c_void_p),
                                         C.POINTER(C.c_void_p), C.POINTER(C.c_longlong), C.POINTER(C.c_longlong), vp]
        _lib = L
    return _lib


PROF_FAMILIES = ["raster.project", "raster.scan", "raster.emit_keys", "raster.sort", "raster.tile_ranges",
                 "raster.blend_fwd", "raster.blend_bwd", "raster.geometry_bwd", "dit.input", "dit.conditioning",
                 "dit.ln_modulate", "dit.gemm_qkv", "dit.attention", "dit.gemm_proj", "dit.gemm_fc1", "dit.gemm_fc2",
                 "dit.heads", "dit.bwd_elementwise", "dit.bwd_gemm_wgrad", "dit.bwd_gemm_dgrad", "dit.bwd_attention"]


def profile_read():
    """-> {family: (total_ms, spans)} of everything recorded since the last read (synchronises)."""
    n = len(PROF_FAMILIES)
    ms = (C.c_float * n)()
    cnt = (C.c_int * n)()
    lib().dgs_profile_read(ms, cnt, n)
    return {f: (float(ms[i]), int(cnt[i])) for i, f in enumerate(PROF_FAMILIES)}


def check(rc):
    if rc != 0:
        raise DgsError(f"libdgs_b200 status {rc}: {lib().dgs_last_error().decode()}")


EXPORTED = [  # every symbol include/dgs_b200.h declares (checked by tests/test_abi.py)
    "dgs_version", "dgs_last_error", "dgs_kernel_launch_count", "dgs_profile_enable", "dgs_profile_read",
    "dgs_raster_geom_bytes", "dgs_raster_binning_bytes",
    "dgs_raster_image_bytes", "dgs_raster_forward", "dgs_raster_backward", "dgs_mark_visible",
    "dgs_render_batch_forward", "dgs_render_batch_backward", "dgs_raster_export_state",
    "dgs_dit_workspace_bytes", "dgs_dit_forward", "dgs_gemm_bf16", "dgs_attention_fwd", "dgs_ln_modulate",
    "dgs_rays_from_cameras", "dgs_q_sample", "dgs_p_sample_step",
    "dgs_dit_train_state_bytes", "dgs_dit_backward", "dgs_transpose_bf16", "dgs_adamw_step", "dgs_attention_fwd_train",
    "dgs_attention_bwd", "dgs_gemm_bf16_ex", "dgs_ln_modulate_bwd", "dgs_gate_bwd", "dgs_cast_transpose_f32", "dgs_gemm_bf16_tn",
    "dgs_dit_train_state_bytes_ex", "dgs_dit_backward_ex", "dgs_event_create", "dgs_event_destroy", "dgs_stream_wait_event",
    "dgs_adamw_ema_step", "dgs_render_batch_forward_mse", "dgs_render_batch_backward_mse", "dgs_dit_export_state",
    "dgs_dit_export_ends", "dgs_lpips_workspace_bytes", "dgs_lpips_state_bytes", "dgs_lpips_forward", "dgs_lpips_backward",
    "dgs_ssim_workspace_bytes", "dgs_ssim_state_bytes", "dgs_ssim_forward", "dgs_ssim_backward",
    "dgs_dit_workspace_bytes_fp8", "dgs_dit_forward_fp8", "dgs_quantize_rows_e4m3", "dgs_ln_modulate_fp8", "dgs_gemm_fp8",
    "dgs_mesh_field", "dgs_marching_cubes",
]
