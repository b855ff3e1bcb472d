"""The FP8 inference path as tests/test_fp8_gpu.py and test_fp8_attention_gpu.py drive it: the C ABI's quantizers, FP8
GEMM and FP8 attention, one DiT block built from them, and the models and error measure of the end-to-end checks."""
import gc

import torch

from dgs_b200 import _lib
from util import rel_l2 as rel

DEV = "cuda:0"
D = 1024
ATT_OPERANDS = ("q8", "k8", "vt8", "sq", "sk", "sv")  # the FP8 attention's operands, in C ABI order


def ms(M):
    return (M + 3) // 4 * 4


def quantize_rows(x):
    """dgs_quantize_rows_e4m3: x [R, K] fp32 -> (q uint8 [R, K], s [R])."""
    R, K = x.shape
    q = torch.empty(R, K, dtype=torch.uint8, device=DEV)
    s = torch.empty(R, dtype=torch.float32, device=DEV)
    _lib.check(_lib.lib().dgs_quantize_rows_e4m3(x.data_ptr(), R, K, q.data_ptr(), s.data_ptr(), _lib.stream(None)))
    return q, s


def deq_act(q, sa, M):
    """e4m3 [M, K] with group scales [K/128][ms(M)] -> fp64 [M, K]"""
    K = q.shape[1]
    return (q.view(torch.float8_e4m3fn).double().reshape(M, K // 128, 128) *
            sa[:, :M].t().double()[:, :, None]).reshape(M, K)


def deq_w(q, s):
    return q.view(torch.float8_e4m3fn).double() * s.double()[:, None]


def gemm_fp8(A, sa, Wq, sw, M, epi, bias=None, gate=None, x=None, rows_per_sample=1, gate_stride=0):
    N, K = Wq.shape
    out_scale = None
    if epi == 0:
        out = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    elif epi == 2:
        out = x
    elif epi == 3:
        out = torch.empty(M, N, dtype=torch.float32, device=DEV)
    else:
        out = torch.empty(M, N, dtype=torch.uint8, device=DEV)
        out_scale = torch.full((N // 128, ms(M)), float("nan"), device=DEV)
    _lib.check(_lib.lib().dgs_gemm_fp8(A.data_ptr(), sa.data_ptr(), Wq.data_ptr(), sw.data_ptr(),
                                       None if bias is None else bias.data_ptr(),
                                       None if gate is None else gate.data_ptr(), out.data_ptr(),
                                       None if out_scale is None else out_scale.data_ptr(), M, N, K, epi, N,
                                       gate_stride, rows_per_sample, _lib.stream(None)))
    return out, out_scale


def quantize_attention(qkv, B, N, H):
    """dgs_attention_quantize_e4m3 -> the dict of oracle.fp8_attention.quantize_attention_operands."""
    Nk = (N + 127) // 128 * 128
    u8 = lambda *s: torch.empty(*s, dtype=torch.uint8, device=DEV)  # noqa: E731
    ops = dict(q8=u8(B, N, H, 64), k8=u8(B, N, H, 64), vt8=u8(B, H, 64, Nk).fill_(0xAB),  # pads must be written
               sq=torch.empty(B, H, N, device=DEV), sk=torch.empty(B, H, Nk // 128, device=DEV),
               sv=torch.empty(B, H, Nk // 128, device=DEV))
    _lib.check(_lib.lib().dgs_attention_quantize_e4m3(qkv.data_ptr(), *(ops[k].data_ptr() for k in ATT_OPERANDS), B, N,
                                                      H, _lib.stream(None)))
    return ops


def attention_fwd_fp8(ops, B, N, H):
    out = torch.zeros(B, N, H * 64, dtype=torch.bfloat16, device=DEV)
    _lib.check(_lib.lib().dgs_attention_fwd_fp8(*(ops[k].data_ptr() for k in ATT_OPERANDS), out.data_ptr(), B, N, H,
                                                _lib.stream(None)))
    return out


def block_product(blk, x, mod32, N, attention_fp8=False):
    """One FP8 block from the exported building blocks, in the sequence of dgs_dit_forward_fp8; attention_fp8: with
    the attention on e4m3 operands, as the "fp8_attention" precision runs it.  -> every intermediate: h1q, qkv, attn,
    x_mid, h2q, uq, x_out."""
    B = x.shape[0]
    M = B * N
    L = _lib.lib()
    st = _lib.stream(None)
    m = mod32.data_ptr()
    f = 4  # bytes per float
    out = {}
    q1 = torch.empty(M, D, dtype=torch.uint8, device=DEV)
    s1 = torch.zeros(D // 128, ms(M), device=DEV)
    _lib.check(L.dgs_ln_modulate_fp8(x.data_ptr(), m, m + f * D, 6 * D, q1.data_ptr(), s1.data_ptr(), B, N, D, 1e-6,
                                     st))
    out["h1q"] = deq_act(q1, s1, M).reshape(B, N, D)
    wq = {k: quantize_rows(getattr(blk.attn if k == "qkv" else blk.mlp, k).weight.detach().float().contiguous())
          for k in ("qkv", "fc1", "fc2")}
    bias = {k: getattr(blk.attn if k in ("qkv", "proj") else blk.mlp, k).bias.detach().float().contiguous()
            for k in ("qkv", "proj", "fc1", "fc2")}
    qkv, _ = gemm_fp8(q1, s1, *wq["qkv"], M, 0, bias=bias["qkv"])
    out["qkv"] = qkv.reshape(B, N, 3 * D)
    if attention_fp8:
        attn = attention_fwd_fp8(quantize_attention(qkv, B, N, 16), B, N, 16).reshape(M, D)
    else:
        attn = torch.empty(M, D, dtype=torch.bfloat16, device=DEV)
        _lib.check(L.dgs_attention_fwd(qkv.data_ptr(), attn.data_ptr(), B, N, 16, st))
    out["attn"] = attn.reshape(B, N, D)
    x_mid = x.reshape(M, D).clone()
    wp = blk.attn.proj.weight.detach().to(torch.bfloat16).contiguous()
    _lib.check(L.dgs_gemm_bf16(attn.data_ptr(), wp.data_ptr(), bias["proj"].data_ptr(), m + f * 2 * D, x_mid.data_ptr(),
                               M, D, D, 2, D, 6 * D, N, st))
    out["x_mid"] = x_mid.reshape(B, N, D).clone()
    q2 = torch.empty(M, D, dtype=torch.uint8, device=DEV)
    s2 = torch.zeros(D // 128, ms(M), device=DEV)
    _lib.check(L.dgs_ln_modulate_fp8(x_mid.data_ptr(), m + f * 3 * D, m + f * 4 * D, 6 * D, q2.data_ptr(),
                                     s2.data_ptr(), B, N, D, 1e-6, st))
    out["h2q"] = deq_act(q2, s2, M).reshape(B, N, D)
    u8, su = gemm_fp8(q2, s2, *wq["fc1"], M, 6, bias=bias["fc1"])
    out["uq"] = deq_act(u8, su, M).reshape(B, N, 4 * D)
    gemm_fp8(u8, su, *wq["fc2"], M, 2, bias=bias["fc2"], gate=mod32[:, 5 * D:], x=x_mid, rows_per_sample=N,
             gate_stride=6 * D)
    out["x_out"] = x_mid.reshape(B, N, D)
    torch.cuda.synchronize()
    return out


def _models(layers, scene, trained, seed):
    from dgs_b200.denoiser import DGSDenoiser, DGSDenoiserScene
    from dit_regime import apply_trained_scale
    from oracle.dit import DenoiserOracle
    gc.collect()
    torch.cuda.empty_cache()
    torch.manual_seed(seed)
    cfg = dict(patch_size=8, num_layers=layers, ray_pe_type="plk" if scene else "relative_plk")
    model = (DGSDenoiserScene if scene else DGSDenoiser)(cfg)
    if trained:
        apply_trained_scale(model, seed)
    model = model.to(DEV).eval()
    oracle = DenoiserOracle(layers=layers, scene=scene).to(DEV)
    oracle.load_state_dict(model.state_dict(), strict=True)
    return model, oracle


def _views(model, out, V, H, W):
    from dgs_b200 import synth
    c2w, fx = synth.orbit_cameras(V, W, H)
    return model.render_gaussians(out, torch.tensor(c2w[None], device=DEV), torch.tensor(fx[None], device=DEV), H, W)


def _attr(d):
    from dgs_b200.denoiser import AttrDict
    return AttrDict(d)


def _err(out, ia, views, ref):
    r_out, r_ia, r_views = ref
    return max([rel(out[k], r_out[k]) for k in r_out] + [rel(ia, r_ia), rel(views, r_views)])
