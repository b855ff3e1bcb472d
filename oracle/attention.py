"""oracle/attention.py -- TEST INFRASTRUCTURE: the bf16 attention kernels (attention_sm90.cu, attention_bwd_sm90.cu) as
a model of their own arithmetic in fp64, block by block, the way oracle/fp8_attention.py models the e4m3 path.

* attention_fwd_matched: the forward's online softmax over 128-key blocks -- scores rounded to fp32, the running max
  in score units, P = 2^(fmaf(s, c, -fp32(m c))) in fp32, row sums of the unrounded P, P rounded to bf16 for P V,
  out = bf16(O fp32(1 / l)) and lse2 = fmaf(m, c, log2 l);
* attention_bwd_matched: the backward's two kernels from the forward's out and lse2 -- Dsum = rowsum(O dO), P from
  lse2, dS in the dQ kernel's form bf16(P fmaf(dP, 1/8, -Dsum/8)) and in the dK/dV kernel's form
  bf16(P (dP - Dsum) 1/8), bf16(P)^T dO, and dQ / dK / dV stored in bf16.
Accumulations (row sums, P V, the backward's products) are exact fp64 sums: the kernels' fp32 accumulation order is
the one thing not modelled.  rounding=False drops every rounding: the plain fp64 softmax and its gradient.
`defects` plant named defects (ATTENTION_DEFECTS) so that tests/test_attention_cpu.py can show that the GPU bounds of
tests/test_attention_gpu.py would see them.  Both functions chunk over heads and query rows, so N = 16386 never forms
a whole score matrix.  Never imported by the product path.
"""
import collections
import math

import numpy as np
import torch

BLOCK = 128       # keys per block of the forward's online softmax
BWD_QBLOCK = 64   # queries per block of the dK/dV kernel
HD = 64
SCALE = 0.125     # 1 / sqrt(64)
C = float(np.float32(SCALE) * np.float32(1.4426950408889634))  # sl2 = 0.125f * 1.4426950408889634f (fp32)
C_EXACT = SCALE / math.log(2.0)                                 # rounding=False: the exact log2(e) / 8
CHUNK = 1 << 24   # score elements per chunk (128 MB of fp64)

_Defects = collections.namedtuple("AttentionDefects", [
    "pad_key_unmasked",        # forward: the last key block admits one zero-filled key (score 0, value 0)
    "alpha_not_on_l",          # forward: the row sum is not rescaled at block 1
    "exp2_bias",               # forward: the exponentials of one column pair in eight (keys 0, 1 of every 16) 1e-3 high
    "lse_natural_log",         # forward: lse2 written in natural-log units
    "l_from_rounded_p",        # forward: the row sum adds up bf16(P) instead of the fp32 P
    "dkv_query_tail_dropped",  # backward: the dK/dV kernel skips the last 64-query block
    "ds_scale_dropped_in_dq",  # backward: the dQ kernel's dS leaves out the 1/8
])
ATTENTION_DEFECTS = _Defects(*_Defects._fields)


def _f32(t):
    return t.float().double()


def _f32_ftz(t):
    """fp32 with subnormals flushed to zero, as ex2.approx.ftz.f32 returns them."""
    x = t.float()
    return torch.where(x.abs() < 2.0 ** -126, torch.zeros_like(x), x).double()


def _bf16(t):
    return t.to(torch.bfloat16).double()


def _split(qkv):
    """qkv [B, N, 3, H, 64] (bf16 values, any dtype) -> q, k, v [B, H, N, 64] fp64."""
    B, N, three, H, hd = qkv.shape
    assert three == 3 and hd == HD, qkv.shape
    return qkv.double().permute(2, 0, 3, 1, 4).unbind(0)


def _query_chunk(B, n_cols):
    """Query rows per chunk: a multiple of 128 with B * rows * n_cols <= CHUNK."""
    return max(BLOCK, (CHUNK // max(1, B * n_cols)) // BLOCK * BLOCK)


def _fwd_rows(q, k, v, N, defects, rounding):
    """q [B, R, 64], k / v [B, N, 64] of one head -> out [B, R, 64] (fp64), lse2 [B, R] (fp64)."""
    B, R, _ = q.shape
    nb = (N + BLOCK - 1) // BLOCK
    Nk = nb * BLOCK
    rnd = _f32 if rounding else (lambda t: t)
    rnd_ftz = _f32_ftz if rounding else (lambda t: t)
    c = C if rounding else C_EXACT
    s = q.new_full((B, R, Nk), -math.inf)
    s[..., :N] = rnd(q @ k.transpose(-1, -2))           # exact dot products of the bf16 operands, then fp32
    vp = v.new_zeros(B, Nk, HD)
    vp[:, :N] = v
    if "pad_key_unmasked" in defects and N < Nk:
        s[..., N] = 0.0                                  # the zero-filled key: score 0, value 0
    sb = s.view(B, R, nb, BLOCK)
    m = sb.amax(-1).cummax(-1).values                    # running max (score units) after each block
    m_old = torch.cat([torch.full_like(m[..., :1], -math.inf), m[..., :-1]], -1)
    alpha = rnd_ftz(torch.exp2(rnd(rnd(m_old - m) * c)))  # 0 at block 0
    moff = rnd(m * c)
    p = rnd_ftz(torch.exp2(rnd(sb * c - moff[..., None])))  # fmaf(s, c, -moff): one rounding
    if "exp2_bias" in defects:
        col = torch.arange(BLOCK, device=p.device) % 16
        p = p * torch.where(col < 2, 1.0 + 1e-3, 1.0).to(p)
    pv = _bf16(p) if rounding else p                     # the A operand of the P V wgmma
    ls = (pv if "l_from_rounded_p" in defects else p).sum(-1)
    # O_j = O_{j-1} alpha_j + P_j V_j (the same for l) unrolled: block j's terms are scaled by w_j = prod_{i>j} alpha_i
    w = torch.ones_like(alpha)
    if nb > 1:
        w[..., :-1] = alpha[..., 1:].flip(-1).cumprod(-1).flip(-1)
    wl = w.clone()
    if "alpha_not_on_l" in defects and nb > 1:
        wl[..., 0] = w[..., 1]                           # l after block 1 = l_0 + ls_1: block 0 misses alpha_1
    o = (pv * w[..., None]).view(B, R, Nk) @ vp
    l = (ls * wl).sum(-1)
    if rounding:
        out = _f32(o * _f32(1.0 / _f32(l))[..., None])   # o * (1.0f / l) in fp32, rounded to bf16 by the caller
        lse2 = _f32(m[..., -1] * c + _f32(torch.log2(_f32(l))))
    else:
        out = o / l[..., None]
        lse2 = m[..., -1] * c + torch.log2(l)
    if "lse_natural_log" in defects:
        lse2 = lse2 * math.log(2.0)
    return out, lse2


@torch.no_grad()
def attention_fwd_matched(qkv, defects=(), rounding=True):
    """The bf16 attention forward (attention_fwd_kernel<ATT_BF16>) in fp64.  qkv [B, N, 3, H, 64] with bf16 values ->
    (out [B, N, H * 64], lse2 [B, H, N]): out is bf16 (fp64 when rounding=False), lse2 fp64 holding the kernel's fp32
    values (log2 units)."""
    q, k, v = _split(qkv)
    B, H, N, _ = q.shape
    out = torch.empty(B, H, N, HD, dtype=torch.float64, device=q.device)
    lse2 = torch.empty(B, H, N, dtype=torch.float64, device=q.device)
    rows = _query_chunk(B, N + BLOCK)
    for h in range(H):
        for r0 in range(0, N, rows):
            r1 = min(N, r0 + rows)
            out[:, h, r0:r1], lse2[:, h, r0:r1] = _fwd_rows(q[:, h, r0:r1], k[:, h], v[:, h], N, defects, rounding)
    out = out.permute(0, 2, 1, 3).reshape(B, N, H * HD)
    return (out.to(torch.bfloat16) if rounding else out), lse2


@torch.no_grad()
def attention_bwd_matched(qkv, out, dout, lse2, defects=(), rounding=True):
    """The bf16 attention backward (attn_bwd_prep_kernel, attn_bwd_dq_kernel, attn_bwd_dkv_kernel) in fp64.
    qkv [B, N, 3, H, 64], out / dout [B, N, H * 64] (bf16 values), lse2 [B, H, >= N] (the forward's, log2 units) ->
    (dqkv [B, N, 3, H, 64], dsum [B, H, N]): dqkv is bf16 (fp64 when rounding=False), dsum fp64 holding fp32 values."""
    q, k, v = _split(qkv)
    B, H, N, _ = q.shape
    rnd = _f32 if rounding else (lambda t: t)
    rnd_ftz = _f32_ftz if rounding else (lambda t: t)
    c = C if rounding else C_EXACT
    o = out.double().reshape(B, N, H, HD).permute(0, 2, 1, 3)
    do = dout.double().reshape(B, N, H, HD).permute(0, 2, 1, 3)
    dsum = rnd((o * do).sum(-1))                         # [B, H, N]
    lse = lse2.double()[..., :N]
    dqkv = torch.empty(3, B, H, N, HD, dtype=torch.float64, device=q.device)
    keep_q = N if "dkv_query_tail_dropped" not in defects else (N - 1) // BWD_QBLOCK * BWD_QBLOCK
    rows = _query_chunk(B, N)
    for h in range(H):
        qh, kh, vh, doh = q[:, h], k[:, h], v[:, h], do[:, h]
        dk = torch.zeros(B, N, HD, dtype=torch.float64, device=q.device)
        dv = torch.zeros_like(dk)
        for r0 in range(0, N, rows):
            r1 = min(N, r0 + rows)
            s = rnd(qh[:, r0:r1] @ kh.transpose(-1, -2))
            p = rnd_ftz(torch.exp2(rnd(s * c - lse[:, h, r0:r1, None])))  # fmaf(s, c, -lse2)
            del s
            dp = rnd(doh[:, r0:r1] @ vh.transpose(-1, -2))
            d = dsum[:, h, r0:r1, None]
            # dQ kernel: dS = bf16(P * fmaf(dP, 1/8, -Dsum/8)), dQ += dS K
            if "ds_scale_dropped_in_dq" in defects:
                ds = rnd(p * rnd(dp - d))
            else:
                ds = rnd(p * rnd(dp * SCALE - d * SCALE))
            dqkv[0, :, h, r0:r1] = (_bf16(ds) if rounding else ds) @ kh
            # dK/dV kernel: P^T and dS^T = bf16(P * (dP - Dsum) * 1/8), dV += bf16(P)^T dO, dK += dS^T Q
            ds = rnd(rnd(p * rnd(dp - d)) * SCALE)
            del dp
            k1 = max(r0, min(r1, keep_q))
            if k1 > r0:
                pb = (_bf16(p) if rounding else p)[:, :k1 - r0]
                dv += pb.transpose(-1, -2) @ doh[:, r0:k1]
                dk += (_bf16(ds) if rounding else ds)[:, :k1 - r0].transpose(-1, -2) @ qh[:, r0:k1]
            del p, ds
        dqkv[1, :, h], dqkv[2, :, h] = dk, dv
    dqkv = dqkv.permute(1, 3, 0, 2, 4)
    if rounding:
        dqkv = _f32(dqkv).to(torch.bfloat16)
    return dqkv.contiguous(), dsum
