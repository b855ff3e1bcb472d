"""oracle/fp8_attention.py -- TEST INFRASTRUCTURE: the FP8 attention of the "fp8_attention" inference precision
(DGS_FP8_ATTENTION) in plain PyTorch, on top of oracle/fp8.py's number format.

* quantize_attention_operands: the bitwise reference of the quantize pass (q8, k8, the transposed and key-permuted
  vt8, and the scales sq, sk, sv);
* attention_fp8_matched: the kernel's arithmetic in fp64 -- 128-key blocks, running max, P = 2^(x - m + 8) rounded to
  e4m3, O kept in units of the current block's V scale, fp64 row sums of the unrounded P;
* dit_block_fp8_matched / emulate_fp8: oracle/fp8.py's functions with an `attention_fp8` / `attention` switch that
  replaces the bf16 attention by the FP8 one.
`defects` plant named defects (FP8_ATTENTION_DEFECTS) so that tests/test_fp8_attention_cpu.py can show the GPU bounds
would see them.  Never imported by the product path.
"""
import copy
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import fp8 as _fp8
from oracle.dit import _bf16

FP8_ATTENTION_DEFECTS = ("v_scale_not_rebased", "key_order_dropped", "p_offset_kept")
BLOCK = 128
HD = 64


def key_of_slot(a):
    """Slot a (0..15) of every 16 keys of vt8 holds this key: the thread of a quad that owns score columns {2u, 2u+1,
    8+2u, 9+2u} supplies the e4m3 A fragment's k = 4u..4u+3."""
    return 2 * (a // 4) + (a % 2) + 8 * ((a // 2) % 2)


def _slot_keys(n, device):
    a = torch.arange(n, device=device)
    return (a // 16) * 16 + key_of_slot(a % 16)


def quantize_attention_operands(qkv, heads):
    """qkv [B, N, 3 * heads * 64] (any float dtype; the product passes bf16) -> dict of
    q8, k8 uint8 (e4m3 bits) [B, N, heads, 64]; vt8 uint8 [B, heads, 64, Nk] (V transposed, keys of every 16 in the
    key_of_slot order, zero past N); sq fp32 [B, heads, N]; sk, sv fp32 [B, heads, Nk / 128]."""
    B, N, _ = qkv.shape
    t = qkv.float().reshape(B, N, 3, heads, HD)
    nkb = (N + BLOCK - 1) // BLOCK
    Nk = nkb * BLOCK
    q8, sq = _fp8.quantize_e4m3(t[:, :, 0], HD)

    def per_block(x):  # [B, N, H, 64] -> (e4m3 [B, H, nkb, 128, 64], s [B, H, nkb])
        xp = torch.zeros(B, Nk, heads, HD, dtype=torch.float32, device=x.device)
        xp[:, :N] = x
        xb = xp.reshape(B, nkb, BLOCK, heads, HD).permute(0, 3, 1, 2, 4).reshape(B, heads, nkb, BLOCK * HD)
        q, s = _fp8.quantize_e4m3(xb, BLOCK * HD)
        return q.view(torch.uint8).reshape(B, heads, nkb, BLOCK, HD), s[..., 0]

    k8b, sk = per_block(t[:, :, 1])
    v8b, sv = per_block(t[:, :, 2])
    k8 = k8b.permute(0, 2, 3, 1, 4).reshape(B, Nk, heads, HD)[:, :N]
    vt = v8b.permute(0, 1, 4, 2, 3).reshape(B, heads, HD, Nk)  # [B, H, 64, Nk], keys in natural order
    vt8 = vt[..., _slot_keys(Nk, vt.device)]
    return dict(q8=q8.view(torch.uint8).contiguous(), k8=k8.contiguous(), vt8=vt8.contiguous(),
                sq=sq[..., 0].permute(0, 2, 1).contiguous(), sk=sk.contiguous(), sv=sv.contiguous())


def _e4m3(bits):
    return bits.view(torch.float8_e4m3fn).double()


@torch.no_grad()
def attention_fp8_matched(ops, N, defects=()):
    """The FP8 attention forward in fp64 from quantize_attention_operands' output -> [B, N, heads * 64] (fp64; the
    kernel rounds it to bf16).  Defects: "v_scale_not_rebased" (O is not moved into the new block's V scale),
    "key_order_dropped" (vt8 read as if its keys were in natural order), "p_offset_kept" (the 2^8 of P not divided out)."""
    q = _e4m3(ops["q8"]).permute(0, 2, 1, 3)  # [B, H, N, 64]
    k = _e4m3(ops["k8"]).permute(0, 2, 1, 3)
    vt = _e4m3(ops["vt8"])                    # [B, H, 64, Nk]
    if "key_order_dropped" not in defects:    # back to the natural key order
        inv = torch.empty(vt.shape[-1], dtype=torch.long, device=vt.device)
        inv[_slot_keys(vt.shape[-1], vt.device)] = torch.arange(vt.shape[-1], device=vt.device)
        vt = vt[..., inv]
    sq, sk, sv = ops["sq"].double(), ops["sk"].double(), ops["sv"].double()
    B, H = q.shape[:2]
    cq = sq[..., None] * (0.125 / math.log(2.0))  # the score factor without the block's K scale (log2 units)
    m = torch.full((B, H, N, 1), -math.inf, dtype=torch.float64, device=q.device)
    l = torch.zeros_like(m)
    o = torch.zeros(B, H, N, HD, dtype=torch.float64, device=q.device)
    sv_prev = None
    for j in range((N + BLOCK - 1) // BLOCK):
        k0, k1 = j * BLOCK, min(N, (j + 1) * BLOCK)
        x = (q @ k[:, :, k0:k1].transpose(-1, -2)) * (cq * sk[:, :, j, None, None])
        m_new = torch.maximum(m, x.amax(-1, keepdim=True))
        alpha = torch.exp2(m - m_new)
        p = torch.exp2(x - m_new + 8.0)
        l = l * alpha + (p if "p_offset_kept" not in defects else torch.exp2(x - m_new)).sum(-1, keepdim=True)
        p8 = p.float().to(torch.float8_e4m3fn).double()  # p <= 256: inside e4m3's range, round to nearest even
        svj = sv[:, :, j, None, None]
        rebase = alpha if sv_prev is None or "v_scale_not_rebased" in defects else alpha * sv_prev / svj
        o = o * rebase + p8 @ vt[..., k0:k1].transpose(-1, -2)
        m, sv_prev = m_new, svj
    out = o * sv_prev / l
    return out.permute(0, 2, 1, 3).reshape(B, N, H * HD)


def _ln(t):
    mu = t.mean(-1, keepdim=True)
    return (t - mu) / torch.sqrt((t - mu).pow(2).mean(-1, keepdim=True) + 1e-6)


@torch.no_grad()
def dit_block_fp8_matched(blk, x, mod, head_chunk=None, feed=None, defects=(), attention_fp8=False):
    """oracle.fp8.dit_block_fp8_matched; attention_fp8=True: the "fp8_attention" block, its attention being
    attention_fp8_matched on the quantized bf16 qkv (the rest as in oracle/fp8.py: qkv / fc1 / fc2 on quantize-
    dequantized operands, bf16 rounding of qkv, the attention output and attn.proj's weight).  feed: as there (h1q,
    x_mid, h2q, uq).  Returns h1q, qkv, attn, proj_out, x_mid, h2q, u, uq, x_out (fp64)."""
    if not attention_fp8:
        return _fp8.dit_block_fp8_matched(blk, x, mod, head_chunk=head_chunk, feed=feed, defects=defects)
    feed = dict(feed or {})
    B, N, D = x.shape
    heads = D // HD
    x, mod = x.double(), mod.double()
    s1, c1, g1, s2, c2, g2 = (m[:, None, :] for m in mod.chunk(6, dim=1))
    q = lambda t: _fp8.qdq_act(t, defects).double()  # noqa: E731
    w8 = lambda lin: _fp8.qdq_weight(lin.weight.detach().float(), defects).double()  # noqa: E731
    bias = lambda lin: lin.bias.detach().double()  # noqa: E731
    out = {}
    h1q = feed["h1q"].double() if "h1q" in feed else q(_ln(x) * (1 + c1) + s1)
    out["qkv"] = _bf16(F.linear(h1q, w8(blk.attn.qkv), bias(blk.attn.qkv)))
    ops = quantize_attention_operands(out["qkv"], heads)
    out["attn"] = _bf16(attention_fp8_matched(ops, N, defects))
    proj = F.linear(out["attn"], _bf16(blk.attn.proj.weight.detach().double()), bias(blk.attn.proj))
    out["proj_out"] = _bf16(proj)
    out["x_mid"] = x + g1 * proj
    x_mid = feed["x_mid"].double() if "x_mid" in feed else out["x_mid"]
    h2q = feed["h2q"].double() if "h2q" in feed else q(_ln(x_mid) * (1 + c2) + s2)
    out["u"] = F.gelu(F.linear(h2q, w8(blk.mlp.fc1), bias(blk.mlp.fc1)), approximate="tanh")
    uq = feed["uq"].double() if "uq" in feed else q(out["u"])
    out["x_out"] = x_mid + g2 * F.linear(uq, w8(blk.mlp.fc2), bias(blk.mlp.fc2))
    out.update(h1q=h1q, h2q=h2q, uq=uq)
    return out


class _Fp8Attention(nn.Module):
    """An oracle Attention whose softmax(q k^T / 8) v is attention_fp8_matched on the quantized q / k / v."""

    def __init__(self, attn, defects=()):
        super().__init__()
        self.qkv, self.proj, self.num_heads, self.defects = attn.qkv, attn.proj, attn.num_heads, defects

    def forward(self, x):
        B, N, C = x.shape
        ops = quantize_attention_operands(self.qkv(x), self.num_heads)
        return self.proj(attention_fp8_matched(ops, N, self.defects).to(x.dtype))


def emulate_fp8(oracle, defects=(), attention=False):
    """oracle.fp8.emulate_fp8; attention=True: the blocks' attention runs as attention_fp8_matched as well."""
    em = _fp8.emulate_fp8(oracle, defects)
    if attention:
        for blk in em.transformer:
            blk.attn = _Fp8Attention(blk.attn, defects)
    return em
