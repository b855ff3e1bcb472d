"""oracle/fp8.py -- TEST INFRASTRUCTURE: the FP8 (e4m3) inference path's number format in plain PyTorch.

* quantize_e4m3: power-of-two scales 2^ceil(log2(amax / 448)) per group of `group` columns (1 for an all-zero group),
  then x / s rounded to nearest even into torch.float8_e4m3fn -- the bytes the kernels produce from the same fp32 input;
* dit_block_fp8_matched: oracle/dit.py's dit_block_matched with the qkv / fc1 / fc2 inputs and weights
  quantize-dequantized instead of bf16-rounded (each product GEMM then differs from it by its accumulation only);
* emulate_fp8: a DenoiserOracle whose qkv / fc1 / fc2 linears quantize-dequantize their input and weight: the FP8
  model's output with exact accumulation, the yardstick of the end-to-end tests.
`defects` plant named defects (FP8_DEFECTS) so that tests/test_fp8_cpu.py can show the GPU bounds would see them.
Never imported by the product path.
"""
import copy

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.dit import dit_block_matched

E4M3_MAX = 448.0
FP8_DEFECTS = ("group_scale_from_wrong_group", "weight_scale_dropped")


def scale_exponent(amax):
    """e with amax <= 448 * 2^e minimal (clamped to [-126, 126]; 0 where amax == 0), from amax's fp32 bits exactly as
    the kernels do: amax = m 2^E, m in [0.5, 1) -> e = E - 9 + (m > 0.875)."""
    m, E = torch.frexp(amax.float())
    e = E - 9 + (m > 0.875).to(E.dtype)
    e = e.clamp(-126, 126)
    return torch.where(amax > 0, e, torch.zeros_like(e))


def quantize_e4m3(t, group):
    """t [..., K] (fp32; K % group == 0) -> (q float8_e4m3fn [..., K], s fp32 [..., K / group]) with
    t ~ q * s per group.  Scaling by a power of two is exact, so the cast's round-to-nearest-even is the only rounding."""
    t = t.float()
    g = t.reshape(*t.shape[:-1], t.shape[-1] // group, group)
    e = scale_exponent(g.abs().amax(-1))
    s = torch.ldexp(torch.ones_like(e, dtype=torch.float32), e)
    q = (g * torch.ldexp(torch.ones_like(e, dtype=torch.float32), -e)[..., None]).clamp(-E4M3_MAX, E4M3_MAX)
    return q.to(torch.float8_e4m3fn).reshape(t.shape), s


def dequantize_e4m3(q, s, group):
    g = q.float().reshape(*q.shape[:-1], q.shape[-1] // group, group)
    return (g * s[..., None]).reshape(q.shape)


def qdq_act(t, defects=()):
    """Activation format: 1 x 128 groups.  Defect "group_scale_from_wrong_group": k-block 1 is multiplied by k-block
    0's scale."""
    q, s = quantize_e4m3(t, 128)
    if "group_scale_from_wrong_group" in defects:
        s = s.clone()
        s[..., 1] = s[..., 0]
    return dequantize_e4m3(q, s, 128).to(t.dtype)


def qdq_weight(w, defects=()):
    """Weight format: one scale per output channel (row).  Defect "weight_scale_dropped": channel 5's scale is 1."""
    q, s = quantize_e4m3(w, w.shape[-1])
    if "weight_scale_dropped" in defects:
        s = s.clone()
        s[5] = 1.0
    return dequantize_e4m3(q, s, w.shape[-1]).to(w.dtype)


class _QdqLinearView(nn.Module):
    """The weight and bias of a linear, its weight quantize-dequantized (what dit_block_matched reads)."""

    def __init__(self, lin, defects=()):
        super().__init__()
        self.weight = nn.Parameter(qdq_weight(lin.weight.detach().float(), defects).to(lin.weight.dtype),
                                   requires_grad=False)
        self.bias = lin.bias


@torch.no_grad()
def dit_block_fp8_matched(blk, x, mod, head_chunk=None, feed=None, defects=()):
    """One DiTBlock as the FP8 path computes it, in fp64: dit_block_matched's arithmetic (bf16 rounding of qkv, P,
    the attention output and attn.proj's weight) with h1, h2 and u -- the A operands of qkv, fc1 and fc2 -- and those
    three weights quantize-dequantized in the FP8 format instead of bf16-rounded.  The quantizers see the unrounded
    values (the kernels quantize their fp32 results), so the block is composed from dit_block_matched in stages, each
    stage fed the quantized output of the one before.  feed: {name: tensor} for x_mid / h1q / h2q / uq replaces this
    function's own value (teacher forcing).  Returns dit_block_matched's dict plus h1q, h2q, uq (the dequantized
    GEMM inputs)."""
    feed = dict(feed or {})
    blk8 = copy.copy(blk)
    blk8.attn = copy.copy(blk.attn)
    blk8.mlp = copy.copy(blk.mlp)
    blk8.attn.qkv = _QdqLinearView(blk.attn.qkv, defects)
    blk8.mlp.fc1 = _QdqLinearView(blk.mlp.fc1, defects)
    blk8.mlp.fc2 = _QdqLinearView(blk.mlp.fc2, defects)
    q = lambda t: qdq_act(t, defects)  # noqa: E731
    run = lambda rounding, **fd: dit_block_matched(blk8, x, mod, feed=fd, rounding=rounding, head_chunk=head_chunk)  # noqa: E731
    h1q = feed.get("h1q")
    if h1q is None:
        h1q = q(run(False)["h1"])
    att = run(True, h1=h1q)  # bf16 attention as in the product, x_mid from the FP8 qkv
    x_mid = feed.get("x_mid", att["x_mid"])
    h2q = feed.get("h2q")
    if h2q is None:
        h2q = q(run(False, h1=h1q, x_mid=x_mid)["h2"])
    mlp = run(False, h1=h1q, x_mid=x_mid, h2=h2q)
    uq = feed.get("uq")
    if uq is None:
        uq = q(mlp["u"])
    out = run(False, h1=h1q, x_mid=x_mid, h2=h2q, u=uq)
    for k in ("qkv", "attn", "lse", "proj_out"):
        out[k] = att[k]
    out["x_mid"] = att["x_mid"]
    out.update(h1q=h1q, h2q=h2q, uq=uq)
    return out


class _Fp8Linear(nn.Module):
    def __init__(self, lin, defects=()):
        super().__init__()
        self.lin, self.defects = lin, defects

    def forward(self, x):
        return F.linear(qdq_act(x, self.defects), qdq_weight(self.lin.weight, self.defects), self.lin.bias)


def emulate_fp8(oracle, defects=()):
    """-> a copy of the DenoiserOracle `oracle` whose blocks run qkv / fc1 / fc2 on quantize-dequantized operands."""
    em = copy.deepcopy(oracle)
    for blk in em.transformer:
        blk.attn.qkv = _Fp8Linear(blk.attn.qkv, defects)
        blk.mlp.fc1 = _Fp8Linear(blk.mlp.fc1, defects)
        blk.mlp.fc2 = _Fp8Linear(blk.mlp.fc2, defects)
    return em
