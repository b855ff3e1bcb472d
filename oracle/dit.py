"""oracle/dit.py -- TEST INFRASTRUCTURE: plain-PyTorch fp32 restatement of the reference denoiser.

Follows diffusionGS/models/denoiser/denoiser.py:21-22,26-72,76-164,199-253,306-416 (object model),
denoiser_scene.py:232-263,314-429 (scene differences) and
diffusionGS/models/transformers/utils_transformer.py:26-36,246-290 (DiTBlock).
The block's arithmetic lives in a third-party dependency that is NOT under /root/reference:
timm==0.9.16 (requirement.txt:25) `timm.models.vision_transformer.Attention` and `Mlp`; their published
forward is restated here (qkv Linear -> reshape [B,N,3,H,hd] -> softmax(q k^T / sqrt(hd)) v -> proj;
fc1 -> GELU(tanh) -> fc2; dropout 0; qk_norm off).
PINNED: tests/test_oracle_dit_vs_reference.py (through tests/golden/make_dit_golden.py) executes the reference's OWN denoiser.py /
denoiser_scene.py / utils_transformer.py (loaded by path, tests/golden/ref_import.py; only the absent third-party
packages are stubbed -- timm's Attention there is an independent restatement over F.scaled_dot_product_attention)
and holds this file to it at 1e-6 (object + scene model, both ray_pe_type values); the same run's inputs/outputs are
committed as tests/golden/dit_ref_*.npz (tests/golden/make_dit_golden.py) for boxes without /root/reference.
Same module tree / state_dict keys as the reference so a reference checkpoint loads with strict=True.
Never imported by the product path.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F


def modulate(x, shift, scale):
    return x * (1 + scale.unsqueeze(1)) + shift.unsqueeze(1)


class Attention(nn.Module):  # timm 0.9.16 semantics
    def __init__(self, dim, num_heads):
        super().__init__()
        self.num_heads, self.head_dim = num_heads, dim // num_heads
        self.qkv = nn.Linear(dim, dim * 3, bias=True)
        self.proj = nn.Linear(dim, dim)

    def forward(self, x):
        B, N, C = x.shape
        qkv = self.qkv(x).reshape(B, N, 3, self.num_heads, self.head_dim).permute(2, 0, 3, 1, 4)
        q, k, v = qkv.unbind(0)
        att = (q * self.head_dim ** -0.5) @ k.transpose(-2, -1)
        x = att.softmax(dim=-1) @ v
        return self.proj(x.transpose(1, 2).reshape(B, N, C))


class Mlp(nn.Module):  # timm 0.9.16 semantics, act = GELU(tanh)
    def __init__(self, dim, hidden):
        super().__init__()
        self.fc1, self.fc2 = nn.Linear(dim, hidden), nn.Linear(hidden, dim)

    def forward(self, x):
        return self.fc2(F.gelu(self.fc1(x), approximate="tanh"))


class DiTBlock(nn.Module):
    def __init__(self, dim, heads, mlp_ratio=4.0):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, elementwise_affine=False, eps=1e-6)
        self.attn = Attention(dim, heads)
        self.norm2 = nn.LayerNorm(dim, elementwise_affine=False, eps=1e-6)
        self.mlp = Mlp(dim, int(dim * mlp_ratio))
        self.adaLN_modulation = nn.Sequential(nn.SiLU(), nn.Linear(dim, 6 * dim, bias=True))

    def forward(self, x, c):
        s1, c1, g1, s2, c2, g2 = self.adaLN_modulation(c).chunk(6, dim=1)
        x = x + g1.unsqueeze(1) * self.attn(modulate(self.norm1(x), s1, c1))
        x = x + g2.unsqueeze(1) * self.mlp(modulate(self.norm2(x), s2, c2))
        return x


class TimestepEmbedder(nn.Module):
    def __init__(self, hidden, freq=256):
        super().__init__()
        self.mlp = nn.Sequential(nn.Linear(freq, hidden), nn.SiLU(), nn.Linear(hidden, hidden))
        self.freq = freq

    def forward(self, t):
        half = self.freq // 2
        freqs = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32, device=t.device) / half)
        args = t[:, None].float() * freqs[None]
        emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
        return self.mlp(emb.to(self.mlp[0].weight.dtype))


class _Head(nn.Module):
    def __init__(self, dim, out):
        super().__init__()
        self.layernorm = nn.LayerNorm(dim, bias=False)
        self.linear = nn.Linear(dim, out, bias=False)
        self.adaLN_modulation = nn.Sequential(nn.SiLU(), nn.Linear(dim, 2 * dim, bias=True))

    def forward(self, x, c):
        shift, scale = self.adaLN_modulation(c).chunk(2, dim=1)
        return self.linear(modulate(self.layernorm(x), shift, scale))


def _bf16(t):
    return t.to(torch.bfloat16).to(t.dtype)


def cond64(model, t, fp32_args=False, defects=()):
    """c = t_embedder(t) in fp64 (the adaLN input before its SiLU), differentiable in the module's parameters.
    fp32_args: the timestep argument t * freq is formed in fp32, as the reference (TimestepEmbedder.forward) and the
    kernel do; at t ~ 1e3 that moves c by ~1e-5 against the fp64 argument.  defects: see END_DEFECTS."""
    te = model.t_embedder.mlp
    half = te[0].weight.shape[1] // 2
    if fp32_args:
        freqs = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32, device=t.device) / half)
        args = (t[:, None].float() * freqs[None]).double()
    else:
        freqs = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float64, device=t.device) / half)
        args = t[:, None].double() * freqs[None]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    if "cos_sin_swapped" in defects:
        emb = torch.cat([torch.sin(args), torch.cos(args)], dim=-1)
    h = F.silu(F.linear(emb, te[0].weight.double(), te[0].bias.double()))
    return F.linear(h, te[2].weight.double(), te[2].bias.double())


@torch.no_grad()
def conditioning64(model, t):
    """c = t_embedder(t) in fp64 (the adaLN input before its SiLU) for any module with the reference's tree."""
    return cond64(model, t)


@torch.no_grad()
def block_modulation64(blk, c):
    """[B, 6*width] fp64: shift_msa | scale_msa | gate_msa | shift_mlp | scale_mlp | gate_mlp of one DiTBlock."""
    lin = blk.adaLN_modulation[1]
    return F.linear(F.silu(c.double()), lin.weight.double(), lin.bias.double())


@torch.no_grad()
def dit_block_matched(blk, x, mod, feed=None, rounding=True, softmax_scale=None, head_chunk=None):
    """One DiTBlock (same arithmetic as DiTBlock.forward) in fp64 from given inputs, rounding to bf16 where the CUDA
    kernels round: the LayerNorm+modulate outputs h1 / h2, the GEMM weights, the qkv GEMM output, the unnormalised
    softmax probabilities P (scaled by the row max, normalised after P.V by the fp64 sum of the unrounded ones), the
    attention output and the GELU output u.  The gated residual updates use the unrounded branch outputs, as the
    fused GEMM epilogues do.  rounding=False: the plain fp64 block.

    blk: a DiTBlock-shaped module (attn.qkv, attn.proj, mlp.fc1, mlp.fc2; the adaLN linear is not read), x [B, N, w],
    mod [B, 6w] (block_modulation64).  feed: {name: tensor} replaces this function's own value of that intermediate by
    the given one before it is used downstream (teacher forcing: each stage is fed the product's previous tensor);
    keys out of x_mid, h1, qkv, attn, h2, u.  head_chunk: heads per attention pass (bounds the fp64 score memory).
    Returns every intermediate (fp64): h1, qkv, attn, lse (log2-domain log-sum-exp of the scaled scores, [B, heads, N]),
    proj_out, x_mid, h2, u_pre, u, fc2_out, x_out."""
    feed = feed or {}
    rnd = _bf16 if rounding else (lambda t: t)
    B, N, D = x.shape
    heads = blk.attn.num_heads if hasattr(blk.attn, "num_heads") else D // 64
    hd = D // heads
    scale = hd ** -0.5 if softmax_scale is None else softmax_scale
    x = x.double()
    mod = mod.double()
    s1, c1, g1, s2, c2, g2 = (m[:, None, :] for m in mod.chunk(6, dim=1))
    W = lambda lin: rnd(lin.weight.detach().double())  # noqa: E731
    b = lambda lin: lin.bias.detach().double()  # noqa: E731
    get = lambda k, v: feed[k].double() if k in feed else v  # noqa: E731
    out = {}

    def ln(t):
        mu = t.mean(-1, keepdim=True)
        var = (t - mu).pow(2).mean(-1, keepdim=True)
        return (t - mu) / torch.sqrt(var + 1e-6)

    out["h1"] = rnd(ln(x) * (1 + c1) + s1)
    h1 = get("h1", out["h1"])
    out["qkv"] = rnd(F.linear(h1, W(blk.attn.qkv), b(blk.attn.qkv)))
    qkv = get("qkv", out["qkv"]).reshape(B, N, 3, heads, hd).permute(2, 0, 3, 1, 4)  # [3, B, H, N, hd]
    attn = torch.empty(B, heads, N, hd, dtype=torch.float64, device=x.device)
    lse = torch.empty(B, heads, N, dtype=torch.float64, device=x.device)
    step = head_chunk or heads
    for h0 in range(0, heads, step):
        q, k, v = (qkv[i, :, h0:h0 + step] for i in range(3))
        s = (q @ k.transpose(-1, -2)) * scale
        mx = s.amax(-1, keepdim=True)
        p = torch.exp(s - mx)
        den = p.sum(-1, keepdim=True)
        attn[:, h0:h0 + step] = (rnd(p) @ v) / den
        lse[:, h0:h0 + step] = (mx + torch.log(den)).squeeze(-1) / math.log(2.0)
        del s, p
    out["attn"] = rnd(attn.permute(0, 2, 1, 3).reshape(B, N, D))
    out["lse"] = lse
    a = get("attn", out["attn"])
    proj = F.linear(a, W(blk.attn.proj), b(blk.attn.proj))
    out["proj_out"] = rnd(proj)
    out["x_mid"] = x + g1 * proj
    x_mid = get("x_mid", out["x_mid"])
    out["h2"] = rnd(ln(x_mid) * (1 + c2) + s2)
    h2 = get("h2", out["h2"])
    pre = F.linear(h2, W(blk.mlp.fc1), b(blk.mlp.fc1))
    out["u_pre"] = rnd(pre)
    out["u"] = rnd(F.gelu(pre, approximate="tanh"))
    u = get("u", out["u"])
    fc2 = F.linear(u, W(blk.mlp.fc2), b(blk.mlp.fc2))
    out["fc2_out"] = rnd(fc2)
    out["x_out"] = x_mid + g2 * fc2
    return out


# named defects of the block backward (see dit_block_backward_matched); tests/test_dit_block_bwd_power_cpu.py shows the GPU
# checks would see each one; the product path never sets one
BWD_DEFECTS = ("gate_sample0_everywhere", "wgrad_tail_dropped", "last_key_dropped", "gelu_erf_grad", "ln_bwd_no_mean",
               "dscale_sample1_into_0")


def _gelu_tanh_grad(x):
    k0, k1 = math.sqrt(2.0 / math.pi), 0.044715
    t = torch.tanh(k0 * (x + k1 * x ** 3))
    return 0.5 * (1.0 + t) + 0.5 * x * (1.0 - t * t) * k0 * (1.0 + 3.0 * k1 * x * x)


def _gelu_erf_grad(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


@torch.no_grad()
def dit_block_backward_matched(blk, fwd, mod, c, dx_out, feed=None, rounding=True, head_chunk=None, defects=()):
    """Backward of one DiTBlock in fp64 from the forward tensors `fwd` and the gradient dx_out [B, N, w] of its output,
    rounding to bf16 where the backward kernels round:
      d_fc2_out = bf16(gate_mlp dx) and d_proj_out = bf16(gate_msa dx_mid) (gate_bwd);
      du_pre = bf16((d_fc2_out W2) gelu'(u_pre)) with the tanh GELU (the fc2 dgrad's dGELU epilogue);
      dh2, d_attn, dh1 = bf16 of the fc1 / attn.proj / qkv dgrads, the weights in bf16 (the transposed copies);
      attention: P = exp2(S log2(e) / 8 - lse2) from the forward's lse2, Dsum = rowsum(attn d_attn), dV = bf16(P)^T dO,
      dS = P (dP - Dsum) / 8 rounded to bf16 before dQ = dS K and dK = dS^T Q, dqkv stored in bf16.
    The weight and bias gradients are fp64 sums of the same bf16 operands the kernels multiply; dx_mid and dx (fp32 in the
    kernels) are not rounded.  rounding=False: the plain fp64 backward (then `fwd` should be the plain forward's).

    blk: a DiTBlock-shaped module (its fp32 weights are read); fwd: {x, x_mid, h1, qkv, attn, lse, proj_out, h2, u_pre, u,
    fc2_out} as dgs_dit_export_state / dit_block_matched give them (lse [B, heads, >= N] in log2 units); mod [B, 6w] the
    block's adaLN modulation, c [B, w] the conditioning before the SiLU.  feed: {name: tensor} replaces this function's
    own value of an intermediate gradient by the given one before it is used downstream (teacher forcing), keys out of
    d_fc2_out, du_pre, dh2, dx_mid, d_proj_out, d_attn, dqkv, dh1.  head_chunk: heads per attention pass (bounds the fp64
    score memory).  defects: names out of BWD_DEFECTS.
    Returns every gradient (fp64): d_fc2_out, du_pre, dh2, dx_mid, d_proj_out, d_attn, dsum [B, heads, N], dqkv, dh1, dx,
    dmod [B, 6w], and the parameter gradients under the block's parameter names (attn.qkv.weight, ...,
    adaLN_modulation.1.bias)."""
    feed = feed or {}
    rnd = _bf16 if rounding else (lambda t: t)
    f = {k: v.double() for k, v in fwd.items()}
    dx = dx_out.double()
    B, N, D = dx.shape
    heads = blk.attn.num_heads if hasattr(blk.attn, "num_heads") else D // 64
    hd = D // heads
    scale = hd ** -0.5
    mod = mod.double()
    s1, c1, g1, s2, c2, g2 = (m[:, None, :] for m in mod.chunk(6, dim=1))
    W = lambda lin: rnd(lin.weight.detach().double())  # noqa: E731
    get = lambda k, v: feed[k].double() if k in feed else v  # noqa: E731
    M = B * N
    keep = (M // 128) * 128 if "wgrad_tail_dropped" in defects else M
    out, dmod = {}, torch.zeros(B, 6 * D, dtype=torch.float64, device=dx.device)

    def linear_grads(name, dy, a):  # dW = dy^T a, db = sum dy over the rows
        dy2, a2 = dy.reshape(M, -1), a.reshape(M, -1)
        out[name + ".weight"] = dy2[:keep].t() @ a2[:keep]
        out[name + ".bias"] = dy2.sum(0)

    def gate(g, t):
        return rnd((g[:1] if "gate_sample0_everywhere" in defects else g) * t)

    def ln_modulate_bwd(x, dh, c_):  # -> dx, dshift, dscale of h = LN(x; 1e-6) (1 + c_) + shift
        mu = x.mean(-1, keepdim=True)
        rstd = 1.0 / torch.sqrt((x - mu).pow(2).mean(-1, keepdim=True) + 1e-6)
        xh = (x - mu) * rstd
        dxh = dh * (1 + c_)
        m1 = 0.0 if "ln_bwd_no_mean" in defects else dxh.mean(-1, keepdim=True)
        dscale = (dh * xh).sum(1)
        if "dscale_sample1_into_0" in defects and B > 1:
            dscale = torch.cat([dscale[:1] + dscale[1:2], torch.zeros_like(dscale[1:2]), dscale[2:]])
        return rstd * (dxh - m1 - xh * (dxh * xh).mean(-1, keepdim=True)), dh.sum(1), dscale

    # -- MLP branch: x_out = x_mid + gate_mlp * fc2(gelu(fc1(h2)))
    out["d_fc2_out"] = gate(g2, dx)
    d_fc2 = get("d_fc2_out", out["d_fc2_out"])
    dmod[:, 5 * D:] = (dx * f["fc2_out"]).sum(1)
    linear_grads("mlp.fc2", d_fc2, f["u"])
    dgelu = _gelu_erf_grad if "gelu_erf_grad" in defects else _gelu_tanh_grad
    out["du_pre"] = rnd((d_fc2 @ W(blk.mlp.fc2)) * dgelu(f["u_pre"]))
    du_pre = get("du_pre", out["du_pre"])
    linear_grads("mlp.fc1", du_pre, f["h2"])
    out["dh2"] = rnd(du_pre @ W(blk.mlp.fc1))
    ddx, dmod[:, 3 * D:4 * D], dmod[:, 4 * D:5 * D] = ln_modulate_bwd(f["x_mid"], get("dh2", out["dh2"]), c2)
    out["dx_mid"] = dx + ddx
    dx_mid = get("dx_mid", out["dx_mid"])
    # -- attention branch: x_mid = x_in + gate_msa * proj(attention(qkv(h1)))
    out["d_proj_out"] = gate(g1, dx_mid)
    d_proj = get("d_proj_out", out["d_proj_out"])
    dmod[:, 2 * D:3 * D] = (dx_mid * f["proj_out"]).sum(1)
    linear_grads("attn.proj", d_proj, f["attn"])
    out["d_attn"] = rnd(d_proj @ W(blk.attn.proj))
    d_attn = get("d_attn", out["d_attn"])
    split = lambda t: t.reshape(B, N, heads, hd).permute(0, 2, 1, 3)  # noqa: E731  [B, H, N, hd]
    q, k, v = f["qkv"].reshape(B, N, 3, heads, hd).permute(2, 0, 3, 1, 4)
    o, do = split(f["attn"]), split(d_attn)
    dsum = (o * do).sum(-1)
    out["dsum"] = dsum
    lse2 = f["lse"][:, :, :N]
    dqkv = torch.empty(3, B, heads, N, hd, dtype=torch.float64, device=dx.device)
    step = head_chunk or heads
    for h0 in range(0, heads, step):
        hs = slice(h0, h0 + step)
        s = q[:, hs] @ k[:, hs].transpose(-1, -2)
        p = torch.exp2(s * (scale / math.log(2.0)) - lse2[:, hs, :, None])
        del s
        ds = p * (do[:, hs] @ v[:, hs].transpose(-1, -2) - dsum[:, hs, :, None]) * scale
        dqkv[2, :, hs] = rnd(p).transpose(-1, -2) @ do[:, hs]
        del p
        ds = rnd(ds)
        dqkv[0, :, hs] = ds @ k[:, hs]
        dqkv[1, :, hs] = ds.transpose(-1, -2) @ q[:, hs]
        del ds
    if "last_key_dropped" in defects:
        dqkv[1:, :, :, N - 1] = 0.0
    out["dqkv"] = rnd(dqkv.permute(1, 3, 0, 2, 4).reshape(B, N, 3 * D))
    dqkv = get("dqkv", out["dqkv"])
    linear_grads("attn.qkv", dqkv, f["h1"])
    out["dh1"] = rnd(dqkv @ W(blk.attn.qkv))
    ddx, dmod[:, :D], dmod[:, D:2 * D] = ln_modulate_bwd(f["x"], get("dh1", out["dh1"]), c1)
    out["dx"] = dx_mid + ddx
    # -- adaLN: mod = Linear(silu(c))
    out["dmod"] = dmod
    out["adaLN_modulation.1.weight"] = dmod.t() @ F.silu(c.double())
    out["adaLN_modulation.1.bias"] = dmod.sum(0)
    return out


# ---- the stages on either side of the blocks, in fp64 and differentiable (fp64 autograd gives their backward) ----
# matched=True rounds where the kernels round; plain fp64 otherwise.  `defects` plants a named defect (END_DEFECTS) so
# that tests/test_dit_ends_power_cpu.py can show the GPU checks would see it; the product path never sets one.
END_DEFECTS = ("lo_dropped_tokenizer", "lo_dropped_upsampler", "lo_dropped_decoder", "cross_swapped",
               "clamp_grad_everywhere", "depth_third_dropped", "pos_grad_sample0", "cos_sin_swapped")


def _hi_lo(t):
    hi = _bf16(t)
    return hi, _bf16(t - hi)


class _SplitLinear(torch.autograd.Function):
    """y = a W^T as the split-bf16 GEMMs compute it: hi(a) hi(W) + lo(a) hi(W) + hi(a) lo(W) (lo(a) lo(W) is the
    ~2^-18 term they leave out), and its backward as the kernels compute it: the output gradient g rounded to bf16
    first when g_bf16, da = bf16(g W_d) with W_d = hi(W) if dgrad_hi else W, dW = g^T hi(a) if wgrad_hi else
    g^T (hi(a) + lo(a)).  drop_lo: the two lo terms left out (a planted defect)."""

    @staticmethod
    def forward(ctx, a, w, g_bf16, dgrad_hi, wgrad_hi, drop_lo):
        ah, al = _hi_lo(a)
        wh, wl = _hi_lo(w)
        y = ah @ wh.t()
        if not drop_lo:
            y = y + al @ wh.t() + ah @ wl.t()
        ctx.save_for_backward(a, w)
        ctx.flags = (g_bf16, dgrad_hi, wgrad_hi)
        return y

    @staticmethod
    def backward(ctx, gy):
        a, w = ctx.saved_tensors
        g_bf16, dgrad_hi, wgrad_hi = ctx.flags
        g = _bf16(gy) if g_bf16 else gy
        da = dw = None
        if ctx.needs_input_grad[0]:
            da = _bf16(g @ (_bf16(w) if dgrad_hi else w))
        if ctx.needs_input_grad[1]:
            ah, al = _hi_lo(a)
            aw = ah if wgrad_hi else ah + al
            dw = g.reshape(-1, g.shape[-1]).t() @ aw.reshape(-1, a.shape[-1])
        return da, dw, None, None, None, None


def _linear64(a, w, matched, g_bf16, dgrad_hi, wgrad_hi, drop_lo=False):
    if matched:
        return _SplitLinear.apply(a, w.double(), g_bf16, dgrad_hi, wgrad_hi, drop_lo)
    return F.linear(a, w.double())


def _layernorm64(x, w, eps):
    mu = x.mean(-1, keepdim=True)
    var = (x - mu).pow(2).mean(-1, keepdim=True)
    y = (x - mu) / torch.sqrt(var + eps)
    return y if w is None else y * w.double()


def posed_patches64(images, ray_o, ray_d, ray_pe_type, patch, defects=()):
    """[B, V*(H/p)*(W/p), p*p*9] fp64: the posed image (rgb*2-1 | Pluecker rays) patchified as the tokenizer reads it
    ("b v c (hh ph) (ww pw) -> b (v hh ww) (ph pw c)")."""
    images, ray_o, ray_d = images[:, :, :3].double(), ray_o.double(), ray_d.double()
    if ray_pe_type == "relative_plk":
        o_dot_d = torch.sum(-ray_o * ray_d, dim=2, keepdim=True)
        posed = torch.cat([images * 2.0 - 1.0, ray_d, ray_o + o_dot_d * ray_d], dim=2)
    else:
        cross = torch.cross(ray_d, ray_o, dim=2) if "cross_swapped" in defects else torch.cross(ray_o, ray_d, dim=2)
        posed = torch.cat([images * 2.0 - 1.0, cross, ray_d], dim=2)
    b, v, c, h, w = posed.shape
    p = patch
    return posed.reshape(b, v, c, h // p, p, w // p, p).permute(0, 1, 3, 5, 4, 6, 2).reshape(b, -1, p * p * c)


def input_stage64(model, images, ray_o, ray_d, ray_pe_type, matched=False, eps=1e-5, patches=None, defects=()):
    """The input stage: {patches, tok, x_pre = [pos embedding | tok], x0 = LayerNorm(x_pre) * weight} in fp64.
    matched: the tokenizer product split-bf16 as the kernel computes it, and in the backward the weight gradient
    bf16(d tok)^T hi(patches).  `patches` replaces posed_patches64's (e.g. the product's)."""
    if patches is None:
        p = math.isqrt(model.image_tokenizer[1].weight.shape[1] // 9)
        patches = posed_patches64(images, ray_o, ray_d, ray_pe_type, p, defects)
    tok = _linear64(patches, model.image_tokenizer[1].weight, matched, g_bf16=True, dgrad_hi=True, wgrad_hi=True,
                    drop_lo="lo_dropped_tokenizer" in defects)
    B, D = tok.shape[0], tok.shape[-1]
    pos = model.gaussians_pos_embedding.double().reshape(-1, D)
    pos = pos[None].expand(B, -1, -1)
    if "pos_grad_sample0" in defects:
        pos = torch.cat([pos[:1], pos[1:].detach()], dim=0)
    x_pre = torch.cat([pos, tok], dim=1)
    x0 = _layernorm64(x_pre, model.transformer_input_layernorm.weight, eps)
    return dict(patches=patches, tok=tok, x_pre=x_pre, x0=x0)


def mod_table64(model, c):
    """[B, L*6w + 4w] fp64: the adaLN modulation of every block (shift_msa | scale_msa | gate_msa | shift_mlp |
    scale_mlp | gate_mlp) then of the upsampler and the decoder head (shift | scale each), from c (cond64)."""
    lins = [blk.adaLN_modulation[1] for blk in model.transformer] + \
        [model.upsampler.adaLN_modulation[1], model.image_token_decoder.adaLN_modulation[1]]
    s = F.silu(c.double())
    return torch.cat([F.linear(s, lin.weight.double(), lin.bias.double()) for lin in lins], dim=1)


def head_channels(sh_degree):
    """Channels per Gaussian of both heads: xyz 3 | features 3 (d+1)^2 | scaling 3 | rotation 4 | opacity 1."""
    return 11 + 3 * (sh_degree + 1) ** 2


def gaussians_epilogue(gs_tok, img_gs, ray_o, ray_d, depth_mode, near=0.0, far=500.0, defects=()):
    """The raw head outputs -> the renderer-ready Gaussians (denoiser.py:94-98, 103-120, 145-149, 362-413;
    denoiser_scene.py:263, 406-410) in the dtype of the inputs.  gs_tok [B, G, C], img_gs [B, T, p*p*C] with
    C = head_channels(d) split [xyz 3 | features 3 (d+1)^2 | scaling 3 | rotation 4 | opacity 1]; the features reshape
    coefficient-major, RGB-minor to [B, G + T*p*p, (d+1)^2, 3].  depth_mode 0: (2 sigmoid(m) - 1) * 1.8 + o.(-d)
    (object model, 'relative_plk'), 1: sigmoid(m) * (far - near) + near (scene model), 2: sigmoid(m) (object model,
    'plk').  -> {xyz, features, scaling, rotation, opacity, img_aligned_xyz, depth_m (the sigmoid argument m)}."""
    b, v, _, h, w = ray_o.shape
    C = gs_tok.shape[-1]
    p = math.isqrt(img_gs.shape[-1] // C)
    img_g = img_gs.reshape(b, -1, C)
    allg = torch.cat((gs_tok, img_g), dim=1)
    xyz, features, scaling, rotation, opacity = allg.split([3, C - 11, 3, 4, 1], dim=2)
    features = features.reshape(b, -1, (C - 11) // 3, 3)
    if "clamp_grad_everywhere" in defects:
        scaling = scaling - 2.3 + ((scaling - 2.3).clamp(max=-1.20) - (scaling - 2.3)).detach()
    else:
        scaling = (scaling - 2.3).clamp(max=-1.20)
    opacity = opacity - 2.0
    n_img = img_g.shape[1]
    ia = xyz[:, -n_img:, :].reshape(b, v, h // p, w // p, p, p, 3).permute(0, 1, 6, 2, 4, 3, 5).reshape(b, v, 3, h, w)
    m = ia.mean(dim=2, keepdim=True)
    if "depth_third_dropped" in defects:
        s = ia.sum(dim=2, keepdim=True)
        m = s - (s - m).detach()
    if depth_mode == 1:
        depth = torch.sigmoid(m) * (far - near) + near
    elif depth_mode == 0:
        depth = (2.0 * torch.sigmoid(m) - 1.0) * 1.8 + torch.sum(-ray_o * ray_d, dim=2, keepdim=True)
    else:
        depth = torch.sigmoid(m)
    ia = ray_o + depth * ray_d
    ia_flat = ia.reshape(b, v, 3, h // p, p, w // p, p).permute(0, 1, 3, 5, 4, 6, 2).reshape(b, -1, 3)
    xyz = torch.cat((xyz[:, :-n_img, :], ia_flat), dim=1)
    return dict(xyz=xyz, features=features, scaling=scaling, rotation=rotation, opacity=opacity, img_aligned_xyz=ia,
                depth_m=m)


def gaussians_epilogue64(gs_tok, img_gs, ray_o, ray_d, depth_mode, near=0.0, far=500.0, defects=()):
    """gaussians_epilogue in fp64."""
    return gaussians_epilogue(gs_tok.double(), img_gs.double(), ray_o.double(), ray_d.double(), depth_mode, near, far,
                              defects)


def heads64(model, x, mod_heads, ray_o, ray_d, depth_mode, near=0.0, far=500.0, matched=False, defects=(), feed=None):
    """The two heads on the final residual stream x [B, G + T, w] with their modulation mod_heads [B, 4w] (the last
    4w columns of mod_table64): {gs_tok [B, G, C], img_gs [B, T, p*p*C], h_ups, h_dec} and every output of
    gaussians_epilogue64.  matched: the upsampler and decoder products split-bf16 as the kernels compute them; in the
    backward the decoder's output gradient d_img and both heads' dh rounded to bf16, dh of the decoder through hi(W),
    and its weight gradient through hi(h).  feed: {"gs_tok" / "img_gs": tensor} -- the epilogue runs on the given raw
    outputs (e.g. the product's) while the gradient still flows into this function's own heads, so that a raw value
    within rounding noise of the `scaling` clamp takes the same branch as in the product's backward."""
    x = x.double()
    G = model.gaussians_pos_embedding.numel() // x.shape[-1]
    D = x.shape[-1]
    mu, md = mod_heads[:, :2 * D].double(), mod_heads[:, 2 * D:].double()
    ups, dec = model.upsampler, model.image_token_decoder
    h_ups = modulate(_layernorm64(x[:, :G], ups.layernorm.weight, 1e-5), mu[:, :D], mu[:, D:])
    h_dec = modulate(_layernorm64(x[:, G:], dec.layernorm.weight, 1e-5), md[:, :D], md[:, D:])
    gs_tok = _linear64(h_ups, ups.linear.weight, matched, g_bf16=False, dgrad_hi=False, wgrad_hi=False,
                       drop_lo="lo_dropped_upsampler" in defects)
    img_gs = _linear64(h_dec, dec.linear.weight, matched, g_bf16=True, dgrad_hi=True, wgrad_hi=True,
                       drop_lo="lo_dropped_decoder" in defects)
    feed = feed or {}
    fed = lambda k, v: v + (feed[k].double() - v).detach() if k in feed else v  # noqa: E731
    out = gaussians_epilogue64(fed("gs_tok", gs_tok), fed("img_gs", img_gs), ray_o, ray_d, depth_mode, near, far, defects)
    out.update(gs_tok=gs_tok, img_gs=img_gs, h_ups=h_ups, h_dec=h_dec)
    return out


def _init_linear(m):
    if isinstance(m, nn.Linear):
        nn.init.normal_(m.weight, mean=0.0, std=0.02)
        if m.bias is not None:
            nn.init.zeros_(m.bias)


class DenoiserOracle(nn.Module):
    def __init__(self, width=1024, heads=16, layers=24, patch=8, n_gaussians=2, scene=False, near=0.0, far=500.0,
                 ray_pe_type=None, sh_degree=0):
        super().__init__()
        self.width, self.patch, self.G, self.scene, self.near, self.far = width, patch, n_gaussians, scene, near, far
        # yaml defaults: object configs leave the class default 'relative_plk' (denoiser.py:186), scene configs set 'plk'
        self.ray_pe_type = ray_pe_type or ("plk" if scene else "relative_plk")
        self.t_embedder = TimestepEmbedder(width)
        nn.init.normal_(self.t_embedder.mlp[0].weight, std=0.02)
        nn.init.normal_(self.t_embedder.mlp[2].weight, std=0.02)
        self.image_tokenizer = nn.Sequential(nn.Identity(), nn.Linear(9 * patch * patch, width, bias=False))
        self.image_tokenizer.apply(_init_linear)
        shape = (1, n_gaussians, width) if scene else (n_gaussians, width)
        self.gaussians_pos_embedding = nn.Parameter(torch.randn(*shape))
        nn.init.trunc_normal_(self.gaussians_pos_embedding, std=0.02)
        self.transformer_input_layernorm = nn.LayerNorm(width, bias=False)
        self.transformer = nn.ModuleList([DiTBlock(width, heads) for _ in range(layers)])
        self.transformer.apply(_init_linear)
        C = head_channels(sh_degree)
        self.upsampler = _Head(width, C)
        self.upsampler.apply(_init_linear)
        self.image_token_decoder = _Head(width, patch * patch * C)
        self.image_token_decoder.apply(_init_linear)

    def image_to_gaussians(self, images, ray_o, ray_d, t, return_tokens=False):
        p = self.patch
        o_dot_d = torch.sum(-ray_o * ray_d, dim=2, keepdim=True)
        if self.ray_pe_type == "relative_plk":  # denoiser.py:312-322 == denoiser_scene.py:319-331
            posed = torch.cat([images[:, :, :3] * 2.0 - 1.0, ray_d, ray_o + o_dot_d * ray_d], dim=2)
        else:
            posed = torch.cat([images[:, :, :3] * 2.0 - 1.0, torch.cross(ray_o, ray_d, dim=2), ray_d], dim=2)
        b, v, c, h, w = posed.shape
        # "b v c (hh ph) (ww pw) -> (b v) (hh ww) (ph pw c)"
        tok = posed.reshape(b, v, c, h // p, p, w // p, p).permute(0, 1, 3, 5, 4, 6, 2).reshape(b * v, -1, p * p * c)
        tok = self.image_tokenizer(tok).reshape(b, -1, self.width)
        temb = self.t_embedder(t)
        pos = self.gaussians_pos_embedding.reshape(self.G, self.width).expand(b, -1, -1)
        x = self.transformer_input_layernorm(torch.cat((pos, tok), dim=1))
        for blk in self.transformer:
            x = blk(x, temb)
        tokens = x
        g_tok, i_tok = x.split([self.G, x.shape[1] - self.G], dim=1)
        # the scene model's range_func whatever ray_pe_type is (denoiser_scene.py:263,406-410); denoiser.py:381-388
        depth_mode = 1 if self.scene else (0 if self.ray_pe_type == "relative_plk" else 2)
        g = gaussians_epilogue(self.upsampler(g_tok, temb), self.image_token_decoder(i_tok, temb), ray_o, ray_d,
                               depth_mode, self.near, self.far)
        out = {k: g[k] for k in ("xyz", "features", "scaling", "rotation", "opacity")}
        ia = g["img_aligned_xyz"]
        return (out, ia, tokens) if return_tokens else (out, ia)
