"""Trained-scale weights for the DiT block tests.

At the reference's init (weights N(0, 0.02), zero biases) the adaLN gates have rms ~0.025 and the 24 blocks barely
change the residual stream, so an end-to-end comparison says little about any one block.  `apply_trained_scale`
rescales a DGSDenoiser (or the oracle's DenoiserOracle: same module tree) in place, deterministically from `seed`:

* timestep embedder at unit gain, so the conditioning varies with t;
* adaLN: bias N(0, 0.2^2) plus a t-dependent part of rms ~0.2: shift / scale / gate of rms ~0.3;
* attention: q and k rows of every head scaled by a per-head factor, so that the logit std of the heads spreads from
  ~1 (flat rows) to ~8 (peaky rows); which head gets which factor is permuted per layer;
* non-zero biases on every linear layer, LayerNorm weights 1 + N(0, 0.2^2);
* fc1 / fc2 at unit gain, so the branch outputs are O(1) and the gated updates keep the residual stream O(1-3)
  through 24 layers.

tests/test_dit_block_power_cpu.py pins the resulting statistics on the oracle.

Also the seeded DiT inputs of the GPU tests (`dit_inputs`) and the oracle of a product model (`oracle_like`).
"""
import math

import torch

DEV = "cuda:0"

ADALN_BIAS_STD = 0.2
ADALN_DYNAMIC_RMS = 0.2
LOGIT_STD_RANGE = (0.8, 8.0)  # per-head q.k/sqrt(64) std for unit-rms LayerNorm outputs


def _fill(p, g, std, mean=0.0):
    with torch.no_grad():
        p.copy_((torch.randn(p.shape, generator=g, dtype=torch.float64) * std + mean).to(p.dtype))


def apply_trained_scale(model, seed=0):
    g = torch.Generator().manual_seed(1000 + seed)
    w = model.transformer_input_layernorm.weight.shape[0]
    heads = w // 64
    te = model.t_embedder.mlp
    _fill(te[0].weight, g, 2.0 / math.sqrt(te[0].weight.shape[1]))
    _fill(te[0].bias, g, 0.1)
    _fill(te[2].weight, g, 1.0 / math.sqrt(w))
    _fill(te[2].bias, g, 0.1)
    # silu(c) has rms ~0.5 for the embedder above; the adaLN weight turns it into the t-dependent part of the modulation
    adaln_w_std = ADALN_DYNAMIC_RMS / (0.5 * math.sqrt(w))
    _fill(model.transformer_input_layernorm.weight, g, 0.2, 1.0)
    for blk in model.transformer:
        _fill(blk.adaLN_modulation[1].weight, g, adaln_w_std)
        _fill(blk.adaLN_modulation[1].bias, g, ADALN_BIAS_STD)
        qkv = blk.attn.qkv
        _fill(qkv.weight, g, 1.0 / math.sqrt(w))
        _fill(qkv.bias, g, 0.1)
        lo, hi = LOGIT_STD_RANGE
        logit_std = torch.exp(torch.linspace(math.log(lo), math.log(hi), heads, dtype=torch.float64))
        gain = logit_std.sqrt()[torch.randperm(heads, generator=g)]  # q and k each carry sqrt(logit std)
        with torch.no_grad():
            rows = gain.repeat_interleave(64).to(qkv.weight.dtype)
            qkv.weight[:w] *= rows[:, None]
            qkv.weight[w:2 * w] *= rows[:, None]
        _fill(blk.attn.proj.weight, g, 1.0 / math.sqrt(w))
        _fill(blk.attn.proj.bias, g, 0.5)
        _fill(blk.mlp.fc1.weight, g, 1.0 / math.sqrt(w))
        _fill(blk.mlp.fc1.bias, g, 0.3)
        _fill(blk.mlp.fc2.weight, g, 1.5 / math.sqrt(blk.mlp.fc2.weight.shape[1]))
        _fill(blk.mlp.fc2.bias, g, 0.3)
    for head in (model.upsampler, model.image_token_decoder):
        _fill(head.layernorm.weight, g, 0.2, 1.0)
        _fill(head.adaLN_modulation[1].weight, g, adaln_w_std)
        _fill(head.adaLN_modulation[1].bias, g, ADALN_BIAS_STD)
    return model


def oracle_like(model, **kw):
    """A DenoiserOracle with the configuration of the product model `model` (DGSDenoiser[Scene]), its parameters
    loaded strictly."""
    from oracle.dit import DenoiserOracle
    c = model.cfg
    o = DenoiserOracle(width=c.width, heads=c.width // c.dim_heads, layers=c.num_layers, patch=c.patch_size,
                       n_gaussians=c.n_gaussians, scene=model.SCENE, near=c.range_setting_near, far=c.range_setting_far,
                       ray_pe_type=c.ray_pe_type, sh_degree=c.gaussians_sh_degree, **kw)
    o.load_state_dict({k: v.detach() for k, v in model.state_dict().items()}, strict=True)
    return o.to(model.device)


def dit_inputs(B, V, H, W, seed=0):
    """Seeded (images, ray_o, ray_d, t) on the device: view 0 in [0, 1), the other views N(0, 1)."""
    g = torch.Generator(DEV).manual_seed(seed)
    images = torch.rand(B, V, 3, H, W, device=DEV, generator=g)
    images[:, 1:] = torch.randn(B, V - 1, 3, H, W, device=DEV, generator=g)
    ray_o = torch.randn(B, V, 3, 1, 1, device=DEV, generator=g).expand(B, V, 3, H, W).contiguous() * 1.5
    ray_d = torch.nn.functional.normalize(torch.randn(B, V, 3, H, W, device=DEV, generator=g), dim=2)
    t = torch.randint(0, 1000, (B,), device=DEV, generator=g)
    return images, ray_o, ray_d, t
