"""CPU checks of the DiT block tests' own machinery (no GPU):

* the trained-scale regime (tests/dit_regime.py) has the statistics it promises, on the oracle, so it cannot drift
  back to the near-identity blocks of the reference init;
* the rounding-matched block reference (oracle.dit.dit_block_matched) computes the same block as the fp32 oracle class;
* power: with the matched reference standing in for the kernels, defects planted in one block move that block's
  increment by at least twice the bound tests/test_dit_blocks_gpu.py applies on the H100, i.e. the per-block check
  would catch them.
"""
import copy
import math

import pytest
import torch

from test_dit_blocks_gpu import BLOCK_MATCHED
from util import rel_l2 as rel

D = 1024


@pytest.fixture(scope="module")
def oracle24():
    from dit_regime import apply_trained_scale
    from oracle.dit import DenoiserOracle
    torch.manual_seed(0)
    return apply_trained_scale(DenoiserOracle(layers=24), seed=0)


def _inputs(B=2, V=4, H=32, W=32):
    g = torch.Generator().manual_seed(0)
    images = torch.rand(B, V, 3, H, W, generator=g)
    ray_o = torch.randn(B, V, 3, 1, 1, generator=g).expand(B, V, 3, H, W).contiguous() * 1.5
    ray_d = torch.nn.functional.normalize(torch.randn(B, V, 3, H, W, generator=g), dim=2)
    return images, ray_o, ray_d, torch.tensor([100, 800])


def test_trained_scale_regime_statistics(oracle24):
    from oracle.dit import block_modulation64, conditioning64
    o = oracle24
    images, ray_o, ray_d, t = _inputs()
    seen = []
    hooks = [b.register_forward_hook(lambda m, inp, out: seen.append((m, inp[0].detach(), out.detach())))
             for b in o.transformer]
    with torch.no_grad():
        o.image_to_gaussians(images, ray_o, ray_d, t)
    for h in hooks:
        h.remove()
    c = conditioning64(o, t)
    mod_rms, gate_dt, logit_std, x_rms = [], [], [], []
    for blk, x, _ in seen:
        chunks = block_modulation64(blk, c).chunk(6, dim=1)
        mod_rms.append([float(m.pow(2).mean().sqrt()) for m in chunks])
        gate_dt.append(min(float((chunks[i][0] - chunks[i][1]).pow(2).mean().sqrt()) for i in (2, 5)))
        with torch.no_grad():
            h1 = torch.nn.functional.layer_norm(x, (D,), eps=1e-6) * (1 + chunks[1][:, None].float()) + chunks[0][:, None].float()
            qkv = blk.attn.qkv(h1).reshape(x.shape[0], x.shape[1], 3, 16, 64)
            logits = torch.einsum("bnhd,bmhd->bhnm", qkv[:, :, 0], qkv[:, :, 1]) / 8
        logit_std.append(logits.std(dim=(0, 2, 3)))
        x_rms.append(float(x.pow(2).mean().sqrt()))
    x_rms.append(float(seen[-1][2].pow(2).mean().sqrt()))
    ls = torch.stack(logit_std)
    print("modulation rms per chunk: min %.3f max %.3f" % (min(map(min, mod_rms)), max(map(max, mod_rms))))
    print("gate change between t=100 and t=800 (rms): min %.3f" % min(gate_dt))
    print("head logit std: min %.2f max %.2f; heads above 5: %d / %d" % (ls.min(), ls.max(), int((ls > 5).sum()), ls.numel()))
    print("residual stream rms per layer: " + " ".join(f"{v:.2f}" for v in x_rms))
    # shift / scale / gate of every block: rms ~0.3 (reference init: 0.025), and they depend on t
    assert all(0.2 < v < 0.45 for row in mod_rms for v in row), mod_rms
    assert min(gate_dt) > 0.15, gate_dt
    # every layer has peaky heads (logit std > 5) and near-flat ones (std < 1.5)
    assert bool((ls.amax(1) > 5).all()) and bool((ls.amin(1) < 1.5).all()), ls
    assert 0.15 < float((ls > 5).float().mean()) < 0.6
    # the residual stream stays O(1-3) through 24 layers, and every block moves it
    assert all(0.8 < v < 3.5 for v in x_rms), x_rms
    incr = [rel(out, x) for _, x, out in seen]
    assert min(incr) > 0.1, incr
    # non-zero biases everywhere, LayerNorm weights other than 1
    for name, p in o.named_parameters():
        if name.endswith("bias"):
            assert float(p.abs().mean()) > 0.05, name
        if "layernorm" in name:
            assert float((p - 1).abs().mean()) > 0.05, name


def _block_case(oracle24, B=2, N=130, layer=5):
    from oracle.dit import block_modulation64, conditioning64
    g = torch.Generator().manual_seed(1)
    blk = oracle24.transformer[layer]
    x = torch.randn(B, N, D, generator=g, dtype=torch.float64) * 1.5
    mod = block_modulation64(blk, conditioning64(oracle24, torch.tensor([100, 800][:B])))
    return blk, x, mod


def test_matched_reference_is_the_oracle_block(oracle24):
    """rounding=False is the fp32 DiTBlock in fp64; rounding=True differs from it by bf16 noise only; feeding the
    reference its own intermediates changes nothing."""
    from oracle.dit import conditioning64, dit_block_matched
    blk, x, mod = _block_case(oracle24)
    c = conditioning64(oracle24, torch.tensor([100, 800]))
    with torch.no_grad():
        ref32 = blk(x.float(), c.float()).double()
    plain = dit_block_matched(blk, x, mod, rounding=False)
    assert rel(plain["x_out"] - x, ref32 - x) < 1e-5
    matched = dit_block_matched(blk, x, mod)
    e = rel(matched["x_out"] - x, plain["x_out"] - x)
    print(f"matched vs plain block increment: {e:.2e}")
    assert 1e-4 < e < 2e-2
    fed = dit_block_matched(blk, x, mod, feed={k: matched[k] for k in ("h1", "qkv", "attn", "x_mid", "h2", "u")})
    for k in matched:
        assert torch.equal(fed[k], matched[k]), k
    chunked = dit_block_matched(blk, x, mod, head_chunk=3)
    assert rel(chunked["x_out"], matched["x_out"]) < 1e-12


def _power(clean, bad, x):
    return rel(bad["x_out"] - x, clean["x_out"] - x)


def test_planted_block_defects_exceed_the_gpu_bound(oracle24):
    from oracle.dit import dit_block_matched
    blk, x, mod = _block_case(oracle24)
    B, N, _ = x.shape
    clean = dit_block_matched(blk, x, mod)
    incr = clean["x_out"] - x
    power = {}

    # the gate of the wrong sample: sample 1's rows gated with sample 0's gate_msa / gate_mlp
    m = mod.clone()
    for i in (2, 5):
        m[1, i * D:(i + 1) * D] = mod[0, i * D:(i + 1) * D]
    power["gate of the wrong sample"] = _power(clean, dit_block_matched(blk, x, m), x)

    # the last two rows of the last sample not updated (the 2-row tail tile of M = 4098).  Norm-wise the defect shrinks
    # with the row count, so it is scaled to one sample of N = 4098 rows with this block's mean row increment.
    row2 = incr.pow(2).sum(-1)
    power["last two rows not updated"] = float(row2[-1, -2:].sum().sqrt() / (row2.mean() * 4098).sqrt())

    # attn.proj bias dropped
    nb = copy.deepcopy(blk)
    with torch.no_grad():
        nb.attn.proj.bias.zero_()
    power["proj bias dropped"] = _power(clean, dit_block_matched(nb, x, mod), x)

    # shift and scale swapped in both LayerNorm+modulate calls
    m = mod.clone()
    for a, b in ((0, 1), (3, 4)):
        m[:, a * D:(a + 1) * D], m[:, b * D:(b + 1) * D] = mod[:, b * D:(b + 1) * D], mod[:, a * D:(a + 1) * D]
    power["shift and scale swapped"] = _power(clean, dit_block_matched(blk, x, m), x)

    # the attention gate used for the MLP branch
    m = mod.clone()
    m[:, 5 * D:] = mod[:, 2 * D:3 * D]
    power["gate_msa used for the MLP"] = _power(clean, dit_block_matched(blk, x, m), x)

    # one head's attention output 5 % off
    def head_off(f, h=3):
        a = clean["attn"].clone()
        a[..., h * 64:(h + 1) * 64] *= f
        return dit_block_matched(blk, x, mod, feed={"attn": a.to(torch.bfloat16).double()})
    power["one head 5 % off"] = _power(clean, head_off(1.05), x)

    for k, v in power.items():
        print(f"{k:28s} {v:.2e}  ({v / BLOCK_MATCHED:.1f} x the bound {BLOCK_MATCHED:.1e})")
    for k, v in power.items():
        assert v >= 2 * BLOCK_MATCHED, (k, v)

    # Finer than the bound resolves with a 2x margin (the kernels' own per-block noise is up to 1.7e-3):
    # * the softmax scale 1 % off moves the increment by ~3.7e-3: above the bound, so usually flagged, but not 2x above;
    # * one head's output 1 % off moves it by ~2.0e-3: below the bound, inside the kernels' noise, not caught.
    scale_1pct = _power(clean, dit_block_matched(blk, x, mod, softmax_scale=1.01 / math.sqrt(64)), x)
    one_pct = _power(clean, head_off(1.01), x)
    print(f"softmax scale 1 % off {scale_1pct:.2e}; one head 1 % off {one_pct:.2e}")
    assert BLOCK_MATCHED < scale_1pct < 2 * BLOCK_MATCHED
    assert one_pct < BLOCK_MATCHED
