"""CPU checks of the block-backward tests' own machinery (no GPU), on a synthetic trained-scale block at width 1024,
B = 2, N = 130 tokens per sample (M = 260 rows: a 4-row tail past the last full 128-row tile, and sample 1 starting at
row 130, inside a tile):

* oracle.dit.dit_block_backward_matched(rounding=False) equals torch fp64 autograd through the oracle's DiTBlock;
  with rounding=True it stays within bf16 level of it;
* power: with the rounding-matched reference standing in for the kernels, each planted defect (BWD_DEFECTS) moves the
  tensor it touches by at least twice the bound tests/test_dit_blocks_bwd_gpu.py applies on the H100.
"""
import copy

import pytest
import torch

from test_dit_blocks_bwd_gpu import BWD
from util import rel_l2 as _rel

D, B, N = 1024, 2, 130


@pytest.fixture(scope="module")
def case():
    """-> (block, c, mod, x, dx_out) in fp64: a trained-scale block, a residual stream of the trained-scale size."""
    from dit_regime import apply_trained_scale
    from oracle.dit import DenoiserOracle, block_modulation64, cond64
    torch.manual_seed(0)
    model = apply_trained_scale(DenoiserOracle(layers=1), 0)
    blk = model.transformer[0]
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():
        c = cond64(model, torch.tensor([100.0, 900.0]))
    mod = block_modulation64(blk, c)
    x = torch.randn(B, N, D, generator=g, dtype=torch.float64) * 1.5 + torch.randn(D, generator=g, dtype=torch.float64) * 0.5
    dx_out = torch.randn(B, N, D, generator=g, dtype=torch.float64) * 1e-3
    return blk, c, mod, x, dx_out


def _fwd(blk, x, mod, rounding):
    from oracle.dit import dit_block_matched
    r = dit_block_matched(blk, x, mod, rounding=rounding)
    return dict(r, x=x)


def _autograd(blk, c, x, dx_out):
    """fp64 autograd through the oracle's DiTBlock: {x, the block's parameters, dmod}."""
    b64 = copy.deepcopy(blk).double()
    xr, cr = x.clone().requires_grad_(), c.clone().requires_grad_()
    mods = []

    def keep(module, args, o):
        o.retain_grad()
        mods.append(o)
    hook = b64.adaLN_modulation.register_forward_hook(keep)
    with torch.enable_grad():
        b64(xr, cr).backward(dx_out)
    hook.remove()
    out = {n: p.grad for n, p in b64.named_parameters()}
    out.update(dx=xr.grad, dmod=mods[0].grad)
    return out


def test_plain_backward_is_fp64_autograd(case):
    from oracle.dit import dit_block_backward_matched
    blk, c, mod, x, dx_out = case
    ref = _autograd(blk, c, x, dx_out)
    plain = dit_block_backward_matched(blk, _fwd(blk, x, mod, False), mod, c, dx_out, rounding=False, head_chunk=5)
    matched = dit_block_backward_matched(blk, _fwd(blk, x, mod, True), mod, c, dx_out)
    e_plain = {k: _rel(plain[k], v) for k, v in ref.items()}
    e_matched = {k: _rel(matched[k], v) for k, v in ref.items()}
    print("plain   " + "  ".join(f"{k}={v:.1e}" for k, v in e_plain.items()))
    print("matched " + "  ".join(f"{k}={v:.1e}" for k, v in e_matched.items()))
    assert set(ref) == {n for n, _ in blk.named_parameters()} | {"dx", "dmod"}
    assert max(e_plain.values()) < 1e-12, e_plain
    # bf16 rounding of the operands and stored gradients: ~1e-3 .. 1e-2, never 0 (the rounding is really applied)
    assert max(e_matched.values()) < 3e-2, e_matched
    assert min(e_matched.values()) > 1e-5, e_matched


def _checked(r, dx_out):
    """The quantities tests/test_dit_blocks_bwd_gpu.py checks, by the name of the bound it applies."""
    dx_mid = r["dx_mid"]
    out = {k: r[k] for k in ("d_fc2_out", "du_pre", "dh2", "d_proj_out", "d_attn", "dsum", "dqkv", "dh1", "dmod")}
    out["dx_mid"] = dx_mid - dx_out  # the increments, as on the GPU
    out["dx"] = r["dx"] - dx_mid
    for fam in ("attn.qkv", "attn.proj", "mlp.fc1", "mlp.fc2"):
        out[fam + ".weight"] = r[fam + ".weight"]
    out["adaLN"] = r["adaLN_modulation.1.weight"]
    return out


def _bound(name):
    return BWD["weight"] if name.endswith(".weight") else BWD[name]


def test_planted_backward_defects_exceed_the_gpu_bound(case):
    from oracle.dit import BWD_DEFECTS, dit_block_backward_matched
    blk, c, mod, x, dx_out = case
    fwd = _fwd(blk, x, mod, True)
    clean = _checked(dit_block_backward_matched(blk, fwd, mod, c, dx_out), dx_out)
    touches = {"gate_sample0_everywhere": ("d_fc2_out", "d_proj_out"),
               "wgrad_tail_dropped": ("attn.qkv.weight", "attn.proj.weight", "mlp.fc1.weight", "mlp.fc2.weight"),
               "last_key_dropped": ("dqkv",),
               "gelu_erf_grad": ("du_pre",),
               "ln_bwd_no_mean": ("dx_mid", "dx"),
               "dscale_sample1_into_0": ("dmod",)}
    assert set(touches) == set(BWD_DEFECTS)
    power = {}
    for defect, names in touches.items():
        bad = _checked(dit_block_backward_matched(blk, fwd, mod, c, dx_out, defects=(defect,)), dx_out)
        for k in names:
            power[f"{defect}: {k}"] = (_rel(bad[k], clean[k]), _bound(k))
    for k, (v, bound) in power.items():
        print(f"{k:40s} {v:.2e}  " + (f"({v / bound:.1f} x the bound {bound:.1e})" if bound else "(checked for equality)"))
    for k, (v, bound) in power.items():
        assert v >= 2 * bound and v > 0, (k, v, bound)
