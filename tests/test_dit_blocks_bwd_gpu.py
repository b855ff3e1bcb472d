"""Teacher-forced block-by-block tests of the DiT BACKWARD (dgs_dit_backward_ex) in the trained-scale weight regime
(tests/dit_regime.py), against oracle/dit.py's fp64 block backward (dit_block_backward_matched) on the device.

The end-to-end gradient tests (tests/test_dit_bwd_gpu.py) bound the whole gradient at ~2e-2: over 24 bf16 blocks they
cannot tell kernel noise from a 1 % defect in one block.  Here the backward's per-block gradients are read out with
the backward trace (DitTrainer.trace_backward, dgs_dit_bwd_opts.trace) and every stage of every block is compared
against the rounding-matched reference fed the product's previous tensor (d_fc2_out <- dx[l+1], du_pre <- d_fc2_out,
dh2 <- du_pre, dx_mid <- dh2, d_proj_out <- dx_mid, d_attn <- d_proj_out, dsum / dqkv <- d_attn, dh1 <- dqkv,
dx[l] <- dh1) and the product's own stored forward tensors (dgs_dit_export_state):

* every traced tensor, the block's eight linear weight / bias gradients, its 6w rows of dmod and its adaLN gradients;
* dx[l] against the plain fp64 backward of the plain fp64 forward of the product's x[l], fed dx[l+1];
* recompute mode (the backward re-runs each block's forward into the single slot first) against store mode;
* the obj-512 / scene-512 token count (N = 16386) on two layers.

Every bound below was set from the errors measured on an H100 80GB HBM3 over seeds 0, 1, 2; the measured worst case is
written next to it.  Errors are norm-wise relative; dx and dx_mid are compared as increments (dx[l] - dx_mid[l] and
dx_mid[l] - dx[l+1]), as the forward tests compare the residual updates.
"""
import gc

import pytest
import torch

from util import rel_l2 as _rel

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
OBJ256 = (1, 4, 256, 256)  # N = 4098 tokens: 32 full 128-row tiles and a 2-row tail
OUTS = ("xyz", "features", "scaling", "rotation", "opacity")
LINEARS = ("attn.qkv", "attn.proj", "mlp.fc1", "mlp.fc2")
FEED = ("d_fc2_out", "du_pre", "dh2", "dx_mid", "d_proj_out", "d_attn", "dqkv", "dh1")
STATE = ("x", "x_mid", "h1", "qkv", "attn", "lse", "proj_out", "h2", "u_pre", "u", "fc2_out")

# ---- bounds against the rounding-matched reference fed the product's previous tensor; measured worst in the comment ----
# (over every block of obj-256 B = 1 and B = 2 and of N = 16386).  d_fc2_out / d_proj_out = bf16(gate * dx) are
# bitwise those of the reference (0 measured): the fp32 product of two fp32 numbers is the fp64 one correctly rounded,
# and both sides then round it to bf16 the same way.
BWD = dict(d_fc2_out=0.0,
           du_pre=2.5e-4,    # 1.07e-4 (bf16 output; gelu' with tanh.approx)
           dh2=4e-4,         # 1.62e-4 (bf16 output of a K = 4096 product)
           dx_mid=5e-7,      # 2.12e-7 (increment dx_mid - dx[l+1]: the fp32 LayerNorm backward)
           d_proj_out=0.0,
           d_attn=2e-4,      # 8.2e-5
           dsum=1e-7,        # 4.1e-8
           dqkv=1.5e-3,      # 6.4e-4 (P and dS rounded to bf16 before their MMAs, exp2.approx)
           dh1=5e-4,         # 2.08e-4
           dx=8e-7,          # 3.05e-7 (increment dx[l] - dx_mid)
           weight=6e-5,      # 2.68e-5 at N = 16386, 1.95e-5 at N = 4098 (the four linears; fp32 sums over the tokens)
           bias=3e-7,        # 1.29e-7
           dmod=8e-7,        # 3.20e-7 (worst of the six 1w chunks)
           adaLN=8e-7)       # 2.94e-7
PLAIN_DX = 4e-2  # dx[l] - dx[l+1] against the plain fp64 backward (all bf16 rounding counted as error): 1.68e-2
# recompute mode against store mode: dx and dx_mid are bitwise equal (the refill reproduces store mode's forward tensors
# bit for bit); the parameter gradients differ by the order of their fp32 atomic sums: 2.09e-7
RECOMPUTE_PARAM = 5e-7


def backward_run(model, trainer, shape, seed, recompute, names=None):
    """One training forward + traced backward of the loss tests/test_dit_bwd_gpu._grad_compare uses (seeded random
    weights on the five outputs) -> ({name: stacked trace}, {parameter name: gradient copy})."""
    from dit_regime import dit_inputs
    trainer.recompute = recompute
    inputs = dit_inputs(*shape, seed=seed)
    tr = trainer.trace_backward() if names is None else trainer.trace_backward(names)
    with torch.enable_grad():
        out, _ = model.image_to_gaussians(*inputs)
        g = torch.Generator(DEV).manual_seed(11)
        wts = {k: torch.randn(out[k].shape, device=DEV, generator=g) for k in OUTS}
        trainer.zero_grad()
        sum((out[k] * wts[k]).sum() for k in OUTS).backward()
    grads = {n: p.grad.detach().clone() for n, p in model.named_parameters()}
    return tr, grads


def block_bwd_errors(model, trainer, ref, shape, seed=0, head_chunk=4, plain=True):
    """Store mode: per block {check: error} against dit_block_backward_matched fed the product's tensors."""
    from oracle.dit import dit_block_backward_matched, dit_block_matched
    B, V, H, W = shape
    tr, grads = backward_run(model, trainer, shape, seed, recompute=False)
    ex = trainer.export_ends(B, V, H, W, ("c", "mod", "dmod"))
    D = ex["c"].shape[1]
    errs = []
    for l, blk in enumerate(ref.transformer):
        st = trainer.export_state(B, V, H, W, l, STATE)
        N = st["x"].shape[1]
        m = ex["mod"][:, l * 6 * D:(l + 1) * 6 * D]
        dx_out = tr["dx"][l + 1].double()
        r = dit_block_backward_matched(blk, st, m, ex["c"], dx_out, feed={k: tr[k][l] for k in FEED},
                                       head_chunk=head_chunk)
        e = {k: _rel(tr[k][l], r[k]) for k in ("d_fc2_out", "du_pre", "dh2", "d_proj_out", "d_attn", "dqkv", "dh1")}
        e["dsum"] = _rel(tr["dsum"][l][:, :, :N], r["dsum"])
        dx_mid = tr["dx_mid"][l].double()
        e["dx_mid"] = _rel(dx_mid - dx_out, r["dx_mid"] - dx_out)
        e["dx"] = _rel(tr["dx"][l].double() - dx_mid, r["dx"] - dx_mid)
        p = f"transformer.{l}."
        e["weight"] = max(_rel(grads[p + n + ".weight"], r[n + ".weight"]) for n in LINEARS)
        e["bias"] = max(_rel(grads[p + n + ".bias"], r[n + ".bias"]) for n in LINEARS)
        dm = ex["dmod"][:, l * 6 * D:(l + 1) * 6 * D]
        e["dmod"] = max(_rel(dm[:, i * D:(i + 1) * D], r["dmod"][:, i * D:(i + 1) * D]) for i in range(6))
        e["adaLN"] = max(_rel(grads[p + "adaLN_modulation.1." + s], r["adaLN_modulation.1." + s]) for s in ("weight", "bias"))
        del r
        if plain:
            x = st["x"].double()
            fwd = dict(dit_block_matched(blk, x, m, rounding=False, head_chunk=head_chunk), x=x)
            rp = dit_block_backward_matched(blk, fwd, m, ex["c"], dx_out, rounding=False, head_chunk=head_chunk)
            e["plain_dx"] = _rel(tr["dx"][l].double() - dx_out, rp["dx"] - dx_out)
            del fwd, rp
        errs.append(e)
        del st
    return errs


def recompute_errors(model, trainer, shape, seed=0):
    """Per block {dx, dx_mid, param}: recompute mode's backward against store mode's on the same model and inputs."""
    tr_s, g_s = backward_run(model, trainer, shape, seed, recompute=False, names=("dx", "dx_mid"))
    tr_r, g_r = backward_run(model, trainer, shape, seed, recompute=True, names=("dx", "dx_mid"))
    errs = []
    for l in range(tr_s["dx_mid"].shape[0]):
        p = f"transformer.{l}."
        errs.append(dict(dx=_rel(tr_r["dx"][l], tr_s["dx"][l]), dx_mid=_rel(tr_r["dx_mid"][l], tr_s["dx_mid"][l]),
                         param=max(_rel(g_r[n], g_s[n]) for n in g_s if n.startswith(p))))
    return errs


def _report(tag, errs):
    names = list(errs[0])
    print(f"[{tag}] per block:")
    for l, e in enumerate(errs):
        print(f"  block {l:2d}: " + "  ".join(f"{k}={e[k]:.2e}" for k in names))
    worst = {k: max(e[k] for e in errs) for k in names}
    print(f"[{tag}] worst: " + "  ".join(f"{k}={v:.2e}" for k, v in worst.items()))
    return worst


def _check(errs):
    for l, e in enumerate(errs):
        for k, bound in BWD.items():
            assert e[k] <= bound, (l, k, e)
        if "plain_dx" in e:
            assert e["plain_dx"] < PLAIN_DX, (l, e)


@pytest.fixture(scope="module")
def obj24():
    from test_dit_blocks_gpu import build_models
    model, trainer, ref = build_models(24)
    yield model, trainer, ref
    del model, trainer, ref
    gc.collect()
    torch.cuda.empty_cache()


def test_blocks_backward_obj256_b1(obj24):
    """M = 4098 rows: the last 128-row tile of every GEMM and the last 64-key block of the attention hold 2 rows."""
    errs = block_bwd_errors(*obj24, OBJ256)
    _report("obj-256 B=1 backward", errs)
    _check(errs)


def test_blocks_backward_obj256_b2(obj24):
    """B = 2: sample 1 starts at row 4098, inside a 64-row and a 128-row tile, so gate_bwd's and the LayerNorm
    backward's per-sample sums (dmod) and the per-sample attention decide which sample's rows a tile's row gets."""
    errs = block_bwd_errors(*obj24, (2, 4, 256, 256), seed=1)
    _report("obj-256 B=2 backward", errs)
    _check(errs)


def test_blocks_backward_recompute_matches_store(obj24):
    """Recompute mode refills block l's forward (into slot 0, with dx_pre as the scratch output) right before
    differentiating it; its gradients must be those of store mode."""
    errs = recompute_errors(*obj24[:2], OBJ256, seed=2)
    worst = _report("obj-256 recompute vs store", errs)
    assert worst["dx"] == 0 and worst["dx_mid"] == 0, worst
    assert worst["param"] < RECOMPUTE_PARAM, worst


def test_trace_does_not_change_the_backward(obj24):
    """The trace only copies: with it armed, the gradients written by one GEMM are bitwise those of an untraced backward,
    the atomically accumulated ones equal to 1e-6.  At M = 4098 the qkv, fc1 and fc2 weight gradients are written tile by
    tile; attn.proj's (64 output tiles of 128 x 128) runs split-K with fp32 atomics, like the biases, the LayerNorm
    weights and the adaLN table's gradients, so its summation order varies from run to run."""
    from dit_regime import dit_inputs
    model, trainer, _ = obj24
    grads = []
    for traced in (False, True):
        trainer.recompute = False
        inputs = dit_inputs(*OBJ256, seed=4)
        if traced:
            trainer.trace_backward()
        with torch.enable_grad():
            out, _ = model.image_to_gaussians(*inputs)
            trainer.zero_grad()
            sum(out[k].double().square().sum() for k in OUTS).backward()
        grads.append({n: p.grad.detach().clone() for n, p in model.named_parameters()})
    gemm = [n for n in grads[0] if n.endswith(("attn.qkv.weight", "mlp.fc1.weight", "mlp.fc2.weight"))]
    assert len(gemm) == 3 * len(model.transformer)
    differ = [n for n in gemm if not torch.equal(grads[0][n], grads[1][n])]
    assert not differ, differ
    worst = max(_rel(grads[1][n], grads[0][n]) for n in grads[0])
    print(f"[trace on / off] worst parameter gradient difference {worst:.1e}")
    assert worst < 1e-6


def test_block_backward_n16386_two_layers():
    """The obj-512 / scene-512 token count (4 views at 512 x 512: N = 16386); the reference attention runs head by head so
    that the fp64 scores fit in memory."""
    from test_dit_blocks_gpu import build_models
    model, trainer, ref = build_models(2)
    errs = block_bwd_errors(model, trainer, ref, (1, 4, 512, 512), seed=3, head_chunk=1)
    _report("N=16386 backward", errs)
    _check(errs)


def test_localises_a_one_percent_fc1_dgrad_weight_error(obj24):
    """The backward runs with layer 7's transposed fc1 weight copy (read only by the fc1 dgrad) 1 % off: the per-block
    check flags block 7's dh2 and nothing else (every later stage is fed the product's own, already different, tensor)."""
    model, trainer, ref = obj24
    with torch.no_grad():
        trainer._wT_keep["fc1_wT"][7].mul_(1.01)
    try:
        errs = block_bwd_errors(model, trainer, ref, OBJ256, plain=False)
    finally:
        trainer.refresh_weights()
    _report("obj-256 fc1_wT[7] x 1.01", errs)
    flagged = [(l, k) for l, e in enumerate(errs) for k, bound in BWD.items() if e[k] > bound]
    assert flagged == [(7, "dh2")], flagged
