"""Teacher-forced tests of the DiT stages on either side of the blocks, forward and backward, against oracle/dit.py's
fp64 end-stage reference (input_stage64, cond64 / mod_table64, heads64, gaussians_epilogue64) on the device:

* the input stage (posed-image patchify in both Pluecker modes, the split-bf16 tokenizer GEMM, token assembly, the input
  LayerNorm), the conditioning (timestep embedding, timestep MLP, the adaLN table of every block and both heads) and
  the heads (LayerNorm + modulate, the split-bf16 upsampler and decoder products, the Gaussian epilogue);
* the backward of all of these, fed the product's own gradient at the stage boundary (dgs_dit_export_ends).

Each stage gets the product's own tensor at its input and only that stage is compared, so the bounds are those of the
stage (fp32-accurate by design) rather than of the 24 bf16 blocks around it.  The weights are in an end-stage regime
(apply_end_scale below) where the `scaling` clamp and the saturated depth sigmoid are actually reached.

Every bound below was set from the errors measured on an H100 80GB HBM3 over seeds 0, 1, 2 at every shape here; the
measured worst case is written next to it.  Errors are norm-wise relative unless noted.
"""
import gc
import math

import pytest
import torch

from dit_regime import dit_inputs
from util import rel_l2 as _rel

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# ---- end-stage regime ----
# target std of the raw head output per channel (xyz | features | scaling | rotation | opacity): the xyz channels so
# that the depth sigmoid's argument m (their mean) has |m| > 4 for ~15 % of the pixels, the scaling channels so that
# ~25 % of the raw values a clamp (a - 2.3 > -1.2), the rest O(1)
HEAD_CHANNEL_STD = (4.8,) * 3 + (1.0,) * 3 + (1.6,) * 3 + (1.0,) * 4 + (1.0,)
HEAD_INPUT_RMS = 1.1  # rms of LayerNorm * weight * (1 + scale) + shift in the trained-scale regime


def apply_end_scale(model, seed=0):
    """tests/dit_regime.apply_trained_scale, then the end stages at trained scale too: tokenizer at unit gain,
    Gaussian position embedding of std 1, and head linear rows scaled per output channel (HEAD_CHANNEL_STD)."""
    from dit_regime import apply_trained_scale
    apply_trained_scale(model, seed)
    g = torch.Generator().manual_seed(2000 + seed)
    fill = lambda p, std: p.copy_((torch.randn(p.shape, generator=g, dtype=torch.float64) * std).to(p.dtype))  # noqa: E731
    with torch.no_grad():
        tw = model.image_tokenizer[1].weight
        fill(tw, 1.0 / math.sqrt(tw.shape[1]))
        fill(model.gaussians_pos_embedding, 1.0)
        for head in (model.upsampler, model.image_token_decoder):
            w = head.linear.weight
            std = torch.tensor(HEAD_CHANNEL_STD, dtype=torch.float64).repeat(w.shape[0] // 14)
            fill(w, 1.0)
            w.mul_((std / (math.sqrt(w.shape[1]) * HEAD_INPUT_RMS)).to(w.dtype)[:, None])
    return model


# kind -> (scene model, ray_pe_type, depth mode of gaussians_epilogue)
KINDS = {"obj-rel": (False, "relative_plk", 0), "obj-plk": (False, "plk", 2),
         "scene-rel": (True, "relative_plk", 1), "scene-plk": (True, "plk", 1)}
OUTS = ("xyz", "features", "scaling", "rotation", "opacity")

# ---- bounds, against the rounding-matched reference; measured worst (H100, seeds 0-2, every shape) in the comment ----
# The split-bf16 products are left with the fp32 accumulation of the tensor cores over K = 3 * 576 (tokenizer) and
# K = 3 * 1024 (decoder), ~3e-6 and ~5e-6: the reference reproduces the split itself, not the order of the sums.
FWD = dict(x_pre=6e-6,     # tokenizer GEMM (split-bf16) + assembly: 2.92e-6
           x0=2e-7,        # input LayerNorm of the product's x_pre: 6.6e-8
           c=4e-7,         # timestep embedding + MLP: 1.65e-7
           mod=3e-7,       # every 6w block segment and the two 2w head segments of the adaLN table: 1.00e-7
           gs_tok=3e-6,    # upsampler (split-bf16 tiny_linear): 1.16e-6
           img_gs=1e-5,    # decoder GEMM (split-bf16): 5.27e-6
           epilogue=2e-7)  # the five outputs and img_aligned_xyz, on the product's raw head outputs: 6.3e-8
# against the plain fp64 reference, what "fp32-accurate" promises: x_pre 5.25e-6, c 8.06e-6 (the fp32 t * freq),
# gs_tok 6.67e-6, img_gs 6.93e-6
PLAIN = dict(x_pre=1.5e-5, c=2e-5, gs_tok=1.5e-5, img_gs=1.5e-5)
BWD = dict(upsampler=3e-6,     # upsampler linear + LayerNorm weights, d_gs_tok: 1.02e-6
           # decoder linear + LayerNorm weights and the head rows of dmod: the decoder's dh is rounded to bf16 from a
           # K = 896 product whose fp32 noise puts ~0.1 % of the roundings on the other side: 1.25e-4
           decoder=4e-4,
           cond=2e-6,          # every adaLN weight / bias, t_embedder.*, dc (fed the product's dmod): 6.3e-7
           input=6e-6,         # input LayerNorm weight, pos embedding, dx_pre (fed the product's dx0): 2.8e-6
           tokenizer=4e-4,     # tokenizer weight fed the product's dx0 (likewise, bf16 rounding of d tok): 1.46e-4
           # tokenizer weight fed the product's bf16(d tok): 1.53e-5, from hi(patches) -- the fp32 o x d of the 'plk'
           # mode cancels, and a few of its bf16 roundings differ from those of the fp64 patches (<= 2.4e-7 otherwise)
           tokenizer_fed=4e-5)
# the regime must reach the clamp and the saturated sigmoid at every shape
CLAMP_FRAC = (0.1, 0.4)
SATURATED_FRAC = (0.03, 0.35)


def build(kind, layers, seed=0):
    """-> (product DGSDenoiser with a DitTrainer, fp64 DenoiserOracle on the device with the same weights)."""
    from dgs_b200.denoiser import DGSDenoiser, DGSDenoiserScene
    from dgs_b200.train import DitTrainer
    from oracle.dit import DenoiserOracle
    gc.collect()
    torch.cuda.empty_cache()
    scene, pe, _ = KINDS[kind]
    torch.manual_seed(seed)
    cfg = dict(patch_size=8, num_layers=layers, ray_pe_type=pe)
    model = apply_end_scale((DGSDenoiserScene if scene else DGSDenoiser)(cfg), seed)
    ref = DenoiserOracle(layers=layers, scene=scene, ray_pe_type=pe)
    ref.load_state_dict(model.state_dict(), strict=True)
    model, ref = model.to(DEV), ref.to(DEV).double()
    trainer = DitTrainer(model)
    model.train()
    return model, trainer, ref


def _depth_args(model, kind):
    c = model.cfg
    return KINDS[kind][2], float(c.range_setting_near), float(c.range_setting_far)


def forward_errors(model, trainer, ref, kind, shape, seed=0, recompute=False):
    """One training forward, then every forward stage against the reference fed the product's tensor at its input.
    -> ({check: matched error}, {check: plain error}, {"mod_segments": [...], "clamp": frac, "saturated": frac})."""
    from oracle.dit import cond64, gaussians_epilogue64, heads64, input_stage64, mod_table64, _layernorm64
    B, V, H, W = shape
    images, ray_o, ray_d, t = inputs = dit_inputs(B, V, H, W, seed=seed)
    trainer.recompute = recompute
    with torch.enable_grad():
        out, img_xyz = model.image_to_gaussians(*inputs)
    trainer.reset()
    L, D = len(ref.transformer), ref.width
    ex = trainer.export_ends(B, V, H, W, ("x_pre", "c", "mod", "gs_tok", "img_gs"))
    x0 = trainer.export_state(B, V, H, W, 0)["x"]
    xL = trainer.export_state(B, V, H, W, L)["x"]
    mode, near, far = _depth_args(model, kind)
    pe = KINDS[kind][1]
    e, p, info = {}, {}, {}
    with torch.no_grad():
        e["x_pre"] = _rel(ex["x_pre"], input_stage64(ref, images, ray_o, ray_d, pe, matched=True)["x_pre"])
        p["x_pre"] = _rel(ex["x_pre"], input_stage64(ref, images, ray_o, ray_d, pe)["x_pre"])
        e["x0"] = _rel(x0, _layernorm64(ex["x_pre"].double(), ref.transformer_input_layernorm.weight, 1e-5))
        e["c"] = _rel(ex["c"], cond64(ref, t, fp32_args=True))
        p["c"] = _rel(ex["c"], cond64(ref, t))
        mod = mod_table64(ref, ex["c"])
        bounds = [(l * 6 * D, (l + 1) * 6 * D) for l in range(L)] + [(L * 6 * D, L * 6 * D + 2 * D),
                                                                     (L * 6 * D + 2 * D, L * 6 * D + 4 * D)]
        info["mod_segments"] = [_rel(ex["mod"][:, a:b], mod[:, a:b]) for a, b in bounds]
        e["mod"] = max(info["mod_segments"])
        hd = heads64(ref, xL, mod[:, L * 6 * D:], ray_o, ray_d, mode, near, far, matched=True)
        hp = heads64(ref, xL, mod[:, L * 6 * D:], ray_o, ray_d, mode, near, far)
        for k in ("gs_tok", "img_gs"):
            e[k] = _rel(ex[k], hd[k])
            p[k] = _rel(ex[k], hp[k])
        epi = gaussians_epilogue64(ex["gs_tok"], ex["img_gs"], ray_o, ray_d, mode, near, far)
        got = dict(out, img_aligned_xyz=img_xyz)
        info["epilogue"] = {k: _rel(got[k], epi[k]) for k in OUTS + ("img_aligned_xyz",)}
        e["epilogue"] = max(info["epilogue"].values())
        raw = torch.cat([ex["gs_tok"], ex["img_gs"].reshape(B, -1, 14)], dim=1)[..., 6:9]
        info["clamp"] = float((raw - 2.3 > -1.2).double().mean())
        info["saturated"] = float((epi["depth_m"].abs() > 4).double().mean())
    return e, p, info


def _cotangents(out, seed):
    g = torch.Generator(DEV).manual_seed(100 + seed)
    return {k: torch.randn(out[k].shape, device=DEV, generator=g) for k in OUTS}


def backward_errors(model, trainer, ref, kind, shape, seed=0, recompute=False):
    """One training forward + backward with a seeded cotangent on the five outputs, then each backward stage against
    fp64 autograd through the reference fed the product's tensors at the stage boundary.  -> {check: {tensor: error}}."""
    from oracle.dit import _bf16, cond64, heads64, input_stage64, mod_table64
    B, V, H, W = shape
    images, ray_o, ray_d, t = inputs = dit_inputs(B, V, H, W, seed=seed)
    trainer.recompute = recompute
    with torch.enable_grad():
        out, _ = model.image_to_gaussians(*inputs)
        wts = _cotangents(out, seed)
        trainer.zero_grad()
        sum((out[k] * wts[k]).sum() for k in OUTS).backward()
    L, D = len(ref.transformer), ref.width
    ex = trainer.export_ends(B, V, H, W, trainer.ENDS_FIELDS)
    xL = trainer.export_state(B, V, H, W, L)["x"]
    ours = dict(model.named_parameters())
    refp = dict(ref.named_parameters())
    mode, near, far = _depth_args(model, kind)
    pe = KINDS[kind][1]
    errs = {}
    with torch.enable_grad():
        # heads: fp64 autograd through heads64 on the product's final stream and head modulation
        ref.zero_grad(set_to_none=True)
        mod_h = ex["mod"][:, L * 6 * D:].double().requires_grad_()
        hd = heads64(ref, xL, mod_h, ray_o, ray_d, mode, near, far, matched=True,
                     feed={k: ex[k] for k in ("gs_tok", "img_gs")})
        hd["gs_tok"].retain_grad()
        sum((hd[k] * wts[k].double()).sum() for k in OUTS).backward()
        for fam in ("upsampler", "image_token_decoder"):
            names = [n for n in refp if n.startswith(fam + ".") and "adaLN" not in n]
            errs[fam.split("_")[-1]] = {n: _rel(ours[n].grad, refp[n].grad) for n in names}
        errs["decoder"]["dmod[heads]"] = _rel(ex["dmod"][:, L * 6 * D:], mod_h.grad)
        errs["upsampler"]["d_gs_tok"] = _rel(ex["d_gs_tok"], hd["gs_tok"].grad)
        # conditioning: fp64 autograd through mod_table64(cond64(t)) fed the product's dmod
        ref.zero_grad(set_to_none=True)
        c = cond64(ref, t, fp32_args=True)
        c.retain_grad()
        mod_table64(ref, c).backward(ex["dmod"].double())
        names = [n for n in refp if "adaLN_modulation" in n or n.startswith("t_embedder.")]
        e = {n: _rel(ours[n].grad, refp[n].grad) for n in names}
        e["dc"] = _rel(ex["dc"], c.grad)
        errs["cond"] = e
        # input stage: fp64 autograd through input_stage64 fed the product's dx0
        ref.zero_grad(set_to_none=True)
        st = input_stage64(ref, images, ray_o, ray_d, pe, matched=True)
        st["x_pre"].retain_grad()
        st["x0"].backward(ex["dx0"].double())
        names = ("transformer_input_layernorm.weight", "gaussians_pos_embedding")
        e = {n: _rel(ours[n].grad, refp[n].grad) for n in names}
        e["dx_pre"] = _rel(ex["dx_pre"], st["x_pre"].grad)
        errs["input"] = e
        # the tokenizer weight gradient rounds d tok to bf16: fed through the reference's own d tok (which differs by
        # the fp32 noise of the LayerNorm backward) ~0.1 % of the roundings land on the other side
        tw = "image_tokenizer.1.weight"
        errs["tokenizer"] = {tw: _rel(ours[tw].grad, refp[tw].grad)}
        # teacher-forced at the rounding: bf16(the product's d tok)^T hi(patches)
        G = ex["dx_pre"].shape[1] - st["patches"].shape[1]
        dtok = _bf16(ex["dx_pre"][:, G:].double()).reshape(-1, D)
        dw = dtok.t() @ _bf16(st["patches"].detach()).reshape(dtok.shape[0], -1)
        errs["tokenizer_fed"] = {tw: _rel(ours[tw].grad, dw)}
    ref.zero_grad(set_to_none=True)
    return errs


def _check_forward(tag, e, p, info):
    print(f"[{tag}] matched " + "  ".join(f"{k}={v:.2e}" for k, v in e.items()))
    print(f"[{tag}] plain   " + "  ".join(f"{k}={v:.2e}" for k, v in p.items()))
    print(f"[{tag}] epilogue " + "  ".join(f"{k}={v:.2e}" for k, v in info["epilogue"].items()) +
          f"; clamp {info['clamp']:.3f} saturated {info['saturated']:.3f}")
    segs = info["mod_segments"]
    for k, bound in FWD.items():
        if k == "mod":
            bad = [i for i, v in enumerate(segs) if v >= bound]
            n = len(segs) - 2
            assert not bad, (tag, [f"block {i}" if i < n else ("upsampler", "decoder")[i - n] for i in bad], segs)
        else:
            assert e[k] < bound, (tag, k, e)
    for k, bound in PLAIN.items():
        assert p[k] < bound, (tag, k, p)
    assert CLAMP_FRAC[0] < info["clamp"] < CLAMP_FRAC[1], (tag, info["clamp"])
    assert SATURATED_FRAC[0] < info["saturated"] < SATURATED_FRAC[1], (tag, info["saturated"])


def _check_backward(tag, errs):
    for fam, e in errs.items():
        worst = max(e, key=e.get)
        print(f"[{tag}] bwd {fam}: worst {worst} {e[worst]:.2e}  " + "  ".join(f"{k}={v:.1e}" for k, v in e.items()))
    for fam, e in errs.items():
        for k, v in e.items():
            assert v < BWD[fam], (tag, fam, k, v)


SHAPE_B2 = (2, 4, 32, 48)  # non-square; N = 2 + 4 * 4 * 6 = 98 tokens per sample (the backward needs >= 64)
SHAPE_V1 = (1, 1, 32, 48)  # one view: N = 26


@pytest.mark.parametrize("kind", list(KINDS))
def test_ends_two_layers(kind):
    model, trainer, ref = build(kind, 2)
    for shape, recompute in ((SHAPE_B2, False), (SHAPE_V1, True)):
        _check_forward(f"{kind} L=2 {shape}", *forward_errors(model, trainer, ref, kind, shape, recompute=recompute))
    for recompute in (False, True):
        tag = f"{kind} L=2 {SHAPE_B2} {'recompute' if recompute else 'store'}"
        _check_backward(tag, backward_errors(model, trainer, ref, kind, SHAPE_B2, recompute=recompute))


def test_ends_24_layers():
    """The full depth: mod_stride = 24*6w + 4w, so the head segments sit behind all 24 block segments."""
    model, trainer, ref = build("obj-rel", 24)
    _check_forward("obj-rel L=24", *forward_errors(model, trainer, ref, "obj-rel", SHAPE_B2, seed=1))
    _check_backward("obj-rel L=24 store", backward_errors(model, trainer, ref, "obj-rel", SHAPE_B2, seed=1))


def test_ends_batch_of_nine():
    """B = 9 > 8: the conditioning's skinny linears run as two launches (8 + 1 samples)."""
    model, trainer, ref = build("obj-rel", 2)
    _check_forward("obj-rel L=2 B=9", *forward_errors(model, trainer, ref, "obj-rel", (9, 1, 32, 32), seed=2))
    with pytest.raises(ValueError, match="unknown end-stage tensors"):
        trainer.export_ends(9, 1, 32, 32, ("x_pre", "hdec"))


@pytest.mark.parametrize("kind", ["obj-rel", "scene-plk"])
def test_inference_matches_recompute_bitwise(kind):
    """Inference and a recompute-mode training forward run the same kernels on the same inputs (the decoder's A
    operand lives in the workspace in one and in the train state in the other), so they agree to the bit."""
    model, trainer, ref = build(kind, 2)
    inputs = dit_inputs(*SHAPE_B2, seed=3)
    with torch.no_grad():
        a, a_img = model.image_to_gaussians(*inputs)
        a = {k: v.clone() for k, v in a.items()}
        a_img = a_img.clone()
    trainer.recompute = True
    with torch.enable_grad():
        b, b_img = model.image_to_gaussians(*inputs)
    trainer.reset()
    for k in OUTS:
        assert torch.equal(a[k], b[k].detach()), (kind, k, _rel(b[k], a[k]))
    assert torch.equal(a_img, b_img), (kind, _rel(b_img, a_img))

