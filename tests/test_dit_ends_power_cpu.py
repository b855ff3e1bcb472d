"""CPU checks of the DiT end-stage tests' own machinery (no GPU):

* the fp64 end-stage reference (oracle.dit.input_stage64 -> the oracle blocks -> heads64) composes to exactly the
  oracle's image_to_gaussians, for the object and the scene model and both Pluecker modes;
* the end-stage regime (tests/test_dit_ends_gpu.apply_end_scale) reaches the `scaling` clamp and the saturated depth
  sigmoid as often as it promises;
* power: with the rounding-matched reference standing in for the kernels, each planted defect moves the quantity
  tests/test_dit_ends_gpu.py checks by at least twice the bound it applies on the H100.
"""
import pytest
import torch

from test_dit_ends_gpu import BWD, CLAMP_FRAC, FWD, OUTS, SATURATED_FRAC, apply_end_scale
from util import rel_l2 as _rel

D = 1024


def _oracle(scene=False, pe="relative_plk", seed=0):
    from oracle.dit import DenoiserOracle
    torch.manual_seed(seed)
    return apply_end_scale(DenoiserOracle(layers=2, scene=scene, ray_pe_type=pe), seed).double()


@pytest.fixture(scope="module")
def obj2():
    return _oracle()


def _inputs(B=2, V=2, H=32, W=48, seed=0):
    g = torch.Generator().manual_seed(seed)
    images = torch.rand(B, V, 3, H, W, generator=g, dtype=torch.float64)
    ray_o = torch.randn(B, V, 3, 1, 1, generator=g, dtype=torch.float64).expand(B, V, 3, H, W).contiguous() * 1.5
    ray_d = torch.nn.functional.normalize(torch.randn(B, V, 3, H, W, generator=g, dtype=torch.float64), dim=2)
    return images, ray_o, ray_d, torch.tensor([100, 999][:B])


def _compose(o, images, ray_o, ray_d, t, depth_mode, **kw):
    """input_stage64 -> the oracle's own blocks -> heads64, conditioned on the oracle's own t_embedder."""
    from oracle.dit import heads64, input_stage64, mod_table64
    c = o.t_embedder(t)
    mod = mod_table64(o, c)
    x = input_stage64(o, images, ray_o, ray_d, o.ray_pe_type, **kw)["x0"]
    for blk in o.transformer:
        x = blk(x, c)
    return heads64(o, x, mod[:, len(o.transformer) * 6 * D:], ray_o, ray_d, depth_mode, o.near, o.far, **kw), mod, c


@pytest.mark.parametrize("scene,pe", [(False, "relative_plk"), (False, "plk"), (True, "relative_plk"), (True, "plk")])
def test_end_stage_reference_composes_to_the_oracle(scene, pe):
    from oracle.dit import cond64
    o = _oracle(scene, pe)
    images, ray_o, ray_d, t = _inputs()
    depth_mode = 1 if scene else (0 if pe == "relative_plk" else 2)
    with torch.no_grad():
        ref, ref_ia = o.image_to_gaussians(images, ray_o, ray_d, t)
        got, mod, c = _compose(o, images, ray_o, ray_d, t, depth_mode)
        for k in OUTS:
            assert _rel(got[k], ref[k]) < 1e-12, k
        assert _rel(got["img_aligned_xyz"], ref_ia) < 1e-12
        for l, blk in enumerate(o.transformer):
            assert _rel(mod[:, l * 6 * D:(l + 1) * 6 * D], blk.adaLN_modulation(c)) < 1e-12
        # the oracle forms t * freq in fp32 and takes cos / sin in fp32: cond64(fp32_args) differs from it by the fp32
        # rounding of cos / sin only; the fp64 argument differs at t = 999 by ~1e-5
        e32, e64 = _rel(cond64(o, t, fp32_args=True), c), _rel(cond64(o, t), c)
        print(f"cond64 vs the oracle's t_embedder: fp32 args {e32:.1e}, fp64 args {e64:.1e}")
        assert e32 < 1e-6 < e64
        # matched differs from plain by the split-bf16 rounding only
        m, _, _ = _compose(o, images, ray_o, ray_d, t, depth_mode, matched=True)
        e = _rel(m["img_gs"], got["img_gs"])
        assert 1e-8 < e < 1e-4, e


def test_end_stage_regime_statistics(obj2):
    images, ray_o, ray_d, t = _inputs(V=4)
    with torch.no_grad():
        out, _, _ = _compose(obj2, images, ray_o, ray_d, t, 0)
    raw = torch.cat([out["gs_tok"], out["img_gs"].reshape(2, -1, 14)], dim=1)
    clamp = float((raw[..., 6:9] - 2.3 > -1.2).double().mean())
    sat = float((out["depth_m"].abs() > 4).double().mean())
    rms = {k: float(raw[..., a:b].pow(2).mean().sqrt()) for k, (a, b) in
           dict(features=(3, 6), rotation=(9, 13), opacity=(13, 14)).items()}
    print(f"clamped {clamp:.3f}  saturated {sat:.3f}  rms " + "  ".join(f"{k}={v:.2f}" for k, v in rms.items()))
    assert 0.2 < clamp < 0.3 and CLAMP_FRAC[0] < clamp < CLAMP_FRAC[1]
    assert 0.05 < sat < 0.3 and SATURATED_FRAC[0] < sat < SATURATED_FRAC[1]
    assert all(0.5 < v < 2.0 for v in rms.values()), rms
    tok = obj2.image_tokenizer[1].weight.detach()
    assert 0.9 < float(tok.std() * tok.shape[1] ** 0.5) < 1.1
    assert 0.9 < float(obj2.gaussians_pos_embedding.detach().std()) < 1.1


def _head_grads(o, x, mod_h, ray_o, ray_d, wts, depth_mode, defects=()):
    from oracle.dit import heads64
    o.zero_grad(set_to_none=True)
    with torch.enable_grad():
        hd = heads64(o, x, mod_h, ray_o, ray_d, depth_mode, matched=True, defects=defects)
        sum((hd[k] * wts[k]).sum() for k in OUTS).backward()
    return {n: p.grad.clone() for n, p in o.named_parameters()
            if n.startswith(("upsampler.", "image_token_decoder.")) and "adaLN" not in n}


def _input_grads(o, images, ray_o, ray_d, dx0, defects=()):
    from oracle.dit import input_stage64
    o.zero_grad(set_to_none=True)
    with torch.enable_grad():
        input_stage64(o, images, ray_o, ray_d, "relative_plk", matched=True, defects=defects)["x0"].backward(dx0)
    return {n: o.get_parameter(n).grad.clone() for n in
            ("transformer_input_layernorm.weight", "gaussians_pos_embedding", "image_tokenizer.1.weight")}


def _worst(a, b):
    return max(_rel(a[k], b[k]) for k in b)


def test_planted_end_defects_exceed_the_gpu_bound(obj2):
    from oracle.dit import cond64, gaussians_epilogue64, heads64, input_stage64, mod_table64
    o = obj2
    L = len(o.transformer)
    images, ray_o, ray_d, t = _inputs()
    B = images.shape[0]
    power = {}  # defect -> (measured change of the checked quantity, the GPU bound on it)
    with torch.no_grad():
        ins = lambda pe, **kw: input_stage64(o, images, ray_o, ray_d, pe, matched=True, **kw)  # noqa: E731
        clean = ins("relative_plk")
        power["tokenizer lo dropped"] = (_rel(ins("relative_plk", defects=("lo_dropped_tokenizer",))["x_pre"],
                                              clean["x_pre"]), FWD["x_pre"])
        power["o x d computed as d x o"] = (_rel(ins("plk", defects=("cross_swapped",))["x_pre"], ins("plk")["x_pre"]),
                                            FWD["x_pre"])
        power["input LayerNorm eps 1e-6"] = (_rel(ins("relative_plk", eps=1e-6)["x0"], clean["x0"]), FWD["x0"])
        c = cond64(o, t, fp32_args=True)
        power["cos and sin swapped"] = (_rel(cond64(o, t, fp32_args=True, defects=("cos_sin_swapped",)), c), FWD["c"])
        mod = mod_table64(o, c)
        u0, d0 = L * 6 * D, L * 6 * D + 2 * D
        swapped = torch.cat([mod[:, :u0], mod[:, d0:], mod[:, u0:d0]], dim=1)
        power["head adaLN rows swapped"] = (min(_rel(swapped[:, a:a + 2 * D], mod[:, a:a + 2 * D]) for a in (u0, d0)),
                                            FWD["mod"])
        # the heads on a final stream of the trained-scale size (rms ~2.4 after 24 blocks)
        g = torch.Generator().manual_seed(5)
        N = o.G + images.shape[1] * (images.shape[3] // 8) * (images.shape[4] // 8)
        x = torch.randn(B, N, D, generator=g, dtype=torch.float64) * 2.4
        mod_h = mod[:, u0:]
        hd = heads64(o, x, mod_h, ray_o, ray_d, 0, matched=True)
        for stage, k in (("upsampler", "gs_tok"), ("decoder", "img_gs")):
            bad = heads64(o, x, mod_h, ray_o, ray_d, 0, matched=True, defects=(f"lo_dropped_{stage}",))
            power[f"{stage} lo dropped"] = (_rel(bad[k], hd[k]), FWD[k])
        swap = gaussians_epilogue64(hd["gs_tok"], hd["img_gs"], ray_o, ray_d, 2)
        power["depth modes 0 and 2 swapped"] = (max(_rel(swap[k], hd[k]) for k in OUTS + ("img_aligned_xyz",)),
                                                FWD["epilogue"])
    wts = {k: torch.randn(hd[k].shape, generator=g, dtype=torch.float64) for k in OUTS}
    clean_g = _head_grads(o, x, mod_h, ray_o, ray_d, wts, 0)
    for name, defect in (("clamp gradient passed everywhere", "clamp_grad_everywhere"),
                         ("1/3 dropped in the depth gradient", "depth_third_dropped")):
        power[name] = (_worst(_head_grads(o, x, mod_h, ray_o, ray_d, wts, 0, (defect,)), clean_g), BWD["decoder"])
    dx0 = torch.randn(clean["x0"].shape, generator=g, dtype=torch.float64)
    clean_in = _input_grads(o, images, ray_o, ray_d, dx0)
    power["pos_embed gradient from sample 0 only"] = (_worst(_input_grads(o, images, ray_o, ray_d, dx0,
                                                                          ("pos_grad_sample0",)), clean_in), BWD["input"])
    for k, (v, bound) in power.items():
        print(f"{k:40s} {v:.2e}  ({v / bound:.1f} x the bound {bound:.1e})")
    for k, (v, bound) in power.items():
        assert v >= 2 * bound, (k, v, bound)
