"""The DiT's Gaussian heads at gaussians_sh_degree 1..3 on the device, forward and backward: the epilogue kernels
teacher-forced against oracle/dit.py's fp64 epilogue, the GEMM at the decoder head's shapes against torch,
the whole denoiser against the degree-aware fp32 oracle (outputs, renders, parameter gradients in both train modes),
a training step through the rasterizer's SH backward, and the FP8 inference path at degree 3.

Bounds: those of the degree-0 tests the same checks copy (tests/test_dit_gpu.py, test_dit_bwd_gpu.py,
test_dit_ends_gpu.py, test_fp8_gpu.py) unless a comment says otherwise; each run prints what it measured."""
import gc
import math

import pytest
import torch

from dgs_b200 import _lib
from dit_regime import dit_inputs, oracle_like
from oracle.dit import gaussians_epilogue64, head_channels
from util import rel_l2 as rel

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
OUTS = ("xyz", "features", "scaling", "rotation", "opacity")
# raw channel std of the epilogue inputs, as test_dit_ends_gpu's end-stage regime: the depth sigmoid saturates for part
# of the pixels and about a quarter of the scaling channels hit the clamp
XYZ_STD, SCALING_STD = 4.8, 1.6


def _raw(n_rows, C_, g):
    std = torch.ones(C_, device=DEV)
    std[:3], std[C_ - 8:C_ - 5] = XYZ_STD, SCALING_STD
    return torch.randn(n_rows, C_, device=DEV, generator=g) * std


# (B, G, V, H, W): 1 x (3 + 256) = 259 and 3 x (1 + 768) = 2307 Gaussians, so the last CTA of 256 threads holds an odd
# number of rows (3); with an odd G the image rows start at both parities of the odd-C row pitch
EPI_SHAPES = [(1, 3, 1, 16, 16), (3, 1, 2, 16, 24), (2, 2, 3, 8, 16)]


@pytest.mark.parametrize("degree", [1, 2, 3])
def test_epilogue_teacher_forced(degree):
    L = _lib.lib()
    C_, M = head_channels(degree), (degree + 1) ** 2
    p = 8
    for si, (B, G, V, H, W) in enumerate(EPI_SHAPES):
        for mode in (0, 1, 2):
            g = torch.Generator(DEV).manual_seed(100 * degree + 10 * si + mode)
            T = V * (H // p) * (W // p)
            P = G + V * H * W
            gs = _raw(B * G, C_, g).reshape(B, G, C_)
            ig = _raw(B * T * p * p, C_, g).reshape(B, T, p * p * C_)
            ro = (torch.randn(B, V, 3, 1, 1, device=DEV, generator=g) * 1.5).expand(B, V, 3, H, W).contiguous()
            rd = torch.nn.functional.normalize(torch.randn(B, V, 3, H, W, device=DEV, generator=g), dim=2)
            near, far = 0.5, 6.0
            out = {k: torch.full((B, P) + s, float("nan"), device=DEV)
                   for k, s in dict(xyz=(3,), features=(M, 3), scaling=(3,), rotation=(4,), opacity=(1,)).items()}
            ia = torch.full((B, V, 3, H, W), float("nan"), device=DEV)
            _lib.check(L.dgs_gaussians_epilogue(gs.data_ptr(), ig.data_ptr(), ro.data_ptr(), rd.data_ptr(),
                                                *(out[k].data_ptr() for k in OUTS), ia.data_ptr(), B, G, V, H, W, p,
                                                degree, mode, near, far, _lib.stream(None)))
            gs64, ig64 = gs.double().requires_grad_(), ig.double().requires_grad_()
            ref = gaussians_epilogue64(gs64, ig64, ro, rd, mode, near, far)
            raw = torch.cat([gs, ig.reshape(B, -1, C_)], dim=1)
            # the features are copies of raw channels 3 + 3k + c: bit-exact
            assert torch.equal(out["features"], raw[..., 3:C_ - 8].reshape(B, P, M, 3)), (degree, si, mode)
            errs = {k: rel(out[k], ref[k]) for k in OUTS}
            errs["img_aligned_xyz"] = rel(ia, ref["img_aligned_xyz"])
            # the scaling clamp and the saturated depth sigmoid are reached
            clamp = float((raw[..., C_ - 8:C_ - 5] - 2.3 > -1.2).double().mean())
            sat = float((ref["depth_m"].abs() > 4).double().mean())
            print(f"[epilogue d={degree} {(B, G, V, H, W)} mode={mode}] " +
                  "  ".join(f"{k}={v:.1e}" for k, v in errs.items()) + f"  clamp {clamp:.2f} saturated {sat:.2f}")
            assert all(v < 2e-7 for v in errs.values()), errs  # test_dit_ends_gpu FWD["epilogue"]
            assert 0.1 < clamp < 0.4 and sat > 0.03
            # backward: fp64 autograd through the reference epilogue with seeded output gradients
            cot = {k: torch.randn(out[k].shape, device=DEV, generator=g) for k in OUTS}
            d_gs = torch.full((B * G, C_), float("nan"), device=DEV)
            d_img = torch.full((B * T, p * p * C_), float("nan"), device=DEV).to(torch.bfloat16)
            _lib.check(L.dgs_gaussians_epilogue_bwd(gs.data_ptr(), ig.data_ptr(), rd.data_ptr(),
                                                    *(cot[k].data_ptr() for k in OUTS), d_gs.data_ptr(),
                                                    d_img.data_ptr(), B, G, V, H, W, p, degree, mode, near, far,
                                                    _lib.stream(None)))
            r_gs, r_img = torch.autograd.grad(sum((ref[k] * cot[k].double()).sum() for k in OUTS), [gs64, ig64])
            # free tokens: every channel's gradient is a copy (or a masked copy) of an output gradient
            assert torch.equal(d_gs.double(), r_gs.reshape(B * G, C_)), (degree, si, mode)
            r_img = r_img.reshape(-1, C_)
            d_img = d_img.reshape(-1, C_)
            # image tokens, channels 3..C-1: copies, so the bf16 gradient is the exact rounding of the fp64 one
            assert torch.equal(d_img[:, 3:], r_img[:, 3:].to(torch.bfloat16)), (degree, si, mode)
            # xyz channels: the fp32 depth chain rule, then one bf16 rounding; only the roundings whose fp32 input
            # straddles a bf16 rounding boundary may differ from those of the fp64 gradient
            e_xyz = rel(d_img[:, :3], r_img[:, :3].to(torch.bfloat16))
            print(f"    backward: d_img_gs xyz channels vs bf16(fp64) {e_xyz:.1e}")
            assert e_xyz < 1e-3, (degree, si, mode, e_xyz)


def _gemm_operands(M, N, K, seed):
    g = torch.Generator(DEV).manual_seed(seed)
    A = torch.randn(M, K, device=DEV, generator=g).to(torch.bfloat16)
    Wt = (torch.randn(N, K, device=DEV, generator=g) * 0.03).to(torch.bfloat16)
    return A, Wt


@pytest.mark.parametrize("Ndec", [1472, 2432, 3776])
def test_gemm_at_decoder_head_shapes(Ndec):
    """The decoder head's three GEMMs at obj-256 (Mt = 4096 image tokens, K = 3 * 1024 split-bf16): the forward
    Mt x Ndec x 3w with the fp32 epilogue (Ndec = 64 C: a 64-column N tail for odd C), the dgrad Mt x w x Ndec (bf16
    out) and the weight gradient Ndec x w over the Mt tokens (TN, the hi third of the [hi|lo|hi] operand)."""
    L = _lib.lib()
    Mt, D = 4096, 1024
    A, Wd = _gemm_operands(Mt, Ndec, 3 * D, Ndec)
    out = torch.full((Mt, Ndec), float("nan"), device=DEV)
    _lib.check(L.dgs_gemm_bf16(A.data_ptr(), Wd.data_ptr(), None, None, out.data_ptr(), Mt, Ndec, 3 * D, 3, Ndec, 0, 0,
                               _lib.stream(None)))
    e_fwd = rel(out, A.float() @ Wd.float().t())
    dimg, WdT = _gemm_operands(Mt, D, Ndec, Ndec + 1)
    dh = torch.empty(Mt, D, dtype=torch.bfloat16, device=DEV)
    _lib.check(L.dgs_gemm_bf16(dimg.data_ptr(), WdT.data_ptr(), None, None, dh.data_ptr(), Mt, D, Ndec, 0, D, 0, 0,
                               _lib.stream(None)))
    ref_dh = dimg.float() @ WdT.float().t()
    e_dgrad = rel(dh.float(), ref_dh.to(torch.bfloat16).float())
    d_img = torch.randn(Mt, Ndec, device=DEV, generator=torch.Generator(DEV).manual_seed(Ndec + 2)).to(torch.bfloat16)
    dw = torch.full((Ndec, D), float("nan"), device=DEV)
    _lib.check(L.dgs_gemm_bf16_tn(d_img.data_ptr(), A.data_ptr(), dw.data_ptr(), Ndec, D, Mt, Ndec, 3 * D, D,
                                  _lib.stream(None)))
    torch.cuda.synchronize()
    e_wgrad = rel(dw, d_img.float().t() @ A[:, :D].float())
    print(f"decoder GEMMs Ndec={Ndec}: fwd {e_fwd:.2e}  dgrad (vs bf16 of fp32) {e_dgrad:.2e}  wgrad {e_wgrad:.2e}")
    assert e_fwd < 1e-5 and e_wgrad < 4e-5  # fp32 accumulation order (test_gemm_tn_mn_major_operands: 4e-5)
    # only the bf16 roundings whose fp32 inputs straddle a rounding boundary differ, more of them as K grows: measured
    # 9.0e-5 / 1.1e-4 / 1.5e-4 at K = 1472 / 2432 / 3776 (H100 80GB HBM3, 700 W)
    assert e_dgrad < 3e-4


def _pair(degree, scene=False, layers=2, seed=0):
    from dgs_b200.denoiser import DGSDenoiser, DGSDenoiserScene
    gc.collect()
    torch.cuda.empty_cache()
    torch.manual_seed(seed)
    cfg = dict(patch_size=8, num_layers=layers, ray_pe_type="plk" if scene else "relative_plk",
               gaussians_sh_degree=degree)
    model = (DGSDenoiserScene if scene else DGSDenoiser)(cfg).to(DEV)
    return model, oracle_like(model)


def _compare(model, oracle, shape, tag, seed=0):
    images, ray_o, ray_d, t = dit_inputs(*shape, seed=seed)
    with torch.no_grad():
        ref, ref_ia = oracle.image_to_gaussians(images, ray_o, ray_d, t)
        out, ia = model.image_to_gaussians(images, ray_o, ray_d, t)
    torch.cuda.synchronize()
    assert out.features.shape == ref["features"].shape == (shape[0], 2 + shape[1] * shape[2] * shape[3],
                                                           (model.cfg.gaussians_sh_degree + 1) ** 2, 3)
    errs = {k: rel(out[k], ref[k]) for k in OUTS}
    errs["img_aligned_xyz"] = rel(ia, ref_ia)
    print(f"[{tag}] " + "  ".join(f"{k}={v:.2e}" for k, v in errs.items()))
    return errs, out, ref


@pytest.mark.parametrize("scene", [False, True], ids=["obj", "scene"])
@pytest.mark.parametrize("degree", [1, 3])
def test_denoiser_small_vs_oracle(degree, scene):
    model, oracle = _pair(degree, scene)
    errs, _, _ = _compare(model, oracle, (2, 4, 64, 64), f"small d={degree} scene={scene}")
    assert all(v < 1e-3 for v in errs.values()), errs  # accuracy bound of the bf16 path (test_dit_gpu)


def _psnr(a, b):
    mse = float((a.double() - b.double()).pow(2).mean())
    return 10 * math.log10(float(b.double().abs().max()) ** 2 / max(mse, 1e-30))


def test_denoiser_full_depth_obj256_degree3_vs_oracle():
    """obj-256 at degree 3: 24 layers, 4 views 256x256, features [1, 262146, 16, 3]; outputs and the rendered views of
    both sets of Gaussians (the rasterizer evaluating degree-3 SH per view)."""
    from dgs_b200 import synth
    model, oracle = _pair(3, layers=24)
    errs, out, ref = _compare(model, oracle, (1, 4, 256, 256), "obj-256 x24 d=3")
    assert all(v < 1e-3 for v in errs.values()), errs
    c2w, fx = synth.orbit_cameras(4, 256, 256)
    c2w, fx = torch.tensor(c2w[None], device=DEV), torch.tensor(fx[None], device=DEV)
    with torch.no_grad():
        r_ref = model.gs_renderer(ref["xyz"], ref["features"], ref["scaling"], ref["rotation"], ref["opacity"], 256, 256,
                                  c2w, fx)
        r_out = model.render_gaussians(out, c2w, fx, 256, 256)
    e, psnr = rel(r_out, r_ref), _psnr(r_out, r_ref)
    print(f"[obj-256 x24 d=3] rendered views: rel={e:.2e}  PSNR {psnr:.1f} dB")
    assert e < 1e-3  # as test_denoiser_full_depth_obj256_vs_oracle at degree 0


def _grad_compare(degree, recompute, shape=(2, 4, 32, 32), scene=False, seed=0):
    from dgs_b200.train import DitTrainer
    model, oracle = _pair(degree, scene, seed=seed)
    trainer = DitTrainer(model)
    trainer.recompute = recompute
    model.train()
    images, ray_o, ray_d, t = dit_inputs(*shape)
    g = torch.Generator(DEV).manual_seed(11)
    out, _ = model.image_to_gaussians(images, ray_o, ray_d, t)
    wts = {k: torch.randn(out[k].shape, device=DEV, generator=g) for k in OUTS}
    trainer.zero_grad()
    sum((out[k] * wts[k]).sum() for k in wts).backward()
    ref, _ = oracle.image_to_gaussians(images, ray_o, ray_d, t)
    sum((ref[k] * wts[k]).sum() for k in wts).backward()
    torch.cuda.synchronize()
    ours = dict(model.named_parameters())
    errs, num, den = {}, 0.0, 0.0
    for name, p in oracle.named_parameters():
        errs[name] = rel(ours[name].grad, p.grad)
        num += float((ours[name].grad.double() - p.grad.double()).pow(2).sum())
        den += float(p.grad.double().pow(2).sum())
    return (num / den) ** 0.5, errs


@pytest.mark.parametrize("recompute", [False, True], ids=["store", "recompute"])
@pytest.mark.parametrize("degree", [1, 3])
def test_backward_vs_oracle_autograd(degree, recompute):
    total, errs = _grad_compare(degree, recompute)
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:4]
    print(f"[bwd d={degree} recompute={recompute}] whole-gradient rel={total:.2e}  worst: " +
          "  ".join(f"{k}={v:.2e}" for k, v in worst))
    for k in ("upsampler.linear.weight", "image_token_decoder.linear.weight"):
        assert k in errs
    # test_dit_backward_small_vs_oracle_autograd's bounds
    assert total < 1e-2, total
    assert max(errs.values()) < 3e-2, errs


def test_training_step_through_renderer_sh_backward():
    """image_to_gaussians -> Renderer.forward_mse -> loss.backward() -> DitTrainer.optimizer_step() at degree 3: the
    rasterizer's SH backward hands d_features [B, P, 16, 3] to dgs_dit_backward.  Three steps on ours and on the oracle
    (torch.optim.AdamW, the same rasterizer): the losses decrease and track each other."""
    from dgs_b200 import synth
    from dgs_b200.train import DitTrainer
    model, oracle = _pair(3)
    trainer = DitTrainer(model, lr=1e-4, clip=0.0)
    opt = torch.optim.AdamW(oracle.parameters(), lr=1e-4, betas=(0.9, 0.99), eps=1e-8, weight_decay=0.01)
    model.train()
    B, V, H, W = 2, 4, 32, 32
    images, ray_o, ray_d, t = dit_inputs(B, V, H, W)
    c2w, fx = synth.orbit_cameras(V, W, H)
    c2w = torch.tensor(c2w[None], device=DEV).expand(B, -1, -1, -1).contiguous()
    fx = torch.tensor(fx[None], device=DEV).expand(B, -1, -1).contiguous()
    target = torch.rand(B, V, 3, H, W, device=DEV, generator=torch.Generator(DEV).manual_seed(5))
    losses, ref_losses = [], []
    for step in range(3):
        out, _ = model.image_to_gaussians(images, ray_o, ray_d, t)
        _, l2 = model.gs_renderer.forward_mse(out.xyz, out.features, out.scaling, out.rotation, out.opacity, H, W, c2w,
                                              fx, target)
        loss = l2.mean()
        trainer.zero_grad()
        loss.backward()
        if step == 0:
            assert out.features.shape == (B, 2 + V * H * W, 16, 3)
            dec = model.image_token_decoder.linear.weight.grad.reshape(64, -1, model.cfg.width)
            # the decoder rows of the higher-order SH coefficients (channels 6 .. 50) receive gradient
            assert float(dec[:, 6:51].abs().sum()) > 0
        trainer.optimizer_step(allreduce=False)
        ref, _ = oracle.image_to_gaussians(images, ray_o, ray_d, t)
        _, ref_l2 = model.gs_renderer.forward_mse(ref["xyz"], ref["features"], ref["scaling"], ref["rotation"],
                                                  ref["opacity"], H, W, c2w, fx, target)
        ref_loss = ref_l2.mean()
        opt.zero_grad()
        ref_loss.backward()
        opt.step()
        losses.append(float(loss))
        ref_losses.append(float(ref_loss))
    print("train steps d=3: ours", losses, "oracle", ref_losses)
    assert losses[2] < losses[1] < losses[0]
    assert all(abs(a - b) <= 5e-3 * abs(b) for a, b in zip(losses, ref_losses))


def test_fp8_inference_at_degree3():
    """set_inference_precision("fp8") at degree 3 (the heads stay split-bf16): within the FP8 path's end-to-end bound
    against its emulation (test_fp8_gpu.test_end_to_end_fp8)."""
    from oracle.fp8 import emulate_fp8
    from test_fp8_gpu import E2E_SLACK
    model, oracle = _pair(3, layers=24)
    model.eval()
    inputs = dit_inputs(1, 4, 256, 256)
    with torch.no_grad():
        r_out, r_ia = oracle.image_to_gaussians(*inputs)
        e_out, e_ia = emulate_fp8(oracle).image_to_gaussians(*inputs)
        model.set_inference_precision("fp8")
        f_out, f_ia = model.image_to_gaussians(*inputs)
    e_em = max([rel(e_out[k], r_out[k]) for k in OUTS] + [rel(e_ia, r_ia)])
    e_f8 = max([rel(f_out[k], r_out[k]) for k in OUTS] + [rel(f_ia, r_ia)])
    print(f"fp8 d=3 obj-256 x24: fp8 {e_f8:.2e}  emulated-fp8 {e_em:.2e}  gate {1.5 * e_em + E2E_SLACK:.2e}")
    assert f_out.features.shape == (1, 2 + 4 * 256 * 256, 16, 3)
    assert e_f8 <= 1.5 * e_em + E2E_SLACK
