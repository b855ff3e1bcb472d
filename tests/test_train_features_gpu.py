"""GPU tests of the round-2 training-side features: activation recompute, EMA inside AdamW, the MSE fused into the
blend kernels, gradient accumulation and the trainer's misuse guards (all through the C ABI)."""
import ctypes as C

import numpy as np
import pytest
import torch

from util import rel_l2 as rel

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _model_and_inputs(layers=2, B=2, V=4, H=32, W=32, scene=False, **trainer_kw):
    from dgs_b200.denoiser import DGSDenoiser, DGSDenoiserScene
    from dgs_b200.train import DitTrainer
    from dit_regime import dit_inputs
    torch.manual_seed(0)
    cfg = dict(patch_size=8, num_layers=layers, ray_pe_type="plk" if scene else "relative_plk")
    model = (DGSDenoiserScene if scene else DGSDenoiser)(cfg).to(DEV)
    # non-zero biases / adaLN so every gradient path is exercised (the reference initialises them to zero)
    with torch.no_grad():
        g = torch.Generator(DEV).manual_seed(5)
        for n, p in model.named_parameters():
            if n.endswith(".bias"):
                p.copy_(0.05 * torch.randn(p.shape, device=DEV, generator=g))
    trainer = DitTrainer(model, **trainer_kw)
    model.train()
    return model, trainer, dit_inputs(B, V, H, W)


def _backward_once(model, trainer, inputs, seed=11):
    images, ray_o, ray_d, t = inputs
    out, _ = model.image_to_gaussians(images, ray_o, ray_d, t)
    g = torch.Generator(DEV).manual_seed(seed)
    wts = {k: torch.randn(out[k].shape, device=DEV, generator=g) for k in ("xyz", "features", "scaling", "rotation", "opacity")}
    loss = sum((out[k] * wts[k]).sum() for k in wts)
    loss.backward()
    return {k: out[k].detach().clone() for k in wts}


@pytest.mark.parametrize("scene", [False, True])
def test_recompute_mode_equals_store_mode(scene):
    """The reference checkpoints every block (denoiser.py:348-354): same outputs, same gradients, a fraction of the memory."""
    m0, t0, inp = _model_and_inputs(layers=3, scene=scene)
    o0 = _backward_once(m0, t0, inp)
    g0 = t0.arena.flat.clone()
    s0 = t0._state.numel()
    m1, t1, _ = _model_and_inputs(layers=3, scene=scene, recompute=True)
    o1 = _backward_once(m1, t1, inp)
    torch.cuda.synchronize()
    # 3 layers: 4 residual snapshots + ONE layer's activations + the backward scratch vs 3 layers' activations; the ratio
    # falls with depth (24 layers at N = 4098: 0.6 vs 4.05 GB per sample, checked in test_recompute_state_bytes_full_model)
    assert t1._state.numel() < 0.7 * s0, (t1._state.numel(), s0)
    for k in o0:
        assert rel(o1[k], o0[k]) < 1e-6, k  # forward: in-place reduce-add epilogue vs separate residual source (<= 1 ulp)
    e = rel(t1.arena.flat, g0)
    print(f"recompute vs store (scene={scene}): whole-gradient rel={e:.2e}, state {t1._state.numel() / 2**20:.0f} vs {s0 / 2**20:.0f} MiB")
    assert e < 2e-3  # the recomputed activations differ from the stored ones by bf16 rounding of 1-ulp different fp32 inputs


def test_recompute_state_bytes_full_model():
    """Sizes only (no allocation): the obj-256 model at batch 1 -- what lets the yaml batch sizes fit."""
    from dgs_b200 import _lib
    from dgs_b200.denoiser import DGSDenoiser
    m = DGSDenoiser(dict(patch_size=8)).to(DEV)
    w, _ = m.packed_weights()
    L = _lib.lib()
    store = L.dgs_dit_train_state_bytes_ex(C.byref(w), 1, 4, 256, 256, _lib.TRAIN_STORE)
    rec = L.dgs_dit_train_state_bytes_ex(C.byref(w), 1, 4, 256, 256, _lib.TRAIN_RECOMPUTE)
    print(f"train state per sample at N=4098: store {store / 2**30:.2f} GiB, recompute {rec / 2**30:.2f} GiB")
    assert store > 3.5 * 2 ** 30 and rec < 0.9 * 2 ** 30
    assert L.dgs_dit_train_state_bytes_ex(C.byref(w), 1, 4, 256, 256, 7) == 0 and b"train_mode" in L.dgs_last_error()


def test_recompute_full_depth_vs_oracle():
    from oracle.dit import DenoiserOracle
    model, trainer, inp = _model_and_inputs(layers=6, B=1, V=4, H=64, W=64, recompute=True)
    oracle = DenoiserOracle(layers=6).to(DEV)
    oracle.load_state_dict(model.state_dict(), strict=True)
    images, ray_o, ray_d, t = inp
    out, _ = model.image_to_gaussians(images, ray_o, ray_d, t)
    g = torch.Generator(DEV).manual_seed(2)
    wts = {k: torch.randn(out[k].shape, device=DEV, generator=g) for k in ("xyz", "features", "scaling", "rotation", "opacity")}
    sum((out[k] * wts[k]).sum() for k in wts).backward()
    ref, _ = oracle.image_to_gaussians(images, ray_o, ray_d, t)
    sum((ref[k] * wts[k]).sum() for k in wts).backward()
    ours = dict(model.named_parameters())
    num = sum(float((ours[n].grad.double() - p.grad.double()).pow(2).sum()) for n, p in oracle.named_parameters())
    den = sum(float(p.grad.double().pow(2).sum()) for _, p in oracle.named_parameters())
    e = (num / den) ** 0.5
    print(f"recompute 6 layers vs fp32 autograd: whole-gradient rel={e:.2e}")
    assert e < 1e-2


def test_ema_inside_adamw_matches_reference_formula():
    """ema = decay * ema + (1 - decay) * p after every optimizer step (diffusionGS/utils/ema.py:82-101), fused into AdamW."""
    decay = 0.9
    model, trainer, inp = _model_and_inputs(ema_decay=decay, lr=1e-3, clip=0.0)
    ema_ref = trainer.master.clone()
    for step in range(3):
        _backward_once(model, trainer, inp, seed=step)
        trainer.optimizer_step(allreduce=False)
        ema_ref = decay * ema_ref + (1 - decay) * trainer.master
    torch.cuda.synchronize()
    assert rel(trainer.ema, ema_ref) < 1e-6
    assert rel(trainer.ema, trainer.master) > 1e-6  # the EMA really lags the weights
    sd = trainer.ema_state_dict()
    assert list(sd) == [n for n, _ in model.named_parameters()]
    live = trainer.master.clone()
    with trainer.swap_ema_weights():
        assert torch.equal(trainer.master, trainer.ema)
        with torch.no_grad():
            model.eval()
            model.image_to_gaussians(*inp)
            model.train()
    assert torch.equal(trainer.master, live)


def test_ema_checkpoint_roundtrip(tmp_path):
    from dgs_b200 import checkpoint as ck
    from dgs_b200.denoiser import DGSDenoiser
    model, trainer, inp = _model_and_inputs(ema_decay=0.5, lr=1e-3)
    _backward_once(model, trainer, inp)
    trainer.optimizer_step(allreduce=False)
    reg = str(tmp_path / "step1.ckpt")
    ck.save_system_checkpoint(model, reg, epoch=1, global_step=1)
    path = ck.save_ema_checkpoint(trainer, reg, epoch=1, global_step=1)
    assert path.endswith("step1-EMA.ckpt")
    m2 = DGSDenoiser(dict(patch_size=8, num_layers=2))
    meta = ck.load_checkpoint(m2, path)
    assert meta["global_step"] == 1
    for (n, p), (_, e) in zip(m2.named_parameters(), trainer.ema_state_dict().items()):
        assert torch.equal(p.detach(), e.cpu()), n


def test_trainer_guards():
    """One training forward may be outstanding; every way of breaking that raises instead of corrupting state."""
    model, trainer, inp = _model_and_inputs()
    images, ray_o, ray_d, t = inp
    out, _ = model.image_to_gaussians(images, ray_o, ray_d, t)
    with pytest.raises(RuntimeError, match="already pending"):
        model.image_to_gaussians(images, ray_o, ray_d, t)          # second grad-enabled forward
    with pytest.raises(RuntimeError, match="pending"):
        with torch.no_grad():
            model.image_to_gaussians(images, ray_o, ray_d, t)      # inference would overwrite the shared workspace
    with pytest.raises(RuntimeError, match="still pending"):
        trainer.optimizer_step(allreduce=False)                      # step before backward
    loss = out.xyz.sum()
    loss.backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="already backpropagated"):
        loss.backward()                                              # the activation state was consumed
    trainer.optimizer_step(allreduce=False)
    with pytest.raises(RuntimeError, match="no backward"):
        trainer.optimizer_step(allreduce=False)
    out, _ = model.image_to_gaussians(images, ray_o, ray_d, t)      # a dropped forward ...
    trainer.reset()
    out, _ = model.image_to_gaussians(images, ray_o, ray_d, t)      # ... does not block the next one
    out.xyz.sum().backward()
    trainer.optimizer_step(allreduce=False)


def test_gradient_accumulation_is_the_mean_of_micro_batches():
    m0, t0, inp = _model_and_inputs(clip=0.0, lr=1e-3)
    _backward_once(m0, t0, inp, seed=1)
    g1 = t0.arena.flat.clone()
    _backward_once(m0, t0, inp, seed=2)
    g2 = t0.arena.flat.clone()
    m1, t1, _ = _model_and_inputs(clip=0.0, lr=1e-3, accumulate_grad_batches=2)
    _backward_once(m1, t1, inp, seed=1)
    _backward_once(m1, t1, inp, seed=2)
    assert rel(t1._accum, g1 + g2) < 1e-5  # split-K weight gradients add their partial sums in arrival order
    # one AdamW step from zero moments: update = -lr * sign-ish(mean grad); compare against a single step on the mean
    t1.optimizer_step(allreduce=False)
    t0.arena.flat.copy_((g1 + g2) / 2)
    t0._micro = 1
    t0.optimizer_step(allreduce=False)
    torch.cuda.synchronize()
    assert rel(t1.master, t0.master) < 1e-6


def _render_inputs(B=2, V=3, P=2000, W=64, H=48):
    from dgs_b200 import synth
    gs = [synth.make_gaussians(P, i, "trained") for i in range(B)]
    names = ("xyz", "features", "scaling", "rotation", "opacity")
    raw = {k: np.stack([g[k] for g in gs]) for k in names}
    cams = [synth.orbit_cameras(V, W, H, az0=15.0 * i) for i in range(B)]
    c2w, fx = np.stack([c[0] for c in cams]), np.stack([c[1] for c in cams])
    return names, raw, torch.tensor(c2w, device=DEV), torch.tensor(fx, device=DEV)


@pytest.mark.parametrize("tc,with_image_grad", [(3, False), (4, False), (3, True)])
def test_fused_mse_matches_unfused(tc, with_image_grad):
    """Renderer.forward_mse == Renderer.forward + F.mse_loss per sample (losses.py:279-281), values and gradients."""
    from dgs_b200.renderer import Renderer
    B, V, W, H = 2, 3, 64, 48
    names, raw, c2w, fx = _render_inputs(B, V, 2000, W, H)

    class Cfg:
        gaussians_sh_degree = 0
        use_gssplat = False
    r = Renderer(Cfg())
    g = torch.Generator(DEV).manual_seed(3)
    target = torch.rand(B, V, tc, H, W, device=DEV, generator=g)
    lam = torch.tensor([0.7, 1.3], device=DEV)           # per-sample weights: dL/dl2_loss[b]
    gimg = torch.randn(B, V, 3, H, W, device=DEV, generator=g) * 1e-3
    pa = [torch.tensor(raw[k], device=DEV, requires_grad=True) for k in names]
    img_a = r(*pa, H, W, c2w, fx)
    l2_a = ((img_a - target[:, :, :3]) ** 2).mean(dim=(1, 2, 3, 4))
    loss_a = (l2_a * lam).sum() + ((img_a * gimg).sum() if with_image_grad else 0.0)
    loss_a.backward()
    pb = [torch.tensor(raw[k], device=DEV, requires_grad=True) for k in names]
    img_b, l2_b = r.forward_mse(*pb, H, W, c2w, fx, target)
    loss_b = (l2_b * lam).sum() + ((img_b * gimg).sum() if with_image_grad else 0.0)
    loss_b.backward()
    torch.cuda.synchronize()
    assert torch.equal(img_a.detach(), img_b.detach())
    assert rel(l2_b, l2_a) < 1e-6
    for k, a, b in zip(names, pa, pb):
        e = rel(b.grad, a.grad)
        print(f"fused mse tc={tc} img_grad={with_image_grad} d{k}: rel={e:.2e}")
        assert e < 1e-5, k


def test_fused_mse_two_phase_binning_counts_every_pixel_once():
    """Dense scene (R >= 2^21) -> the near/far two-phase path: phase A counts the tiles it finished, phase B the open ones."""
    from dgs_b200 import raster, synth
    B, V, P, W, H = 1, 2, 60000, 256, 256
    g = synth.make_gaussians(P, 0, "init")
    names = ("xyz", "features", "scaling", "rotation", "opacity")
    t = [torch.tensor(g[k][None], device=DEV) for k in names]
    t[2] = t[2] + 1.2  # bigger splats: tens of tiles per Gaussian
    c2w, fx = synth.orbit_cameras(V, W, H)
    c2w, fx = torch.tensor(c2w[None], device=DEV), torch.tensor(fx[None], device=DEV)
    target = torch.rand(B, V, 3, H, W, device=DEV)
    for near in (0, 3):
        ls = torch.zeros(B, dtype=torch.float64, device=DEV)
        img, st = raster.render_batch_forward(*t, H, W, c2w, fx, near_log2=near, mse_target=target, mse_loss_sum=ls)
        ref = ((img - target) ** 2).double().sum(dim=(1, 2, 3, 4))
        print(f"near_log2={near}: R={st['R']} chunks={st['chunks']} loss_sum={float(ls[0]):.6f} ref={float(ref[0]):.6f}")
        assert st["R"] >= (1 << 21)
        assert rel(ls, ref) < 1e-6


def test_loss_stage_end_to_end_training_step():
    """DiT -> fused render + MSE -> backward -> AdamW: same loss value and same gradients as the unfused torch loss."""
    from dgs_b200 import losses, synth
    m0, t0, inp = _model_and_inputs(B=1, V=4, H=32, W=32, clip=0.0)
    images, ray_o, ray_d, t = inp
    c2w, fx = synth.orbit_cameras(5, 32, 32)
    c2w, fx = torch.tensor(c2w[None], device=DEV), torch.tensor(fx[None], device=DEV)
    target = torch.rand(1, 5, 3, 32, 32, device=DEV)
    out, _ = m0.image_to_gaussians(images, ray_o, ray_d, t)
    res, renders = losses.fused_render_and_loss(m0, out, c2w, fx, 32, 32, target, lambdas=dict(lambda_diffusion=1.0))
    res["loss"].backward()
    g_fused = t0.arena.flat.clone()
    m1, t1, _ = _model_and_inputs(B=1, V=4, H=32, W=32, clip=0.0)
    out1, _ = m1.image_to_gaussians(images, ray_o, ray_d, t)
    r1 = m1.render_gaussians(out1, c2w, fx, 32, 32)
    loss1 = torch.nn.functional.mse_loss(r1, target)
    loss1.backward()
    torch.cuda.synchronize()
    assert rel(res["loss"], loss1) < 1e-6
    e = rel(g_fused, t1.arena.flat)
    print(f"fused loss stage: loss={float(res['loss']):.6f} whole-gradient rel vs unfused={e:.2e}")
    assert e < 1e-4
