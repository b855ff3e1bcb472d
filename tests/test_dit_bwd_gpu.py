"""GPU parity tests of the DiT BACKWARD: the operator kernels against plain PyTorch fp32
autograd of the same op, and the whole dgs_dit_backward (through DGSDenoiser + DitTrainer, i.e. the C ABI) against
torch autograd over the fp32 oracle (oracle/dit.py) with the same fp32 master weights.

Tolerances: the backward runs its GEMMs / attention with bf16 operands (gradient activations rounded to bf16, like
torch autocast), fp32 accumulation, fp32 residual-stream gradient and fp32 weight gradients.  Expected norm-wise error
per tensor ~ a few 1e-3; each bound is written at its assert."""
import pytest
import torch

from util import rel_l2 as rel

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def ptr(t):
    return None if t is None else t.data_ptr()


@pytest.mark.parametrize("M,Cc,f32", [(200, 128, False), (4098, 1024, False), (66, 64, True), (8196, 3072, False)])
def test_transpose_bf16(M, Cc, f32):
    from dgs_b200 import _lib
    g = torch.Generator(DEV).manual_seed(M)
    x = torch.randn(M, Cc, device=DEV, generator=g)
    if not f32:
        x = x.to(torch.bfloat16)
    Mp = (M + 63) // 64 * 64
    out = torch.full((Cc, Mp), 7.0, dtype=torch.bfloat16, device=DEV)
    cs = torch.zeros(Cc, device=DEV)
    _lib.check(_lib.lib().dgs_transpose_bf16(x.data_ptr(), int(f32), M, Cc, out.data_ptr(), cs.data_ptr(),
                                             _lib.stream(None)))
    xb = x.to(torch.bfloat16)
    assert torch.equal(out[:, :M], xb.t())
    assert torch.all(out[:, M:] == 0)
    assert rel(cs, xb.float().sum(0)) < 1e-5


@pytest.mark.parametrize("B,N,H", [(1, 4098, 16), (2, 1026, 16), (1, 128, 2), (2, 200, 2), (1, 77, 4), (1, 64, 2), (1, 130, 1),
                                   (1, 16386, 1)])
def test_attention_backward_vs_autograd(B, N, H):
    from dgs_b200 import _lib
    L = _lib.lib()
    g = torch.Generator(DEV).manual_seed(N + H)
    qkv = (torch.randn(B, N, 3, H, 64, device=DEV, generator=g) * 1.2).to(torch.bfloat16)
    dout = torch.randn(B, N, H * 64, device=DEV, generator=g).to(torch.bfloat16)
    Np = (N + 127) // 128 * 128
    out = torch.zeros(B, N, H * 64, dtype=torch.bfloat16, device=DEV)
    lse = torch.full((B, H, Np), float("nan"), device=DEV)
    dsum = torch.full((B, H, Np), float("nan"), device=DEV)
    dqkv = torch.full((B, N, 3, H, 64), float("nan"), dtype=torch.bfloat16, device=DEV)
    _lib.check(L.dgs_attention_fwd_train(ptr(qkv), ptr(out), ptr(lse), B, N, H, _lib.stream(None)))
    _lib.check(L.dgs_attention_bwd(ptr(qkv), ptr(out), ptr(dout), ptr(lse), ptr(dsum), ptr(dqkv), B, N, H,
                                   _lib.stream(None)))
    torch.cuda.synchronize()
    x = qkv.float().requires_grad_(True)
    q, k, v = [t.permute(0, 2, 1, 3) for t in x.unbind(2)]
    s = (q @ k.transpose(-1, -2)) * 0.125
    ref = (torch.softmax(s, dim=-1) @ v).permute(0, 2, 1, 3).reshape(B, N, H * 64)
    ref.backward(dout.float())
    lse_ref = torch.logsumexp(s.detach(), dim=-1) * 1.4426950408889634
    assert rel(out.float(), ref.detach()) < 4e-3
    assert float((lse[:, :, :N] - lse_ref).abs().max()) < 2e-3
    assert not torch.isnan(dqkv.float()).any()
    errs = [rel(dqkv[:, :, i].float(), x.grad[:, :, i]) for i in range(3)]
    print(f"attention bwd B={B} N={N} H={H}: dq={errs[0]:.2e} dk={errs[1]:.2e} dv={errs[2]:.2e}")
    # P and dS enter the MMAs rounded to bf16 and the result is stored in bf16: a few 1e-3 norm-wise
    assert max(errs) < 8e-3


def test_ln_modulate_backward():
    from dgs_b200 import _lib
    B, R, D = 2, 515, 1024
    g = torch.Generator(DEV).manual_seed(5)
    x = (torch.randn(B, R, D, device=DEV, generator=g) * 3 + 1).requires_grad_(True)
    mod = torch.randn(B, 6 * D, device=DEV, generator=g).requires_grad_(True)
    lnw = torch.randn(D, device=DEV, generator=g).requires_grad_(True)
    dh = torch.randn(B, R, D, device=DEV, generator=g).to(torch.bfloat16)
    stats = torch.empty(B * R * 2, device=DEV)
    for w_, eps, f32 in ((None, 1e-6, False), (lnw, 1e-5, False), (lnw, 1e-5, True)):
        for t in (x, mod, lnw):
            t.grad = None
        ln = torch.nn.functional.layer_norm(x, (D,), w_, None, eps)
        (ln * (1 + mod[:, None, D:2 * D]) + mod[:, None, :D]).backward(dh.float())
        dx = torch.ones(B, R, D, device=DEV)  # accumulate = 1 on top of ones
        dmod = torch.zeros(B, 6 * D, device=DEV)
        dw = torch.zeros(D, device=DEV)
        dh_in = dh.float().contiguous() if f32 else dh
        _lib.check(_lib.lib().dgs_ln_modulate_bwd(ptr(x), ptr(dh_in), int(f32), ptr(w_), mod[:, D:].data_ptr(), 6 * D, B, R,
                                                  D, eps, ptr(dx), 1, ptr(dmod), dmod[:, D:].data_ptr(),
                                                  ptr(dw) if w_ is not None else None, ptr(stats), _lib.stream(None)))
        assert rel(dx - 1, x.grad) < 1e-4
        assert rel(dmod[:, :2 * D], mod.grad[:, :2 * D]) < 1e-4
        if w_ is not None:
            assert rel(dw, lnw.grad) < 1e-4
    # no modulation (the input LayerNorm): scale = NULL
    x.grad = None
    lnw.grad = None
    torch.nn.functional.layer_norm(x, (D,), lnw, None, 1e-5).backward(dh.float())
    dx = torch.zeros(B, R, D, device=DEV)
    dw = torch.zeros(D, device=DEV)
    _lib.check(_lib.lib().dgs_ln_modulate_bwd(ptr(x), ptr(dh), 0, ptr(lnw), None, 0, B, R, D, 1e-5, ptr(dx), 0, None, None,
                                              ptr(dw), ptr(stats), _lib.stream(None)))
    assert rel(dx, x.grad) < 1e-4 and rel(dw, lnw.grad) < 1e-4


def test_gate_backward():
    from dgs_b200 import _lib
    B, R, Cc = 3, 150, 256
    M, Mp = B * R, (B * R + 63) // 64 * 64
    g = torch.Generator(DEV).manual_seed(6)
    dx = torch.randn(M, Cc, device=DEV, generator=g)
    y = torch.randn(M, Cc, device=DEV, generator=g).to(torch.bfloat16)
    mod = torch.randn(B, 3 * Cc, device=DEV, generator=g)
    dy = torch.empty(M, Cc, dtype=torch.bfloat16, device=DEV)
    dyT = torch.empty(Cc, Mp, dtype=torch.bfloat16, device=DEV)
    dmod = torch.zeros(B, 3 * Cc, device=DEV)
    db = torch.zeros(Cc, device=DEV)
    _lib.check(_lib.lib().dgs_gate_bwd(ptr(dx), ptr(y), mod[:, Cc:].data_ptr(), 3 * Cc, R, M, Cc, ptr(dy), ptr(dyT),
                                       dmod[:, Cc:].data_ptr(), ptr(db), _lib.stream(None)))
    gate = mod[:, Cc:2 * Cc].repeat_interleave(R, dim=0)
    ref_dy = (gate * dx).to(torch.bfloat16)
    assert torch.equal(dy, ref_dy)
    assert torch.equal(dyT[:, :M], ref_dy.t()) and torch.all(dyT[:, M:] == 0)
    assert rel(db, ref_dy.float().sum(0)) < 1e-5
    ref_dg = (dx * y.float()).reshape(B, R, Cc).sum(1)
    assert rel(dmod[:, Cc:2 * Cc], ref_dg) < 1e-5
    assert float(dmod[:, :Cc].abs().max()) == 0 and float(dmod[:, 2 * Cc:].abs().max()) == 0


def test_adamw_matches_torch():
    from dgs_b200 import _lib
    g = torch.Generator(DEV).manual_seed(7)
    n = 100003
    p = torch.randn(n, device=DEV, generator=g)
    ref_p = torch.nn.Parameter(p.clone())
    opt = torch.optim.AdamW([ref_p], lr=1e-3, betas=(0.9, 0.99), eps=1e-8, weight_decay=0.01)
    m, v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    two = torch.full((1,), 2.0, device=DEV)  # host scale 0.5 x device scale 2.0 = 1
    for step in range(1, 4):
        grad = torch.randn(n, device=DEV, generator=g)
        ref_p.grad = grad.clone()
        opt.step()
        _lib.check(_lib.lib().dgs_adamw_step(ptr(p), ptr(grad), ptr(m), ptr(v), n, 1e-3, 0.9, 0.99, 1e-8, 0.01, step, 0.5,
                                             ptr(two), _lib.stream(None)))
    assert rel(p, ref_p.data) < 1e-6


def _grad_compare(layers, B, V, H, W, scene, tag, seed=0, regime=None, sq_errs=None):
    """-> (whole-gradient rel error, {parameter: rel error}); `regime(model, seed)` rescales the weights first;
    sq_errs (a dict) receives {parameter: (squared error norm, squared reference norm)}."""
    from dgs_b200.denoiser import DGSDenoiser, DGSDenoiserScene
    from dgs_b200.train import DitTrainer
    from oracle.dit import DenoiserOracle
    from dit_regime import dit_inputs
    torch.manual_seed(seed)
    cfg = dict(patch_size=8, num_layers=layers, ray_pe_type="plk" if scene else "relative_plk")
    model = (DGSDenoiserScene if scene else DGSDenoiser)(cfg)
    if regime is not None:
        regime(model, seed)
    model = model.to(DEV)
    oracle = DenoiserOracle(layers=layers, scene=scene).to(DEV)
    oracle.load_state_dict(model.state_dict(), strict=True)
    trainer = DitTrainer(model)
    model.train()
    images, ray_o, ray_d, t = dit_inputs(B, V, H, W)
    g = torch.Generator(DEV).manual_seed(11)
    out, _ = model.image_to_gaussians(images, ray_o, ray_d, t)
    assert out.xyz.requires_grad
    wts = {k: torch.randn(out[k].shape, device=DEV, generator=g) for k in ("xyz", "features", "scaling", "rotation", "opacity")}
    loss = sum((out[k] * wts[k]).sum() for k in wts)
    trainer.zero_grad()
    loss.backward()
    ref, _ = oracle.image_to_gaussians(images, ray_o, ray_d, t)
    ref_loss = sum((ref[k] * wts[k]).sum() for k in wts)
    ref_loss.backward()
    torch.cuda.synchronize()
    ours = dict(model.named_parameters())
    errs, num, den = {}, 0.0, 0.0
    for name, p in oracle.named_parameters():
        gg = ours[name].grad
        assert gg is not None and p.grad is not None, name
        errs[name] = rel(gg, p.grad)
        n2, d2 = float((gg.double() - p.grad.double()).pow(2).sum()), float(p.grad.double().pow(2).sum())
        num += n2
        den += d2
        if sq_errs is not None:
            sq_errs[name] = (n2, d2)
    total = (num / den) ** 0.5
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:6]
    print(f"[{tag}] loss ours={float(loss):.6e} ref={float(ref_loss):.6e}  whole-gradient rel={total:.2e}  worst: " +
          "  ".join(f"{k}={v:.2e}" for k, v in worst))
    return total, errs


@pytest.mark.parametrize("scene", [False, True])
def test_dit_backward_small_vs_oracle_autograd(scene):
    total, errs = _grad_compare(2, 2, 4, 32, 32, scene, f"bwd small scene={scene}")
    # bf16 gradient activations through 2 blocks: whole-gradient error well under 1e-2, no tensor above 3e-2
    assert total < 1e-2, total
    assert max(errs.values()) < 3e-2, errs


def test_dit_backward_full_depth_obj256_vs_oracle_autograd():
    """The obj-256 training model at one sample: 24 layers, 4 views 256x256 (N = 4098 tokens)."""
    total, errs = _grad_compare(24, 1, 4, 256, 256, False, "bwd obj-256 x24")
    assert total < 2e-2, total
    assert max(errs.values()) < 6e-2, errs


def test_train_steps_reduce_loss_and_track_oracle():
    """3 optimizer steps (forward -> render-free surrogate loss -> backward -> AdamW) on ours and on the oracle with
    torch.optim.AdamW: the losses must decrease and stay within 5e-3 relative of each other."""
    from dgs_b200.denoiser import DGSDenoiser
    from dgs_b200.train import DitTrainer
    from oracle.dit import DenoiserOracle
    from dit_regime import dit_inputs
    torch.manual_seed(0)
    model = DGSDenoiser(dict(patch_size=8, num_layers=2)).to(DEV)
    oracle = DenoiserOracle(layers=2).to(DEV)
    oracle.load_state_dict(model.state_dict(), strict=True)
    trainer = DitTrainer(model, lr=1e-4, clip=0.0)
    opt = torch.optim.AdamW(oracle.parameters(), lr=1e-4, betas=(0.9, 0.99), eps=1e-8, weight_decay=0.01)
    model.train()
    images, ray_o, ray_d, t = dit_inputs(2, 4, 32, 32)
    target = {k: None for k in ("xyz", "features", "opacity")}
    g = torch.Generator(DEV).manual_seed(3)
    losses, ref_losses = [], []
    for step in range(3):
        out, _ = model.image_to_gaussians(images, ray_o, ray_d, t)
        ref, _ = oracle.image_to_gaussians(images, ray_o, ray_d, t)
        if step == 0:
            target = {k: ref[k].detach() + 0.5 * torch.randn(ref[k].shape, device=DEV, generator=g) for k in target}
        loss = sum(((out[k] - target[k]) ** 2).mean() for k in target)
        ref_loss = sum(((ref[k] - target[k]) ** 2).mean() for k in target)
        trainer.zero_grad()
        loss.backward()
        trainer.optimizer_step(allreduce=False)
        opt.zero_grad()
        ref_loss.backward()
        opt.step()
        losses.append(float(loss))
        ref_losses.append(float(ref_loss))
    print("train steps: ours", losses, "oracle", ref_losses)
    assert losses[2] < losses[1] < losses[0]
    assert all(abs(a - b) <= 5e-3 * abs(b) for a, b in zip(losses, ref_losses))
