"""The geometry loss terms on the H100 (dgs_b200.geometry_loss over dgs_geometry_loss_forward / _backward) against the
fp64 oracle and the reference's fixture, and their gradient through the DiT backward (dgs_dit_out_grads.d_img_aligned_xyz)
into the model: the exact fold into the image Gaussians' d xyz, the whole model against torch autograd on the oracle
model, and the object recipe's loss schedule (diffusionGS_rel.yaml) through fused_render_and_loss."""
import os

import numpy as np
import pytest
import torch

from util import rel_l2 as rel

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HERE = os.path.dirname(os.path.abspath(__file__))
G_XYZ = 0.025
# diffusionGS_rel.yaml's loss block, lambda_lpips set to 0 (no LPIPS checkpoint here)
REL_LAMBDAS = dict(lambda_diffusion=[150, 0.0, 1.0, 151], lambda_lpips=0.0, lambda_ssim=0.0,
                   lambda_pointsdist=[150, 1.0, 0.0, 151], lambda_xyz=[150, 0.0, 0.025, 151], lambda_depth=0.0)


def kernel_run(x, o, gt, m, g_pd, g_xyz):
    """-> (pointsdist, l2_xyz, d_img) of the kernels through the autograd Function"""
    from dgs_b200.geometry_loss import geometry_losses
    x = x.detach().clone().requires_grad_(True)
    pd, l2 = geometry_losses(x, o, gt, m, pointsdist=g_pd is not None)
    loss = 0.0
    if g_pd is not None:
        loss = loss + (pd * g_pd).sum()
    if g_xyz is not None:
        loss = loss + g_xyz * l2
    d, = torch.autograd.grad(loss, x)
    return (None if pd is None else pd.detach()), (None if l2 is None else l2.detach()), d


def training_shape_inputs(B, V, H, W, seed=0):
    """rays of one camera per view, centres at positive depth along them, binary masks as the datasets give"""
    g = torch.Generator(DEV).manual_seed(seed)
    o = (torch.randn(B, V, 3, 1, 1, device=DEV, generator=g) * 1.5).expand(B, V, 3, H, W).contiguous()
    d = torch.nn.functional.normalize(torch.randn(B, V, 3, H, W, device=DEV, generator=g), dim=2)
    x = o + d * (2.7 + 0.3 * torch.randn(B, V, 1, H, W, device=DEV, generator=g))
    gt = o + d * (2.7 + 0.3 * torch.rand(B, V, 1, H, W, device=DEV, generator=g))
    m = (torch.rand(B, V, 1, H, W, device=DEV, generator=g) > 0.4).float()
    return x, o, gt, m


@pytest.mark.parametrize("name", ["tc3", "tc4", "ragged", "edge"])
def test_kernels_against_fixture_and_oracle(name):
    """Bounds: the values are fp32 per-pixel terms summed in fp64 (measured against fp64 at fp32 rounding, ~1e-7);
    d_img is one fp32 expression per pixel."""
    from oracle.geometry_loss import geometry_grad64
    z = np.load(os.path.join(HERE, "golden", "geometry_loss_ref.npz"))
    x, o, gt, m = (torch.from_numpy(z[f"{name}/{k}"]).to(DEV) for k in ("img_xyz", "ray_o", "gt_xyz", "masks"))
    g_pd = torch.from_numpy(z[f"{name}/g_pd"]).to(DEV)
    pd, l2, d = kernel_run(x, o, gt, m, g_pd, G_XYZ)
    rpd, rl2, rd = geometry_grad64(x, o, gt, m, g_pd=g_pd, g_xyz=G_XYZ)
    ref = lambda k: torch.from_numpy(z[f"{name}/{k}"]).to(DEV)  # noqa: E731
    e = dict(pd_oracle=rel(pd, rpd), l2_oracle=rel(l2, rl2), d_oracle=rel(d, rd),
             pd_ref=rel(pd, ref("pointsdist")), l2_ref=rel(l2, ref("l2_xyz")),
             d_ref=rel(d, ref("d_img")))
    print(name, {k: f"{v:.1e}" for k, v in e.items()})
    assert max(e["pd_oracle"], e["l2_oracle"], e["pd_ref"], e["l2_ref"]) < 1e-6, e
    assert max(e["d_oracle"], e["d_ref"]) < 1e-5, e
    if name == "edge":
        _, _, d_pd = kernel_run(x, o, gt, m, g_pd, None)
        assert torch.all(d_pd[1, 0, :, 3:9, 5:17] == 0)  # dist == 0: no pointsdist gradient
        assert torch.isfinite(d_pd).all()


@pytest.mark.parametrize("H", [256, 512])
def test_kernels_at_training_shapes(H):
    """obj-256 (B = 4, V = 4, 256^2) and 512^2: against fp64, the same bits on a second run, and each sample's
    pointsdist and its part of d_img the same bits from a B = 1 call (l2_xyz is one number over the batch)."""
    from oracle.geometry_loss import geometry_grad64
    B, V = 4, 4
    x, o, gt, m = training_shape_inputs(B, V, H, H)
    g_pd = torch.full((B,), 0.25, device=DEV)  # pointsdist.mean()
    pd, l2, d = kernel_run(x, o, gt, m, g_pd, G_XYZ)
    rpd, rl2, rd = geometry_grad64(x, o, gt, m, g_pd=g_pd, g_xyz=G_XYZ)
    e = (rel(pd, rpd), rel(l2, rl2), rel(d, rd))
    print(f"{H}^2: pointsdist {e[0]:.1e} l2_xyz {e[1]:.1e} d_img {e[2]:.1e}")
    assert e[0] < 1e-6 and e[1] < 1e-6 and e[2] < 1e-5, e
    pd2, l22, d2 = kernel_run(x, o, gt, m, g_pd, G_XYZ)
    assert torch.equal(pd, pd2) and torch.equal(l2, l22) and torch.equal(d, d2)
    _, _, d_pd = kernel_run(x, o, gt, m, g_pd, None)
    for b in range(B):
        pb, _, db = kernel_run(x[b:b + 1], o[b:b + 1], gt[b:b + 1], m[b:b + 1], g_pd[b:b + 1], None)
        assert torch.equal(pb, pd[b:b + 1]), b
        assert torch.equal(db, d_pd[b:b + 1]), b


def test_all_zero_mask_gives_nan_like_the_reference():
    x, o, gt, m = training_shape_inputs(1, 2, 32, 48)
    pd, l2, _ = kernel_run(x, o, gt, torch.zeros_like(m), torch.ones(1, device=DEV), None)
    assert torch.isnan(l2) and torch.isfinite(pd).all()


# ---- through the DiT backward ----------------------------------------------------------------------------------------

KINDS = {"obj-rel": (False, "relative_plk"), "obj-plk": (False, "plk"), "scene-plk": (True, "plk")}


def build(kind, layers, recompute):
    from dgs_b200.denoiser import DGSDenoiser, DGSDenoiserScene
    from dgs_b200.train import DitTrainer
    scene, pe = KINDS[kind]
    torch.manual_seed(0)
    model = (DGSDenoiserScene if scene else DGSDenoiser)(dict(patch_size=8, num_layers=layers, ray_pe_type=pe)).to(DEV)
    with torch.no_grad():  # non-zero biases so that every gradient path carries signal
        g = torch.Generator(DEV).manual_seed(5)
        for n, p in model.named_parameters():
            if n.endswith(".bias"):
                p.copy_(0.05 * torch.randn(p.shape, device=DEV, generator=g))
    trainer = DitTrainer(model, recompute=recompute)
    model.train()
    return model, trainer


def scatter_img(d_img, G, p):
    """[B, V, 3, H, W] -> the [B, G + V H W, 3] xyz layout of the image Gaussians ((v, hh, ww, ph, pw) order)"""
    B, V, _, H, W = d_img.shape
    rows = d_img.reshape(B, V, 3, H // p, p, W // p, p).permute(0, 1, 3, 5, 4, 6, 2).reshape(B, -1, 3)
    return torch.cat((torch.zeros(B, G, 3, device=DEV), rows), dim=1)


def _arena_after(model, trainer, inputs, wts, w_img):
    out, img = model.image_to_gaussians(*inputs)
    loss = sum((out[k] * w).sum() for k, w in wts.items())
    if w_img is not None:
        loss = loss + (img * w_img).sum()
    trainer.zero_grad()
    loss.backward()
    torch.cuda.synchronize()
    return trainer.arena.flat.clone()


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("recompute", [False, True])
def test_dit_backward_folds_d_img_exactly(kind, recompute):
    """(d_xyz, d_img) and (d_xyz + scatter(d_img), NULL) give the epilogue the same fp32 sums, so the same parameter
    gradients.  The backward accumulates some of them (biases, LayerNorm weights, the adaLN and conditioning path) with
    float atomics, whose order varies from run to run, so the claim is made per parameter tensor: every tensor the
    (d_xyz + scatter, NULL) call reproduces bit for bit on a second run (the GEMM weight gradients among them) must come
    out bit for bit, and the whole arena within that call's run-to-run spread."""
    from dit_regime import dit_inputs
    model, trainer = build(kind, 2, recompute)
    inputs = dit_inputs(2, 4, 32, 48)
    B, V, _, H, W = inputs[0].shape
    G, p = model.cfg.n_gaussians, model.cfg.patch_size
    P = G + V * H * W
    g = torch.Generator(DEV).manual_seed(3)
    n_sh = (model.cfg.gaussians_sh_degree + 1) ** 2
    shapes = dict(xyz=(B, P, 3), features=(B, P, n_sh, 3), scaling=(B, P, 3), rotation=(B, P, 4), opacity=(B, P, 1))
    wts = {k: torch.randn(s, device=DEV, generator=g) for k, s in shapes.items()}
    w_img = torch.randn(B, V, 3, H, W, device=DEV, generator=g)
    folded = _arena_after(model, trainer, inputs, wts, w_img)
    pre = dict(wts, xyz=wts["xyz"] + scatter_img(w_img, G, p))
    ref = _arena_after(model, trainer, inputs, pre, None)
    ref2 = _arena_after(model, trainer, inputs, pre, None)
    spread, exact, off = rel(ref2, ref), [], 0
    for name, q in model.named_parameters():
        sl = slice(off, off + q.numel())
        off += q.numel()
        if q.numel() >= 4096 and torch.equal(ref[sl], ref2[sl]):
            exact.append(name)
            assert torch.equal(folded[sl], ref[sl]), name
    print(f"{kind} {'recompute' if recompute else 'store'}: {len(exact)} tensors reproducible bit for bit, run-to-run "
          f"{spread:.1e}, folded vs pre-scattered {rel(folded, ref):.1e}")
    assert "image_token_decoder.linear.weight" in exact and any("attn.qkv.weight" in n for n in exact)
    assert rel(folded, ref) <= max(4 * spread, 1e-6)
    base = _arena_after(model, trainer, inputs, wts, None)
    assert rel(base, ref) > 1e-3  # the d_img term is really there


def test_geometry_terms_through_the_model_vs_oracle_autograd():
    """0.7 pointsdist.mean() + 0.025 l2_xyz through the product (kernels + dgs_dit_backward) vs torch autograd through
    DenoiserOracle and the fp64 oracle of the two terms: the bound test_recompute_full_depth_vs_oracle uses."""
    from dgs_b200.geometry_loss import geometry_losses
    from oracle.dit import DenoiserOracle
    from oracle.geometry_loss import geometry_losses64
    from dit_regime import dit_inputs
    model, trainer = build("obj-rel", 4, True)
    oracle = DenoiserOracle(layers=4).to(DEV)
    oracle.load_state_dict(model.state_dict(), strict=True)
    images, ray_o, ray_d, t = dit_inputs(1, 4, 64, 64)
    gen = torch.Generator(DEV).manual_seed(9)
    gt = ray_o + ray_d * (2.7 + 0.3 * torch.rand(1, 4, 1, 64, 64, device=DEV, generator=gen))
    m = (torch.rand(1, 4, 1, 64, 64, device=DEV, generator=gen) > 0.4).float()
    _, img = model.image_to_gaussians(images, ray_o, ray_d, t)
    pd, l2 = geometry_losses(img, ray_o, gt, m)
    trainer.zero_grad()
    (0.7 * pd.mean() + G_XYZ * l2).backward()
    _, ref_img = oracle.image_to_gaussians(images, ray_o, ray_d, t)
    rpd, rl2 = geometry_losses64(ref_img, ray_o, gt, m)
    (0.7 * rpd.mean() + G_XYZ * rl2).backward()
    ours = dict(model.named_parameters())
    num = sum(float((ours[n].grad.double() - q.grad.double()).pow(2).sum()) for n, q in oracle.named_parameters())
    den = sum(float(q.grad.double().pow(2).sum()) for _, q in oracle.named_parameters())
    e = (num / den) ** 0.5
    print(f"geometry terms through 4 layers vs fp32 autograd: whole-gradient rel={e:.2e}, den={den:.2e}")
    assert den > 0 and e < 1e-2


def _recipe_setup():
    from dgs_b200 import synth
    from dit_regime import dit_inputs
    model, trainer = build("obj-rel", 2, True)
    B, V, H, W = 2, 4, 64, 64
    images, ray_o, ray_d, t = dit_inputs(B, V, H, W)
    c2w, fx = synth.orbit_cameras(V, W, H)
    c2w = torch.tensor(c2w[None], device=DEV).expand(B, -1, -1, -1).contiguous()
    fx = torch.tensor(fx[None], device=DEV).expand(B, -1, -1).contiguous()
    gen = torch.Generator(DEV).manual_seed(4)
    target = torch.rand(B, V, 3, H, W, device=DEV, generator=gen)
    gt = ray_o + ray_d * (2.7 + 0.3 * torch.rand(B, V, 1, H, W, device=DEV, generator=gen))
    m = (torch.rand(B, V, 1, H, W, device=DEV, generator=gen) > 0.4).float()
    return model, trainer, (images, ray_o, ray_d, t), (c2w, fx, H, W, target, gt, m)


def _fused_grad(model, trainer, inputs, scene, step, lambdas=REL_LAMBDAS):
    from dgs_b200.losses import LossComputer, fused_render_and_loss
    c2w, fx, H, W, target, gt, m = scene
    out, img = model.image_to_gaussians(*inputs)
    trainer.zero_grad()
    losses, _ = fused_render_and_loss(model, out, c2w, fx, H, W, target, loss_computer=LossComputer(compute_pointsdist=True),
                                      lambdas=lambdas, ray_o=inputs[1], masks_all=m, masks=m, img_aligned_xyz=img,
                                      gt_img_aligned_xyz=gt, global_step=step)
    losses["loss"].backward()
    torch.cuda.synchronize()
    return trainer.arena.flat.clone(), losses


def _unfused_grad(model, trainer, inputs, scene, w_mse, w_pd, w_xyz):
    """the same weighted loss from torch ops: the renderer's forward + F.mse_loss, the reference's geometry formulas"""
    c2w, fx, H, W, target, gt, m = scene
    o = inputs[1]
    out, img = model.image_to_gaussians(*inputs)
    loss = 0.0
    if w_mse:
        r = model.render_gaussians(out, c2w, fx, H, W)
        loss = loss + w_mse * ((r - target) ** 2).mean(dim=(1, 2, 3, 4)).mean()
    if w_pd:
        dist = (img - o).norm(dim=2, p=2, keepdim=True)
        dd = dist.detach()
        trgt = (dd - dd.mean(dim=(2, 3, 4), keepdim=True)) / (dd.std(dim=(2, 3, 4), keepdim=True) + 1e-8) * 0.5 + \
            torch.norm(o, dim=2, p=2, keepdim=True)
        loss = loss + w_pd * ((dist - trgt) ** 2).mean(dim=(1, 2, 3, 4)).mean()
    if w_xyz:
        loss = loss + w_xyz * torch.nn.functional.mse_loss(img * m, gt * m, reduction="sum") / m.sum()
    trainer.zero_grad()
    loss.backward()
    torch.cuda.synchronize()
    return trainer.arena.flat.clone()


def test_object_recipe_trains_at_every_step():
    """diffusionGS_rel.yaml through fused_render_and_loss.  Step 0: pointsdist is the only weighted term, and the
    gradient reaches the model.  Step 151: MSE + 0.025 xyz.  Against the same losses from torch ops; the bound covers
    bf16 rounding flips of the decoder's output gradient (1 bf16 ulp = 2^-8 on the flipped entries)."""
    model, trainer, inputs, scene = _recipe_setup()
    g0, l0 = _fused_grad(model, trainer, inputs, scene, 0)
    assert float(l0["loss"].detach()) == float(l0["loss_pointsdist"].detach()) and float(g0.abs().max()) > 0
    u0 = _unfused_grad(model, trainer, inputs, scene, 0.0, 1.0, 0.0)
    e0 = rel(g0, u0)
    g151, l151 = _fused_grad(model, trainer, inputs, scene, 151)
    assert float(l151["loss"]) == pytest.approx(float(l151["loss_diffusion"]) + 0.025 * float(l151["loss_xyz"]), rel=1e-6)
    u151 = _unfused_grad(model, trainer, inputs, scene, 1.0, 0.0, 0.025)
    mse = _unfused_grad(model, trainer, inputs, scene, 1.0, 0.0, 0.0)
    g_mse, _ = _fused_grad(model, trainer, inputs, scene, 151, lambdas=dict(lambda_diffusion=1.0))
    e151, e_term = rel(g151, u151), rel(g151 - g_mse, u151 - mse)
    print(f"recipe: step 0 rel={e0:.1e}; step 151 rel={e151:.1e}, xyz term rel={e_term:.1e}, "
          f"|xyz term| / |mse| = {float((u151 - mse).norm() / mse.norm()):.2e}")
    assert e0 < 1e-3 and e151 < 1e-3 and e_term < 2e-2
