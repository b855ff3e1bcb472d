"""GPU parity tests of the DiT kernels (wgmma attention, LN+modulate; the GEMM is tested in test_gemm_gpu.py) and of
the whole DGSDenoiser.image_to_gaussians against the fp32 PyTorch oracle (oracle/dit.py).
Tolerance: 1e-3 relative in bf16, measured norm-wise against fp32 on the SAME
(bf16-representable where the kernel consumes bf16) inputs; the exact bound per check is written below."""
import numpy as np
import pytest
import torch

from dit_regime import dit_inputs
from util import rel_l2 as rel

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


# (1, 2050, 20) / (1, 1500, 16) / (3, 4098, 16): ragged query/key tails at other head counts and batch sizes
# (1, 16386, 2): the 512x512 configurations (obj-512 / scene-512 / the pipline_obj.py demo), two heads bound the fp32 reference
@pytest.mark.parametrize("B,N,H", [(1, 4098, 16), (2, 1026, 16), (1, 128, 2), (1, 130, 1), (2, 77, 4), (1, 1, 1), (1, 16386, 2),
                                   (1, 2050, 20), (1, 1500, 16), (3, 4098, 16)])
def test_attention_vs_fp32_softmax(B, N, H):
    from dgs_b200 import _lib
    g = torch.Generator(DEV).manual_seed(N)
    qkv = (torch.randn(B, N, 3, H, 64, device=DEV, generator=g) * 1.5).to(torch.bfloat16)
    out = torch.zeros(B, N, H * 64, dtype=torch.bfloat16, device=DEV)
    _lib.check(_lib.lib().dgs_attention_fwd(qkv.data_ptr(), out.data_ptr(), B, N, H, _lib.stream(None)))
    q, k, v = [t.float().permute(0, 2, 1, 3) for t in qkv.unbind(2)]  # [B,H,N,64]
    ref = torch.softmax((q @ k.transpose(-1, -2)) * 0.125, dim=-1) @ v
    ref = ref.permute(0, 2, 1, 3).reshape(B, N, H * 64)
    e = rel(out.float(), ref)
    print(f"attention B={B} N={N} H={H}: rel={e:.2e}")
    # Operator-level bound, not the model-level one: the inputs here are N(0, 1.5^2) q/k (logit std 2.25, peaky rows) and
    # BOTH P (before the PV MMA) and the output are rounded to bf16 (2^-9 relative each, uncorrelated): ~2e-3 norm-wise.
    # Against the fp32 result rounded to bf16 the kernel must be within the P rounding alone.
    assert e < 3e-3
    assert rel(out.float(), ref.to(torch.bfloat16).float()) < 2.5e-3


def test_ln_modulate():
    from dgs_b200 import _lib
    B, R, D = 2, 515, 1024
    g = torch.Generator(DEV).manual_seed(5)
    x = torch.randn(B, R, D, device=DEV, generator=g) * 3 + 1
    mod = torch.randn(B, 6 * D, device=DEV, generator=g)
    lnw = torch.randn(D, device=DEV, generator=g)
    h = torch.empty(B, R, D, dtype=torch.bfloat16, device=DEV)
    for w_, eps in ((None, 1e-6), (lnw, 1e-5)):
        _lib.check(_lib.lib().dgs_ln_modulate(x.data_ptr(), None if w_ is None else w_.data_ptr(), mod.data_ptr(),
                                              mod[:, D:].data_ptr(), 6 * D, h.data_ptr(), B, R, D, eps,
                                              _lib.stream(None)))
        ln = torch.nn.functional.layer_norm(x, (D,), w_, None, eps)
        ref = ln * (1 + mod[:, None, D:2 * D]) + mod[:, None, :D]
        assert rel(h.float(), ref) < 2.5e-3
        assert rel(h.float(), ref.to(torch.bfloat16).float()) < 3e-4


def _compare_models(model, oracle, B, V, H, W, tag):
    images, ray_o, ray_d, t = dit_inputs(B, V, H, W)
    with torch.no_grad():
        ref, ref_xyz, ref_tok = oracle.image_to_gaussians(images, ray_o, ray_d, t, return_tokens=True)
        out, xyz_img, tok = model.image_to_gaussians(images, ray_o, ray_d, t, return_tokens=True)
    torch.cuda.synchronize()
    errs = {k: rel(out[k], ref[k]) for k in ref}
    errs["tokens"] = rel(tok, ref_tok)
    errs["img_aligned_xyz"] = rel(xyz_img, ref_xyz)
    print(f"[{tag}] " + "  ".join(f"{k}={v:.2e}" for k, v in errs.items()))
    return errs


@pytest.mark.parametrize("scene", [False, True])
def test_denoiser_small_vs_oracle(scene):
    from dgs_b200.denoiser import DGSDenoiser, DGSDenoiserScene
    from oracle.dit import DenoiserOracle
    torch.manual_seed(0)
    cfg = dict(patch_size=8, num_layers=2, ray_pe_type="plk" if scene else "relative_plk")
    model = (DGSDenoiserScene if scene else DGSDenoiser)(cfg).to(DEV)
    oracle = DenoiserOracle(layers=2, scene=scene).to(DEV)
    oracle.load_state_dict(model.state_dict(), strict=True)
    errs = _compare_models(model, oracle, 2, 4, 64, 64, f"small scene={scene}")
    assert all(v < 1e-3 for v in errs.values()), errs  # accuracy bound of the bf16 path


def test_denoiser_full_depth_obj256_vs_oracle():
    """The obj-256 model: 24 layers, 4 views at 256x256 (N = 4098 tokens, P = 262,146 Gaussians),
    random-init weights by the reference's init rules; bf16 tensor-core path vs the fp32 oracle."""
    from dgs_b200.denoiser import DGSDenoiser
    from oracle.dit import DenoiserOracle
    torch.manual_seed(0)
    model = DGSDenoiser(dict(patch_size=8)).to(DEV)
    oracle = DenoiserOracle().to(DEV)
    oracle.load_state_dict(model.state_dict(), strict=True)
    errs = _compare_models(model, oracle, 1, 4, 256, 256, "obj-256 x24")
    # accuracy bound: DiT outputs within 1e-3 rel in bf16 (vs the fp32 oracle with the same fp32 master weights).
    # The two GEMMs at the ends of the network run split-bf16 and the conditioning runs fp32, so what is left is
    # the bf16 operand rounding inside the 24 blocks, entering through the gated residual updates.
    assert all(v < 1e-3 for v in errs.values()), errs
    # the hot path's final product: the rendered views from both sets of Gaussians
    from dgs_b200 import synth
    c2w, fx = synth.orbit_cameras(4, 256, 256)
    c2w, fx = torch.tensor(c2w[None], device=DEV), torch.tensor(fx[None], device=DEV)
    images, ray_o, ray_d, t = dit_inputs(1, 4, 256, 256)
    with torch.no_grad():
        ref, _ = oracle.image_to_gaussians(images, ray_o, ray_d, t)
        out, _ = model.image_to_gaussians(images, ray_o, ray_d, t)
        r_ref = model.gs_renderer(ref["xyz"], ref["features"], ref["scaling"], ref["rotation"], ref["opacity"], 256,
                                  256, c2w, fx)
        r_out = model.render_gaussians(out, c2w, fx, 256, 256)
    e = rel(r_out, r_ref)
    print(f"[obj-256 x24] rendered views (ours DiT vs oracle DiT, same rasterizer): rel={e:.2e}")
    assert e < 1e-3
