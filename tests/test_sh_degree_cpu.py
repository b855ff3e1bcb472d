"""The denoiser at gaussians_sh_degree 0..3 without a GPU: the module tree against the reference's, the configuration
checks of the Python modules and of the C ABI, the degree-aware oracle (oracle/dit.py) against outputs of the
reference's own code (tests/golden/make_dit_sh_golden.py), and the degree-3 Gaussians through prepare_to_save and the
PLY files."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_dit_sh_golden as msg  # noqa: E402
import ref_import as ri  # noqa: E402
from util import rel_l2 as rel  # noqa: E402

from oracle import dit as od  # noqa: E402

SMALL = [n for n in msg.DIT_SH_CASES if n.startswith("s_")]
WIDE = [n for n in msg.DIT_SH_CASES if n.startswith("w1024_")]


def _model(scene, **cfg):
    from dgs_b200.denoiser import DGSDenoiser, DGSDenoiserScene
    return (DGSDenoiserScene if scene else DGSDenoiser)(dict(cfg, in_channels=9, n_gaussians=2))


@pytest.mark.parametrize("scene", [False, True], ids=["obj", "scene"])
@pytest.mark.parametrize("degree", [0, 1, 2, 3])
def test_state_dict_keys_and_shapes_equal_reference(scene, degree):
    z = np.load(os.path.join(HERE, "golden", "dit_sh_keys.npz"))
    pre = f"{'scene' if scene else 'obj'}_sh{degree}/"
    sd = _model(scene, **msg.KEYS_CFG, gaussians_sh_degree=degree).state_dict()
    assert list(sd) == [str(k) for k in z[pre + "keys"]]
    for k, v in sd.items():
        assert tuple(v.shape) == tuple(z[pre + "shape/" + k]), k
    C_ = od.head_channels(degree)
    assert tuple(sd["upsampler.linear.weight"].shape) == (C_, 64)
    assert tuple(sd["image_token_decoder.linear.weight"].shape) == (64 * C_, 64)


def test_degree_d_checkpoint_loads_strictly(tmp_path):
    from dgs_b200 import checkpoint  # noqa: F401  (the module the trainer saves through; keys only)
    a = _model(False, **msg.KEYS_CFG, gaussians_sh_degree=3)
    path = tmp_path / "sh3.pt"
    torch.save(a.state_dict(), path)
    b = _model(False, **msg.KEYS_CFG, gaussians_sh_degree=3)
    b.load_state_dict(torch.load(path), strict=True)
    assert all(torch.equal(a.state_dict()[k], v) for k, v in b.state_dict().items())
    with pytest.raises(RuntimeError):
        _model(False, **msg.KEYS_CFG, gaussians_sh_degree=1).load_state_dict(torch.load(path), strict=True)


@pytest.mark.parametrize("degree", [-1, 4])
def test_degree_out_of_range_is_rejected(degree):
    with pytest.raises(ValueError, match="gaussians_sh_degree"):
        _model(False, **msg.KEYS_CFG, gaussians_sh_degree=degree)


def test_patch4_with_odd_channel_count_is_rejected():
    """patch 4: 16 C outputs per token, a multiple of 32 only for even C (degrees 0 and 2)."""
    for d in (1, 3):
        with pytest.raises(ValueError, match="multiple of 32"):
            _model(True, width=64, dim_heads=16, num_layers=1, patch_size=4, gaussians_sh_degree=d)
    _model(True, width=64, dim_heads=16, num_layers=1, patch_size=4, gaussians_sh_degree=2)


def _abi_weights(**kw):
    from dgs_b200._lib import DitWeights
    return DitWeights(**dict(dict(width=1024, heads=16, layers=2, patch=8, n_gaussians=2, mlp_hidden=4096), **kw))


def test_c_abi_sh_degree_field_and_checks():
    """sh_degree is appended after every existing field of dgs_dit_weights (their offsets unchanged, a zero-initialised
    struct is degree 0); dgs_dit_workspace_bytes sizes the head buffers by it and refuses what the heads cannot run."""
    from dgs_b200 import _lib
    from dgs_b200._lib import DitWeights
    names = [f[0] for f in DitWeights._fields_]
    assert names[-1] == "sh_degree" and names[-2] == "dec_w"
    assert DitWeights.sh_degree.offset == DitWeights.dec_w.offset + C.sizeof(C.c_void_p)
    assert DitWeights().sh_degree == 0
    L = _lib.lib()
    sizes = [L.dgs_dit_workspace_bytes(C.byref(_abi_weights(sh_degree=d)), 1, 4, 64, 64) for d in range(4)]
    assert sizes[0] == L.dgs_dit_workspace_bytes(C.byref(_abi_weights()), 1, 4, 64, 64) > 0
    T = 4 * 8 * 8
    for d in range(1, 4):  # gs_tok [B*G, C] and img_gs [B*T, 64 C], fp32, up to the carver's alignment
        extra = (2 * (od.head_channels(d) - 14) + T * 64 * (od.head_channels(d) - 14)) * 4
        assert extra - 256 <= sizes[d] - sizes[0] <= extra + 256, d
    for bad in (dict(sh_degree=4), dict(sh_degree=-1)):
        assert L.dgs_dit_workspace_bytes(C.byref(_abi_weights(**bad)), 1, 4, 64, 64) == 0
        assert "sh_degree" in L.dgs_last_error().decode()
    assert L.dgs_dit_workspace_bytes(C.byref(_abi_weights(patch=4, sh_degree=1)), 1, 4, 64, 64) == 0
    assert "multiple of 32" in L.dgs_last_error().decode()
    assert L.dgs_dit_workspace_bytes(C.byref(_abi_weights(patch=4, sh_degree=2)), 1, 4, 64, 64) > 0
    assert L.dgs_dit_train_state_bytes(C.byref(_abi_weights(sh_degree=3)), 1, 4, 64, 64) > \
        L.dgs_dit_train_state_bytes(C.byref(_abi_weights()), 1, 4, 64, 64)


def _oracle_for(name):
    scene, pe, cfg, _, seed = msg.DIT_SH_CASES[name]
    o = od.DenoiserOracle(width=cfg["width"], heads=cfg["width"] // cfg["dim_heads"], layers=cfg["num_layers"],
                          patch=cfg["patch_size"], scene=scene, ray_pe_type=pe, sh_degree=cfg["gaussians_sh_degree"])
    z = np.load(os.path.join(HERE, "golden", f"dit_ref_{name}.npz"))
    keys = [str(k) for k in z["keys"]]
    assert list(o.state_dict()) == keys
    for k, v in o.state_dict().items():
        assert tuple(v.shape) == tuple(z["shape/" + k]), k
    o.load_state_dict(ri.seeded_state_dict(o, seed), strict=True)
    return o, z


@pytest.mark.parametrize("name", SMALL + WIDE)
def test_oracle_reproduces_reference_outputs(name):
    """The degree-aware oracle on the case's seeded parameters and inputs against what the reference's own
    DGSDenoiser[Scene] produced: outputs to 1e-5 relative (BLAS summation order may differ between boxes), and on the
    small cases the parameter gradients of the seeded loss (norms to 1e-4, fixed projections to 1e-3 of the norm)."""
    if name.startswith("w1024") and os.environ.get("DGS_SKIP_WIDE_CPU"):
        pytest.skip("wide cases skipped by request")
    _, _, cfg, (b, v, h, w), seed = msg.DIT_SH_CASES[name]
    o, z = _oracle_for(name)
    img, ro, rd, t = ri.seeded_dit_inputs(b, v, h, w, seed + 1000)
    oo, oia = o.image_to_gaussians(img, ro, rd, t)
    oo = dict(oo, img_aligned_xyz=oia)
    M = (cfg["gaussians_sh_degree"] + 1) ** 2
    assert tuple(oo["features"].shape) == (b, 2 + v * h * w, M, 3)
    for k in [f[4:] for f in z.files if f.startswith("out/")]:
        e = rel(oo[k], torch.from_numpy(z["out/" + k]))
        assert e < 1e-5, (name, k, e)
    if name.startswith("s_"):
        cot = {k: ri.seeded(tuple(oo[k].shape), seed + 2000 + i) for i, k in enumerate(ri.GS_KEYS)}
        loss = sum((oo[k] * cot[k]).sum() for k in cot)
        og = torch.autograd.grad(loss, list(o.parameters()))
        rng = np.random.default_rng(7)
        for (k, _), g in zip(o.named_parameters(), og):
            gg = g.double().numpy().ravel()
            n_ref, p_ref = float(z["gnorm/" + k]), float(z["gproj/" + k])
            proj = float(gg @ rng.standard_normal(gg.size))
            assert abs(np.linalg.norm(gg) - n_ref) <= 1e-4 * n_ref + 1e-12, (name, k)
            assert abs(proj - p_ref) <= 1e-3 * n_ref + 1e-9, (name, k)


@pytest.mark.skipif(not ri.available(), reason="needs a reference checkout (DGS_REFERENCE_ROOT)")
def test_oracle_equals_reference_code_directly():
    """Where the reference is mounted: the oracle against the reference's own module, outputs and every gradient."""
    name = "s_obj_rel_sh3"
    model, outs, grads = msg.reference_sh_case(name)
    _, _, _, (b, v, h, w), seed = msg.DIT_SH_CASES[name]
    o, _ = _oracle_for(name)
    img, ro, rd, t = ri.seeded_dit_inputs(b, v, h, w, seed + 1000)
    oo, oia = o.image_to_gaussians(img, ro, rd, t)
    oo = dict(oo, img_aligned_xyz=oia)
    for k, g in outs.items():
        assert rel(oo[k], g) < 1e-6, k
    cot = {k: ri.seeded(tuple(oo[k].shape), seed + 2000 + i) for i, k in enumerate(ri.GS_KEYS)}
    og = torch.autograd.grad(sum((oo[k] * cot[k]).sum() for k in cot), list(o.parameters()))
    for (k, _), g in zip(o.named_parameters(), og):
        assert rel(g, grads[k]) < 2e-5, k


def test_features_are_coefficient_major_copies():
    """feature (k, c) of a Gaussian is raw channel 3 + 3k + c, for free and image tokens, at every degree."""
    b, v, h, w, p, G = 1, 1, 8, 8, 8, 2
    ro = torch.zeros(b, v, 3, h, w, dtype=torch.float64)
    rd = torch.ones(b, v, 3, h, w, dtype=torch.float64)
    for d in range(4):
        C_ = od.head_channels(d)
        gs = torch.arange(b * G * C_, dtype=torch.float64).reshape(b, G, C_)
        ig = 1000 + torch.arange(b * p * p * C_, dtype=torch.float64).reshape(b, 1, p * p * C_)
        f = od.gaussians_epilogue64(gs, ig, ro, rd, 0)["features"]
        raw = torch.cat([gs, ig.reshape(b, -1, C_)], dim=1)
        for k in range((d + 1) ** 2):
            for c in range(3):
                assert torch.equal(f[:, :, k, c], raw[:, :, 3 + 3 * k + c])


def _read_ply(path):
    with open(path, "rb") as fh:
        data = fh.read()
    head, body = data.split(b"end_header\n", 1)
    props = [ln.split() for ln in head.decode().splitlines() if ln.startswith("property")]
    dt = np.dtype([(p[2], "<f4" if p[1] == "float" else "u1") for p in props])
    return np.frombuffer(body, dtype=dt)


def test_degree3_gaussians_through_prepare_to_save_and_ply(tmp_path):
    """Degree-3 DiT outputs [B, P, 16, 3] go through prepare_to_save into a degree-3 GaussianModel, whose save_ply
    writes f_rest in the reference's order (gs_core.py: features_rest.transpose(1, 2).flatten(1), i.e. f_rest_i =
    feature (1 + i % 15, i // 15)) and whose load_ply reads them back unchanged."""
    from dgs_b200.denoiser import AttrDict
    from dgs_b200.renderer import GaussianModel
    model = _model(False, **msg.KEYS_CFG, gaussians_sh_degree=3)
    g = torch.Generator().manual_seed(3)
    P = 37
    params = AttrDict(xyz=torch.randn(1, P, 3, generator=g), features=torch.randn(1, P, 16, 3, generator=g),
                      scaling=torch.randn(1, P, 3, generator=g) - 3, rotation=torch.randn(1, P, 4, generator=g),
                      opacity=torch.randn(1, P, 1, generator=g))
    gm, = model.prepare_to_save(params)
    assert gm.sh_degree == 3 and torch.equal(gm.get_features, params.features[0])
    path = gm.save_ply(str(tmp_path / "sh3.ply"))
    v = _read_ply(path)
    feats = params.features[0].numpy()
    for i in range(45):
        np.testing.assert_array_equal(v[f"f_rest_{i}"], feats[:, 1 + i % 15, i // 15])
    for c in range(3):
        np.testing.assert_array_equal(v[f"f_dc_{c}"], feats[:, 0, c])
    back = GaussianModel(3).load_ply(path)
    assert torch.equal(back.get_features, params.features[0])
    for k in ("_xyz", "_scaling", "_rotation", "_opacity"):
        assert torch.equal(getattr(back, k), getattr(gm, k)), k
