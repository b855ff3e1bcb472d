"""LPIPS-VGG without a GPU: the fp64 reference against torchvision's VGG16, weight loading from every checkpoint layout,
and the argument checks of the C ABI (dgs_lpips_*)."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from lpips_regime import random_lpips_state_dict
from oracle.lpips import lpips64, weights_from_state_dict


def _images(n, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, 3, H // 4, W // 4, generator=g, dtype=torch.float64)
    return F.interpolate(x, size=(H, W), mode="bilinear") * 2 - 1


def test_oracle_matches_torchvision_vgg16():
    """The unmatched reference equals LPIPS assembled from torchvision's vgg16().features sliced at 4/9/16/23/30, with
    the features' weights moved into the lpips layout: this pins the layer indices and the key mapping."""
    torchvision = pytest.importorskip("torchvision")
    torch.manual_seed(0)
    feats = torchvision.models.vgg16(weights=None).features.double().eval()
    bounds = (0, 4, 9, 16, 23, 30)
    sd = {"scaling_layer.shift": torch.tensor([-.030, -.088, -.188]).view(1, 3, 1, 1),
          "scaling_layer.scale": torch.tensor([.458, .448, .450]).view(1, 3, 1, 1)}
    for i, m in enumerate(feats):
        if isinstance(m, torch.nn.Conv2d):
            s = next(k for k in range(1, 6) if bounds[k - 1] <= i < bounds[k])
            sd[f"net.slice{s}.{i}.weight"] = m.weight.detach().clone()
            sd[f"net.slice{s}.{i}.bias"] = m.bias.detach().clone()
    g = torch.Generator().manual_seed(1)
    lins = [torch.rand(1, c, 1, 1, generator=g, dtype=torch.float64) for c in (64, 128, 256, 512, 512)]
    for k, w in enumerate(lins):
        sd[f"lins.{k}.model.1.weight"] = w
    in0, in1 = _images(2, 32, 48, 2), _images(2, 32, 48, 3)

    def tv_lpips(a, b):
        shift, scale = sd["scaling_layer.shift"].double(), sd["scaling_layer.scale"].double()
        a, b = (a - shift) / scale, (b - shift) / scale
        out = 0
        for k in range(5):
            a, b = feats[bounds[k]:bounds[k + 1]](a), feats[bounds[k]:bounds[k + 1]](b)
            na = a / (torch.sqrt(torch.sum(a ** 2, dim=1, keepdim=True)) + 1e-10)
            nb = b / (torch.sqrt(torch.sum(b ** 2, dim=1, keepdim=True)) + 1e-10)
            out = out + F.conv2d((na - nb) ** 2, lins[k]).mean(dim=(2, 3)).reshape(-1)
        return out

    with torch.no_grad():
        ref = tv_lpips(in0, in1)
        ours = lpips64(weights_from_state_dict(sd), in0, in1)
    assert float((ours - ref).abs().max() / ref.abs().max()) < 1e-12
    assert float(ref.min()) > 0


@pytest.mark.parametrize("prefix", ["", "loss_computer.lpips_loss_module.", "denoiser.loss_computer.lpips_loss_module."])
@pytest.mark.parametrize("lin_keys", [("lin",), ("lins",), ("lin", "lins")])
def test_load_from_every_layout(prefix, lin_keys):
    from dgs_b200 import checkpoint
    from dgs_b200.lpips import LPIPS, parse_state_dict
    sd = random_lpips_state_dict(0, lin_keys=lin_keys)
    ref = parse_state_dict(random_lpips_state_dict(0))
    flat = {prefix + k: v for k, v in sd.items()}
    layouts = [flat]
    if prefix:  # a checkpoint: the denoiser's keys around the LPIPS weights, in the layout that goes with the prefix
        den = {"shape_model.x.weight": torch.zeros(2)} if prefix.startswith("loss") else {"denoiser.x.weight": torch.zeros(2)}
        layouts += [{"state_dict": {**den, **flat}, "epoch": 1, "global_step": 2} if prefix.startswith("loss") else
                    {"model": {**den, **flat}}]
    for obj in layouts:
        for m in ([LPIPS.from_state_dict(obj)] if obj is flat else []) + ([LPIPS.from_checkpoint(obj)] if prefix else []):
            w = m.weights()
            for key in ("conv_w", "conv_b", "lin"):
                assert all(torch.equal(a, b) for a, b in zip(w[key], ref[key]))
            assert torch.equal(w["shift"], ref["shift"]) and torch.equal(w["scale"], ref["scale"])
            assert len(list(m.parameters())) == 0
    if prefix:
        assert set(checkpoint.lpips_state_dict(layouts[-1])) == set(sd)


def test_checkpoint_helper_leaves_denoiser_extraction_alone():
    from dgs_b200 import checkpoint
    lp = {"loss_computer.lpips_loss_module." + k: v for k, v in random_lpips_state_dict(0).items()}
    obj = {"state_dict": {"shape_model.a": torch.ones(1), **lp}, "epoch": 3, "global_step": 4}
    sd, meta, ignored = checkpoint.extract_denoiser_state_dict(obj)
    assert list(sd) == ["a"] and meta == {"epoch": 3, "global_step": 4} and set(ignored) == set(lp)
    assert checkpoint.lpips_state_dict({"state_dict": {"shape_model.a": torch.ones(1)}}) == {}


def test_bad_state_dicts_raise():
    from dgs_b200.lpips import LPIPS
    sd = random_lpips_state_dict(0)
    for drop in ("net.slice3.12.weight", "net.slice5.28.bias", "scaling_layer.scale"):
        bad = {k: v for k, v in sd.items() if k != drop}
        with pytest.raises(KeyError, match=drop.replace(".", r"\.")):
            LPIPS.from_state_dict(bad)
    bad = {k: v for k, v in sd.items() if not k.endswith("2.model.1.weight")}
    with pytest.raises(KeyError, match="lin2"):
        LPIPS.from_state_dict(bad)
    for key, shape in (("net.slice2.7.weight", (128, 128, 3, 1)), ("net.slice1.0.bias", (32,)),
                       ("lin4.model.1.weight", (1, 256, 1, 1))):
        bad = dict(sd)
        bad[key] = torch.zeros(shape)
        with pytest.raises(ValueError, match="shape"):
            LPIPS.from_state_dict(bad)
    bad = dict(sd)
    bad["lins.1.model.1.weight"] = bad["lins.1.model.1.weight"] + 1
    with pytest.raises(ValueError, match="differ"):
        LPIPS.from_state_dict(bad)
    with pytest.raises(ValueError, match="unexpected"):
        LPIPS.from_state_dict({**sd, "net.slice6.30.weight": torch.zeros(1)})
    with pytest.raises(KeyError, match="no LPIPS weights"):
        LPIPS.from_checkpoint({"state_dict": {"shape_model.a": torch.ones(1)}})


def test_target_gradient_is_refused():
    from dgs_b200.lpips import LPIPS
    m = LPIPS.from_state_dict(random_lpips_state_dict(0))
    x = torch.zeros(1, 3, 16, 16)
    with pytest.raises(ValueError, match="second input"):
        m(x, x.clone().requires_grad_(True))


def test_abi_argument_checks_without_gpu():
    """Invalid arguments return DGS_ERR_INVALID_ARGUMENT before any device work (the pointers are never read)."""
    from test_abi import _ensure_built
    from dgs_b200 import _lib
    _ensure_built()
    L = _lib.lib()
    w = _lib.LpipsWeights()
    fake = ctypes.c_void_p(256)
    ws1 = L.dgs_lpips_workspace_bytes(1, 256, 256)
    assert 100e6 < ws1 < 120e6  # ~109 MB per image at 256^2, mostly the im2col operand
    assert L.dgs_lpips_workspace_bytes(4, 256, 256) >= 4 * ws1 - 4096
    st = L.dgs_lpips_state_bytes(1, 256, 256)
    assert abs(st - (35_389_440 + 31_981_568)) < 16 * 256  # bf16 activations + fp32 tap gradients

    def fwd(n=1, H=32, W=32, ws=fake, nbytes=None, state=None):
        nbytes = L.dgs_lpips_workspace_bytes(1, H, W) if nbytes is None else nbytes
        return L.dgs_lpips_forward(ctypes.byref(w), n, H, W, fake, fake, fake, state, ws, nbytes, None)

    def bwd(n=1, H=32, W=32, state=fake, nbytes=None):
        nbytes = L.dgs_lpips_workspace_bytes(1, H, W) if nbytes is None else nbytes
        return L.dgs_lpips_backward(ctypes.byref(w), n, H, W, state, fake, fake, fake, nbytes, None)

    for H, W in ((24, 32), (32, 40), (8, 32), (32, 0), (0, 16)):
        assert fwd(H=H, W=W, nbytes=1 << 30) == 1 and b"multiples of 16" in L.dgs_last_error()
        assert bwd(H=H, W=W, nbytes=1 << 30) == 1 and b"multiples of 16" in L.dgs_last_error()
    for n in (0, -3):
        assert fwd(n=n) == 1 and b"n > 0" in L.dgs_last_error()
        assert bwd(n=n) == 1 and b"n > 0" in L.dgs_last_error()
    small = L.dgs_lpips_workspace_bytes(1, 32, 32) - 1
    assert fwd(nbytes=small) == 1 and b"workspace too small" in L.dgs_last_error()
    assert fwd(ws=None) == 1 and b"workspace too small" in L.dgs_last_error()
    assert bwd(nbytes=small) == 1 and b"workspace too small" in L.dgs_last_error()
    assert bwd(state=None) == 1 and b"state is NULL" in L.dgs_last_error()
    assert L.dgs_lpips_forward(None, 1, 32, 32, fake, fake, fake, None, fake, 1 << 30, None) == 1


def test_inputs_are_read_as_fp32():
    """The kernels read fp32 only: every floating dtype is converted before the C ABI sees a pointer, others raise."""
    from dgs_b200.lpips import prepare_inputs
    x = _images(2, 16, 32, 4)
    for dt in (torch.float16, torch.bfloat16, torch.float64, torch.float32):
        a, b = prepare_inputs(x.to(dt), x.to(dt).flip(0))
        assert a.dtype == b.dtype == torch.float32 and a.is_contiguous() and b.is_contiguous()
        assert torch.equal(a, x.to(dt).float()) and torch.equal(b, x.to(dt).flip(0).float())
    a, _ = prepare_inputs(x.float().permute(0, 1, 3, 2).contiguous().permute(0, 1, 3, 2), x.float())
    assert a.is_contiguous()
    with pytest.raises(TypeError, match="floating-point"):
        prepare_inputs((x * 100).to(torch.uint8), x.float())
    with pytest.raises(ValueError, match="n, 3, H, W"):
        prepare_inputs(x[:, :2].float(), x[:, :2].float())


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float64])
def test_packed_weights_stay_fp32_after_module_conversion(dtype):
    """module.half() / .to(bf16) / .double() converts the buffers; the C struct still receives bf16 conv matrices and
    fp32 biases, lin weights, shift and scale (of the converted values)."""
    from dgs_b200.lpips import LPIPS, pack_weights
    m = LPIPS.from_state_dict(random_lpips_state_dict(0)).to(dtype)
    _, t = pack_weights(m.weights(), "cpu")
    assert all(v.dtype == torch.bfloat16 for v in t["conv_w"] + t["conv_wt"])
    assert all(v.dtype == torch.float32 for v in t["conv_b"] + t["lin"] + [t["shift"], t["scale"]])
    assert torch.equal(t["conv_b"][5], m.conv5_bias.float()) and torch.equal(t["lin"][4], m.lin4_weight.float())
    assert torch.equal(t["scale"], m.scale.float())


def test_weights_round_trip_through_a_system_checkpoint(tmp_path):
    """lpips_state_dict gives the weights back in the lpips layout, so a checkpoint written here carries the
    "loss_computer.lpips_loss_module.*" keys the reference's checkpoints carry and LPIPS.from_checkpoint reads it."""
    from dgs_b200 import checkpoint
    from dgs_b200.lpips import LPIPS
    sd = random_lpips_state_dict(3)
    m = LPIPS.from_state_dict(sd)
    out = m.lpips_state_dict()
    assert set(out) == set(sd) and all(torch.equal(out[k], sd[k].float()) for k in sd)
    path = checkpoint.save_system_checkpoint(torch.nn.Linear(2, 2), str(tmp_path / "last.ckpt"), epoch=1, global_step=9,
                                             extra_state_dict=m.lpips_state_dict("loss_computer.lpips_loss_module."))
    m2 = LPIPS.from_checkpoint(path)
    for a, b in zip(m.buffers(), m2.buffers()):
        assert torch.equal(a, b)
    den, meta, _ = checkpoint.extract_denoiser_state_dict(torch.load(path, weights_only=False))
    assert set(den) == {"weight", "bias"} and meta == {"epoch": 1, "global_step": 9}
