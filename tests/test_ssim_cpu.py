"""SSIM and the evaluation metrics without a GPU: the fp64 reference (oracle/ssim.py) pinned to scipy's filter (what
skimage's structural_similarity runs) and to autograd, the closed-form gradient the kernels implement, the argument
checks of the C ABI (dgs_ssim_*) and of the Python modules, and the file handling of compute_metrics."""
import ctypes
import json

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.ssim import SAMPLE_COV, ssim64, ssim_grad64, window


def smooth_pair(n, H, W, seed, contrast=0.02):
    """A smooth, low-contrast target in [0.4, 0.6] and a blurred perturbation of it of amplitude ~`contrast` (at the
    default, sigma^2 is of the order of C2, where skimage's sample covariance shows)."""
    g = torch.Generator().manual_seed(seed)
    up = lambda t: F.interpolate(t, size=(H, W), mode="bilinear", align_corners=False)  # noqa: E731
    target = 0.4 + 0.2 * up(torch.rand(n, 3, max(2, H // 6), max(2, W // 6), generator=g, dtype=torch.float64))
    pert = up(torch.randn(n, 3, max(2, H // 4), max(2, W // 4), generator=g, dtype=torch.float64))
    return (target + contrast * pert).clamp(0, 1), target


def _scipy_replica(x, y, k):
    """skimage structural_similarity(gaussian_weights=True, win_size=11, channel_axis=0, data_range=1) in fp64:
    scipy.ndimage.gaussian_filter(sigma=1.5, truncate=3.5, mode="reflect"), then a 5-pixel crop."""
    from scipy import ndimage
    out = []
    for a, b in zip(x.numpy(), y.numpy()):
        per = []
        for ca, cb in zip(a, b):
            f = lambda t: ndimage.gaussian_filter(t, sigma=1.5, truncate=3.5, mode="reflect")  # noqa: E731
            ux, uy, uxx, uyy, uxy = f(ca), f(cb), f(ca * ca), f(cb * cb), f(ca * cb)
            vx, vy, vxy = k * (uxx - ux * ux), k * (uyy - uy * uy), k * (uxy - ux * uy)
            S = (2 * ux * uy + 1e-4) * (2 * vxy + 9e-4) / ((ux ** 2 + uy ** 2 + 1e-4) * (vx + vy + 9e-4))
            per.append(S[5:-5, 5:-5].mean())
        out.append(np.mean(per))
    return torch.tensor(out)


@pytest.mark.parametrize("HW", [(11, 11), (37, 61), (64, 96)], ids=lambda s: "x".join(map(str, s)))
def test_metric_variant_equals_scipy_reflect_filter(HW):
    """The reflect-padded filter is only read inside the valid window after the crop: the valid-window mean with
    k = 121/120 is skimage's value (11 x 11 has one valid pixel)."""
    pytest.importorskip("scipy")
    x, y = smooth_pair(2, *HW, seed=0)
    ref = _scipy_replica(x, y, SAMPLE_COV)
    ours = ssim64(x, y, k=SAMPLE_COV)
    assert float((ours - ref).abs().max()) < 1e-12
    assert float((ours - ssim64(x, y, k=1.0)).abs().max()) > 1e-5  # and the sample covariance is visible


def test_window_matches_scipy_and_pytorch_msssim():
    from scipy import ndimage
    g = window()
    impulse = np.zeros(21)
    impulse[10] = 1.0
    sc = ndimage.gaussian_filter1d(impulse, sigma=1.5, truncate=3.5, mode="constant")[5:16]
    assert np.abs(sc - g.numpy()).max() < 1e-15 and abs(float(g.sum()) - 1) < 1e-15
    # pytorch_msssim's _fspecial_gauss_1d(11, 1.5): fp32 arithmetic throughout
    c = torch.arange(11, dtype=torch.float32) - 5
    g32 = torch.exp(-(c ** 2) / (2 * 1.5 ** 2))
    g32 = g32 / g32.sum()
    assert float((g32.double() - g).abs().max()) < 2 * 2.0 ** -24


def test_oracle_gradcheck():
    x, y = smooth_pair(2, 13, 17, seed=1, contrast=0.3)
    x.requires_grad_(True)
    for k in (1.0, SAMPLE_COV):
        assert torch.autograd.gradcheck(lambda a: ssim64(a, y, k=k), (x,), eps=1e-6, atol=1e-9)


@pytest.mark.parametrize("k", [1.0, SAMPLE_COV], ids=["msssim", "skimage"])
@pytest.mark.parametrize("HW", [(11, 11), (13, 17), (37, 61)], ids=lambda s: "x".join(map(str, s)))
def test_closed_form_gradient_equals_autograd(HW, k):
    """alpha / beta / gamma and the transposed stencil, as the backward kernel forms them, are the exact gradient."""
    for pair in (smooth_pair(3, *HW, seed=2), smooth_pair(3, *HW, seed=3, contrast=0.5)):
        x, y = pair
        dout = torch.tensor([0.7, -1.3, 2.0], dtype=torch.float64)
        xg = x.clone().requires_grad_(True)
        (ssim64(xg, y, k=k) * dout).sum().backward()
        cf = ssim_grad64(x, y, dout, k=k)
        assert float((cf - xg.grad).norm() / xg.grad.norm()) < 1e-12


def test_abi_argument_checks_without_gpu():
    """Invalid arguments return DGS_ERR_INVALID_ARGUMENT before any device work (the pointers are never read)."""
    from test_abi import _ensure_built
    from dgs_b200 import _lib
    _ensure_built()
    L = _lib.lib()
    fake = ctypes.c_void_p(256)
    assert L.dgs_ssim_state_bytes(2, 64, 96) == 256 * ((2 * 9 * 54 * 86 * 4 + 255) // 256)  # 3 maps x 3 channels, fp32
    assert L.dgs_ssim_workspace_bytes(5, 256, 256) == 256 * ((5 * 8 * 8 * 2 * 4 + 255) // 256)
    assert L.dgs_ssim_workspace_bytes(1, 10, 64) == 0 and L.dgs_ssim_state_bytes(0, 64, 64) == 0

    def fwd(n=1, H=32, W=32, x=fake, y=fake, dr=1.0, ssim=fake, ws=fake, nbytes=None):
        nbytes = L.dgs_ssim_workspace_bytes(1, 32, 32) if nbytes is None else nbytes
        return L.dgs_ssim_forward(n, H, W, x, y, dr, 0, ssim, None, None, ws, nbytes, None)

    def bwd(n=1, H=32, W=32, x=fake, y=fake, state=fake, dout=fake):
        return L.dgs_ssim_backward(n, H, W, x, y, state, dout, fake, None)

    for n in (0, -2):
        assert fwd(n=n) == 1 and b"n > 0" in L.dgs_last_error()
        assert bwd(n=n) == 1 and b"n > 0" in L.dgs_last_error()
    for H, W in ((10, 32), (32, 10), (0, 0)):
        assert fwd(H=H, W=W) == 1 and b"at least 11" in L.dgs_last_error()
        assert bwd(H=H, W=W) == 1 and b"at least 11" in L.dgs_last_error()
    for kw in (dict(x=None), dict(y=None), dict(ssim=None)):
        assert fwd(**kw) == 1 and b"must not be NULL" in L.dgs_last_error()
    for dr in (0.0, -1.0):
        assert fwd(dr=dr) == 1 and b"data_range" in L.dgs_last_error()
    assert fwd(nbytes=L.dgs_ssim_workspace_bytes(1, 32, 32) - 1) == 1 and b"workspace too small" in L.dgs_last_error()
    assert fwd(ws=None) == 1 and b"workspace too small" in L.dgs_last_error()
    one = L.dgs_ssim_workspace_bytes(1, 256, 256)
    assert fwd(n=2, H=256, W=256, nbytes=one) == 1 and b"workspace too small" in L.dgs_last_error()
    assert bwd(state=None) == 1 and b"state is NULL" in L.dgs_last_error()
    assert bwd(dout=None) == 1 and b"must not be NULL" in L.dgs_last_error()


def test_unsupported_constructor_values_raise():
    from dgs_b200.ssim import SSIM, SsimLoss
    SSIM()
    SSIM(data_range=255.0, size_average=True)
    SsimLoss(data_range=2.0)
    for kw in (dict(win_size=7), dict(win_sigma=1.0), dict(channel=1), dict(spatial_dims=3), dict(K=(0.01, 0.04)),
               dict(nonnegative_ssim=True), dict(data_range=0.0), dict(data_range=-1.0)):
        with pytest.raises(ValueError):
            SSIM(**kw)


def test_bad_inputs_are_rejected():
    from dgs_b200 import _lib
    from dgs_b200.metrics import MetricComputer
    from dgs_b200.ssim import SSIM, prepare_inputs, ssim_psnr
    x = torch.rand(2, 3, 16, 16)
    with pytest.raises(TypeError, match="floating-point"):
        SSIM()((x * 255).to(torch.uint8), x)
    with pytest.raises(ValueError, match="at least 11"):
        SSIM()(x[..., :10], x[..., :10])
    with pytest.raises(ValueError, match="at least 11"):
        ssim_psnr(x[:, :, :10], x[:, :, :10])
    with pytest.raises(ValueError, match="second input"):
        SSIM()(x, x.clone().requires_grad_(True))
    with pytest.raises(ValueError, match="n, 3, H, W"):
        SSIM()(x[:, :2], x[:, :2])
    with pytest.raises(_lib.DgsError, match="no CPU fallback"):
        prepare_inputs(x, x)
    with pytest.raises(_lib.DgsError, match="no CPU fallback"):
        MetricComputer(torch.nn.Identity())(x, x)
    with pytest.raises(ValueError, match="at least 11"):  # PSNR comes out of the SSIM pass, so it shares its limits
        MetricComputer(torch.nn.Identity()).compute_psnr(x[..., :8, :8], x[..., :8, :8])
    with pytest.raises(TypeError, match="floating-point"):
        MetricComputer(torch.nn.Identity()).compute_psnr((x * 255).to(torch.uint8), x)


class _StandIn(torch.nn.Module):
    """Records each call's chunk and returns per-image values computed from the images (not the real metrics)."""

    def __init__(self):
        super().__init__()
        self.calls = []

    def forward(self, target, rendering):
        self.calls.append((tuple(target.shape), tuple(rendering.shape)))
        t = target.reshape(-1, *target.shape[-3:])
        r = rendering.reshape(-1, *rendering.shape[-3:])
        return t.mean(dim=(1, 2, 3)), r.mean(dim=(1, 2, 3)), (t - r).abs().mean(dim=(1, 2, 3))


def test_compute_metrics_file_handling(tmp_path, capsys):
    from dgs_b200.metrics import compute_metrics
    g = torch.Generator().manual_seed(0)
    scenes = []
    for i in range(5):
        pkg = {"render_images": torch.rand(4, 3, 16, 24, generator=g), "image": torch.rand(4, 3, 16, 24, generator=g)}
        torch.save(pkg, tmp_path / f"scene_{i:03d}.pt")
        scenes.append(pkg)
    (tmp_path / "notes.txt").write_text("not a result")
    torch.save({"unused": 1}, tmp_path / "scene_x.pth")
    results = []
    for chunk in (2, 8):
        m = _StandIn()
        res = compute_metrics(str(tmp_path), chunk=chunk, metric_computer=m, device="cpu")
        assert [c[0][0] for c in m.calls] == ([2, 2, 1] if chunk == 2 else [5])
        assert all(c[0] == (c[0][0], 4, 3, 16, 24) for c in m.calls)
        out = capsys.readouterr().out
        assert out.startswith("psnr: ") and ", ssim: " in out and ", lpips: " in out
        text = (tmp_path / "eval_result.json").read_text()
        assert json.loads(text) == res and list(res) == ["psnr", "ssim", "lpips"]
        assert text == json.dumps(res, indent=4)
        results.append(res)
    r = torch.stack([s["render_images"] for s in scenes])
    t = torch.stack([s["image"] for s in scenes])
    # the reference passes (render_images, image) as forward(target, rendering)
    assert abs(results[1]["psnr"] - float(r.mean(dim=(2, 3, 4)).mean())) < 1e-6
    assert abs(results[1]["ssim"] - float(t.mean(dim=(2, 3, 4)).mean())) < 1e-6
    assert all(abs(results[0][k] - results[1][k]) < 1e-6 for k in results[0])
    with pytest.raises(ValueError, match="lpips_checkpoint"):
        compute_metrics(str(tmp_path))
    (tmp_path / "empty").mkdir()
    with pytest.raises(FileNotFoundError, match="no .pt result files"):
        compute_metrics(str(tmp_path / "empty"), metric_computer=_StandIn())


def test_cli_requires_the_lpips_checkpoint():
    from dgs_b200.metrics import main
    with pytest.raises(SystemExit):
        main(["--path", "somewhere"])
