"""SSIM on libdgs_b200.so (dgs_ssim_forward / dgs_ssim_backward): a drop-in for `pytorch_msssim.SSIM` with the arguments
the reference passes, and the reference's `SsimLoss` (diffusionGS/utils/losses.py:216-234) built on it.

    loss = SsimLoss()(rendering, target)       # [n, 3, H, W] -> [n] = 1 - SSIM, differentiable in the rendering
    LossComputer(ssim_module=SsimLoss())       # the ssim term of the training loss

The window is the 11-tap Gaussian with sigma 1.5, filtered over the valid (H-10) x (W-10) pixels; H and W must be at
least 11.  The gradient is taken w.r.t. the first input only.  `ssim_psnr` is the evaluation form (skimage's sample
covariance, and PSNR from the same pass) that `dgs_b200.metrics` uses.
"""

import torch
import torch.nn as nn

from . import _lib
from ._lib import check, stream

WIN_SIZE, WIN_SIGMA, K_DEFAULT = 11, 1.5, (0.01, 0.03)


def prepare_inputs(x, y):
    """Checks two [n, 3, H, W] floating-point images (H, W >= 11) on one CUDA device and returns them as contiguous fp32,
    the only element type the kernels read (fp16 / bf16 / fp64 images are converted; integer images raise)."""
    if x.dim() != 4 or x.shape[1] != 3 or tuple(y.shape) != tuple(x.shape):
        raise ValueError(f"SSIM: expected two [n, 3, H, W] inputs, got {tuple(x.shape)} and {tuple(y.shape)}")
    if not (x.is_floating_point() and y.is_floating_point()):
        raise TypeError(f"SSIM: expected floating-point images, got {x.dtype} and {y.dtype}")
    if x.shape[2] < WIN_SIZE or x.shape[3] < WIN_SIZE:
        raise ValueError(f"SSIM: H and W must be at least {WIN_SIZE}, the window size (got {x.shape[2]}x{x.shape[3]})")
    if x.shape[0] == 0:
        raise ValueError("SSIM: empty batch")
    if not x.is_cuda or y.device != x.device:
        raise _lib.DgsError("SSIM needs both inputs on the same CUDA device (no CPU fallback)")
    return x.to(torch.float32).contiguous(), y.to(torch.float32).contiguous()


def _forward(x, y, data_range, sample_covariance, want_psnr, train):
    """fp32 contiguous CUDA inputs -> (ssim [n], psnr [n] or None, state or None)"""
    n, _, H, W = x.shape
    dev = x.device
    L = _lib.lib()
    out = torch.empty(n, dtype=torch.float32, device=dev)
    psnr = torch.empty(n, dtype=torch.float32, device=dev) if want_psnr else None
    state = torch.empty(L.dgs_ssim_state_bytes(n, H, W), dtype=torch.uint8, device=dev) if train else None
    ws = torch.empty(L.dgs_ssim_workspace_bytes(n, H, W), dtype=torch.uint8, device=dev)
    check(L.dgs_ssim_forward(n, H, W, x.data_ptr(), y.data_ptr(), float(data_range), int(sample_covariance),
                             out.data_ptr(), psnr.data_ptr() if want_psnr else None,
                             state.data_ptr() if train else None, ws.data_ptr(), ws.numel(), stream(dev)))
    return out, psnr, state


class _SsimFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, y, data_range):
        in_dtype = x.dtype
        x, y = prepare_inputs(x, y)
        train = ctx.needs_input_grad[0]
        out, _, state = _forward(x, y, data_range, False, False, train)
        if train:
            ctx.saved = (x, y, state, in_dtype)
        return out

    @staticmethod
    def backward(ctx, dout):
        x, y, state, in_dtype = ctx.saved
        n, _, H, W = x.shape
        d = dout.reshape(n).to(torch.float32).contiguous()
        d_x = torch.empty_like(x)
        check(_lib.lib().dgs_ssim_backward(n, H, W, x.data_ptr(), y.data_ptr(), state.data_ptr(), d.data_ptr(),
                                           d_x.data_ptr(), stream(x.device)))
        ctx.saved = None
        return d_x.to(in_dtype), None, None


@torch.no_grad()
def ssim_psnr(x, y, data_range=1.0, sample_covariance=True, psnr=True):
    """-> (ssim [n], psnr [n] or None), fp32, from one kernel pass.  sample_covariance=True is skimage's
    structural_similarity(gaussian_weights=True, win_size=11, channel_axis=0, data_range); False is pytorch_msssim's SSIM.
    PSNR is -10 log10 of the mean squared difference of the images clamped to [0, 1] (+inf for identical images)."""
    if not data_range > 0:
        raise ValueError(f"SSIM: data_range must be > 0, got {data_range}")
    x, y = prepare_inputs(x, y)
    s, p, _ = _forward(x, y, data_range, sample_covariance, psnr, False)
    return s, p


class SSIM(nn.Module):
    """`pytorch_msssim.SSIM` for the configuration the reference uses: forward(X, Y) -> [n] fp32 (the mean with
    size_average=True), differentiable in X.  Every other argument value raises ValueError; data_range may be any value
    > 0.  Images of any floating dtype are read as fp32 and the gradient comes back in X's dtype."""

    def __init__(self, data_range=1.0, size_average=False, win_size=11, win_sigma=1.5, channel=3, spatial_dims=2,
                 K=(0.01, 0.03), nonnegative_ssim=False):
        super().__init__()
        if not data_range > 0:
            raise ValueError(f"SSIM: data_range must be > 0, got {data_range}")
        for name, got, want in (("win_size", win_size, WIN_SIZE), ("win_sigma", win_sigma, WIN_SIGMA),
                                ("channel", channel, 3), ("spatial_dims", spatial_dims, 2),
                                ("K", tuple(K), K_DEFAULT), ("nonnegative_ssim", nonnegative_ssim, False)):
            if got != want:
                raise ValueError(f"SSIM: {name}={got!r} is not supported (only {want!r})")
        self.data_range = float(data_range)
        self.size_average = bool(size_average)

    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(self, X, Y):
        if Y.requires_grad:
            raise ValueError("SSIM: the gradient w.r.t. the second input (the target) is not computed; pass it detached")
        out = _SsimFunction.apply(X, Y, self.data_range)
        return out.mean() if self.size_average else out


class SsimLoss(nn.Module):
    """The reference's SsimLoss: 1 - SSIM(win_size=11, win_sigma=1.5, data_range, size_average=False, channel=3), [n]."""

    def __init__(self, data_range=1.0):
        super().__init__()
        self.data_range = data_range
        self.ssim_module = SSIM(data_range=data_range, size_average=False, win_size=11, win_sigma=1.5, channel=3)

    def forward(self, x, y):
        return 1 - self.ssim_module(x, y)
