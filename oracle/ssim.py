"""fp64 SSIM and PSNR references, plain torch ops, autograd-capable.

    S = (2 mx my + C1)(2 sxy + C2) / ((mx^2 + my^2 + C1)(sx^2 + sy^2 + C2)),  C1 = (0.01 R)^2, C2 = (0.03 R)^2

with the moments of an 11-tap Gaussian window (sigma 1.5) taken by a VALID separable convolution (H pass, then W pass)
and sx^2 = k (E[xx] - mx^2), sxy = k (E[xy] - mx my); the per-image value is the mean of S over the valid pixels and the
3 channels.  k = 1 is pytorch_msssim.SSIM (the training loss), k = SAMPLE_COV = 121/120 is skimage's
structural_similarity(gaussian_weights=True, win_size=11) (the evaluation metric).

`ssim_grad64` is the closed-form input gradient the kernels implement (coefficient maps alpha / beta / gamma and the
transposed stencil); `ssim_torch32` is pytorch_msssim's own fp32 arithmetic on F.conv2d.  `defects` plants a named defect
(DEFECTS) for the power tests.
"""
import torch
import torch.nn.functional as F

WIN, SIGMA = 11, 1.5
SAMPLE_COV = 121.0 / 120.0
DEFECTS = ("population_cov",   # k = 1 where the sample covariance k = 121/120 was asked for
           "c1_c2_swapped",    # C1 and C2 exchanged
           "same_padding",     # zero-padded "same" filtering (H x W outputs) instead of the valid window
           "win9",             # a 9-tap window (sigma 1.5)
           "no_2x_beta",       # gradient without the 2 x W^T beta term
           "no_y_gamma",       # gradient without the y W^T gamma term
           "bwd_shift",        # backward stencil shifted by one pixel in x
           "psnr_unclamped",   # PSNR of the images without clamping to [0, 1]
           "psnr_frame_twice")  # PSNR counting the 5-pixel border frame twice


def window(size=WIN, sigma=SIGMA, dtype=torch.float64):
    """Normalised 1-D Gaussian taps g[i] ~ exp(-(i - size//2)^2 / (2 sigma^2)) (pytorch_msssim's _fspecial_gauss_1d)."""
    c = torch.arange(size, dtype=dtype) - size // 2
    g = torch.exp(-(c ** 2) / (2 * sigma ** 2))
    return g / g.sum()


def filter_valid(x, g, padding=0):
    """Separable per-channel correlation of [n, C, H, W] with taps g: H pass, then W pass (padding=0: valid)."""
    C = x.shape[1]
    k = g.numel()
    x = F.conv2d(x, g.view(1, 1, k, 1).expand(C, 1, k, 1).to(x), groups=C, padding=(padding, 0))
    return F.conv2d(x, g.view(1, 1, 1, k).expand(C, 1, 1, k).to(x), groups=C, padding=(0, padding))


def _constants(data_range, defects):
    C1, C2 = (0.01 * data_range) ** 2, (0.03 * data_range) ** 2
    return (C2, C1) if "c1_c2_swapped" in defects else (C1, C2)


def _taps(defects, dtype=torch.float64):
    return window(9 if "win9" in defects else WIN, SIGMA, dtype)


def moments(x, y, defects=()):
    g = _taps(defects, x.dtype)
    pad = g.numel() // 2 if "same_padding" in defects else 0
    return [filter_valid(t, g, pad) for t in (x, y, x * x, y * y, x * y)]


def ssim_map(x, y, k=1.0, data_range=1.0, defects=()):
    """-> S [n, 3, H-10, W-10] (fp64 for fp64 inputs)."""
    if "population_cov" in defects:
        k = 1.0
    C1, C2 = _constants(data_range, defects)
    mx, my, exx, eyy, exy = moments(x, y, defects)
    vx, vy, vxy = k * (exx - mx * mx), k * (eyy - my * my), k * (exy - mx * my)
    return (2 * mx * my + C1) * (2 * vxy + C2) / ((mx * mx + my * my + C1) * (vx + vy + C2))


def ssim64(x, y, k=1.0, data_range=1.0, defects=()):
    """-> [n] per-image SSIM in fp64; differentiable in both inputs."""
    return ssim_map(x.double(), y.double(), k, data_range, defects).mean(dim=(1, 2, 3))


def ssim_grad64(x, y, dout, k=1.0, data_range=1.0, defects=()):
    """Closed-form d (sum_i dout[i] ssim[i]) / d x in fp64, as the kernels form it:
        alpha = S (2my/A1 - 2mx/B1 + 2k mx/B2 - 2k my/A2),  beta = -k S/B2,  gamma = 2k S/A2,
        dx = dout / (3 Hv Wv) [W^T alpha + 2 x W^T beta + y W^T gamma]
    (alpha and gamma formed as the kernels form them, without dividing by A1 or A2)
    with W^T the transposed valid stencil (a full correlation with the flipped taps)."""
    x, y, dout = x.double(), y.double(), torch.as_tensor(dout).double().to(x.device)
    C1, C2 = _constants(data_range, defects)
    mx, my, exx, eyy, exy = moments(x, y)
    vx, vy, vxy = k * (exx - mx * mx), k * (eyy - my * my), k * (exy - mx * my)
    A1, A2, B1, B2 = 2 * mx * my + C1, 2 * vxy + C2, mx * mx + my * my + C1, vx + vy + C2
    l, cs = A1 / B1, A2 / B2
    S = l * cs
    # S/A1 = cs/B1 and S/A2 = l/B2 substituted, so nothing divides by A1 or A2 (either may be 0)
    alpha = 2 * (my * cs - mx * S) / B1 + 2 * k * (mx * S - my * l) / B2
    beta, gamma = -k * S / B2, 2 * k * l / B2
    g = window(WIN, SIGMA, torch.float64).flip(0)
    n, c, hv, wv = S.shape

    def wt(m):
        out = filter_valid(m, g, WIN - 1)  # full correlation with the flipped taps: [n, 3, H, W]
        if "bwd_shift" in defects:
            out = torch.roll(out, 1, dims=3)
        return out
    dx = wt(alpha)
    if "no_2x_beta" not in defects:
        dx = dx + 2 * x * wt(beta)
    if "no_y_gamma" not in defects:
        dx = dx + y * wt(gamma)
    return dx * (dout / (c * hv * wv)).view(-1, 1, 1, 1)


def psnr64(x, y, defects=()):
    """-> [n] -10 log10(mean over c, h, w of (clamp(x) - clamp(y))^2) in fp64 (+inf for identical images)."""
    x, y = x.double(), y.double()
    if "psnr_unclamped" not in defects:
        x, y = x.clamp(0, 1), y.clamp(0, 1)
    d2 = (x - y) ** 2
    sse = d2.sum(dim=(1, 2, 3))
    if "psnr_frame_twice" in defects:
        sse = sse + d2.sum(dim=(1, 2, 3)) - d2[..., 5:-5, 5:-5].sum(dim=(1, 2, 3))
    return -10 * torch.log10(sse / d2[0].numel())


def ssim_torch32(x, y, data_range=1.0, k=1.0):
    """pytorch_msssim.SSIM(win_size=11, win_sigma=1.5, size_average=False, channel=3)'s arithmetic in fp32 on F.conv2d
    (groups=3): the numbers the reference's training loss computes (k = 121/120 gives the metric variant)."""
    x, y = x.float(), y.float()
    g = window(WIN, SIGMA, torch.float32).to(x.device)
    C1, C2 = (0.01 * data_range) ** 2, (0.03 * data_range) ** 2
    mu1, mu2 = filter_valid(x, g), filter_valid(y, g)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    s1 = k * (filter_valid(x * x, g) - mu1_sq)
    s2 = k * (filter_valid(y * y, g) - mu2_sq)
    s12 = k * (filter_valid(x * y, g) - mu1_mu2)
    cs = (2 * s12 + C2) / (s1 + s2 + C2)
    return (((2 * mu1_mu2 + C1) / (mu1_sq + mu2_sq + C1)) * cs).flatten(2).mean(-1).mean(1)


def ssim_scipy32(x, y, data_range=1.0):
    """skimage structural_similarity(gaussian_weights=True, win_size=11, channel_axis=0, data_range) as skimage computes
    it: float32 arrays through scipy.ndimage.gaussian_filter(sigma=1.5, truncate=3.5, mode="reflect"), sample covariance,
    a 5-pixel crop and the mean in float64.  x, y: CPU [n, 3, H, W] -> [n] float64 numpy."""
    import numpy as np
    from scipy import ndimage
    C1, C2 = (0.01 * data_range) ** 2, (0.03 * data_range) ** 2
    out = []
    for a, b in zip(x.detach().cpu().numpy().astype(np.float32), y.detach().cpu().numpy().astype(np.float32)):
        per = []
        for ca, cb in zip(a, b):
            f = lambda t: ndimage.gaussian_filter(t, sigma=SIGMA, truncate=3.5, mode="reflect")  # noqa: E731
            ux, uy, uxx, uyy, uxy = f(ca), f(cb), f(ca * ca), f(cb * cb), f(ca * cb)
            cov = np.float32(SAMPLE_COV)
            vx, vy, vxy = cov * (uxx - ux * ux), cov * (uyy - uy * uy), cov * (uxy - ux * uy)
            A1, A2, B1, B2 = 2 * ux * uy + C1, 2 * vxy + C2, ux ** 2 + uy ** 2 + C1, vx + vy + C2
            S = (A1 * A2) / (B1 * B2)
            per.append(S[5:-5, 5:-5].mean(dtype=np.float64))
        out.append(float(np.mean(per)))
    return np.array(out)

