"""fp64 LPIPS-VGG reference (lpips 0.1, net="vgg", eval mode), plain torch.nn.functional ops, autograd-capable.

    d[n] = sum_k mean_hw sum_c lin_k[c] (f0 - f1)^2,   f = a / (sqrt(sum_c a^2) + 1e-10)

with a the relu1_2 .. relu5_3 activations of torchvision VGG16 features[0:30] applied to (x - shift) / scale.

`weights_from_state_dict` reads the lpips-layout state dict (net.slice{s}.{i}.*, lin{k} / lins.{k}, scaling_layer.*).
matched=True rounds where the kernels (dgs_lpips_*) round: bf16 conv weights, bf16 input after the ScalingLayer, bf16
post-ReLU activations, and dz = d/dz (pre-ReLU) rounded to bf16 in the backward.  The max-pool sends its gradient to the
first maximum of each window in row-major order, in both modes (torch's max_pool2d rule; ties are real in bf16).
`defects` plants a named defect (DEFECTS) for the power tests.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

CONV_INDEX = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)
SLICE = (1, 1, 2, 2, 3, 3, 3, 4, 4, 4, 5, 5, 5)
TAP_AFTER = (1, 3, 6, 9, 12)   # conv (0..12) after whose ReLU each of the 5 taps is taken
POOL_BEFORE = (2, 4, 7, 10)    # convs preceded by a 2x2 / 2 max-pool
DEFECTS = ("eps_1e-6",         # normalisation eps 1e-6 instead of 1e-10
           "lin_swapped",      # lin weights of taps 3 and 4 (both 512 channels) swapped
           "no_scaling",       # ScalingLayer skipped
           "pool_tie_last",    # max-pool gradient to the LAST maximum of a tied window
           "dgrad_one_axis",   # input gradient of every conv through a kernel flipped in x only
           "tap_pre_relu")     # tap 2 (relu3_3) taken before its ReLU


def weights_from_state_dict(sd, dtype=torch.float64):
    g = lambda k: torch.as_tensor(sd[k]).detach().to(dtype)  # noqa: E731
    lin = []
    for k in range(5):
        key = f"lin{k}.model.1.weight" if f"lin{k}.model.1.weight" in sd else f"lins.{k}.model.1.weight"
        lin.append(g(key).reshape(-1))
    return dict(conv_w=[g(f"net.slice{SLICE[l]}.{CONV_INDEX[l]}.weight") for l in range(13)],
                conv_b=[g(f"net.slice{SLICE[l]}.{CONV_INDEX[l]}.bias") for l in range(13)],
                lin=lin, shift=g("scaling_layer.shift").reshape(3), scale=g("scaling_layer.scale").reshape(3))


def _bf16(x):
    """Round to bf16 in the forward, identity in the backward."""
    return x + (x.to(torch.bfloat16).to(x.dtype) - x).detach()


class _RoundGrad(torch.autograd.Function):
    """Identity in the forward; the incoming gradient is rounded to bf16 (the kernels' bf16 dz operand)."""
    @staticmethod
    def forward(ctx, x):
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return g.to(torch.bfloat16).to(g.dtype)


class _ConvOneAxis(torch.autograd.Function):
    """Defect: a 3x3 conv whose input gradient uses the kernel flipped in x only (the correct one flips both axes)."""
    @staticmethod
    def forward(ctx, x, w, b):
        ctx.save_for_backward(w)
        return F.conv2d(x, w, b, padding=1)

    @staticmethod
    def backward(ctx, g):
        (w,) = ctx.saved_tensors
        return F.conv2d(g, w.transpose(0, 1).flip(3), padding=1), None, None


def maxpool(x, last=False):
    """2x2 / 2 max-pool; the gradient goes to the first (last=True: the last) maximum in row-major window order."""
    n, c, h, w = x.shape
    v = x.reshape(n, c, h // 2, 2, w // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(n, c, h // 2, w // 2, 4)
    idx = 3 - v.flip(-1).argmax(-1) if last else v.argmax(-1)  # argmax returns the first maximal index
    return v.gather(-1, idx.unsqueeze(-1)).squeeze(-1)


def features(wts, x, matched=False, defects=()):
    """-> the 5 tap activations of one input [n, 3, H, W] in [-1, 1]."""
    if "no_scaling" not in defects:
        x = (x - wts["shift"].view(1, 3, 1, 1)) / wts["scale"].view(1, 3, 1, 1)
    if matched:
        x = _bf16(x)
    taps = []
    for l in range(13):
        if l in POOL_BEFORE:
            x = maxpool(x, last="pool_tie_last" in defects)
        w = wts["conv_w"][l]
        if matched:
            w = w.to(torch.bfloat16).to(w.dtype)
        if "dgrad_one_axis" in defects:
            z = _ConvOneAxis.apply(x, w, wts["conv_b"][l])
        else:
            z = F.conv2d(x, w, wts["conv_b"][l], padding=1)
        if matched:
            z = _RoundGrad.apply(z)
        a = F.relu(z)
        if matched:
            a = _bf16(a)
        if l in TAP_AFTER:
            taps.append(z if ("tap_pre_relu" in defects and l == TAP_AFTER[2]) else a)
        x = a
    return taps


def lpips64(wts, in0, in1, matched=False, defects=()):
    """-> [n] LPIPS distances in the dtype of `wts` (weights_from_state_dict)."""
    dt = wts["conv_w"][0].dtype
    in0, in1 = in0.to(dt), in1.to(dt)
    eps = 1e-6 if "eps_1e-6" in defects else 1e-10
    lin = list(wts["lin"])
    if "lin_swapped" in defects:
        lin[3], lin[4] = lin[4], lin[3]
    f0s, f1s = features(wts, in0, matched, defects), features(wts, in1, matched, defects)
    out = 0
    for k, (f0, f1) in enumerate(zip(f0s, f1s)):
        n0 = f0 / (torch.sqrt(torch.sum(f0 ** 2, dim=1, keepdim=True)) + eps)
        n1 = f1 / (torch.sqrt(torch.sum(f1 ** 2, dim=1, keepdim=True)) + eps)
        out = out + ((n0 - n1) ** 2 * lin[k].view(1, -1, 1, 1)).sum(dim=1).mean(dim=(1, 2))
    return out


class LPIPSOracle(nn.Module):
    """lpips.LPIPS(net="vgg")-style module over lpips64: forward(in0, in1) -> [n, 1, 1, 1] in `dtype` (torch ops on
    whatever device the inputs are on), usable as LossComputer(lpips_module=...)."""

    def __init__(self, state_dict, dtype=torch.float64, matched=False):
        super().__init__()
        self.wts = weights_from_state_dict(state_dict, dtype)
        self.matched = matched

    def forward(self, in0, in1):
        dev = in0.device
        if self.wts["shift"].device != dev:
            self.wts = {k: ([t.to(dev) for t in v] if isinstance(v, list) else v.to(dev)) for k, v in self.wts.items()}
        out = lpips64(self.wts, in0, in1, self.matched)
        return out.to(in0.dtype).view(-1, 1, 1, 1)
