"""fp64 LPIPS-VGG reference (lpips 0.1, net="vgg", eval mode), plain torch.nn.functional ops, autograd-capable.

    d[n] = sum_k mean_hw sum_c lin_k[c] (f0 - f1)^2,   f = a / (sqrt(sum_c a^2) + 1e-10)

with a the relu1_2 .. relu5_3 activations of torchvision VGG16 features[0:30] applied to (x - shift) / scale.

`weights_from_state_dict` reads the lpips-layout state dict (net.slice{s}.{i}.*, lin{k} / lins.{k}, scaling_layer.*).
matched=True rounds where the kernels (dgs_lpips_*) round: bf16 conv weights, bf16 input after the ScalingLayer, bf16
post-ReLU activations, and dz = d/dz (pre-ReLU) rounded to bf16 in the backward.  The max-pool sends its gradient to the
first maximum of each window in row-major order, in both modes (torch's max_pool2d rule; ties are real in bf16).
`defects` plants a named defect (DEFECTS) for the power tests.

The stage functions (input_stage32, conv_stage64, head64, backward64) restate one stage of the kernels each, on
activations given as the kernels store them (NHWC [n, h, w, C], bf16 values), on any device: fed the kernels' own
activations, they isolate that one stage's arithmetic.  kernel_model64 chains them into a stand-in for the kernels, with
every rounding where the kernels round; it also takes the STAGE_DEFECTS, which only the stage-level checks can see.
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
STAGE_DEFECTS = ("g_no_projection",  # G = g / s: the normalisation's projection term -a0 (g . a0) / (s^2 r) left out
                 "im2col_wrap",      # im2col's tap right of a row's last pixel reads the next row's first pixel
                 "dout_neighbour")   # the backward scales image i's tap gradients by dout[i + 1] (cyclically)


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


# ---- stage functions: one kernel stage each, on given NHWC activations ----
LEVEL = (0, 0, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4)  # conv l runs at H >> LEVEL[l], W >> LEVEL[l]


def _round_bf16(x):
    return x.to(torch.bfloat16).to(x.dtype)


def _nchw(a):
    return a.permute(0, 3, 1, 2).to(torch.float64)


def _nhwc(x):
    return x.permute(0, 2, 3, 1)


def _w64(wts, name, l, dev):
    return wts[name][l].to(dev, torch.float64)


def _pad(x, defects=()):
    """the 1-pixel zero border im2col reads around [n, C, h, w]"""
    p = F.pad(x, (1, 1, 1, 1))
    if "im2col_wrap" in defects:
        p[:, :, 1:-2, -1] = x[:, :, 1:, 0]
    return p


def maxpool_backward(x, g, last=False):
    """2x2 / 2 max-pool backward: g [n, C, h/2, w/2] -> [n, C, h, w], each value to the first (last=True: the last)
    maximum of its window of x in row-major order, 0 elsewhere"""
    n, c, h, w = x.shape
    v = x.reshape(n, c, h // 2, 2, w // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(n, c, h // 2, w // 2, 4)
    idx = 3 - v.flip(-1).argmax(-1) if last else v.argmax(-1)
    out = torch.zeros(v.shape, dtype=g.dtype, device=g.device).scatter_(-1, idx.unsqueeze(-1), g.unsqueeze(-1))
    return out.reshape(n, c, h // 2, w // 2, 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(n, c, h, w)


def input_stage32(wts, x, defects=()):
    """in [n, 3, H, W] -> conv1_1's input bf16((x - shift) / scale) [n, H, W, 3] (fp64 holding bf16 values), computed in
    fp32 as the kernels do"""
    x = x.to(torch.float32)
    if "no_scaling" not in defects:
        x = (x - wts["shift"].to(x.device, torch.float32).view(1, 3, 1, 1)) / \
            wts["scale"].to(x.device, torch.float32).view(1, 3, 1, 1)
    return _nhwc(_round_bf16(x)).to(torch.float64)


def conv_stage64(wts, l, x, defects=()):
    """conv l (max-pooled first where POOL_BEFORE) on its given input x [n, h, w, C_in] with bf16-rounded weights and the
    bias as given, in fp64 -> (a, z, acc) [n, h', w', C_out]: a = bf16(relu(z)) the post-ReLU activation the kernels
    store, z the fp64 pre-activation, acc = (|x| * |W|) + |b| the magnitude the fp32 accumulation rounds"""
    x = _nchw(x)
    if l in POOL_BEFORE:
        x = maxpool(x)
    w, b = _round_bf16(_w64(wts, "conv_w", l, x.device)), _w64(wts, "conv_b", l, x.device)
    z = F.conv2d(_pad(x, defects), w, b)
    acc = F.conv2d(_pad(x.abs()), w.abs(), b.abs())
    return _nhwc(_round_bf16(F.relu(z))), _nhwc(z), _nhwc(acc)


def head64(lin, a0, a1, defects=()):
    """one tap on the given activations a0, a1 [n, h, w, C] with lin [C], in fp64 -> (d, G, mag):
      d [n]            the tap's distance per image, mean_hw sum_c lin (f0 - f1)^2
      G [n, h, w, C]   d d / d a0 as head_kernel defines it: with g = 2 lin (f0 - f1) / hw, r = |a0|, s = r + 1e-10,
                       G = g / s - a0 (g . a0) / (s^2 r), the second term 0 where r = 0 (a pixel the backward never reads)
      mag [n, h, w, C] the same expression over absolute values, the magnitude G's fp32 arithmetic rounds"""
    a0, a1 = a0.to(torch.float64), a1.to(torch.float64)
    lin = lin.to(a0.device, torch.float64)
    eps = 1e-6 if "eps_1e-6" in defects else 1e-10
    hw = a0.shape[1] * a0.shape[2]
    r0, r1 = a0.square().sum(-1, keepdim=True).sqrt(), a1.square().sum(-1, keepdim=True).sqrt()
    s0 = r0 + eps
    f0, f1 = a0 / s0, a1 / (r1 + eps)
    d = (lin * (f0 - f1).square()).sum(-1).sum((1, 2)) / hw
    g, gmag = 2 / hw * lin * (f0 - f1), 2 / hw * lin * (f0.abs() + f1.abs())
    G, mag = g / s0, gmag / s0
    if "g_no_projection" not in defects:
        den = torch.where(r0 > 0, s0 * s0 * r0, torch.ones_like(r0))
        G = G - a0 * torch.where(r0 > 0, (g * a0).sum(-1, keepdim=True) / den, 0.0)
        mag = mag + a0.abs() * torch.where(r0 > 0, (gmag * a0.abs()).sum(-1, keepdim=True) / den, 0.0)
    return d, G, mag


def backward64(wts, act, G, dout, defects=()):
    """d in0 [n, 3, H, W] (fp64) from the given activations act[13] of in0 ([n, h, w, C], bf16 values), tap gradients
    G[5] and dout [n], through the chain the backward kernels run: every routing decision comes from `act` -- the ReLU
    mask [a > 0] and the first maximum of each pool window in row-major order -- dz = (da + dout G) [a > 0] is rounded
    to bf16 where the kernels round it, everything else is fp64, down to the ScalingLayer's / scale"""
    dev = act[0].device
    dout = dout.to(dev, torch.float64).view(-1, 1, 1, 1)
    if "dout_neighbour" in defects:
        dout = dout.roll(-1, 0)
    da = None
    for l in reversed(range(13)):
        a = _nchw(act[l])
        g = torch.zeros_like(a) if da is None else da
        if l in TAP_AFTER:
            g = g + dout * _nchw(G[TAP_AFTER.index(l)])
        dz = _round_bf16(torch.where(a > 0, g, 0.0))
        w = _round_bf16(_w64(wts, "conv_w", l, dev))
        wt = w.transpose(0, 1).flip(3) if "dgrad_one_axis" in defects else w.transpose(0, 1).flip(2, 3)
        dx = F.conv2d(_pad(dz, defects), wt)
        if l == 0:
            return dx / wts["scale"].to(dev, torch.float64).view(1, 3, 1, 1)
        da = maxpool_backward(_nchw(act[l - 1]), dx, "pool_tie_last" in defects) if l in POOL_BEFORE else dx


def kernel_model64(wts, in0, in1, dout, defects=()):
    """The kernels' computation restated from the stage functions, rounding where they round -> dict(out [n], act0,
    act1 (13 each, [n, h, w, C]), G (5), d_in0 [n, 3, H, W]), with DEFECTS / STAGE_DEFECTS planted"""
    lin = list(wts["lin"])
    if "lin_swapped" in defects:
        lin[3], lin[4] = lin[4], lin[3]
    acts, taps = [], []
    for x in (in0, in1):
        a, act, tap = input_stage32(wts, x, defects), [], []
        for l in range(13):
            a, z, _ = conv_stage64(wts, l, a, defects)
            act.append(a)
            if l in TAP_AFTER:
                tap.append(_round_bf16(z) if "tap_pre_relu" in defects and l == TAP_AFTER[2] else a)
        acts.append(act)
        taps.append(tap)
    out, G = 0, []
    for k in range(5):
        d, g, _ = head64(lin[k], taps[0][k], taps[1][k], defects)
        out = out + d
        G.append(g)
    return dict(out=out, act0=acts[0], act1=acts[1], G=G, d_in0=backward64(wts, acts[0], G, dout, defects))
