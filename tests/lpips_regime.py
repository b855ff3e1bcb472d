"""Synthetic LPIPS-VGG weights in the lpips package's state-dict layout, for tests: He-scaled random convolutions with
non-zero biases, non-negative `lin` weights and the lpips ScalingLayer constants.  The lin weights are scaled so that two
unrelated renderings lie at a distance of about 0.3-0.6, as with the trained weights."""
import math

import torch

CONV_INDEX = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)
SLICE = (1, 1, 2, 2, 3, 3, 3, 4, 4, 4, 5, 5, 5)
CHANNELS = (3, 64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512)
TAP_CHANNELS = (64, 128, 256, 512, 512)
SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)
LIN_SCALE = 0.5


def random_lpips_state_dict(seed=0, lin_keys=("lin", "lins")):
    g = torch.Generator().manual_seed(seed)
    sd = {"scaling_layer.shift": torch.tensor(SHIFT).view(1, 3, 1, 1),
          "scaling_layer.scale": torch.tensor(SCALE).view(1, 3, 1, 1)}
    for l in range(13):
        ci, co = CHANNELS[l], CHANNELS[l + 1]
        key = f"net.slice{SLICE[l]}.{CONV_INDEX[l]}"
        sd[key + ".weight"] = torch.randn(co, ci, 3, 3, generator=g) * math.sqrt(2.0 / (9 * ci))
        sd[key + ".bias"] = torch.randn(co, generator=g) * 0.1
    for k, c in enumerate(TAP_CHANNELS):
        w = torch.rand(1, c, 1, 1, generator=g) * LIN_SCALE
        if "lin" in lin_keys:
            sd[f"lin{k}.model.1.weight"] = w
        if "lins" in lin_keys:
            sd[f"lins.{k}.model.1.weight"] = w.clone()
    return sd


def sparse_lpips_state_dict(seed, images, fire=1.5 / 512):
    """random_lpips_state_dict(seed) with the biases of relu4_3 and relu5_3 (the convs of taps 3 and 4) lowered per
    channel to the (1 - fire) quantile of the channel's fp64 pre-activation over `images` [n, 3, H, W]: each channel then
    fires on about `fire` of the pixels, so many tap pixels of those images are all zero or have one non-zero channel."""
    from oracle.lpips import CONV_INDEX, SLICE, conv_stage64, input_stage32, weights_from_state_dict
    sd = random_lpips_state_dict(seed)
    wts = weights_from_state_dict(sd)
    wts = {k: ([t.to(images.device) for t in v] if isinstance(v, list) else v.to(images.device)) for k, v in wts.items()}
    a = input_stage32(wts, images)
    for l in range(13):
        x = a
        a, z, _ = conv_stage64(wts, l, x)
        if l in (9, 12):
            key = f"net.slice{SLICE[l]}.{CONV_INDEX[l]}.bias"
            sd[key] = (sd[key].double() - torch.quantile(z.reshape(-1, z.shape[-1]), 1 - fire, dim=0).cpu()).float()
            wts["conv_b"][l] = sd[key].double().to(images.device)
            a, _, _ = conv_stage64(wts, l, x)
    return sd


def state_views(state, n, H, W):
    """The training state of dgs_lpips_forward (a uint8 tensor of dgs_lpips_state_bytes(n, H, W) bytes) as the views
    lpips.cu's carve_state lays out, each 256-byte aligned: act[l] [n, H_l, W_l, C_l] bf16 for the 13 convs (in0's
    post-ReLU activations), then G[k] [n, H_k, W_k, C_k] fp32 for the 5 taps (d d[n] / d act at the tap)."""
    from dgs_b200 import _lib
    from oracle.lpips import LEVEL, TAP_AFTER
    off = 0

    def take(dtype, shape):
        nonlocal off
        off = (off + 255) // 256 * 256
        nbytes = math.prod(shape) * dtype.itemsize
        v = state[off:off + nbytes].view(dtype).view(shape)
        off += nbytes
        return v
    act = [take(torch.bfloat16, (n, H >> LEVEL[l], W >> LEVEL[l], CHANNELS[l + 1])) for l in range(13)]
    G = [take(torch.float32, (n, H >> LEVEL[l], W >> LEVEL[l], CHANNELS[l + 1])) for l in TAP_AFTER]
    total = (off + 255) // 256 * 256
    assert total == _lib.lib().dgs_lpips_state_bytes(n, H, W) == state.numel(), "the LPIPS state layout changed"
    return act, G
