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
