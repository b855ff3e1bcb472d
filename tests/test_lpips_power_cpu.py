"""Power of the LPIPS GPU checks, on the CPU: with the rounding-matched fp64 reference standing in for the kernels, each
defect planted in it (oracle.lpips.DEFECTS) must move the quantity it corrupts -- the value or d in0 -- by at least twice
the bound tests/test_lpips_gpu.py applies on the H100.  Defects that stay below that are recorded at the assert."""
import pytest
import torch
import torch.nn.functional as F

from lpips_regime import random_lpips_state_dict
from test_lpips_gpu import GRAD_BLOCK_MATCHED, GRAD_MATCHED, VALUE_MATCHED, grad_errors

H, W = 64, 96


@pytest.fixture(scope="module")
def setup():
    from oracle.lpips import lpips64, weights_from_state_dict
    wts = weights_from_state_dict(random_lpips_state_dict(0))
    g = torch.Generator().manual_seed(0)
    smooth = lambda: F.interpolate(torch.rand(2, 3, H // 8, W // 8, generator=g, dtype=torch.float64),  # noqa: E731
                                   size=(H, W), mode="bilinear")
    target = smooth()
    white = torch.zeros(1, 1, H, W, dtype=torch.bool)
    white[..., :, : W // 4] = True                   # a background strip where both inputs are identical
    target = torch.where(white, torch.ones_like(target), target)
    blocks = lambda x: F.interpolate(F.avg_pool2d(x, 16), scale_factor=16, mode="nearest")  # noqa: E731
    other = torch.where(white, target, smooth())
    pairs = {"independent": other,
             "noise": torch.where(white, target, (target + 0.05 * torch.randn(target.shape, generator=g,
                                                                              dtype=torch.float64)).clamp(0, 1)),
             "flat": blocks(other)}
    targets = {"independent": target, "noise": target, "flat": blocks(target)}
    dout = torch.tensor([0.7, 1.3], dtype=torch.float64)

    def run(kind, defects=()):
        x = (pairs[kind] * 2 - 1).clone().requires_grad_(True)
        v = lpips64(wts, x, targets[kind] * 2 - 1, matched=True, defects=defects)
        (v * dout).sum().backward()
        return v.detach(), x.grad
    clean = {k: run(k) for k in pairs}
    return run, clean


# defect -> (checked quantity, recorded factor below 2x the bound or None)
CASES = {
    # 1e-10 -> 1e-6 next to channel norms of O(1-10) moves the value by ~4e-7 relative (2e-4 x the 2e-3 bound): a
    # wrong eps of this size is invisible to any bf16 implementation and is recorded here rather than checked.
    "eps_1e-6": ("value", "below"),
    # the lin weights of taps 3 and 4 are drawn from one distribution, so swapping them moves the value by only ~3e-3
    # relative (1.45x the 2e-3 bound): caught, but without a 2x margin; recorded.
    "lin_swapped": ("value", "below"),
    "no_scaling": ("value", None),
    "tap_pre_relu": ("value", None),
    "dgrad_one_axis": ("grad", None),
    # only windows with equal activations are affected: scattered bf16 ties in smooth images (2.1x the full-gradient
    # bound), every window inside a block of the piecewise-constant "flat" pair (far above)
    "pool_tie_last": ("grad", None),
}


@pytest.mark.parametrize("defect", list(CASES))
def test_defect_moves_checked_quantity(setup, defect):
    run, clean = setup
    what, recorded = CASES[defect]
    worst = 0.0
    for kind in ("independent", "noise", "flat"):
        v0, g0 = clean[kind]
        v, g = run(kind, (defect,))
        if what == "value":
            factor = float(((v - v0) / v0).abs().max()) / VALUE_MATCHED
        else:
            full, block = grad_errors(g, g0)
            factor = max(full / GRAD_MATCHED, block / GRAD_BLOCK_MATCHED)
        worst = max(worst, factor)
    print(f"\n{defect}: moves the {what} by {worst:.3g}x the GPU bound")
    if recorded == "below":
        assert worst < 2.0  # recorded: see CASES
        if defect == "lin_swapped":
            assert worst > 1.0  # still above the bound itself
    else:
        assert worst >= 2.0
