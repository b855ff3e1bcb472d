"""Power of the LPIPS stage checks (tests/test_lpips_layers_gpu.py), on the CPU.  The stand-in for correct kernels is
oracle.lpips.kernel_model64: the stage functions chained, rounding where the kernels round, at 2 x 32 x 48.  Each defect
planted in it -- the end-to-end test's DEFECTS and the STAGE_DEFECTS only stage checks can see -- must move at least one
check by at least twice the bound the GPU test applies on the H100.  A defect that stays below that is recorded at the
assert with its factor."""
import pytest
import torch
import torch.nn.functional as F

from lpips_regime import random_lpips_state_dict
from test_lpips_layers_gpu import BOUNDS, stage_errors

N, H, W = 2, 32, 48


@pytest.fixture(scope="module")
def setup():
    from oracle.lpips import kernel_model64, weights_from_state_dict
    wts = weights_from_state_dict(random_lpips_state_dict(0))
    g = torch.Generator().manual_seed(0)
    smooth = lambda: F.interpolate(torch.rand(N, 3, H // 8, W // 8, generator=g, dtype=torch.float64),  # noqa: E731
                                   size=(H, W), mode="bilinear")
    target = smooth()
    white = torch.zeros(1, 1, H, W, dtype=torch.bool)
    white[..., :, : W // 4] = True                   # a background strip where both inputs are identical
    target = torch.where(white, torch.ones_like(target), target)
    blocks = lambda x: F.interpolate(F.avg_pool2d(x, 16), scale_factor=16, mode="nearest")  # noqa: E731
    other = torch.where(white, target, smooth())
    pairs = {"independent": (other, target),
             "noise": (torch.where(white, target, (target + 0.05 * torch.randn(target.shape, generator=g,
                                                                               dtype=torch.float64)).clamp(0, 1)),
                       target),
             "flat": (blocks(other), blocks(target))}   # every max-pool window inside a block is a four-way tie
    dout = torch.tensor([0.7, 1.3], dtype=torch.float64)

    def run(kind, defects=()):
        in0, in1 = (x * 2 - 1 for x in pairs[kind])
        r = kernel_model64(wts, in0, in1, dout, defects)
        return stage_errors(wts, in0, in1, dout, r)[0]
    return run


def test_clean_stand_in_passes(setup):
    for kind in ("independent", "noise", "flat"):
        err = setup(kind)
        assert all(v <= BOUNDS[k] for k, v in err.items()), (kind, err)


# defect -> recorded factor below 2x the bound (None: caught with the 2x margin)
CASES = {
    # 1e-10 -> 1e-6 next to tap norms of O(1-10) moves G by ~1e-6 of its magnitude: 1.17x the head bound, caught but
    # without the 2x margin; recorded.
    "eps_1e-6": 1.17,
    "lin_swapped": None,
    "no_scaling": None,
    "pool_tie_last": None,
    "dgrad_one_axis": None,
    "tap_pre_relu": None,
    "g_no_projection": None,
    "im2col_wrap": None,
    "dout_neighbour": None,
}


@pytest.mark.parametrize("defect", list(CASES))
def test_defect_moves_a_check(setup, defect):
    worst, where = 0.0, None
    for kind in ("independent", "noise", "flat"):
        for check, v in setup(kind, (defect,)).items():
            if v / BOUNDS[check] > worst:
                worst, where = v / BOUNDS[check], f"{check} ({kind})"
    print(f"\n{defect}: moves {where} by {worst:.3g}x its GPU bound")
    if CASES[defect] is not None:
        assert 1.0 < worst < 2.0  # recorded: see CASES
    else:
        assert worst >= 2.0
