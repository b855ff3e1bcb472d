"""Power of the SSIM / PSNR GPU checks, on the CPU: each defect planted in the fp64 reference (oracle.ssim.DEFECTS) must
move the quantity it corrupts -- a per-image SSIM, PSNR, or d x -- by at least twice the bound tests/test_ssim_gpu.py
applies on the H100, on every CPU pair that stands in for a kind of pair the GPU suite feeds and that the defect
depends on (listed in CASES).  Defects that stay below that are recorded at the assert."""
import pytest
import torch

from oracle.ssim import SAMPLE_COV, psnr64, ssim64, ssim_grad64
from test_ssim_cpu import smooth_pair
from test_ssim_gpu import GRAD_F64, KINDS, PSNR_F64, SSIM_F64

H, W = 37, 61


@pytest.fixture(scope="module")
def pairs():
    """Stand-ins for the GPU suite's kinds of pair, built the same way on smooth random images:
    "smooth": sigma^2 ~ C2 (where the sample covariance shows); "noise": the target plus a stronger perturbation,
    clamped to [0, 1]; "overshoot": the target plus an unclamped perturbation, so the rendering leaves [0, 1]."""
    sx, sy = smooth_pair(3, H, W, seed=0)
    nx, ny = smooth_pair(3, H, W, seed=1, contrast=0.5)
    g = torch.Generator().manual_seed(2)
    ox = ny + 0.2 * torch.randn(ny.shape, generator=g, dtype=torch.float64)
    assert bool(((ox < 0) | (ox > 1)).flatten(1).any(1).all())
    return {"smooth": (sx, sy), "noise": (nx, ny), "overshoot": (ox, ny)}


ALL = ("smooth", "noise", "overshoot")
# defect -> (checked quantity, k of the variant it is planted in, the pairs on which it must move that quantity)
CASES = {
    "population_cov": ("ssim", SAMPLE_COV, ALL),
    "c1_c2_swapped": ("ssim", 1.0, ALL),
    "same_padding": ("ssim", 1.0, ALL),
    "win9": ("ssim", 1.0, ALL),
    "no_2x_beta": ("grad", 1.0, ALL),
    "no_y_gamma": ("grad", 1.0, ALL),
    "bwd_shift": ("grad", 1.0, ALL),
    # the clamp only acts on a rendering that leaves [0, 1]: the GPU suite's "overshoot" kind (every image of which the
    # GPU test also checks leaves [0, 1]); on the in-range pairs a missing clamp changes nothing
    "psnr_unclamped": ("psnr", None, ("overshoot",)),
    "psnr_frame_twice": ("psnr", None, ALL),
}


def test_stand_ins_are_kinds_the_gpu_suite_feeds():
    assert set(ALL) <= set(KINDS)


@pytest.mark.parametrize("defect", list(CASES))
def test_defect_moves_checked_quantity(pairs, defect):
    what, k, kinds = CASES[defect]
    dout = torch.tensor([0.7, 1.3, 1.0], dtype=torch.float64)
    factors = {}
    for kind in kinds:
        x, y = pairs[kind]
        if what == "ssim":
            d = (ssim64(x, y, k=k, defects=(defect,)) - ssim64(x, y, k=k)).abs()
            factor = float(d.min()) / SSIM_F64  # every image, not just the most affected one
        elif what == "psnr":
            factor = float((psnr64(x, y, (defect,)) - psnr64(x, y)).abs().min()) / PSNR_F64
        else:
            g0, g = ssim_grad64(x, y, dout, k=k), ssim_grad64(x, y, dout, k=k, defects=(defect,))
            factor = float((g - g0).norm() / g0.norm()) / GRAD_F64
        factors[kind] = factor
    print(f"\n{defect}: " + ", ".join(f"{kind} {f:.3g}x" for kind, f in factors.items()) + " the GPU bound")
    assert min(factors.values()) >= 2.0
