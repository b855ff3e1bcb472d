"""Writes tests/golden/geometry_loss_ref.npz: the pointsdist and l2_xyz outputs of the REFERENCE's own LossComputer
(diffusionGS/utils/losses.py:239-369, the absent lpips / pytorch_msssim / skimage packages stubbed as in
tests/test_losses_cpu.py) and the gradient of sum_b g_pd[b] pointsdist[b] + g_xyz l2_xyz w.r.t. img_aligned_xyz, with
the inputs, for the cases of geometry_cases().
    DGS_REFERENCE_ROOT=<reference checkout> python tests/golden/make_geometry_loss_golden.py"""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "open-diffusiongs_b200"), os.path.join(ROOT, "tests"), HERE):
    sys.path.insert(0, p)

import ref_import as ri  # noqa: E402
import test_losses_cpu as tl  # noqa: E402

G_XYZ = 0.025  # lambda_xyz of diffusionGS_rel.yaml


def geometry_cases():
    """{name: (img_xyz, ray_o, gt_xyz, masks)} fp32 CPU tensors [b, v, 3 / 1, h, w]:
    tc3 / tc4: the inputs of test_losses_cpu.py (binary masks);  ragged: 37 x 53 with fractional masks;
    edge: view (0, 1) at one constant distance (std = 0), view (1, 0) with a block of pixels at img == o (dist = 0),
    fractional masks."""
    out = {}
    for tc in tl.TCS:
        _, _, masks, _, ray_o, xyz, gt_xyz = tl.loss_inputs(tc)
        out[f"tc{tc}"] = (xyz.detach(), ray_o, gt_xyz, masks)
    g = torch.Generator().manual_seed(7)
    b, v, h, w = 2, 2, 37, 53
    ray_o = torch.randn(b, v, 3, 1, 1, generator=g).expand(b, v, 3, h, w).contiguous() * 1.5
    xyz = ray_o + torch.randn(b, v, 3, h, w, generator=g)
    out["ragged"] = (xyz, ray_o, torch.randn(b, v, 3, h, w, generator=g), torch.rand(b, v, 1, h, w, generator=g))
    b, v, h, w = 2, 2, 20, 28
    ray_o = torch.round(torch.randn(b, v, 3, h, w, generator=g) * 8) / 8  # eighths: o + 0.75 e_k is exact
    xyz = ray_o + torch.randn(b, v, 3, h, w, generator=g)
    axis = torch.randint(0, 3, (h, w), generator=g)
    sign = torch.where(torch.rand(h, w, generator=g) < 0.5, -1.0, 1.0)
    step = torch.nn.functional.one_hot(axis, 3).permute(2, 0, 1).float() * sign * 0.75
    xyz[0, 1] = ray_o[0, 1] + step
    xyz[1, 0, :, 3:9, 5:17] = ray_o[1, 0, :, 3:9, 5:17]
    out["edge"] = (xyz, ray_o, torch.randn(b, v, 3, h, w, generator=g), torch.rand(b, v, 1, h, w, generator=g))
    return out


def g_pd_of(b):
    return torch.linspace(0.7, 1.3, b)


def main():
    tl.stub_packages()
    spec = importlib.util.spec_from_file_location("_ref_losses", os.path.join(ri.REF, "diffusionGS/utils/losses.py"))
    ref_mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref_mod)
    lc = ref_mod.LossComputer()
    out = {}
    for name, (xyz, ray_o, gt_xyz, masks) in geometry_cases().items():
        b, v, _, h, w = xyz.shape
        x = xyz.clone().requires_grad_(True)
        rendering = torch.zeros(b, v, 3, h, w)
        _, _, _, pd, l2 = lc(rendering, rendering, masks, masks, ray_o, x, gt_xyz)
        g_pd = g_pd_of(b)
        ((pd * g_pd).sum() + G_XYZ * l2).backward()
        out.update({f"{name}/img_xyz": xyz.numpy(), f"{name}/ray_o": ray_o.numpy(), f"{name}/gt_xyz": gt_xyz.numpy(),
                    f"{name}/masks": masks.numpy(), f"{name}/g_pd": g_pd.numpy(), f"{name}/pointsdist": pd.detach().numpy(),
                    f"{name}/l2_xyz": l2.detach().numpy(), f"{name}/d_img": x.grad.numpy()})
    out["g_xyz"] = np.float32(G_XYZ)
    np.savez_compressed(os.path.join(HERE, "geometry_loss_ref.npz"), **out)


if __name__ == "__main__":
    main()
