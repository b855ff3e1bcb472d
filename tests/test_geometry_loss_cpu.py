"""The geometry loss terms without a GPU: the fp64 oracle (oracle/geometry_loss.py) against the reference's own
LossComputer (tests/golden/geometry_loss_ref.npz, values and the gradient w.r.t. img_aligned_xyz; losses_ref.npz,
values), and the argument checks of the C ABI (dgs_geometry_loss_*)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from dgs_b200 import _lib
from oracle.geometry_loss import geometry_grad64, geometry_losses64
from util import rel_l2 as rel

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = ("tc3", "tc4", "ragged", "edge")


def fixture_case(z, name):
    return [torch.from_numpy(z[f"{name}/{k}"]) for k in ("img_xyz", "ray_o", "gt_xyz", "masks")]


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_reference_fixture(name):
    """fp64 autograd on the reference's formulas vs the reference's fp32 LossComputer + backward: fp32 rounding apart
    (measured: <= 1e-7 on the values, 1.5e-7 on the gradient)."""
    z = np.load(os.path.join(HERE, "golden", "geometry_loss_ref.npz"))
    x, o, gt, m = fixture_case(z, name)
    pd, l2, d = geometry_grad64(x, o, gt, m, g_pd=torch.from_numpy(z[f"{name}/g_pd"]), g_xyz=float(z["g_xyz"]))
    e = dict(pointsdist=rel(pd, z[f"{name}/pointsdist"]), l2_xyz=rel(l2, z[f"{name}/l2_xyz"]), d_img=rel(d, z[f"{name}/d_img"]))
    print(name, {k: f"{v:.1e}" for k, v in e.items()})
    assert e["pointsdist"] < 1e-6 and e["l2_xyz"] < 1e-6 and e["d_img"] < 1e-6, e


def test_fixture_edge_cases_are_what_they_claim():
    z = np.load(os.path.join(HERE, "golden", "geometry_loss_ref.npz"))
    x, o, _, m = fixture_case(z, "edge")
    dist = (x - o).norm(dim=2)
    assert torch.all(dist[0, 1] == 0.75)                      # one constant distance: std 0
    assert int((dist[1, 0] == 0).sum()) == 6 * 12              # img == o
    assert 0 < float(m.min()) and float(m.max()) < 1 and len(torch.unique(m)) > 100  # fractional masks
    _, _, d = geometry_grad64(x, o, g_pd=torch.ones(2))
    assert torch.all(d[1, 0, :, 3:9, 5:17] == 0)               # pointsdist gradient 0 where dist == 0


def test_oracle_reproduces_losses_ref_values():
    import test_losses_cpu as tl
    z = np.load(os.path.join(HERE, "golden", "losses_ref.npz"))
    for tc in tl.TCS:
        _, _, masks, _, ray_o, xyz, gt_xyz = tl.loss_inputs(tc)
        pd, l2 = geometry_losses64(xyz.detach(), ray_o, gt_xyz, masks)
        assert rel(pd, z[f"tc{tc}/pointsdist"]) < 1e-6 and rel(l2, z[f"tc{tc}/l2_xyz"]) < 1e-6, tc


def test_abi_argument_checks_without_gpu():
    L = _lib.lib()
    assert L.dgs_geometry_loss_workspace_bytes(4, 4) == 16 * 64 * 5 * 8  # 64 parts per view: 4 + 1 fp64 sums each
    assert L.dgs_geometry_loss_workspace_bytes(0, 4) == 0
    fake = C.c_void_p(256)
    ws = L.dgs_geometry_loss_workspace_bytes(1, 2)

    def fwd(B=1, V=2, H=8, W=8, o=fake, gt=fake, m=fake, pd=fake, l2=fake, nbytes=ws):
        return L.dgs_geometry_loss_forward(B, V, H, W, fake, o, gt, m, pd, l2, fake, fake, nbytes, None)
    assert fwd(B=0) == 1 and b"must be > 0" in L.dgs_last_error()
    assert fwd(B=300, V=300) == 1 and b"65535" in L.dgs_last_error()
    assert fwd(o=None) == 1 and b"needs ray_o" in L.dgs_last_error()
    assert fwd(m=None) == 1 and b"needs gt_xyz and masks" in L.dgs_last_error()
    assert fwd(nbytes=ws - 1) == 1 and b"workspace too small" in L.dgs_last_error()
    bwd = L.dgs_geometry_loss_backward
    assert bwd(1, 2, 8, 8, fake, None, fake, fake, fake, fake, None, fake, None) == 1 and b"needs ray_o" in L.dgs_last_error()
    assert bwd(1, 2, 8, 8, fake, fake, fake, fake, fake, None, None, None, None) == 1 and b"NULL" in L.dgs_last_error()


def test_python_checks_without_gpu():
    from dgs_b200.geometry_loss import geometry_losses
    x = torch.zeros(1, 2, 3, 4, 4)
    with pytest.raises(ValueError, match="img_xyz"):
        geometry_losses(torch.zeros(1, 2, 4, 4, 4), x)
    with pytest.raises(ValueError, match="masks"):
        geometry_losses(x, x, x, torch.zeros(1, 2, 3, 4, 4))
    with pytest.raises(_lib.DgsError, match="CUDA"):
        geometry_losses(x, x)
