"""`distCUDA2` of the reference's simple_knn extension (simple_knn.cu:148-184, spatial.cu) over dgs_knn."""
import os
import sys

import torch

_PKG_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _PKG_ROOT not in sys.path:  # make the sibling host package importable when only this one is on the path
    sys.path.insert(0, _PKG_ROOT)

from dgs_b200 import mesh as _mesh  # noqa: E402

FLT_MAX = 3.4028234663852886e38


def distCUDA2(points):
    """points fp32 [P, 3] CUDA -> fp32 [P]: per point (b0 + b1 + b2) / 3 over its three smallest squared distances to
    other indices (the exact k = 4 neighbours of dgs_knn, less the point itself), a missing neighbour counting as
    FLT_MAX, so that P <= 3 gives inf as the reference does.  Squared distances are rounded product by product."""
    if not (isinstance(points, torch.Tensor) and points.is_cuda):
        raise TypeError("distCUDA2: points must be a CUDA tensor")
    P = points.shape[0]
    if P == 0:
        return torch.zeros(0, dtype=torch.float32, device=points.device)
    idx, d2 = _mesh.knn(points, 4)
    other = idx != torch.arange(P, dtype=torch.int32, device=idx.device)[:, None]
    other[:, 3] &= ~other.all(1)  # a point that is not among its own four (duplicates) drops its fourth instead
    d = torch.where(idx < 0, torch.full_like(d2, FLT_MAX), d2)[other].view(P, 3)
    s = d[:, 0] + d[:, 1] + d[:, 2]
    return s / torch.full_like(s, 3.0)  # a true division: torch multiplies by the reciprocal of a scalar divisor
