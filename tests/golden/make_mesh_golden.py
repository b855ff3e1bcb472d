"""Writes tests/golden/mesh_fields_ref.npz: the REFERENCE's own GaussianModel.extract_fields (gs_core.py:786-852),
executed by path from a reference checkout on CPU tensors, for seeded Gaussians.  Stored per case: the raw inputs, the
occupancy field, mesh_center and mesh_scale.  The Gaussians sit in a few compact clusters spread over the grid, so most
blocks hold none and their field is exactly 0: the fixture compresses to a few hundred kB while every case still has
blocks cut by the truncation and, at resolution 100, the short last chunk.

    python tests/golden/make_mesh_golden.py        # needs a reference checkout (DGS_REFERENCE_ROOT)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [HERE, ROOT, os.path.join(ROOT, "open-diffusiongs_b200")]
import ref_import as ri  # noqa: E402
from dgs_b200 import synth  # noqa: E402

NAMES = ("xyz", "scaling", "rotation", "opacity")
# name -> (P, resolution, num_blocks, relax_ratio, scaling_modifier, seed)
CASES = {"r64_b16": (800, 64, 16, 1.5, None, 31), "r100_b16": (800, 100, 16, 1.5, None, 32),
         "r64_b16_smod": (600, 64, 16, 1.5, 0.7, 33), "r48_b8_relax1": (500, 48, 8, 1.0, None, 34)}
CLUSTERS, SPREAD = 3, 0.01  # clusters per case; standard deviation of the centres around a cluster's centre


def inputs(case):
    P, _, _, _, _, seed = CASES[case]
    g = synth.make_gaussians(P, seed, "trained")
    rng = np.random.default_rng(seed + 100)
    centres = rng.uniform(-1.0, 1.0, (CLUSTERS, 3))
    g["xyz"] = (centres[rng.integers(0, CLUSTERS, P)] + rng.normal(0, SPREAD, (P, 3))).astype(np.float32)
    g["rotation"] = (g["rotation"] * rng.uniform(0.5, 2.0, (P, 1))).astype(np.float32)  # un-normalised on purpose
    return {k: g[k] for k in NAMES}


def run_reference(case):
    ns = ri.load("oracle")
    sys.modules["kiui"].lo = lambda *a, **k: None  # extract_fields logs the field through kiui.lo
    P, res, nb, relax, smod, _ = CASES[case]
    raw = inputs(case)
    gm = ns.gs_core.GaussianModel(0, scaling_modifier=smod)
    gm._xyz, gm._scaling, gm._rotation, gm._opacity = (torch.from_numpy(raw[k]) for k in NAMES)
    occ = gm.extract_fields(resolution=res, num_blocks=nb, relax_ratio=relax)
    return raw, occ.numpy(), gm.mesh_center.numpy(), float(gm.mesh_scale)


def main():
    rec = {}
    for case in CASES:
        raw, occ, center, scale = run_reference(case)
        rec.update({f"{case}/in/{k}": v for k, v in raw.items()})
        rec.update({f"{case}/occ": occ, f"{case}/mesh_center": center, f"{case}/mesh_scale": np.float64(scale)})
        print(case, occ.shape, f"nonzero={np.count_nonzero(occ)}", f"max={occ.max():.4f}")
    path = os.path.join(HERE, "mesh_fields_ref.npz")
    np.savez_compressed(path, **rec)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
