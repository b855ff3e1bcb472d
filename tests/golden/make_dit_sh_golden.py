"""Writes the fixtures of the DiT at gaussians_sh_degree > 0 from the REFERENCE's own denoiser code (executed through
tests/golden/ref_import.py, as tests/golden/make_dit_golden.py does at degree 0):

  dit_ref_<case>.npz for every case of DIT_SH_CASES: the outputs (features [b, n, (d+1)^2, 3]), a digest of the
      parameter gradients of the seeded loss (per-parameter L2 norm and a fixed random projection, as dit_ref_*.npz),
      and the reference model's state_dict keys and shapes;
  dit_sh_keys.npz: the reference's state_dict keys and shapes of both model classes at d = 0..3.

Parameters and inputs are regenerated from the seed on any box (ref_import.seeded_*).  The degree-0 cases and their
fixtures stay with make_dit_golden.py; this script writes none of them.

    DGS_REFERENCE_ROOT=<reference checkout> python tests/golden/make_dit_sh_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_import as ri  # noqa: E402

# name -> (scene, ray_pe_type, model config, (b, v, h, w), seed), as ref_import.DIT_CASES
_S = dict(width=64, dim_heads=16, patch_size=8)
DIT_SH_CASES = {
    "s_obj_rel_sh1": (False, "relative_plk", dict(_S, num_layers=2, gaussians_sh_degree=1), (2, 2, 16, 16), 31),
    "s_scene_plk_sh2": (True, "plk", dict(_S, num_layers=3, gaussians_sh_degree=2), (1, 3, 16, 24), 32),
    "s_obj_rel_sh3": (False, "relative_plk", dict(_S, num_layers=2, gaussians_sh_degree=3), (2, 2, 16, 16), 33),
    "w1024_obj_rel_sh3": (False, "relative_plk", dict(width=1024, dim_heads=64, num_layers=2, patch_size=8,
                                                      gaussians_sh_degree=3), (2, 2, 32, 32), 34),
}
# the configuration of dit_sh_keys.npz
KEYS_CFG = dict(_S, num_layers=2)


def reference_model(scene, cfg, pe="relative_plk"):
    ns = ri.load("stub")
    cls = (ns.denoiser_scene if scene else ns.denoiser).DGSDenoiser
    return cls(dict(cfg, in_channels=9, n_gaussians=2, ray_pe_type=pe))


def reference_sh_case(name):
    """ref_import.reference_dit_case for a case of DIT_SH_CASES."""
    scene, pe, cfg, (b, v, h, w), seed = DIT_SH_CASES[name]
    model = reference_model(scene, cfg, pe)
    model.load_state_dict(ri.seeded_state_dict(model, seed), strict=True)
    img, ro, rd, t = ri.seeded_dit_inputs(b, v, h, w, seed + 1000)
    out, ia = model.image_to_gaussians(img, ro, rd, t)
    outs = {k: out[k] for k in ri.GS_KEYS}
    outs["img_aligned_xyz"] = ia
    cot = {k: ri.seeded(tuple(o.shape), seed + 2000 + i) for i, (k, o) in enumerate(outs.items()) if k != "img_aligned_xyz"}
    loss = sum((outs[k] * cot[k]).sum() for k in cot)
    grads = torch.autograd.grad(loss, list(model.parameters()))
    grads = {k: g for (k, _), g in zip(model.named_parameters(), grads)}
    return model, {k: o.detach() for k, o in outs.items()}, grads


def _keys_and_shapes(model, prefix=""):
    sd = model.state_dict()
    rec = {prefix + "keys": np.array(list(sd))}
    rec.update({prefix + "shape/" + k: np.array(tuple(v.shape), np.int64) for k, v in sd.items()})
    return rec


def main():
    torch.set_num_threads(8)
    for name in DIT_SH_CASES:
        model, outs, grads = reference_sh_case(name)
        rec = {"out/" + k: v.numpy() for k, v in outs.items()}
        rng = np.random.default_rng(7)
        for k, g in grads.items():
            gg = g.double().numpy().ravel()
            rec["gnorm/" + k] = np.float64(np.linalg.norm(gg))
            rec["gproj/" + k] = np.float64(gg @ rng.standard_normal(gg.size))
        rec.update(_keys_and_shapes(model))
        path = os.path.join(HERE, f"dit_ref_{name}.npz")
        np.savez_compressed(path, **rec)
        print(name, {k: tuple(v.shape) for k, v in outs.items()}, os.path.getsize(path), "bytes")
    rec = {}
    for scene in (False, True):
        for d in range(4):
            rec.update(_keys_and_shapes(reference_model(scene, dict(KEYS_CFG, gaussians_sh_degree=d)),
                                        f"{'scene' if scene else 'obj'}_sh{d}/"))
    np.savez_compressed(os.path.join(HERE, "dit_sh_keys.npz"), **rec)


if __name__ == "__main__":
    main()
