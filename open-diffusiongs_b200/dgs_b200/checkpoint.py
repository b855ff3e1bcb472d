"""On-disk checkpoint compatibility with the reference: host-side key mapping only, no arithmetic.

The reference stores three layouts that contain the denoiser's parameters:
  * a Lightning system checkpoint  {"state_dict": {"shape_model.<key>": ..., "loss_computer.lpips_loss_module.<...>": ...},
    "epoch": e, "global_step": s, ...}   -- what `DiffusionGSPipeline.from_pretrained` and `BaseSystem.load_weights` read
    (diffusionGS/pipline_obj.py:66-71, systems/base.py:51-57, utils/misc.py:40-70);
  * the original release format {"model": {"denoiser.<key>": ..., "denoiser.loss_computer.<...>": ...}} handled inside
    `DGSDenoiser.__init__` (diffusionGS/models/denoiser/denoiser.py:259-268);
  * a bare denoiser `state_dict`.
`extract_denoiser_state_dict` reduces all three to the bare form (the keys identical to
`dgs_b200.denoiser.DGSDenoiser.state_dict()`), `load_checkpoint` loads it strictly, and `system_checkpoint` /
`save_system_checkpoint` write the Lightning layout back so that the reference's `system.load_state_dict(..., strict=False)`
and `load_module_weights(path, module_name="shape_model")` accept a model trained here."""
import re

import torch

SYSTEM_PREFIX = "shape_model."           # attribute name of the denoiser inside the reference's systems
RELEASE_PREFIX = "denoiser."             # original (Adobe) release format
_LOSS_PREFIXES = ("loss_computer.", "denoiser.loss_computer.")
LPIPS_PREFIXES = ("loss_computer.lpips_loss_module.", "denoiser.loss_computer.lpips_loss_module.")


def extract_denoiser_state_dict(obj):
    """-> (bare denoiser state_dict, meta dict with 'epoch' / 'global_step' when present, list of ignored keys)."""
    meta = {}
    if isinstance(obj, dict) and "state_dict" in obj and isinstance(obj["state_dict"], dict):
        meta = {k: obj[k] for k in ("epoch", "global_step") if k in obj}
        sd = obj["state_dict"]
    elif isinstance(obj, dict) and "model" in obj and isinstance(obj["model"], dict):
        sd = obj["model"]
    else:
        sd = obj
    if not isinstance(sd, dict) or not sd:
        raise ValueError("not a checkpoint: expected a (nested) dict of tensors")
    keys = list(sd.keys())
    ignored = [k for k in keys if k.startswith(_LOSS_PREFIXES)]
    keep = [k for k in keys if k not in set(ignored)]
    if any(k.startswith(SYSTEM_PREFIX) for k in keep):
        other = [k for k in keep if not k.startswith(SYSTEM_PREFIX)]
        ignored += other                      # other sub-modules of the system (none in the shipped configs)
        out = {k[len(SYSTEM_PREFIX):]: sd[k] for k in keep if k.startswith(SYSTEM_PREFIX)}
    elif any(k.startswith(RELEASE_PREFIX) for k in keep):
        other = [k for k in keep if not k.startswith(RELEASE_PREFIX)]
        ignored += other
        out = {k[len(RELEASE_PREFIX):]: sd[k] for k in keep if k.startswith(RELEASE_PREFIX)}
    else:
        out = {k: sd[k] for k in keep}
    out = {k: v for k, v in out.items() if not k.startswith("loss_computer.")}
    return out, meta, ignored


def lpips_state_dict(obj):
    """-> the frozen LPIPS-VGG weights a checkpoint holds under "loss_computer.lpips_loss_module.*" (Lightning layout, or a
    bare dict) or "denoiser.loss_computer.lpips_loss_module.*" (release layout), with that prefix removed: the keys of
    `lpips.LPIPS(net="vgg").state_dict()`.  These are among the keys `extract_denoiser_state_dict` drops; {} when the
    checkpoint has none."""
    if isinstance(obj, dict) and "state_dict" in obj and isinstance(obj["state_dict"], dict):
        sd = obj["state_dict"]
    elif isinstance(obj, dict) and "model" in obj and isinstance(obj["model"], dict):
        sd = obj["model"]
    else:
        sd = obj
    if not isinstance(sd, dict):
        raise ValueError("not a checkpoint: expected a (nested) dict of tensors")
    out = {}
    for k, v in sd.items():
        for p in LPIPS_PREFIXES:
            if k.startswith(p):
                out[k[len(p):]] = v
                break
    return out


def load_checkpoint(model, path_or_obj, strict=True, map_location="cpu"):
    """Load any of the three layouts into a `DGSDenoiser[Scene]`; returns the meta dict (epoch / global_step).
    Tensors are cast to the parameters' dtype (released checkpoints are fp16/bf16, the master weights here are fp32)."""
    obj = path_or_obj if isinstance(path_or_obj, dict) else torch.load(path_or_obj, map_location=map_location,
                                                                        weights_only=False)  # path, PathLike or file object
    sd, meta, _ = extract_denoiser_state_dict(obj)
    own = model.state_dict()
    sd = {k: (v.to(own[k].dtype) if k in own and torch.is_tensor(v) else v) for k, v in sd.items()}
    missing, unexpected = model.load_state_dict(sd, strict=False)
    if strict and (missing or unexpected):
        raise RuntimeError(f"checkpoint does not match the denoiser: missing {sorted(missing)[:8]} unexpected {sorted(unexpected)[:8]}")
    if getattr(model, "_trainer", None) is not None:   # flat fp32 master arena + bf16 GEMM operands follow the new values
        model._trainer.refresh_weights()               # (updates the packed stacks in place and re-keys them)
        if model._trainer.ema is not None:             # the EMA restarts from the loaded weights, as EMA.on_train_start's
            model._trainer.ema.copy_(model._trainer.master)   # copy does in the reference (ema.py:69-72)
    else:
        model._packed = None                           # inference-only model: repack lazily on the next forward
    return meta


def system_checkpoint(model, epoch=0, global_step=0, extra_state_dict=None):
    """The Lightning layout the reference reads: {"state_dict": {"shape_model.<key>": tensor}, "epoch", "global_step"}.
    `extra_state_dict` (e.g. the frozen LPIPS weights, `dgs_b200.lpips.LPIPS.lpips_state_dict(
    "loss_computer.lpips_loss_module.")`) is merged in unchanged."""
    sd = {SYSTEM_PREFIX + k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    if extra_state_dict:
        clash = [k for k in extra_state_dict if k in sd]
        if clash:
            raise ValueError(f"extra_state_dict overrides denoiser keys: {clash[:4]}")
        sd.update(extra_state_dict)
    return {"state_dict": sd, "epoch": int(epoch), "global_step": int(global_step)}


def save_system_checkpoint(model, path, epoch=0, global_step=0, extra_state_dict=None):
    torch.save(system_checkpoint(model, epoch, global_step, extra_state_dict), path)
    return path


def ema_checkpoint_path(path):
    """EMAModelCheckpoint._ema_format_filepath (diffusionGS/utils/ema.py:205-206): "x.ckpt" -> "x-EMA.ckpt"."""
    path = str(path)
    return path.replace(".ckpt", "-EMA.ckpt") if ".ckpt" in path else path + "-EMA"


def save_ema_checkpoint(trainer, path, epoch=0, global_step=0, extra_state_dict=None):
    """What EMAModelCheckpoint._save_checkpoint adds next to every checkpoint (ema.py:191-203): the same Lightning layout
    with the EMA weights in place of the trained ones, written to "<name>-EMA.ckpt".  `path` is the REGULAR checkpoint's
    path; returns the EMA file's path."""
    sd = {SYSTEM_PREFIX + k: v.detach().cpu().clone() for k, v in trainer.ema_state_dict().items()}
    for k, v in trainer.model.state_dict().items():  # non-parameter entries (none today) keep their live values
        sd.setdefault(SYSTEM_PREFIX + k, v.detach().cpu().clone())
    if extra_state_dict:
        sd.update(extra_state_dict)
    out = ema_checkpoint_path(path)
    torch.save({"state_dict": sd, "epoch": int(epoch), "global_step": int(global_step)}, out)
    return out


def module_weights(path_or_obj, module_name="shape_model", map_location="cpu"):
    """Same contract as the reference's `load_module_weights(path, module_name=...)` (utils/misc.py:40-70)."""
    ckpt = torch.load(path_or_obj, map_location=map_location, weights_only=False) if isinstance(path_or_obj, (str, bytes)) \
        else path_or_obj
    out = {}
    for k, v in ckpt["state_dict"].items():
        m = re.match(rf"^{re.escape(module_name)}\.(.*)$", k)
        if m is not None:
            out[m.group(1)] = v
    return out, ckpt.get("epoch", 0), ckpt.get("global_step", 0)
