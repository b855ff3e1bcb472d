"""LPIPS-VGG perceptual distance on libdgs_b200.so (dgs_lpips_forward / dgs_lpips_backward): a drop-in for
`lpips.LPIPS(net="vgg")` (lpips 0.1, eval mode) as `LossComputer(lpips_module=...)`, without the `lpips` package.

    lp = LPIPS.from_checkpoint("obj_ckpt.ckpt")     # the reference's checkpoints carry the LPIPS weights
    d = lp(rendering * 2 - 1, target * 2 - 1)       # [n, 3, H, W] in [-1, 1] -> [n, 1, 1, 1]

The distance is differentiated w.r.t. the first input (the rendering) only, as in the reference's training loss.  H and W
must be multiples of 16.  The VGG convolutions run on the library's wgmma GEMM with bf16 operands and fp32 accumulation.
"""
import ctypes as C

import torch
import torch.nn as nn

from . import _lib
from ._lib import LpipsWeights, check, stream
from .checkpoint import LPIPS_PREFIXES, lpips_state_dict

CONV_INDEX = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)   # torchvision vgg16().features indices of the 13 convs
_SLICE = (1, 1, 2, 2, 3, 3, 3, 4, 4, 4, 5, 5, 5)                 # lpips.pretrained_networks.vgg16 slice of each
CONV_CHANNELS = (3, 64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512)  # C_in of conv l = [l], C_out = [l+1]
TAP_CHANNELS = (64, 128, 256, 512, 512)
WORKSPACE_BYTES = 2 << 30  # default cap on the per-call workspace; the images are processed in chunks that fit


def conv_key(l):
    return f"net.slice{_SLICE[l]}.{CONV_INDEX[l]}"


def parse_state_dict(sd):
    """lpips-layout state dict (bare, or under either checkpoint prefix) -> {"conv_w": [13], "conv_b": [13], "lin": [5],
    "shift", "scale"} of fp32 CPU tensors.  lin{k} and lins.{k} keys are both accepted (equal when both present).
    Missing, unexpected or mis-shaped entries raise."""
    if any(k.startswith(LPIPS_PREFIXES) for k in sd):
        sd = lpips_state_dict(sd)
    sd = dict(sd)
    used = set()

    def take(key, shape):
        if key not in sd:
            raise KeyError(f"LPIPS state dict: missing {key!r}")
        v = torch.as_tensor(sd[key]).detach().to("cpu", torch.float32)
        if tuple(v.shape) != tuple(shape):
            raise ValueError(f"LPIPS state dict: {key!r} has shape {tuple(v.shape)}, expected {tuple(shape)}")
        used.add(key)
        return v

    out = dict(conv_w=[], conv_b=[], lin=[])
    for l in range(13):
        ci, co = CONV_CHANNELS[l], CONV_CHANNELS[l + 1]
        out["conv_w"].append(take(conv_key(l) + ".weight", (co, ci, 3, 3)))
        out["conv_b"].append(take(conv_key(l) + ".bias", (co,)))
    for k, c in enumerate(TAP_CHANNELS):
        a, b = f"lin{k}.model.1.weight", f"lins.{k}.model.1.weight"
        if a not in sd and b not in sd:
            raise KeyError(f"LPIPS state dict: missing {a!r} (or {b!r})")
        vals = [take(key, (1, c, 1, 1)) for key in (a, b) if key in sd]
        if len(vals) == 2 and not torch.equal(vals[0], vals[1]):
            raise ValueError(f"LPIPS state dict: {a!r} and {b!r} differ")
        out["lin"].append(vals[0].reshape(c))
    for name in ("shift", "scale"):
        key = f"scaling_layer.{name}"
        if key not in sd:
            raise KeyError(f"LPIPS state dict: missing {key!r}")
        v = torch.as_tensor(sd[key]).detach().to("cpu", torch.float32)
        if v.numel() != 3:
            raise ValueError(f"LPIPS state dict: {key!r} must hold 3 values, got shape {tuple(v.shape)}")
        used.add(key)
        out[name] = v.reshape(3)
    extra = sorted(set(sd) - used)
    if extra:
        raise ValueError(f"LPIPS state dict: unexpected keys {extra[:6]}")
    return out


def pack_weights(p, device):
    """weights (any floating dtype) -> the tensors of dgs_lpips_weights on `device` (see include/dgs_b200.h): bf16 conv
    matrices, everything else fp32, whatever dtype the module's buffers were converted to."""
    f32 = lambda v: v.to(device, torch.float32).contiguous()  # noqa: E731
    t = dict(conv_w=[], conv_wt=[], conv_b=[], lin=[])
    for l, (w, b) in enumerate(zip(p["conv_w"], p["conv_b"])):
        w = f32(w)
        co, ci = w.shape[:2]
        wk = w.permute(0, 2, 3, 1)                                   # [co, ky, kx, ci]
        if l == 0:
            wk = torch.nn.functional.pad(wk, (0, 8 - ci))            # C_in 3 -> 8
        t["conv_w"].append(wk.reshape(co, -1).to(torch.bfloat16).contiguous())
        wt = w.flip(2, 3).permute(1, 2, 3, 0).reshape(ci, 9 * co)    # Wt[ci, (ky, kx, co)] = W[co, ci, 2-ky, 2-kx]
        if l == 0:
            wt = torch.nn.functional.pad(wt, (0, 0, 0, 32 - ci))     # N 3 -> 32 rows for the GEMM
        t["conv_wt"].append(wt.to(torch.bfloat16).contiguous())
        t["conv_b"].append(f32(b))
    t["lin"] = [f32(v) for v in p["lin"]]
    t["shift"], t["scale"] = f32(p["shift"]), f32(p["scale"])
    s = LpipsWeights()
    for name in ("conv_w", "conv_wt", "conv_b", "lin"):
        arr = getattr(s, name)
        for i, v in enumerate(t[name]):
            arr[i] = v.data_ptr()
    s.shift, s.scale = t["shift"].data_ptr(), t["scale"].data_ptr()
    return s, t


def prepare_inputs(in0, in1):
    """Checks two [n, 3, H, W] floating-point images and returns them as contiguous fp32, the only element type the
    kernels read (fp16 / bf16 / fp64 images are converted; integer images raise)."""
    if in0.dim() != 4 or in0.shape[1] != 3 or tuple(in1.shape) != tuple(in0.shape):
        raise ValueError(f"LPIPS: expected two [n, 3, H, W] inputs, got {tuple(in0.shape)} and {tuple(in1.shape)}")
    if not (in0.is_floating_point() and in1.is_floating_point()):
        raise TypeError(f"LPIPS: expected floating-point images, got {in0.dtype} and {in1.dtype}")
    return in0.to(torch.float32).contiguous(), in1.to(torch.float32).contiguous()


class _LpipsFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, in0, in1, module):
        in_dtype = in0.dtype
        in0, in1 = prepare_inputs(in0, in1)
        n, _, H, W = in0.shape
        if not in0.is_cuda or in1.device != in0.device:
            raise _lib.DgsError("LPIPS needs both inputs on the same CUDA device (no CPU fallback)")
        dev = in0.device
        w, keep = module.packed_weights(dev)
        L = _lib.lib()
        out = torch.empty(n, dtype=torch.float32, device=dev)
        train = ctx.needs_input_grad[0]
        state = torch.empty(L.dgs_lpips_state_bytes(n, H, W), dtype=torch.uint8, device=dev) if train else None
        ws = module.workspace(n, H, W, dev)
        check(L.dgs_lpips_forward(C.byref(w), n, H, W, in0.data_ptr(), in1.data_ptr(), out.data_ptr(),
                                  state.data_ptr() if train else None, ws.data_ptr(), ws.numel(), stream(dev)))
        if train:
            ctx.saved = (w, keep, state, module, (n, H, W), in_dtype)
        return out.view(n, 1, 1, 1)

    @staticmethod
    def backward(ctx, dout):
        w, keep, state, module, (n, H, W), in_dtype = ctx.saved
        dev = state.device
        d = dout.reshape(n).to(torch.float32).contiguous()
        d_in0 = torch.empty(n, 3, H, W, dtype=torch.float32, device=dev)
        ws = module.workspace(n, H, W, dev)
        check(_lib.lib().dgs_lpips_backward(C.byref(w), n, H, W, state.data_ptr(), d.data_ptr(), d_in0.data_ptr(),
                                            ws.data_ptr(), ws.numel(), stream(dev)))
        ctx.saved = None
        return d_in0.to(in_dtype), None, None


class LPIPS(nn.Module):
    """`lpips.LPIPS(net="vgg")` in eval mode on the library's kernels: forward(in0, in1) -> [n, 1, 1, 1] fp32.
    Images of any floating dtype are read as fp32; the gradient w.r.t. in0 comes back in in0's dtype.
    Build it with `from_state_dict` / `from_checkpoint`; `lpips_state_dict` gives the weights back in the lpips layout
    (e.g. for the "loss_computer.lpips_loss_module." keys of a system checkpoint).  The weights are frozen, non-persistent
    buffers (no parameters); `max_workspace_bytes` caps the scratch memory of one call (the images are then processed in
    chunks)."""

    def __init__(self, state_dict):
        super().__init__()
        p = parse_state_dict(state_dict)
        for l in range(13):
            self.register_buffer(f"conv{l}_weight", p["conv_w"][l], persistent=False)
            self.register_buffer(f"conv{l}_bias", p["conv_b"][l], persistent=False)
        for k in range(5):
            self.register_buffer(f"lin{k}_weight", p["lin"][k], persistent=False)
        self.register_buffer("shift", p["shift"], persistent=False)
        self.register_buffer("scale", p["scale"], persistent=False)
        self.max_workspace_bytes = WORKSPACE_BYTES
        self._packed, self._packed_key = None, None
        self.eval()

    @classmethod
    def from_state_dict(cls, sd):
        return cls(sd)

    @classmethod
    def from_checkpoint(cls, path_or_obj, map_location="cpu"):
        """Any checkpoint layout `checkpoint.extract_denoiser_state_dict` reads (Lightning, release, bare), with the
        weights under "loss_computer.lpips_loss_module." or "denoiser.loss_computer.lpips_loss_module."."""
        obj = path_or_obj if isinstance(path_or_obj, dict) else torch.load(path_or_obj, map_location=map_location,
                                                                            weights_only=False)
        sd = lpips_state_dict(obj)
        if not sd:
            raise KeyError("checkpoint holds no LPIPS weights (loss_computer.lpips_loss_module.*)")
        return cls(sd)

    def weights(self):
        """-> the fp32 weights in the layout of parse_state_dict."""
        return dict(conv_w=[getattr(self, f"conv{l}_weight") for l in range(13)],
                    conv_b=[getattr(self, f"conv{l}_bias") for l in range(13)],
                    lin=[getattr(self, f"lin{k}_weight") for k in range(5)], shift=self.shift, scale=self.scale)

    def lpips_state_dict(self, prefix=""):
        """-> the weights as `lpips.LPIPS(net="vgg").state_dict()` holds them (fp32, CPU), every key under `prefix`:
        net.slice{s}.{i}.weight / .bias, lin{k}.model.1.weight and its lins.{k} twin, scaling_layer.shift / .scale."""
        w = self.weights()
        cpu = lambda v: v.detach().to("cpu", torch.float32).clone()  # noqa: E731
        sd = {}
        for l in range(13):
            sd[conv_key(l) + ".weight"] = cpu(w["conv_w"][l])
            sd[conv_key(l) + ".bias"] = cpu(w["conv_b"][l])
        for k in range(5):
            sd[f"lin{k}.model.1.weight"] = cpu(w["lin"][k]).view(1, -1, 1, 1)
            sd[f"lins.{k}.model.1.weight"] = sd[f"lin{k}.model.1.weight"].clone()
        sd["scaling_layer.shift"] = cpu(w["shift"]).view(1, 3, 1, 1)
        sd["scaling_layer.scale"] = cpu(w["scale"]).view(1, 3, 1, 1)
        return {prefix + k: v for k, v in sd.items()}

    def packed_weights(self, device):
        bufs = list(self.buffers())
        key = (str(device),) + tuple((b.data_ptr(), b._version) for b in bufs)
        if self._packed is None or self._packed_key != key:
            self._packed, self._packed_key = pack_weights(self.weights(), device), key
        return self._packed

    def workspace(self, n, H, W, device):
        L = _lib.lib()
        per = L.dgs_lpips_workspace_bytes(1, H, W)
        c = max(1, min(n, self.max_workspace_bytes // per))
        return torch.empty(L.dgs_lpips_workspace_bytes(c, H, W), dtype=torch.uint8, device=device)

    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(self, in0, in1, normalize=False):
        if in1.requires_grad:
            raise ValueError("LPIPS: the gradient w.r.t. the second input (the target) is not computed; pass it detached")
        if normalize:  # lpips.LPIPS's option: inputs in [0, 1]
            in0, in1 = 2 * in0 - 1, 2 * in1 - 1
        return _LpipsFunction.apply(in0, in1, self)
