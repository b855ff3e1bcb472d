"""Host-side mirror of the reference denoiser modules (diffusionGS/models/denoiser/denoiser.py:167-446,
denoiser_scene.py:172-457) on top of libdgs_b200.so.

* same registry names ("diffusion-gs-model", "diffusion-gs-model-scene"), same Config fields, same
  `state_dict` keys/shapes so a reference checkpoint loads with strict=True;
* same methods: forward(input_batch, timesteps), image_to_gaussians(images, ray_o, ray_d, t, training=False),
  render_gaussians(params, c2w, fxfycxcy, H, W), prepare_to_save, `dtype`, `gs_renderer`;
* the arithmetic is ONE C-ABI call (dgs_dit_forward: wgmma GEMMs + wgmma attention + fused glue);
  the nn.Linear / nn.LayerNorm objects below only HOLD parameters under the reference's names, their
  forward() is never used.  Training: dgs_b200/train.py (DitTrainer) attaches the backward.
"""
import ctypes as C

import torch
import torch.nn as nn

from . import _lib
from ._lib import DitIO, DitWeights, DitWeightsFp8, check
from .renderer import Renderer

_REGISTRY = {}


def register(name):
    def deco(cls):
        _REGISTRY[name] = cls
        return cls
    return deco


def find(name):
    """Counterpart of `diffusionGS.find` (diffusionGS/__init__.py:19-29) for the two hot-path modules."""
    return _REGISTRY[name]


class AttrDict(dict):
    """Stand-in for easydict.EasyDict (absent offline): attribute access to the Gaussian parameter dict."""
    __getattr__ = dict.__getitem__
    __setattr__ = dict.__setitem__


_DEFAULTS = dict(pretrained_model_name_or_path="", use_downsample=False, num_latents=256, width=1024, in_channels=9,
                 patch_size=16, n_gaussians=2, dim_heads=64, num_layers=24, ray_pe_type="relative_plk",
                 hard_pixelalign=True, clip_xyz=True, gaussians_sh_degree=0, use_gssplat=False,
                 prior_distribution="gaussian", use_flash=False, use_checkpoint=True, grad_checkpoint_every=1,
                 range_setting_type="linear_depth", range_setting_near=0.0, range_setting_far=500.0)
# in_channels: the reference class default is 3 (denoiser.py:181) but its tokenizer is
# Linear(in_channels * patch^2, width) fed with the 9-channel posed image (rgb + 6 Pluecker), so only in_channels == 9
# -- what every shipped yaml sets (configs/*.yaml "in_channels: 9 #rgb+plucker") -- can run; 9 is the default here and
# anything else is rejected.  range_setting_type is carried for config compatibility only: the reference's range_func
# is sigmoid(t)*(far-near)+near whatever it says (denoiser_scene.py:263).


def _cfg(cfg):
    d = dict(_DEFAULTS)
    if cfg is not None:
        items = cfg.items() if hasattr(cfg, "items") else vars(cfg).items()
        for k, v in items:
            if not k.startswith("_"):
                d[k] = v
    return AttrDict(d)


class _AttnParams(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.qkv = nn.Linear(dim, 3 * dim, bias=True)
        self.proj = nn.Linear(dim, dim, bias=True)


class _MlpParams(nn.Module):
    def __init__(self, dim, hidden):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden, bias=True)
        self.fc2 = nn.Linear(hidden, dim, bias=True)


class _BlockParams(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.attn = _AttnParams(dim)
        self.mlp = _MlpParams(dim, 4 * dim)
        self.adaLN_modulation = nn.Sequential(nn.SiLU(), nn.Linear(dim, 6 * dim, bias=True))


class _HeadParams(nn.Module):
    def __init__(self, dim, out):
        super().__init__()
        self.layernorm = nn.LayerNorm(dim, bias=False)
        self.linear = nn.Linear(dim, out, bias=False)
        self.adaLN_modulation = nn.Sequential(nn.SiLU(), nn.Linear(dim, 2 * dim, bias=True))


class _TEmbedParams(nn.Module):
    def __init__(self, dim, freq=256):
        super().__init__()
        self.mlp = nn.Sequential(nn.Linear(freq, dim, bias=True), nn.SiLU(), nn.Linear(dim, dim, bias=True))


def _init_linear(m):  # utils_transformer.py:30-36
    if isinstance(m, nn.Linear):
        nn.init.normal_(m.weight, mean=0.0, std=0.02)
        if m.bias is not None:
            nn.init.zeros_(m.bias)


@register("diffusion-gs-model")
class DGSDenoiser(nn.Module):
    SCENE = False

    def __init__(self, cfg=None):
        super().__init__()
        self.cfg = c = _cfg(cfg)
        w = c.width
        if c.in_channels != 9:
            raise ValueError(f"in_channels={c.in_channels}: the tokenizer consumes the 9-channel posed image (rgb + Pluecker); "
                             "every shipped reference config sets in_channels: 9")
        if c.ray_pe_type not in ("relative_plk", "plk"):
            raise ValueError(f"ray_pe_type={c.ray_pe_type!r} (expected 'relative_plk' or 'plk')")
        if c.gaussians_sh_degree != 0:
            raise NotImplementedError("the DiT heads are built for gaussians_sh_degree == 0 (every shipped config)")
        self.t_embedder = _TEmbedParams(w)
        nn.init.normal_(self.t_embedder.mlp[0].weight, std=0.02)
        nn.init.normal_(self.t_embedder.mlp[2].weight, std=0.02)
        self.image_tokenizer = nn.Sequential(nn.Identity(),
                                             nn.Linear(c.in_channels * c.patch_size ** 2, w, bias=False))  # denoiser.py:216-221
        self.image_tokenizer.apply(_init_linear)
        shape = (1, c.n_gaussians, w) if self.SCENE else (c.n_gaussians, w)
        self.gaussians_pos_embedding = nn.Parameter(torch.randn(*shape))
        nn.init.trunc_normal_(self.gaussians_pos_embedding, std=0.02)
        self.transformer_input_layernorm = nn.LayerNorm(w, bias=False)
        self.transformer = nn.ModuleList([_BlockParams(w) for _ in range(c.num_layers)])
        self.transformer.apply(_init_linear)
        self.upsampler = _HeadParams(w, 14)
        self.upsampler.apply(_init_linear)
        self.image_token_decoder = _HeadParams(w, c.patch_size ** 2 * 14)
        self.image_token_decoder.apply(_init_linear)
        self.gs_renderer = Renderer(c)
        self.register_buffer("_dummy", torch.zeros(0, dtype=torch.float32), persistent=False)  # dGS/utils/base.py:115
        self._packed = None
        self._packed_key = None
        self._packed_fp8 = None
        self._packed_fp8_key = None
        self._precision = "bf16"
        if c.pretrained_model_name_or_path:
            sd = torch.load(c.pretrained_model_name_or_path, map_location="cpu", weights_only=False)
            if "model" in sd:  # denoiser.py:259-268
                sd = {k.replace("denoiser.", ""): v for k, v in sd["model"].items()
                      if k.startswith("denoiser.") and not k.startswith("denoiser.loss_computer")}
            self.load_state_dict(sd, strict=True)

    # ---- weight packing: fp32 master parameters -> the bf16 / stacked layout of dgs_dit_weights ----
    def _pack_key(self):
        return tuple((p.data_ptr(), p._version) for p in self.parameters())

    def _pack_dict(self, skip=()):
        """fp32 master parameters -> {field of dgs_dit_weights: tensor}; `skip` = fields somebody else fills."""
        bf = lambda t: t.detach().to(torch.bfloat16).contiguous()  # noqa: E731

        def split(t):  # split-bf16 weight [n, 3k] = [hi | hi | lo]  (see include/dgs_b200.h)
            t = t.detach().float()
            hi = t.to(torch.bfloat16)
            lo = (t - hi.float()).to(torch.bfloat16)
            return torch.cat([hi, hi, lo], dim=1).contiguous()

        f32 = lambda t: t.detach().float().contiguous()  # noqa: E731
        T = self.transformer
        stack = lambda get: torch.stack([get(b).detach() for b in T])  # noqa: E731
        heads = (self.upsampler, self.image_token_decoder)
        make = dict(
            tokenizer_w=lambda: split(self.image_tokenizer[1].weight), pos_embed=lambda: f32(self.gaussians_pos_embedding),
            in_ln_w=lambda: f32(self.transformer_input_layernorm.weight),
            t0_w=lambda: f32(self.t_embedder.mlp[0].weight), t0_b=lambda: f32(self.t_embedder.mlp[0].bias),
            t2_w=lambda: f32(self.t_embedder.mlp[2].weight), t2_b=lambda: f32(self.t_embedder.mlp[2].bias),
            adaln_w=lambda: f32(torch.cat([b.adaLN_modulation[1].weight.detach() for b in T] +
                                          [h.adaLN_modulation[1].weight.detach() for h in heads], dim=0)),
            adaln_b=lambda: f32(torch.cat([b.adaLN_modulation[1].bias.detach() for b in T] +
                                          [h.adaLN_modulation[1].bias.detach() for h in heads], dim=0)),
            qkv_w=lambda: bf(stack(lambda b: b.attn.qkv.weight)), qkv_b=lambda: f32(stack(lambda b: b.attn.qkv.bias)),
            proj_w=lambda: bf(stack(lambda b: b.attn.proj.weight)), proj_b=lambda: f32(stack(lambda b: b.attn.proj.bias)),
            fc1_w=lambda: bf(stack(lambda b: b.mlp.fc1.weight)), fc1_b=lambda: f32(stack(lambda b: b.mlp.fc1.bias)),
            fc2_w=lambda: bf(stack(lambda b: b.mlp.fc2.weight)), fc2_b=lambda: f32(stack(lambda b: b.mlp.fc2.bias)),
            ups_ln_w=lambda: f32(self.upsampler.layernorm.weight), ups_w=lambda: split(self.upsampler.linear.weight),
            dec_ln_w=lambda: f32(self.image_token_decoder.layernorm.weight),
            dec_w=lambda: split(self.image_token_decoder.linear.weight))
        return {k: fn() for k, fn in make.items() if k not in skip}

    def packed_weights(self, force=False):
        key = self._pack_key()
        if self._packed is not None and self._packed_key == key and not force:
            return self._packed
        t = self._pack_dict()
        c = self.cfg
        w = DitWeights(width=c.width, heads=c.width // c.dim_heads, layers=c.num_layers, patch=c.patch_size,
                       n_gaussians=c.n_gaussians, mlp_hidden=4 * c.width)
        assert tuple(self.image_tokenizer[1].weight.shape) == (c.width, 9 * c.patch_size ** 2), "tokenizer weight shape"
        for k, v in t.items():
            setattr(w, k, v.data_ptr())
        self._packed, self._packed_key = (w, t), key
        return self._packed

    def packed_weights_fp8(self):
        """The qkv / fc1 / fc2 weights of every block in the FP8 format of dgs_dit_weights_fp8 (e4m3 + one power-of-two
        scale per output channel, quantized by dgs_quantize_rows_e4m3), re-packed when any parameter changed."""
        key = self._pack_key()
        if self._packed_fp8 is not None and self._packed_fp8_key == key:
            return self._packed_fp8
        L = _lib.lib()
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        w8, t = DitWeightsFp8(), {}
        for name, get in (("qkv", lambda b: b.attn.qkv.weight), ("fc1", lambda b: b.mlp.fc1.weight),
                          ("fc2", lambda b: b.mlp.fc2.weight)):
            src = torch.stack([get(b).detach().float() for b in self.transformer]).contiguous()
            n_layers, n, k = src.shape
            q = torch.empty(n_layers, n, k, dtype=torch.uint8, device=src.device)
            s = torch.empty(n_layers, n, dtype=torch.float32, device=src.device)
            check(L.dgs_quantize_rows_e4m3(src.data_ptr(), n_layers * n, k, q.data_ptr(), s.data_ptr(), stream))
            t[name + "_w"], t[name + "_s"] = q, s
            setattr(w8, name + "_w", q.data_ptr())
            setattr(w8, name + "_s", s.data_ptr())
        self._packed_fp8, self._packed_fp8_key = (w8, t), key
        return self._packed_fp8

    # ---- inference precision ----
    def set_inference_precision(self, precision):
        """"bf16" (default): every GEMM on bf16 operands.  "fp8": inference runs the qkv, mlp.fc1 and mlp.fc2 GEMMs of
        every block on e4m3 operands with power-of-two scales (dgs_dit_forward_fp8); training refuses to run."""
        if precision not in ("bf16", "fp8"):
            raise ValueError(f"inference precision {precision!r} (expected 'bf16' or 'fp8')")
        self._precision = precision
        return self

    @property
    def inference_precision(self):
        return self._precision

    # ---- reference API ----
    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    def image_to_gaussians(self, images, ray_o, ray_d, t, training: bool = False, return_tokens: bool = False):
        """denoiser.py:306-416.  Inference: one dgs_dit_forward call under no_grad.  With autograd enabled on a module
        in train() mode that has a DitTrainer attached (dgs_b200/train.py), the call is recorded as ONE autograd node
        whose backward is dgs_dit_backward (activations stored, not recomputed)."""
        if torch.is_grad_enabled() and self.training and getattr(self, "_trainer", None) is not None:
            if self._precision == "fp8":
                raise RuntimeError("DGSDenoiser: FP8 is an inference precision; training runs bf16 "
                                   "(set_inference_precision('bf16') before a training forward)")
            from .train import dit_train_forward
            out, img_xyz = dit_train_forward(self, images, ray_o, ray_d, t)
            return (out, img_xyz, None) if return_tokens else (out, img_xyz)
        tr = getattr(self, "_trainer", None)
        if tr is not None and tr._pending:
            raise RuntimeError("DGSDenoiser: a training forward is pending; an inference call would overwrite the workspace "
                               "its backward reads (run backward first, or trainer.reset())")
        with torch.no_grad():
            out, img_xyz, tokens, _ = self._run_dit(images, ray_o, ray_d, t, return_tokens=return_tokens)
            if self.cfg.clip_xyz and training and not self.SCENE:  # denoiser.py:395-396 (never taken by the reference's callers)
                n_img = images.shape[1] * images.shape[3] * images.shape[4]
                out.xyz[:, -n_img:] = out.xyz[:, -n_img:].clamp(-1.0, 1.0)
                img_xyz = img_xyz.clamp(-1.0, 1.0)
        return (out, img_xyz, tokens) if return_tokens else (out, img_xyz)

    def _run_dit(self, images, ray_o, ray_d, t, return_tokens=False, train_state=None, train_mode=0):
        dev = self.device
        if dev.type != "cuda":
            raise _lib.DgsError("DGSDenoiser runs on a CUDA device only (no CPU / PyTorch fallback)")
        c = self.cfg
        images = images[:, :, :3].detach().float().contiguous()
        ray_o, ray_d = ray_o.detach().float().contiguous(), ray_d.detach().float().contiguous()
        B, V, _, H, W = images.shape
        P = c.n_gaussians + V * H * W
        tf = t.to(device=dev, dtype=torch.float32).contiguous()
        w, _keep = self.packed_weights()
        with torch.cuda.device(dev):
            new = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)  # noqa: E731
            out = AttrDict(xyz=new(B, P, 3), features=new(B, P, 1, 3), scaling=new(B, P, 3), rotation=new(B, P, 4),
                           opacity=new(B, P, 1))
            img_xyz = new(B, V, 3, H, W)
            n_tok = c.n_gaussians + V * (H // c.patch_size) * (W // c.patch_size)
            tokens = new(B, n_tok, c.width) if return_tokens else None
            L = _lib.lib()
            fp8 = self._precision == "fp8" and train_state is None
            nbytes = (L.dgs_dit_workspace_bytes_fp8 if fp8 else L.dgs_dit_workspace_bytes)(C.byref(w), B, V, H, W)
            if nbytes == 0:
                raise _lib.DgsError(L.dgs_last_error().decode())
            ws = getattr(self, "_workspace", None)  # grow-only, re-used step after step
            if ws is None or ws.numel() < nbytes or ws.device != dev:
                ws = self._workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            io = DitIO(B=B, V=V, H=H, W=W, plucker_mode=0 if c.ray_pe_type == "relative_plk" else 1,
                       scene_depth=1 if self.SCENE else (0 if c.ray_pe_type == "relative_plk" else 2), range_near=float(c.range_setting_near),
                       range_far=float(c.range_setting_far), images=images.data_ptr(), ray_o=ray_o.data_ptr(),
                       ray_d=ray_d.data_ptr(), t=tf.data_ptr(), xyz=out.xyz.data_ptr(),
                       features=out.features.data_ptr(), scaling=out.scaling.data_ptr(),
                       rotation=out.rotation.data_ptr(), opacity=out.opacity.data_ptr(),
                       img_aligned_xyz=img_xyz.data_ptr(), tokens_out=None if tokens is None else tokens.data_ptr(),
                       train_state=None if train_state is None else train_state.data_ptr(), train_mode=int(train_mode))
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            if fp8:
                w8, _keep8 = self.packed_weights_fp8()
                check(L.dgs_dit_forward_fp8(C.byref(w), C.byref(w8), C.byref(io), ws.data_ptr(), nbytes, stream))
            else:
                check(L.dgs_dit_forward(C.byref(w), C.byref(io), ws.data_ptr(), nbytes, stream))
        keep = (io, ws, nbytes, images, ray_o, ray_d, tf, w, _keep)  # what a later dgs_dit_backward needs alive
        return out, img_xyz, tokens, keep

    def render_gaussians(self, gaussian_params, c2w, fxfycxcy, height, width):
        g = gaussian_params
        return self.gs_renderer(g.xyz, g.features, g.scaling, g.rotation, g.opacity, height, width, C2W=c2w,
                                fxfycxcy=fxfycxcy)

    def prepare_to_save(self, gaussians_parameters):
        out = []
        for b in range(gaussians_parameters.xyz.size(0)):
            m = self.gs_renderer.new_gaussians_model()
            m.empty()
            out.append(m.set_data(*(gaussians_parameters[k][b].detach().float()
                                    for k in ("xyz", "features", "scaling", "rotation", "opacity"))))
        return out

    def forward(self, input_batch, timesteps):
        params, _ = self.image_to_gaussians(input_batch["image"], input_batch["ray_o"], input_batch["ray_d"], timesteps)
        img = input_batch["image"]
        renders = self.render_gaussians(params, input_batch["c2w"], input_batch["fxfycxcy"], img.shape[3], img.shape[4])
        return renders, self.prepare_to_save(params)


@register("diffusion-gs-model-scene")
class DGSDenoiserScene(DGSDenoiser):
    SCENE = True
