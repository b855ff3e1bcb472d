"""Training side of the DiT hot path: the backward of DGSDenoiser.image_to_gaussians as ONE
autograd node over libdgs_b200.so (dgs_dit_backward), flat fp32 master parameters / gradients / Adam moments, the
fused AdamW update (diffusionGS/configs/diffusionGS_rel.yaml:57-62) and the gradient all-reduce (dist.GradArena).

The reference trains through torch autograd with `torch.utils.checkpoint` around every block (denoiser.py:348-354),
i.e. it runs the forward twice.  Here the forward keeps its activations in one big HBM buffer (4 GB per sample at
N = 4098 tokens; an H100 has 80 GB) and the backward consumes them: fwd + 2x bwd FLOPs instead of 2x fwd + 2x bwd.
"""
import ctypes as C

import torch

from . import _lib
import contextlib

import torch.distributed as dist

from ._lib import DitBwdOpts, DitGrads, DitOutGrads, DitWeightsT, check, stream
from .denoiser import head_channels
from .dist import GradArena, gradient_group


class DitTrainer:
    """Owns the flat training state of one DGSDenoiser (one process per GPU).

    * `master`: every parameter, fp32, in module.parameters() order; `p.data` are views of it;
    * `arena`:  the gradients in the same layout (dist.GradArena: `p.grad` are views; one bucket per block);
    * `exp_avg`, `exp_avg_sq`: AdamW moments, same layout -> the optimizer is ONE kernel over the whole model;
    * bf16 / transposed-bf16 GEMM weights are re-derived from `master` after each step (refresh_weights);
    * `ema` (ema_decay given): NeMo-style EMA of the parameters (diffusionGS/utils/ema.py, decay 0.9999 in launch.py:227),
      updated inside the AdamW kernel; `ema_state_dict` / `swap_ema_weights` / checkpoint.save_ema_checkpoint use it;
    * recompute=True: the forward keeps only the residual stream entering each block and the backward re-runs each block
      (the reference's per-block torch.utils.checkpoint, denoiser.py:348-354): 0.6 instead of 4 GB per sample;
    * accumulate_grad_batches=k: k forward/backward pairs per optimizer step (Lightning's option of the same name); each
      backward lands in the arena and is added to a second arena, the step uses their mean;
    * overlap_allreduce: with torch.distributed initialised (world > 1) the per-block buckets are all-reduced on a side
      stream WHILE the remaining blocks are still being differentiated (dgs_dit_backward_ex's block_done events).

    ONE training forward may be outstanding at a time (it owns the activation state and the workspace): a second
    grad-enabled forward before the first one's backward, a second backward through the same forward, or an optimizer step
    with a forward still pending raise instead of corrupting state."""

    def __init__(self, model, lr=1e-5, betas=(0.9, 0.99), eps=1e-8, weight_decay=0.01, clip=0.5, ema_decay=None,
                 recompute=False, accumulate_grad_batches=1, overlap_allreduce=True):
        self.model = model
        self.lr, self.betas, self.eps, self.weight_decay, self.clip = lr, betas, eps, weight_decay, clip
        if ema_decay is not None and not (0.0 <= ema_decay <= 1.0):
            raise ValueError("EMA decay value must be between 0 and 1")  # ema.py:56-57
        if accumulate_grad_batches < 1:
            raise ValueError("accumulate_grad_batches must be >= 1")
        self.ema_decay, self.recompute = ema_decay, bool(recompute)
        self.accumulate, self.overlap = int(accumulate_grad_batches), bool(overlap_allreduce)
        params = [p for p in model.parameters()]
        dev = params[0].device
        if dev.type != "cuda":
            raise _lib.DgsError("DitTrainer needs the model on a CUDA device (no CPU fallback)")
        total = sum(p.numel() for p in params)
        self.master = torch.empty(total, dtype=torch.float32, device=dev)
        off = 0
        for p in params:
            n = p.numel()
            self.master[off:off + n].copy_(p.data.reshape(-1))
            p.data = self.master[off:off + n].view_as(p)
            off += n
        self.arena = GradArena(model)
        assert self.arena.total == total
        self.exp_avg = torch.zeros_like(self.master)
        self.exp_avg_sq = torch.zeros_like(self.master)
        self.ema = self.master.clone() if ema_decay is not None else None  # ema.py:69-72: a copy at train start
        self._accum = torch.zeros_like(self.master) if self.accumulate > 1 else None
        self.steps = 0
        self._state = None
        self._pending = False     # a training forward whose backward has not run yet
        self._micro = 0           # backward passes since the last optimizer step
        self._reduced = False     # the overlapped all-reduce of this step has been issued
        self._events = None
        self._trace = None        # (names, dict) armed by trace_backward for the next backward
        self._group = gradient_group()  # CTA-capped communicator for the gradient exchange (None: default group / 1 rank)
        self._grads = self._grad_struct()
        self.anchor = torch.zeros(1, device=dev, requires_grad=True)  # makes autograd call our backward
        model._trainer = self
        self.refresh_weights()

    # -- pointers into the gradient arena, in the layout dgs_dit_grads wants --
    def _grad_struct(self):
        m = self.model
        T = m.transformer
        g = DitGrads()
        ptr = lambda p: p.grad.data_ptr()  # noqa: E731
        g.tokenizer_w, g.pos_embed, g.in_ln_w = ptr(m.image_tokenizer[1].weight), ptr(m.gaussians_pos_embedding), \
            ptr(m.transformer_input_layernorm.weight)
        g.t0_w, g.t0_b = ptr(m.t_embedder.mlp[0].weight), ptr(m.t_embedder.mlp[0].bias)
        g.t2_w, g.t2_b = ptr(m.t_embedder.mlp[2].weight), ptr(m.t_embedder.mlp[2].bias)
        fields = dict(qkv_w=lambda b: b.attn.qkv.weight, qkv_b=lambda b: b.attn.qkv.bias,
                      proj_w=lambda b: b.attn.proj.weight, proj_b=lambda b: b.attn.proj.bias,
                      fc1_w=lambda b: b.mlp.fc1.weight, fc1_b=lambda b: b.mlp.fc1.bias,
                      fc2_w=lambda b: b.mlp.fc2.weight, fc2_b=lambda b: b.mlp.fc2.bias,
                      adaln_w=lambda b: b.adaLN_modulation[1].weight, adaln_b=lambda b: b.adaLN_modulation[1].bias)
        stride = None
        for name, get in fields.items():
            setattr(g, name, ptr(get(T[0])))
            if len(T) > 1:
                st = (ptr(get(T[1])) - ptr(get(T[0]))) // 4
                assert stride in (None, st), "transformer blocks are not laid out with one common stride"
                stride = st
                assert all(ptr(get(T[i])) == ptr(get(T[0])) + 4 * st * i for i in range(len(T)))
        g.layer_stride = stride or 0
        u, d = m.upsampler, m.image_token_decoder
        g.ups_ln_w, g.ups_w = ptr(u.layernorm.weight), ptr(u.linear.weight)
        g.ups_adaln_w, g.ups_adaln_b = ptr(u.adaLN_modulation[1].weight), ptr(u.adaLN_modulation[1].bias)
        g.dec_ln_w, g.dec_w = ptr(d.layernorm.weight), ptr(d.linear.weight)
        g.dec_adaln_w, g.dec_adaln_b = ptr(d.adaLN_modulation[1].weight), ptr(d.adaLN_modulation[1].bias)
        return g

    _BIG = dict(qkv_w=lambda b: b.attn.qkv.weight, proj_w=lambda b: b.attn.proj.weight,
                fc1_w=lambda b: b.mlp.fc1.weight, fc2_w=lambda b: b.mlp.fc2.weight)

    def refresh_weights(self):
        """fp32 master -> the bf16 stacks the forward reads + the transposed bf16 stacks the dgrad GEMMs read.
        The packed tensors are allocated once and updated IN PLACE (the dgs_dit_weights struct keeps its pointers):
        the four big per-block matrices by one fused cast+transpose launch each (dgs_cast_transpose_f32, batched over
        the blocks through the master arena's block stride), the small vectors / split-bf16 end matrices by torch copies."""
        m = self.model
        T = m.transformer
        dev = self.master.device
        first = m._packed is None or getattr(self, "_wT_keep", None) is None
        if first:
            m.packed_weights(force=True)
            self._wT_keep = {k + "T": torch.empty(len(T), get(T[0]).shape[1], get(T[0]).shape[0], dtype=torch.bfloat16,
                                                  device=dev) for k, get in self._BIG.items()}
        w, t = m._packed
        L = _lib.lib()
        stride = int(self._grads.layer_stride)  # master and gradient arenas share one layout
        with torch.cuda.device(dev):
            for k, get in self._BIG.items():
                p0 = get(T[0])
                check(L.dgs_cast_transpose_f32(p0.data_ptr(), stride, len(T), p0.shape[0], p0.shape[1], t[k].data_ptr(),
                                               self._wT_keep[k + "T"].data_ptr(), stream(dev)))
        if not first:
            for k, v in m._pack_dict(skip=tuple(self._BIG) + ("sh_degree",)).items():
                t[k].copy_(v)
        m._packed_key = m._pack_key()
        self._wT_keep["dec_wT"] = m.image_token_decoder.linear.weight.detach().t().to(torch.bfloat16).contiguous()
        self._wT_keep["ups_w"] = m.upsampler.linear.weight.detach().float().contiguous()
        wT = DitWeightsT()
        for k, v in self._wT_keep.items():
            setattr(wT, k, v.data_ptr())
        self._wT = wT

    @property
    def train_mode(self):
        return _lib.TRAIN_RECOMPUTE if self.recompute else _lib.TRAIN_STORE

    def train_state(self, B, V, H, W):
        w, _ = self.model.packed_weights()
        n = _lib.lib().dgs_dit_train_state_bytes_ex(C.byref(w), B, V, H, W, self.train_mode)
        if n == 0:
            raise _lib.DgsError(_lib.lib().dgs_last_error().decode())
        if self._state is None or self._state.numel() < n:
            self._state = None
            self._state = torch.empty(n, dtype=torch.uint8, device=self.master.device)
        return self._state

    STATE_FIELDS = ("x", "x_mid", "h1", "qkv", "attn", "lse", "proj_out", "h2", "u_pre", "u", "fc2_out")

    def export_state(self, B, V, H, W, layer, names=("x",)):
        """Copies of block `layer`'s tensors from the last training forward at shape (B, V, H, W) (dgs_dit_export_state):
        {name: tensor} for `names` out of STATE_FIELDS.  "x" is the residual stream entering the block ([B, N, width]
        fp32; layer == num_layers: the final stream) in both modes; the others exist in store mode only (not recompute)."""
        unknown = set(names) - set(self.STATE_FIELDS)
        if unknown:
            raise ValueError(f"unknown train-state tensors {sorted(unknown)}; expected a subset of {self.STATE_FIELDS}")
        if self._state is None:
            raise RuntimeError("DitTrainer.export_state: no training forward has run")
        c = self.model.cfg
        w, _ = self.model.packed_weights()
        N = c.n_gaussians + V * (H // c.patch_size) * (W // c.patch_size)
        D, U, heads = c.width, 4 * c.width, c.width // c.dim_heads
        dev = self.master.device
        shapes = dict(x=(B, N, D), x_mid=(B, N, D), h1=(B, N, D), qkv=(B, N, 3 * D), attn=(B, N, D),
                      lse=(B, heads, (N + 127) // 128 * 128), proj_out=(B, N, D), h2=(B, N, D), u_pre=(B, N, U),
                      u=(B, N, U), fc2_out=(B, N, D))
        f32 = ("x", "x_mid", "lse")
        out = {k: torch.empty(shapes[k], dtype=torch.float32 if k in f32 else torch.bfloat16, device=dev) for k in names}
        args = [out[k].data_ptr() if k in out else None for k in self.STATE_FIELDS]
        with torch.cuda.device(dev):
            check(_lib.lib().dgs_dit_export_state(C.byref(w), B, V, H, W, self.train_mode, self._state.data_ptr(), int(layer),
                                                  *args, stream(dev)))
        return out

    ENDS_FIELDS = ("x_pre", "c", "mod", "gs_tok", "img_gs", "dx0", "dx_pre", "dmod", "dc", "d_gs_tok")

    def export_ends(self, B, V, H, W, names=("x_pre",)):
        """Copies of the tensors on either side of the blocks (dgs_dit_export_ends), all fp32: {name: tensor} for
        `names` out of ENDS_FIELDS.  From the last training forward at shape (B, V, H, W): x_pre [B, N, width] (tokens
        before the input LayerNorm), c [B, width] (conditioning before the adaLN SiLU), mod [B, L*6*width + 4*width]
        (adaLN table), gs_tok [B, G, C] and img_gs [B, T, p*p*C] (raw head outputs, C = 11 + 3 (sh_degree+1)^2
        channels per Gaussian).  From the backward that
        followed it (undefined before one): dx0 [B, N, width] (gradient entering block 0), dx_pre, dmod, dc and
        d_gs_tok, the gradients of x_pre, mod, c and gs_tok."""
        unknown = set(names) - set(self.ENDS_FIELDS)
        if unknown:
            raise ValueError(f"unknown end-stage tensors {sorted(unknown)}; expected a subset of {self.ENDS_FIELDS}")
        if self._state is None:
            raise RuntimeError("DitTrainer.export_ends: no training forward has run")
        c = self.model.cfg
        w, _ = self.model.packed_weights()
        p, G, D, Ch = c.patch_size, c.n_gaussians, c.width, head_channels(c.gaussians_sh_degree)
        T = V * (H // p) * (W // p)
        N, R = G + T, c.num_layers * 6 * D + 4 * D
        shapes = dict(x_pre=(B, N, D), c=(B, D), mod=(B, R), gs_tok=(B, G, Ch), img_gs=(B, T, p * p * Ch),
                      dx0=(B, N, D), dx_pre=(B, N, D), dmod=(B, R), dc=(B, D), d_gs_tok=(B, G, Ch))
        dev = self.master.device
        out = {k: torch.empty(shapes[k], dtype=torch.float32, device=dev) for k in names}
        args = [out[k].data_ptr() if k in out else None for k in self.ENDS_FIELDS]
        ws = self.model._workspace
        with torch.cuda.device(dev):
            check(_lib.lib().dgs_dit_export_ends(C.byref(w), B, V, H, W, self.train_mode, self._state.data_ptr(),
                                                 ws.data_ptr(), ws.numel(), *args, stream(dev)))
        return out

    def trace_backward(self, names=_lib.BWD_TRACE_FIELDS):
        """Arms the next backward to read out its per-block gradients (dgs_dit_bwd_opts.trace) and returns a dict that
        this backward fills with {name: tensor} for `names` out of BWD_TRACE_FIELDS, stacked over the layers (M = B*N
        rows as [B, N]): dx [L+1, B, N, width] fp32 (dx[l]: the gradient of the residual stream entering block l,
        dx[L]: the one the heads hand to the blocks), dx_mid [L, B, N, width] fp32, dsum [L, B, heads, round_up(N, 128)]
        fp32, du_pre [L, B, N, 4*width] bf16, dqkv [L, B, N, 3*width] bf16 and d_fc2_out, dh2, d_proj_out, d_attn, dh1
        [L, B, N, width] bf16.  In both train modes; one call traces one backward."""
        unknown = set(names) - set(_lib.BWD_TRACE_FIELDS)
        if unknown:
            raise ValueError(f"unknown backward trace tensors {sorted(unknown)}; expected a subset of {_lib.BWD_TRACE_FIELDS}")
        out = {}
        self._trace = (tuple(names), out)
        return out

    def _take_trace(self, B, V, H, W):
        """The armed trace's buffers for a backward at shape (B, V, H, W) -> DitBwdTrace (None: not armed); disarms."""
        if self._trace is None:
            return None
        names, out = self._trace
        self._trace = None
        c = self.model.cfg
        L, D = c.num_layers, c.width
        N = c.n_gaussians + V * (H // c.patch_size) * (W // c.patch_size)
        shapes = dict(dx=(L + 1, B, N, D), du_pre=(L, B, N, 4 * D), dqkv=(L, B, N, 3 * D),
                      dsum=(L, B, D // c.dim_heads, (N + 127) // 128 * 128))
        for k in names:
            dt = torch.float32 if k in ("dx", "dx_mid", "dsum") else torch.bfloat16
            out[k] = torch.empty(shapes.get(k, (L, B, N, D)), dtype=dt, device=self.master.device)
        return _lib.DitBwdTrace(**{k: out[k].data_ptr() for k in names})

    def zero_grad(self):
        self.arena.zero_()
        if self._accum is not None:
            self._accum.zero_()
        self._micro = 0

    def reset(self):
        """Drop an outstanding training forward (e.g. after an exception between forward and backward)."""
        self._pending, self._reduced = False, False

    # -- hooks called by _DitFunction --
    def _begin_forward(self):
        if self._pending:
            raise RuntimeError("DitTrainer: a training forward is already pending (its backward has not run). The trainer "
                               "holds ONE activation state; run backward first, wrap evaluation in torch.no_grad(), or call "
                               "trainer.reset() to drop the pending forward.")
        if self._reduced:
            raise RuntimeError("DitTrainer: gradients of this step were already all-reduced; call optimizer_step() "
                               "before the next forward")
        self._pending = True

    def _world(self):
        return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1

    def _bwd_opts(self):
        """block_done events for the overlapped all-reduce, or None when there is nothing to overlap with."""
        last_micro = self._micro + 1 >= self.accumulate
        if not (self.overlap and self._world() > 1 and self.accumulate == 1 and last_micro):
            return None
        if self._events is None:
            n = len(self.model.transformer) + 1
            arr = (C.c_void_p * n)()
            for i in range(n):
                ev = C.c_void_p()
                check(_lib.lib().dgs_event_create(C.byref(ev)))
                arr[i] = ev.value
            self._events = arr
        return DitBwdOpts(block_done=C.cast(self._events, C.POINTER(C.c_void_p)))

    def _end_backward(self, overlapped):
        self._pending = False
        self._micro += 1
        if self._accum is not None:
            self._accum.add_(self.arena.flat)
        if overlapped:
            L, ev, n = _lib.lib(), self._events, len(self.model.transformer)
            side = C.c_void_p(self.arena._stream.cuda_stream)

            def gate(block):  # side stream: wait until that block's (or, for the rest, every) gradient is final
                check(L.dgs_stream_wait_event(side, ev[n if block is None else block]))
            self.arena.allreduce_issue_(group=self._group, gate=gate, sync_main=False)
            self._reduced = True

    def optimizer_step(self, allreduce=True):
        """all-reduce (mean) -> clip at `clip` (Lightning gradient_clip_val) -> fused AdamW [+ EMA] -> refresh bf16 weights."""
        if self._pending:
            raise RuntimeError("DitTrainer.optimizer_step: a training forward is still pending (no backward yet)")
        if self._micro == 0:
            raise RuntimeError("DitTrainer.optimizer_step: no backward since the last step")
        grads = self.arena.flat
        gscale = 1.0
        if self._accum is not None:  # mean over the micro-batches (Lightning divides the loss by accumulate_grad_batches)
            grads = self._accum
            gscale = 1.0 / self._micro
            if allreduce and self._world() > 1:
                self.arena.flat.copy_(self._accum)
                grads = self.arena.flat
        if self._reduced:          # issued bucket by bucket during the backward; only the tail can still be in flight
            gscale *= self.arena.allreduce_wait_(scale=False)
        elif allreduce and self._world() > 1:
            self.arena.allreduce_issue_(group=self._group)
            gscale *= self.arena.allreduce_wait_(scale=False)
        self._reduced = False
        norm = scale = None
        if self.clip:  # torch clip_grad_norm_ semantics; the factor stays on the device and is applied inside AdamW
            norm = torch.linalg.vector_norm(grads) * gscale
            scale = torch.clamp(self.clip / (norm + 1e-6), max=1.0).reshape(1).float()
        self.steps += 1
        dev = self.master.device
        with torch.cuda.device(dev):
            check(_lib.lib().dgs_adamw_ema_step(self.master.data_ptr(), grads.data_ptr(), self.exp_avg.data_ptr(),
                                                self.exp_avg_sq.data_ptr(), None if self.ema is None else self.ema.data_ptr(),
                                                self.master.numel(), self.lr, self.betas[0], self.betas[1], self.eps,
                                                self.weight_decay, self.steps, gscale,
                                                None if scale is None else scale.data_ptr(),
                                                0.0 if self.ema_decay is None else float(self.ema_decay), stream(dev)))
        if self._accum is not None:
            self._accum.zero_()
        self._micro = 0
        self.refresh_weights()
        return norm

    # -- EMA (ema.py:94-101 update; 119-160 replace/restore for evaluation and the "-EMA" checkpoint) --
    def ema_state_dict(self):
        """state_dict-shaped views into the EMA arena (same keys / shapes as model.state_dict())."""
        if self.ema is None:
            raise RuntimeError("DitTrainer was built without ema_decay")
        out, off = {}, 0
        for name, p in self.model.named_parameters():
            n = p.numel()
            out[name] = self.ema[off:off + n].view_as(p)
            off += n
        return out

    @contextlib.contextmanager
    def swap_ema_weights(self):
        """with trainer.swap_ema_weights(): evaluate / save with the EMA weights in place of the trained ones
        (EMA.replace_model_weights / restore_original_weights)."""
        if self.ema is None:
            raise RuntimeError("DitTrainer was built without ema_decay")
        if self._pending:
            raise RuntimeError("swap_ema_weights with a training forward pending")
        backup = self.master.clone()
        self.master.copy_(self.ema)
        self.refresh_weights()
        try:
            yield self.model
        finally:
            self.master.copy_(backup)
            self.refresh_weights()


class _DitFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, model, images, ray_o, ray_d, t, anchor):
        tr = model._trainer
        B, V, _, H, W = images.shape
        tr._begin_forward()
        try:
            state = tr.train_state(B, V, H, W)
            out, img_xyz, _, keep = model._run_dit(images, ray_o, ray_d, t, train_state=state, train_mode=tr.train_mode)
        except Exception:
            tr._pending = False
            raise
        ctx.model, ctx.keep = model, keep
        ctx.set_materialize_grads(False)  # an unused output arrives as None: zeros below, NULL for img_xyz
        return out.xyz, out.features, out.scaling, out.rotation, out.opacity, img_xyz

    @staticmethod
    def backward(ctx, d_xyz, d_features, d_scaling, d_rotation, d_opacity, d_img):
        model = ctx.model
        tr = model._trainer
        if ctx.keep is None or not tr._pending:
            raise RuntimeError("DitTrainer: this forward was already backpropagated (or dropped by trainer.reset()); the "
                               "activation state is consumed by the backward -- retain_graph / double backward is not supported")
        io, ws, nbytes, images, *_ = ctx.keep
        w, _k = ctx.keep[7], ctx.keep[8]
        dev = images.device
        B, V, _, H, W = images.shape
        P = model.cfg.n_gaussians + V * H * W
        n_sh = (model.cfg.gaussians_sh_degree + 1) ** 2
        z = lambda g, *s: (torch.zeros(*s, device=dev) if g is None else g.float().contiguous())  # noqa: E731
        gs = [z(d_xyz, B, P, 3), z(d_features, B, P, n_sh, 3), z(d_scaling, B, P, 3), z(d_rotation, B, P, 4),
              z(d_opacity, B, P, 1)]
        # d(img_aligned_xyz) (the geometry loss terms) is added to the image Gaussians' d xyz inside the backward
        d_img = None if d_img is None else d_img.float().contiguous()
        dout = DitOutGrads(*(g.data_ptr() for g in gs), None if d_img is None else d_img.data_ptr())
        opts = tr._bwd_opts()
        overlapped = opts is not None
        trace = tr._take_trace(B, V, H, W)
        if trace is not None:
            opts = opts or DitBwdOpts()
            opts.trace = C.pointer(trace)
        with torch.cuda.device(dev):
            check(_lib.lib().dgs_dit_backward_ex(C.byref(w), C.byref(tr._wT), C.byref(io), C.byref(dout),
                                                 C.byref(tr._grads), None if opts is None else C.byref(opts),
                                                 ws.data_ptr(), nbytes, stream(dev)))
        ctx.keep = None
        tr._end_backward(overlapped=overlapped)
        # parameter gradients were written straight into the arena (p.grad views); nothing to hand to autograd
        return None, None, None, None, None, torch.zeros_like(tr.anchor)


def dit_train_forward(model, images, ray_o, ray_d, t):
    from .denoiser import AttrDict
    xyz, features, scaling, rotation, opacity, img_xyz = _DitFunction.apply(model, images, ray_o, ray_d, t,
                                                                           model._trainer.anchor)
    return AttrDict(xyz=xyz, features=features, scaling=scaling, rotation=rotation, opacity=opacity), img_xyz
