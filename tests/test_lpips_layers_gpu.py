"""LPIPS-VGG on the H100 stage by stage: every stage of dgs_lpips_forward / dgs_lpips_backward against an fp64
restatement of that one stage (oracle/lpips.py: input_stage32, conv_stage64, head64, backward64), fed the kernels' own
activations and tap gradients from the training state (lpips_regime.state_views).  in1's activations come from
forward(in1, in0), which runs the same code with the inputs swapped.  Teacher forcing leaves no bf16 reroute for the bounds
to absorb -- every ReLU and max-pool decision is taken from the kernels' bits on both sides -- so, unlike the end-to-end
comparison of test_lpips_gpu.py, each check sits near fp32 rounding:

  forward   conv l on the kernels' act[l-1] (conv 0 on bf16((x - shift) / scale), computed in fp32) against act[l], for
            in0 and in1: the share of elements whose bits differ, and the element bound
                |act - ref| <= ulp_bf16(max(|act|, |ref|)) + FWD_ACC 2^-24 sqrt(K) (|x| * |W| + |b|),
            K = 9 C_in: one bf16 rounding plus the accumulation-order slack of fp32, the only thing the model leaves out;
  heads     G[k] against head64's G where a0 > 0 (the only place the backward reads G), relative to the magnitude of its
            fp32 arithmetic (head64's `mag`); out[n] against the sum of head64's tap distances;
  gradient  d in0 against backward64 on the same act, G and dout: relative L2 per image.

Each case also runs with the lin weights of every tap but one set to zero, for each of the five taps: the value is then
that tap's distance and the gradient chain has that tap's depth, so a failure names its tap.  Regimes: the independent,
noise and flat pairs of test_lpips_gpu.make_pair (flat gives exact ties in the pools) and "sparse": dark inputs with
relu4_3 / relu5_3 biases lowered until many tap pixels are all zero or have one non-zero channel (head_kernel's r0 = 0
branch and near-zero norms).  tests/test_lpips_layers_power_cpu.py shows which defects these bounds catch."""
import ctypes as C

import pytest
import torch

from lpips_regime import CHANNELS, random_lpips_state_dict, sparse_lpips_state_dict, state_views
from test_lpips_gpu import make_pair

pytestmark = pytest.mark.gpu
DEV = "cuda"

# Worst of every case below (seeds 0-2 on the small shapes, every tap isolation) on an H100 80GB HBM3 (700 W power
# limit), with margin.  The end-to-end bounds of test_lpips_gpu.py are 2e-3 on the value and 0.15 on d in0.
FWD_DIFF_FRAC = 5e-3    # share of a layer's activations whose bits differ from conv_stage64's: measured 1.95e-3 (one
#                         element of relu5_3's 512 at 1x16x16), 1.5e-3 at every other shape
FWD_ACC = 0.5           # multiple of 2^-24 sqrt(K) (|x| * |W| + |b|) beyond one bf16 ulp: measured 0.14
HEAD_G = 1e-6           # |G - G_ref| / mag where a0 > 0: measured 4.3e-7
VALUE_TAPS = 3e-6       # |out - sum of head64 distances| / that sum, per image: measured 1.4e-6 (tap 4 alone at
#                         1x16x16, a single pixel), 1.8e-7 with every tap
# relative L2 of d in0 against backward64, per image: measured 7.0e-3 (tap 4 alone, the deepest chain).  This is the
# floor of the chain, not of the kernels: an fp32 accumulation error that moves one dz across a bf16 rounding midpoint
# changes the da it feeds, which re-draws the bf16 rounding of dz in the layers below.  The kernels and backward64 thus
# end up with independent bf16 roundings of dz in every layer: noise of 1e-3 of an fp32 accumulation error added to
# backward64's own convolutions already moves its d in0 by 3e-3 to 5e-3.
GRAD_CHAIN = 0.015
SPARSE_MIN = 0.04       # share of relu4_3 / relu5_3 pixels that are all zero, and that have one non-zero channel:
#                         measured at least 0.26 and 0.084 (1x512x512)

BOUNDS = dict(fwd_frac=FWD_DIFF_FRAC, fwd_acc=FWD_ACC, head_G=HEAD_G, value=VALUE_TAPS, grad=GRAD_CHAIN)


def bf16_ulp(v):
    """the spacing of bf16 numbers at |v| (v >= 0, fp64); 0 at v = 0"""
    e = torch.frexp(v).exponent
    return torch.where(v > 0, torch.ldexp(torch.ones_like(v), e - 8), torch.zeros_like(v))


def stage_errors(wts, in0, in1, dout, r, forward=True):
    """The checks of this file on one run r = dict(out, act0, act1, G, d_in0) (kernel outputs, or a stand-in's) ->
    (errors: the worst value of each check, keyed as BOUNDS; rows: per-layer forward errors and per-tap G errors)."""
    from oracle.lpips import TAP_AFTER, backward64, conv_stage64, head64, input_stage32
    err, rows = {}, {}
    if forward:
        frac, acc = [0.0] * 13, [0.0] * 13
        for x, act in ((in0, r["act0"]), (in1, r["act1"])):
            a = input_stage32(wts, x)
            for l in range(13):
                ref, _, mag = conv_stage64(wts, l, a)
                k = act[l].double()
                K = 9 * CHANNELS[l]
                excess = ((k - ref).abs() - bf16_ulp(torch.maximum(k.abs(), ref.abs()))).clamp(min=0)
                frac[l] = max(frac[l], float((k != ref).double().mean()))
                acc[l] = max(acc[l], float((excess / (2.0 ** -24 * K ** 0.5 * mag + 1e-300)).max()))
                a = act[l]  # teacher forcing: conv l + 1 reads the kernels' own activation
        err["fwd_frac"], err["fwd_acc"] = max(frac), max(acc)
        rows["frac"], rows["acc"] = frac, acc
    dist, gerr = 0, [0.0] * 5
    for k, l in enumerate(TAP_AFTER):
        d, G, mag = head64(wts["lin"][k], r["act0"][l], r["act1"][l])
        dist = dist + d
        m = r["act0"][l] > 0
        if bool(m.any()):
            gerr[k] = float(((r["G"][k].double() - G).abs() / (mag + 1e-300))[m].max())
    err["head_G"], rows["G"] = max(gerr), gerr
    err["value"] = float(((r["out"].double() - dist) / dist).abs().max())
    ref = backward64(wts, r["act0"], r["G"], dout)
    dif = (r["d_in0"].double() - ref).flatten(1).norm(dim=1)
    err["grad"] = float((dif / ref.flatten(1).norm(dim=1)).max())
    return err, rows


def isolate_tap(sd, k):
    """the state dict with the lin weights of every tap but k set to zero"""
    sd = dict(sd)
    for j in range(5):
        if j != k:
            for key in (f"lin{j}.model.1.weight", f"lins.{j}.model.1.weight"):
                if key in sd:
                    sd[key] = torch.zeros_like(sd[key])
    return sd


class Kernels:
    """dgs_lpips_forward / dgs_lpips_backward called directly, with the test's own state and workspace; `chunk` caps the
    workspace to that many images."""

    def __init__(self, sd, chunk=None):
        from dgs_b200.lpips import pack_weights, parse_state_dict
        self.w, self._keep = pack_weights(parse_state_dict(sd), DEV)
        self.chunk = chunk

    def _workspace(self, n, H, W):
        from dgs_b200 import _lib
        L = _lib.lib()
        nbytes = L.dgs_lpips_workspace_bytes(n, H, W) if self.chunk is None else \
            self.chunk * L.dgs_lpips_workspace_bytes(1, H, W)
        return torch.empty(nbytes, dtype=torch.uint8, device=DEV)

    def forward(self, in0, in1):
        """-> (out [n], the training state)"""
        from dgs_b200 import _lib
        n, _, H, W = in0.shape
        in0, in1 = in0.float().contiguous(), in1.float().contiguous()
        out = torch.empty(n, dtype=torch.float32, device=DEV)
        state = torch.empty(_lib.lib().dgs_lpips_state_bytes(n, H, W), dtype=torch.uint8, device=DEV)
        ws = self._workspace(n, H, W)
        _lib.check(_lib.lib().dgs_lpips_forward(C.byref(self.w), n, H, W, in0.data_ptr(), in1.data_ptr(), out.data_ptr(),
                                                state.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream(DEV)))
        return out, state

    def backward(self, state, dout, H, W):
        from dgs_b200 import _lib
        n = dout.numel()
        dout = dout.float().contiguous()
        d_in0 = torch.empty(n, 3, H, W, dtype=torch.float32, device=DEV)
        ws = self._workspace(n, H, W)
        _lib.check(_lib.lib().dgs_lpips_backward(C.byref(self.w), n, H, W, state.data_ptr(), dout.data_ptr(),
                                                 d_in0.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream(DEV)))
        return d_in0

    def run(self, in0, in1, dout):
        """-> dict(out, act0, act1, G, d_in0): the value, both inputs' activations, in0's tap gradients, d in0"""
        n, _, H, W = in0.shape
        out, s0 = self.forward(in0, in1)
        _, s1 = self.forward(in1, in0)
        d_in0 = self.backward(s0, dout, H, W)
        torch.cuda.synchronize()
        act0, G = state_views(s0, n, H, W)
        act1, _ = state_views(s1, n, H, W)
        return dict(out=out, act0=act0, act1=act1, G=G, d_in0=d_in0)


def _weights(sd):
    from oracle.lpips import weights_from_state_dict
    w = weights_from_state_dict(sd)
    return {k: ([t.to(DEV) for t in v] if isinstance(v, list) else v.to(DEV)) for k, v in w.items()}


def case_inputs(regime, n, H, W, seed):
    """-> (state dict, in0, in1, dout)"""
    if regime == "sparse":
        in0, in1 = make_pair("independent", n, H, W, seed)
        in0, in1 = 0.3 * (in0 + 1) - 1, 0.3 * (in1 + 1) - 1  # dark: [0, 0.3] in image units
        sd = sparse_lpips_state_dict(seed, torch.cat([in0, in1]).double())
    else:
        in0, in1 = make_pair(regime, n, H, W, seed)
        sd = random_lpips_state_dict(seed)
    dout = torch.rand(n, device=DEV, generator=torch.Generator(DEV).manual_seed(seed)) + 0.5
    return sd, in0, in1, dout


SMALL = [(1, 16, 16), (2, 16, 48), (3, 48, 16), (3, 64, 96), (5, 64, 96)]
LARGE = [(1, 256, 256), (2, 256, 256), (1, 512, 512)]
CHUNK = {(5, 64, 96): 2}  # workspace for 2 images: chunks of 2, 2, 1, so the state offsets of later chunks are read


def _cases():
    for shape in SMALL + LARGE:
        seeds = [0, 1, 2] if shape in SMALL else [0]
        # sparse needs enough relu5_3 pixels for the per-channel quantile to leave most of them empty
        regimes = ["independent", "noise", "flat"] + (["sparse"] if shape[0] * shape[1] * shape[2] >= 3 * 64 * 96 else [])
        for regime in regimes:
            for seed in seeds:
                yield pytest.param(shape, regime, seed, id=f"{'x'.join(map(str, shape))}-{regime}-{seed}")


def _check(err, what):
    bad = {k: (v, BOUNDS[k]) for k, v in err.items() if not v <= BOUNDS[k]}
    assert not bad, f"{what}: {bad}"


@pytest.mark.parametrize("shape, regime, seed", list(_cases()))
def test_stages_against_fp64(shape, regime, seed):
    n, H, W = shape
    sd, in0, in1, dout = case_inputs(regime, n, H, W, seed)
    r = Kernels(sd, CHUNK.get(shape)).run(in0, in1, dout)
    err, rows = stage_errors(_weights(sd), in0, in1, dout, r)
    tag = f"{'x'.join(map(str, shape))} {regime} seed={seed}"
    print(f"\nLPSTAT full {tag} lpips={[round(float(v), 4) for v in r['out'][:3]]} "
          + " ".join(f"{k}={v:.3e}" for k, v in err.items()))
    print(f"LPLAYER {tag} frac=[{' '.join(f'{v:.2e}' for v in rows['frac'])}] "
          f"acc=[{' '.join(f'{v:.2f}' for v in rows['acc'])}] G=[{' '.join(f'{v:.2e}' for v in rows['G'])}]")
    if regime == "sparse":
        nz = torch.cat([(a[l] > 0).sum(-1).flatten() for a in (r["act0"], r["act1"]) for l in (9, 12)])
        zero, one = float((nz == 0).double().mean()), float((nz == 1).double().mean())
        print(f"LPSPARSE {tag} zero={zero:.3f} one={one:.3f}")
        assert zero >= SPARSE_MIN and one >= SPARSE_MIN  # the regime the bounds were measured in
    _check(err, tag)
    for k in range(5):
        sdk = isolate_tap(sd, k)
        rk = Kernels(sdk, CHUNK.get(shape)).run(in0, in1, dout)
        assert all(torch.equal(a, b) for a, b in zip(rk["act0"], r["act0"]))  # the lin weights only enter the heads
        ek, _ = stage_errors(_weights(sdk), in0, in1, dout, rk, forward=False)
        print(f"LPSTAT tap{k} {tag} " + " ".join(f"{key}={v:.3e}" for key, v in ek.items()))
        _check(ek, f"{tag} tap {k} alone")


@pytest.mark.parametrize("shape", [(2, 16, 48), (3, 64, 96), (5, 64, 96)], ids=lambda s: "x".join(map(str, s)))
def test_exact_invariants(shape):
    """The value is symmetric in its inputs (which the swapped forward of the stage checks relies on) and the gradient is
    linear in dout image by image, bit for bit: scaling dout by 2 scales d in0 by 2 exactly (powers of two are exact in
    fp32 and bf16 away from subnormals), an image with dout = 0 gets an all-zero gradient and negating one image's dout
    negates that image's gradient and leaves the others alone."""
    n, H, W = shape
    sd, in0, in1, dout = case_inputs("independent", n, H, W, 0)
    k = Kernels(sd, CHUNK.get(shape))
    out, state = k.forward(in0, in1)
    out_swapped, _ = k.forward(in1, in0)
    assert torch.equal(out, out_swapped)
    g = k.backward(state, dout, H, W)
    assert torch.equal(k.backward(state, 2 * dout, H, W), 2 * g)
    d = dout.clone()
    d[1] = 0
    g0 = k.backward(state, d, H, W)
    assert bool((g0[1] == 0).all()) and bool((g[1] != 0).any())
    assert torch.equal(g0[:1], g[:1]) and torch.equal(g0[2:], g[2:])
    d = dout.clone()
    d[-1] = -d[-1]
    gn = k.backward(state, d, H, W)
    assert torch.equal(gn[:-1], g[:-1]) and torch.equal(gn[-1], -g[-1])
