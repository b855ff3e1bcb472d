"""oracle/gemm.py -- TEST INFRASTRUCTURE: the bf16 GEMM (gemm_sm90.cu: gemm_bf16, gemm_bf16_tn) as a model of its own
epilogue arithmetic in fp64, the way oracle/attention.py models the attention kernels.  Never imported by the product.

* The accumulator.  P = A W^T and S = |A| |W|^T are exact fp64 sums of the bf16 products.  wgmma accumulates in fp32 in
  an order the model does not know, so the model gives an interval: acc in [P - delta, P + delta] with
  delta = KAPPA sqrt(K) 2^-24 S, plus splits 2^-24 S for the fp32 atomic adds of split-K partial sums (any order).
  KAPPA is measured (see its definition).
* Each epilogue in the order the code rounds (epilogue_fragment / epilogue_tma):
    v = fl32(acc + b)
    epi 0: bf16(v)        epi 5: bf16(max(v, 0))       epi 1: bf16(gelu_tanh(v))
    epi 4: bf16(fl32(v dgelu_tanh(u))), u the bf16 aux
    epi 2: fl32(x + fl32(g[row / rows_per_sample] v))
    aux (epi 1, 2 in training mode): bf16(v)
    epi 3 and the tn GEMM: v
  bf16() is round-to-nearest-even, fl32() fp32 rounding.
* What the model assumes about the GELU and its derivative.  They run in fp32 with tanh.approx.f32 (PTX: at most
  2^-10.987 relative error) and are compiled without -fmad=false, so the compiler may contract x*x*x + x and the
  final 0.5 x (1 + t) into FMAs.  The model evaluates both in fp64 with the exact tanh and widens the interval by a
  bound on the deviation of the fp32 code: the tanh.approx error |t| 2^-10.987, the rounding of the tanh argument
  (4 ulp of its terms, carried through tanh' = 1 - t^2) and 8 ulp of the terms of the final expression.  Contracted
  or not, the fp32 code stays inside that bound.  GELU is not monotone: its minimum near x = -0.7518 is included when
  the input interval straddles it.
* The admissible output interval of every element is that of its accumulator interval mapped through the epilogue
  and rounded by the same (monotone) roundings; `pt` is the model at acc = fl32(P).
* rounding=False drops every rounding and the interval: the plain fp64 epilogue of P.
* GEMM_DEFECTS: named defects that tests/test_gemm_cpu.py plants in the model's output to show that the checks of
  tests/test_gemm_gpu.py see them.
"""
import collections
import math

import torch

BM, BK = 128, 64
U32 = 2.0 ** -24
TANH_APPROX_REL = 2.0 ** -10.987
K0, K1 = 0.7978845608028654, 0.044715
GELU_XMIN = -0.751791524693564457457   # argmin of gelu_tanh
# KAPPA: |acc - P| <= KAPPA sqrt(K) 2^-24 S element by element.  Measured on an H100 80GB HBM3 (700 W) over every
# case of tests/test_gemm_gpu.py, seeds 0-2: worst 0.290 from EPI_F32 without bias (e3reg256_4, K = 136) and 0.695
# from the tn GEMM (tn128_0, K = 8).  Fixed at 2.0, a margin of 2.9x over the worst.
KAPPA = 2.0

_Defects = collections.namedtuple("GemmDefects", [
    "bias_pair_last_tile",   # the valid columns of the last tile column read the bias pair N-2, N-1
    "gate_row_tile_first",   # the gate row of every row taken from the sample of its tile's first row
    "gelu_erf",              # GELU with erf instead of the tanh approximation
    "bf16_round_to_zero",    # bf16 outputs truncated instead of rounded to nearest even
    "last_kblock_dropped",   # the last, partial k-block left out of the accumulator
    "rows_past_m_stored",    # the rows >= M of the last tile row are stored (past the output)
    "splitk_partial_twice",  # the first split-K partial sum added twice
    "aux_post_activation",   # aux holds gelu(v) instead of v
    "dgelu_no_x2_term",      # dGELU's du/dx without its 3 k1 x^2 term
    "staged_chunk_swapped",  # one 16-byte chunk of the last row swapped with its neighbour
])
GEMM_DEFECTS = _Defects(*_Defects._fields)


def cdiv(a, b):
    return -(-a // b)


def f32(t):
    return t.float().double()


def bf16(t):
    """Round fp64 values holding fp32 numbers (or any fp64) to bf16 by RNE of their fp32 rounding."""
    return t.float().to(torch.bfloat16).double()


def bf16_rtz(t):
    x = t.float().contiguous()
    b = (x.view(torch.int32) & ~0xFFFF).view(torch.float32)
    return b.double()


def f32_down(t):
    x = t.float()
    return torch.where(x.double() > t, torch.nextafter(x, torch.full_like(x, -math.inf)), x).double()


def f32_up(t):
    x = t.float()
    return torch.where(x.double() < t, torch.nextafter(x, torch.full_like(x, math.inf)), x).double()


def bf16_ulp(t):
    """The bf16 ulp of |t| (fp64); 0 where t == 0."""
    _, e = torch.frexp(t)
    return torch.where(t == 0, torch.zeros_like(t), torch.ldexp(torch.ones_like(t), e - 8))


def gelu(x, erf=False):
    if erf:
        return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))
    return 0.5 * x * (1.0 + torch.tanh(K0 * (x + K1 * x * x * x)))


def dgelu(x, no_x2=False):
    t = torch.tanh(K0 * (x + K1 * x * x * x))
    du = K0 * (1.0 if no_x2 else 1.0 + 3.0 * K1 * x * x)
    return 0.5 * (1.0 + t) + 0.5 * x * (1.0 - t * t) * du


def _eps_t(x):
    """Bound on |t_fp32 - tanh(u(x))|: tanh.approx's relative error plus the rounding of its argument."""
    t = torch.tanh(K0 * (x + K1 * x * x * x)).abs()
    return t * TANH_APPROX_REL + (1.0 - t * t) * 4 * U32 * K0 * (x.abs() + K1 * x.abs() ** 3)


def gelu_err(x):
    """Bound on |gelu_fp32(x) - gelu(x)| for the kernel's epi_gelu_tanh."""
    t = torch.tanh(K0 * (x + K1 * x * x * x)).abs()
    return 0.5 * x.abs() * _eps_t(x) + 8 * U32 * 0.5 * x.abs() * (1.0 + t)


def dgelu_err(x):
    """Bound on |dgelu_fp32(x) - dgelu(x)| for the kernel's epi_dgelu_tanh."""
    t = torch.tanh(K0 * (x + K1 * x * x * x)).abs()
    du = K0 * (1.0 + 3.0 * K1 * x * x)
    e = _eps_t(x)
    return e * (0.5 + x.abs() * t * du) + 8 * U32 * (0.5 * (1.0 + t) + 0.5 * x.abs() * (1.0 + t * t) * du)


def products(A, W, tn=False, defects=()):
    """P, S (fp64) of the bf16 operands: A [M, K], W [N, K] (tn: A [K, M], W [K, N])."""
    a, w = A.double(), W.double()
    if tn:
        a, w = a.t(), w.t()
    K = a.shape[1]
    if "last_kblock_dropped" in defects and K % BK:
        a, w = a[:, :K // BK * BK], w[:, :K // BK * BK]
    return a @ w.t(), a.abs() @ w.abs().t()


class Spec:
    """One GEMM call.  epi: 0..5 or "tn"; bias [N] fp32; gate [samples, N] fp32 (the gate vectors, already offset);
    x [M, N] fp32 the residual (epi 2); u [M, N] bf16 the saved pre-activation (epi 4); aux: epi 1 / 2 store aux;
    bn, splits: the tile width and split-K factor of the path the call takes (gemm_path)."""

    def __init__(self, epi, M, N, K, bias=None, gate=None, rows_per_sample=1, x=None, u=None, aux=False, bn=128,
                 splits=1):
        self.epi, self.M, self.N, self.K = epi, M, N, K
        self.bias, self.gate, self.rps, self.x, self.u, self.aux = bias, gate, rows_per_sample, x, u, aux
        self.bn, self.splits = bn, splits

    @property
    def out_bf16(self):
        return self.epi in (0, 1, 4, 5)


def _acc_interval(P, S, spec):
    d = KAPPA * math.sqrt(spec.K) * U32 * S + spec.splits * U32 * S
    return f32_down(P - d), f32_up(P + d), f32(P)


def _bias_rows(spec, r0, r1, defects, like):
    if spec.bias is None:
        return torch.zeros(1, spec.N, dtype=torch.float64, device=like.device)
    b = spec.bias.double().to(like.device).clone()
    if "bias_pair_last_tile" in defects:
        c0 = (cdiv(spec.N, spec.bn) - 1) * spec.bn
        b[c0:] = b[spec.N - 2:].repeat((spec.N - c0) // 2)
    return b[None]


def _gate_rows(spec, r0, r1, defects, device):
    rows = torch.arange(r0, r1, device=device)
    if "gate_row_tile_first" in defects:
        rows = rows // BM * BM
    return spec.gate.double().to(device)[rows // spec.rps]


def model_rows(spec, P, S, r0, defects=(), rounding=True):
    """The model of output rows [r0, r0 + len(P)) from their P and S: a dict of fp64 tensors 'lo', 'hi', 'pt' (the
    output) and, when the call stores one, 'aux_lo', 'aux_hi', 'aux_pt'.  rounding=False: lo = hi = pt = the plain
    fp64 epilogue of P."""
    r1 = r0 + P.shape[0]
    dev = P.device
    epi = spec.epi
    out = {}
    if rounding:
        alo, ahi, apt = _acc_interval(P, S, spec)
        rnd, rbf = f32, (bf16_rtz if "bf16_round_to_zero" in defects else bf16)
    else:
        alo = ahi = apt = P
        rnd = rbf = (lambda t: t)
    if epi == "tn":
        out["lo"], out["hi"], out["pt"] = alo, ahi, apt
        return out
    b = _bias_rows(spec, r0, r1, defects, P)
    v = [rnd(a + b) for a in (alo, ahi, apt)]   # fl32(acc + b): monotone
    if spec.aux and epi in (1, 2):
        f = (lambda t: rbf(gelu(t, "gelu_erf" in defects))) if "aux_post_activation" in defects else rbf
        out["aux_lo"], out["aux_hi"], out["aux_pt"] = f(v[0]), f(v[1]), f(v[2])
        if "aux_post_activation" in defects:
            out["aux_lo"], out["aux_hi"] = torch.minimum(out["aux_lo"], out["aux_hi"]), torch.maximum(out["aux_lo"], out["aux_hi"])
    if epi == 0:
        lo, hi, pt = (rbf(t) for t in v)
    elif epi == 5:
        lo, hi, pt = (rbf(t.clamp(min=0)) for t in v)
    elif epi == 3:
        lo, hi, pt = v
    elif epi == 1:
        erf = "gelu_erf" in defects
        g0, g1 = gelu(v[0], erf), gelu(v[1], erf)
        glo, ghi = torch.minimum(g0, g1), torch.maximum(g0, g1)
        if rounding:
            straddle = (v[0] <= GELU_XMIN) & (v[1] >= GELU_XMIN)
            glo = torch.where(straddle, gelu(torch.tensor(GELU_XMIN, dtype=torch.float64)).to(dev), glo)
            e = torch.maximum(gelu_err(v[0]), gelu_err(v[1]))
            glo, ghi = f32_down(glo - e), f32_up(ghi + e)
        lo, hi, pt = rbf(glo), rbf(ghi), rbf(gelu(v[2], erf))
    elif epi == 4:
        u = spec.u[r0:r1].double().to(dev)
        no_x2 = "dgelu_no_x2_term" in defects
        d = dgelu(u, no_x2)
        if rounding:
            e = dgelu_err(u)
            ends = [a * dd for a in (v[0], v[1]) for dd in (d - e, d + e)]
            plo, phi = torch.stack(ends).amin(0), torch.stack(ends).amax(0)
            plo, phi = f32_down(plo - U32 * plo.abs()), f32_up(phi + U32 * phi.abs())
        else:
            plo = phi = v[2] * d
        lo, hi, pt = rbf(plo), rbf(phi), rbf(v[2] * d)
    elif epi == 2:
        g = _gate_rows(spec, r0, r1, defects, dev)
        x = spec.x[r0:r1].double().to(dev)
        y = [rnd(x + rnd(g * t)) for t in v]   # monotone in v for a fixed sign of g
        lo, hi, pt = torch.minimum(y[0], y[1]), torch.maximum(y[0], y[1]), y[2]
    else:
        raise ValueError(f"unknown epilogue {epi}")
    out["lo"], out["hi"], out["pt"] = lo, hi, pt
    return out


def splitk_first_partial(A, W, K, splits):
    """tn: the partial sum of the first split-K unit (its k-blocks [0, kpb))."""
    num_k = cdiv(K, BK)
    kpb = cdiv(num_k, splits)
    k1 = min(K, kpb * BK)
    return A[:k1].double().t() @ W[:k1].double()


def plant_buffer_defects(out_rows, spec, defects, guard_rows=None):
    """Defects on the stored output: out_rows [M, N] (the model's point values, modified in place) and guard_rows
    [>= 128, N] (the rows past M, modified in place)."""
    if "rows_past_m_stored" in defects and guard_rows is not None and spec.M % BM:
        guard_rows[:BM - spec.M % BM] = 0.0
    if "staged_chunk_swapped" in defects:
        c = 8 if spec.out_bf16 else 4    # elements of a 16-byte chunk
        r = out_rows[-1]
        if spec.N >= 2 * c:
            a = r[:c].clone()
            r[:c] = r[c:2 * c]
            r[c:2 * c] = a


@torch.no_grad()
def model_output(spec, A, W, defects=()):
    """The model's point output of a whole call with `defects` planted: (out [M, N], aux [M, N] or None, guard
    [BM + 2, N]: the rows past M, NaN where nothing was stored)."""
    tn = spec.epi == "tn"
    P, S = products(A, W, tn, defects)
    m = model_rows(spec, P, S, 0, defects)
    out = m["pt"].clone()
    if "splitk_partial_twice" in defects and spec.splits > 1:
        out = f32(out + f32(splitk_first_partial(A, W, spec.K, spec.splits)))
    guard = torch.full((BM + 2, spec.N), math.nan, dtype=torch.float64, device=out.device)
    plant_buffer_defects(out, spec, defects, guard)
    return out, m.get("aux_pt"), guard
