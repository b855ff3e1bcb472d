"""GPU tests of the bf16 GEMM (dgs_gemm_bf16, dgs_gemm_bf16_ex, dgs_gemm_bf16_tn) element by element against a model
of its own epilogue arithmetic (oracle/gemm.py).

Every case of the table (gemm_cases) runs one call and checks:
* hard: every output and aux element inside its admissible interval (the accumulator interval mapped through the
  epilogue and its roundings); not one element may fall outside;
* statistics, for what is smaller than an interval: the share of bf16 outputs whose bits differ from the model at
  acc = P, the mean of sign(model) (out - model) in bf16 ulps, and for fp32 outputs the norm-wise error against the
  model at P;
* guard bands: 130 rows past M, the ldc > N padding and 64 elements before the (offset) output pointer, of the output
  and of aux, keep their sentinel bits; A, W, bias, gate, resid and an input aux are bitwise unchanged;
* determinism: a second launch gives the same bits (paths without split-K), and where the output rows are TMA-storable
  the register epilogue (the same call with an output row stride the TMA store cannot take) gives the same bits.

The table is built for the running device's SM count: gemm_path restates the launcher's tile-width, store-path and
split-K choices, and tests/test_gemm_cpu.py checks that the table reaches every reachable kernel instantiation.
Every bound below is the worst measured on an H100 80GB HBM3 (700 W) over seeds 0, 1, 2, with its margin.
"""
import collections
import math
import zlib

import pytest
import torch

from oracle import gemm as og

DEV = "cuda:0"

# ---- statistics bounds, per epilogue: about 2x the worst measured on the H100 over seeds 0-2 ----
# share of bf16 outputs with other bits than bf16(model at P): the fp32 accumulation order (and for GELU / dGELU
# tanh.approx) now and then puts a value across a rounding midpoint
DIFF_FRAC = {0: 0.005,   # worst 2.35e-3 (fc1_dgrad_8196)
             5: 0.005,   # worst 1.71e-3 (lpips64x96_512_512_4)
             1: 0.15,    # worst 8.93e-2 (e1reg128_4, cancellation: many inputs in the tails)
             4: 0.3}     # worst 0.205 (e4reg128_2, saved pre-activations in saturation)
# |mean of sign(model) (out - model) / ulp| over the nonzero outputs of a case.  GELU and dGELU outputs in the negative
# tail are tiny against the tanh.approx error (2^-11 of t, where 1 + t is small), which moves them by many of their
# own ulps, so their bounds only catch gross biases; erf GELU is caught by DIFF_FRAC instead.
MEAN_ULP = {0: 0.05,     # worst 2.09e-2 (fc1_dgrad_16386)
            5: 0.05,     # worst 3.10e-3 (lpips64x96_512_512_4)
            1: 12.0,     # worst 7.10 (e1reg128_4)
            4: 6.0}      # worst 3.79 (e4reg128_2)
# fp32 outputs: |out - model at P| / |model at P|, norm-wise
REL32 = {2: 8e-6,        # worst 3.68e-6 (tails_1x4096)
         3: 1e-5,        # worst 4.41e-6 (f32nb_4098x1024x4096)
         "tn": 4e-5}     # worst 1.86e-5 (tn_3072x1024x16392: K = 16392)

GUARD_ROWS = 130
PRE = 64
SENT16 = 0x7FA5           # bf16 NaN bits
SENT32 = 0x7FA5A5A5       # fp32 NaN bits
TAILS = (1, 2, 64, 65, 127)

Path = collections.namedtuple("Path", "bn tma splits tiles")
Case = collections.namedtuple("Case", "name M N K epi ldc_pad aux resid mis rps regime bias kpad twin",
                              defaults=(0, False, False, False, 1, "std", True, 0, True))


def cdiv(a, b):
    return -(-a // b)


def gemm_path(M, N, K, epi, ldc, aux=False, resid=False, out_align=16, sms=132):
    """The launcher's choice for one call (gemm_bf16 / gemm_bf16_tn in gemm_sm90.cu): tile width, TMA-store epilogue,
    split-K factor and output tiles.  epi: 0..5, or "tn" for gemm_bf16_tn."""
    if epi == "tn":
        wide = N % 256 == 0 and cdiv(M, 128) * (N // 256) >= sms
        bn = 256 if wide else 128
        tiles, num_k = cdiv(M, 128) * cdiv(N, bn), cdiv(K, 64)
        splits = 1
        if tiles < sms and num_k >= 16 and ldc % 2 == 0 and out_align % 8 == 0:
            splits = min(cdiv(sms, tiles), num_k // 8)
            splits = cdiv(num_k, cdiv(num_k, splits))
        return Path(bn, False, splits, tiles)
    ob = 4 if epi in (2, 3) else 2
    tma = epi != 4 and not aux and not resid and ldc >= N and (ldc * ob) % 16 == 0 and out_align % 16 == 0
    gate_tma = tma and epi == 2
    wide = N % 256 == 0 and (gate_tma or (cdiv(M, 128) * (N // 256) >= 2 * sms and not (tma and ob == 4)))
    bn = 256 if wide else 128
    return Path(bn, tma, 1, cdiv(M, 128) * cdiv(N, bn))


def instantiation(path, epi):
    if epi == "tn":
        return ("tn", path.bn, path.splits > 1)
    return (epi, "tma" if path.tma else "reg", path.bn)


# every gemm_kernel instantiation the ABI can reach (the tn GEMM at BN = 256 never splits K: it takes 256-wide tiles
# only when they fill the SMs, and splits K only when they do not)
REACHABLE = ([(e, s, b) for e in (0, 1, 5) for s in ("tma", "reg") for b in (128, 256)]
             + [(2, s, b) for s in ("tma", "reg") for b in (128, 256)]
             + [(3, "tma", 128), (3, "reg", 128), (3, "reg", 256), (4, "reg", 128), (4, "reg", 256)]
             + [("tn", 128, False), ("tn", 128, True), ("tn", 256, False)])


def case_path(c, sms):
    esize = 4 if c.epi in (2, 3, "tn") else 2
    ldc = c.N + c.ldc_pad
    align = (PRE + (2 if c.mis else 0)) * esize % 16 or 16
    return gemm_path(c.M, c.N, c.K, c.epi, ldc, c.aux or c.epi == 4, c.resid, align, sms)


def _rows_for(nt, sms, few, wide_min=0):
    """Tile rows giving nt * rows tiles: fewer than sms (few), else more than max(sms, wide_min) with a partial last
    wave."""
    if few:
        return max(1, min(2, (sms - 1) // nt))
    r = max(cdiv(sms + 1, nt), cdiv(wide_min, nt))
    while (r * nt) % sms == 0:
        r += 1
    return r


def _instantiation_cases(inst, sms):
    out = []
    for i, tail in enumerate(TAILS):
        few = i in (1, 3)
        if inst[0] == "tn":
            _, bn, split = inst
            K = (1000, 2056, 1096, 4104, 1224)[i] if split else (8, 200, 72, 1000, 136)[i]
            if bn == 256 or (not split and K >= 961):
                few = False
            if split:
                few = True
            N = 2048 if bn == 256 else ((1056, 1120)[i - 1] if i in (1, 2) else 1152)
            if few and N > 1152:
                N = 160
            nt = cdiv(N, bn)
            rows = _rows_for(nt, sms, few)
            M = (rows - 1) * 128 + tail
            out.append(Case(f"tn{bn}{'s' if split else ''}_{i}", M, N, K, "tn", ldc_pad=(0, 8, 0, 2, 0)[i],
                            bias=False, kpad=(0, 8, 0, 0, 16)[i]))
            continue
        epi, store, bn = inst
        K = (8, 200, 72, 1000, 136)[i]
        wide = bn == 256
        gate_tma = epi == 2 and store == "tma"
        if wide:
            N = 256 if (few and gate_tma) else 2048
            if not gate_tma:
                few = False
        else:
            N = (1056, 1120)[i - 1] if i in (1, 2) else (160 if few else 1152)
        nt = cdiv(N, bn)
        rows = _rows_for(nt, sms, few, 2 * sms if wide and not gate_tma else 0)
        M = (rows - 1) * 128 + tail
        fp32 = epi in (2, 3)
        kw = dict(bias=(i != 4) and epi != 4)
        if store == "reg":   # the ways onto the register epilogue: aux / resid, an unaligned row stride or pointer
            way = i % 3
            if epi == 4:
                pass
            elif epi == 1 and way == 0:
                kw["aux"] = True
            elif epi == 2 and way == 0:
                kw.update(aux=True, resid=True)
            elif way == 1:
                kw["ldc_pad"] = 2
            else:
                kw["mis"] = True
        else:
            kw["ldc_pad"] = (0, 16 if not fp32 else 4, 0, 64, 8)[i]
        if epi == 2:
            kw["rps"] = (M + 5, 100, 40, 1, 300)[i]
        if epi in (1, 4):
            kw["regime"] = ("gelu_min", "outlier", "gelu_sat", "zero_rows", "cancel")[i]
        else:
            kw["regime"] = ("std", "outlier", "cancel", "zero_rows", "std")[i]
        if i == 3:
            kw["kpad"] = 16
        out.append(Case(f"e{epi}{store}{bn}_{i}", M, N, K, epi, **kw))
    return out


def product_cases():
    """The library's own shapes: DiT linears at the obj-256 / obj-512 token counts, forward and dgrad, the weight
    gradients, the tokenizer, the decoder head at each SH degree and the LPIPS convolutions."""
    D, U = 1024, 4096
    cs = []
    for M in (4098, 8196, 16386):
        rps = 4098
        cs += [Case(f"qkv_{M}", M, 3 * D, D, 0),
               Case(f"proj_{M}", M, D, D, 2, rps=rps),
               Case(f"fc1_{M}", M, U, D, 1),
               Case(f"fc2_{M}", M, D, U, 2, rps=rps),
               Case(f"qkv_dgrad_{M}", M, D, 3 * D, 0, bias=False),
               Case(f"proj_dgrad_{M}", M, D, D, 0, bias=False),
               Case(f"fc1_dgrad_{M}", M, D, U, 0, bias=False),
               Case(f"fc2_dgrad_{M}", M, U, D, 4, bias=False)]
    cs += [Case("fc1_train_4098", 4098, U, D, 1, aux=True),
           Case("proj_train_4098", 4098, D, D, 2, aux=True, resid=True, rps=4098),
           Case("fc2_train_8196", 8196, D, U, 2, aux=True, resid=True, rps=4098)]
    for K in (4098, 8196):
        cs += [Case(f"qkv_wgrad_{K}", 3 * D, D, K, "tn", bias=False), Case(f"proj_wgrad_{K}", D, D, K, "tn", bias=False),
               Case(f"fc1_wgrad_{K}", U, D, K, "tn", bias=False), Case(f"fc2_wgrad_{K}", D, U, K, "tn", bias=False)]
    cs.append(Case("tokenizer", 4096, D, 3 * 576, 3))
    for deg in range(4):
        nd = 64 * (11 + 3 * (deg + 1) ** 2)
        cs += [Case(f"dec_sh{deg}", 4096, nd, 3 * D, 3, bias=False),
               Case(f"dec_dgrad_sh{deg}", 4096, D, nd, 0, bias=False),
               Case(f"dec_wgrad_sh{deg}", nd, D, 4096, "tn", bias=False)]
    for hw, tag in ((256 * 256, "256"), (64 * 96, "64x96")):
        for cin, cout, lvl in ((8, 64, 0), (64, 64, 0), (64, 128, 1), (128, 128, 1), (128, 256, 2), (256, 256, 2),
                               (256, 512, 3), (512, 512, 3), (512, 512, 4)):
            cs.append(Case(f"lpips{tag}_{cin}_{cout}_{lvl}", hw >> (2 * lvl), cout, 9 * cin, 5, regime="std"))
    return cs


def legacy_cases():
    """The shapes and variants of the GEMM tests this file replaces."""
    cs = []
    for M, N, K in ((4098, 3072, 1024), (4098, 1024, 1024), (4098, 4096, 1024), (4098, 1024, 4096), (4096, 896, 1024),
                    (4096, 1024, 576), (8196, 3072, 1024), (130, 128, 64), (1, 32, 8), (257, 160, 200)):
        cs += [Case(f"f32_{M}x{N}x{K}", M, N, K, 3), Case(f"f32nb_{M}x{N}x{K}", M, N, K, 3, bias=False)]
    for M, N, K in ((4098, 3072, 1024), (4098, 4096, 1024), (300, 256, 128)):
        cs += [Case(f"bias_{M}x{N}x{K}", M, N, K, 0), Case(f"gelu_{M}x{N}x{K}", M, N, K, 1)]
    for pad in (0, 2, 4, 64):
        cs += [Case(f"ldc{pad}_bf16", 4098, 1024, 512, 0, ldc_pad=pad), Case(f"ldc{pad}_f32", 4098, 1024, 512, 3, ldc_pad=pad)]
    for M in (2, 130, 4098):
        for N in (1056, 3072, 4128):
            cs += [Case(f"loads_e{e}_{M}x{N}", M, N, 256, e, ldc_pad=8 if e < 2 else 4, rps=(M + 1) // 2)
                   for e in (0, 1, 2)]
    for M in (4098, 8196, 1, 130, 257):
        for K in (1024, 4096):
            cs.append(Case(f"tails_{M}x{K}", M, 1024, K, 2, rps=4098 if M > 4098 else M))
    for M, N, K in ((4098, 4096, 1024), (300, 256, 128)):
        cs += [Case(f"train_fc1_{M}", M, N, K, 1, aux=True), Case(f"train_dgelu_{M}", M, N, K, 4, bias=False),
               Case(f"train_gate_{M}", M, N, K, 2, aux=True, resid=True, rps=M // 2 + 1),
               Case(f"train_kpad_{M}", M, N, K - 8, 3, bias=False, kpad=72)]
    for M, N, K in ((128, 128, 64), (1024, 1024, 4098), (896, 1024, 4096), (3072, 1024, 16392), (1024, 576, 4096),
                    (200, 160, 104), (4096, 1024, 4098), (1024, 4096, 8196), (4096, 4096, 520)):
        cs.append(Case(f"tn_{M}x{N}x{K}", M, N, K, "tn", bias=False))
    return cs


def gemm_cases(sms):
    cs = [c for inst in REACHABLE for c in _instantiation_cases(inst, sms)]
    return cs + product_cases() + legacy_cases()


def device_sms():
    if torch.cuda.is_available():
        return torch.cuda.get_device_properties(0).multi_processor_count
    return 132


# ---------------------------------------------------------------------------------------------------------------
# inputs, buffers and the checks (device-agnostic: tests/test_gemm_cpu.py runs them on the CPU)
# ---------------------------------------------------------------------------------------------------------------
def make_inputs(c, seed, device=DEV):
    """Operands and epilogue inputs of case c: dict of A, W (bf16, possibly K-padded), bias, gate (the whole adaLN
    table; the gate vectors at column N of its rows), x (residual), u (saved pre-activation)."""
    g = torch.Generator(device).manual_seed(seed * 1000003 + zlib.crc32(c.name.encode()) % 1000003)
    M, N, K = c.M, c.N, c.K
    tn = c.epi == "tn"
    rn = lambda *s: torch.randn(*s, device=device, generator=g)  # noqa: E731
    a = rn(M, K)
    w = rn(N, K) * (1.5 / math.sqrt(K))
    if c.regime in ("gelu_min", "gelu_sat"):
        w = w * (0.05 if c.regime == "gelu_min" else 0.3) / 1.5
    elif c.regime == "outlier":
        a[torch.tensor([0, M // 2, M - 1], device=device)] *= 64
        w[:, torch.tensor([0, K // 2], device=device)] *= 10
    elif c.regime == "cancel" and K >= 16:
        h = K // 2 // 8 * 8
        a[:, h:2 * h] = a[:, :h]
        w[:, h:2 * h] = -w[:, :h] * (1 + 0.01 * rn(N, h))
        w = w * 8
    elif c.regime == "zero_rows":
        a[::7] = 0
    bias = None
    if c.bias:
        if c.regime == "gelu_min":
            bias = og.GELU_XMIN + 0.02 * rn(N)
        elif c.regime == "gelu_sat":
            bias = torch.where(rn(N) > 0, 1.0, -1.0) * (2 + 1.5 * torch.rand(N, device=device, generator=g))
        else:
            bias = 0.5 * rn(N)
    A = a.to(torch.bfloat16)
    W = w.to(torch.bfloat16)
    if tn:
        A, W = A.t().contiguous(), W.t().contiguous()     # [K, M], [K, N]
    # tn: the rows of A [K, M] padded to a multiple of 8 elements (the TMA's 16-byte row stride)
    apad = c.kpad + ((-M) % 8 if tn else 0)
    if apad or c.kpad:
        Ap = torch.full((A.shape[0], A.shape[1] + apad), 9.0, dtype=torch.bfloat16, device=device)
        Wp = torch.full((W.shape[0], W.shape[1] + c.kpad), 9.0, dtype=torch.bfloat16, device=device)
        Ap[:, :A.shape[1]], Wp[:, :W.shape[1]] = A, W
        A, W = Ap, Wp
    d = dict(A=A, W=W, bias=bias)
    if c.epi == 2:
        samples = cdiv(M, c.rps)
        d["gate"] = rn(samples, 6 * N)
        d["x"] = rn(M, N)
    if c.epi == 4:
        if c.regime == "gelu_min":
            u = og.GELU_XMIN + 0.05 * rn(M, N)
        elif c.regime == "gelu_sat":
            u = torch.where(rn(M, N) > 0, 1.0, -1.0) * (2 + 3 * torch.rand(M, N, device=device, generator=g))
        else:
            u = 1.5 * rn(M, N)
        d["u"] = u.to(torch.bfloat16)
    return d


def logical(c, inp):
    """The logical operands (without K padding)."""
    A, W = inp["A"], inp["W"]
    if c.epi == "tn":
        return A[:, :c.M], W[:, :c.N]
    return A[:, :c.K], W[:, :c.K]


def spec_of(c, inp, path):
    gate = inp["gate"][:, c.N:2 * c.N] if c.epi == 2 else None
    return og.Spec(c.epi, c.M, c.N, c.K, bias=inp["bias"], gate=gate, rows_per_sample=c.rps, x=inp.get("x"),
                   u=inp.get("u"), aux=c.aux, bn=path.bn, splits=path.splits)


class Buf:
    """A flat buffer of `PRE (+2 when misaligned)` sentinel elements, then (M + GUARD_ROWS) rows of ldc elements, all
    sentinel; rows() is the [M + GUARD_ROWS, ldc] view that starts at the (offset) pointer."""

    def __init__(self, M, ldc, dtype, mis, device):
        self.M, self.ldc, self.dtype = M, ldc, dtype
        self.off = PRE + (2 if mis else 0)
        n = self.off + (M + GUARD_ROWS) * ldc
        itype = torch.int16 if dtype == torch.bfloat16 else torch.int32
        sent = SENT16 if dtype == torch.bfloat16 else SENT32
        self.t = torch.full((n,), sent, dtype=itype, device=device).view(dtype)

    def rows(self):
        return self.t[self.off:].view(self.M + GUARD_ROWS, self.ldc)

    def ptr(self):
        return self.t.data_ptr() + self.off * self.t.element_size()

    def bits(self):
        return self.t.view(torch.int16 if self.dtype == torch.bfloat16 else torch.int32)


def guard_changes(after, before, M, N):
    """Elements outside the [M, N] output region whose bits changed."""
    a, b = after.bits().clone(), before.bits()
    ra, rb = a[after.off:].view(after.M + GUARD_ROWS, after.ldc), b[before.off:].view(before.M + GUARD_ROWS, before.ldc)
    ra[:M, :N] = rb[:M, :N]
    return int((a != b).sum())


def check_outputs(c, spec, A, W, out, aux=None, defects=(), chunk=2048):
    """Hard check and statistics of out [M, N] (and aux [M, N]) against the model, in row chunks: a dict of counts
    and statistics.  `defects` plants defects in the model's point values, which then stand in for `out`."""
    tn = c.epi == "tn"
    st = collections.Counter()
    sq_err = sq_ref = 0.0
    kappa = 0.0
    for r0 in range(0, c.M, chunk):
        r1 = min(c.M, r0 + chunk)
        Ar = A[:, r0:r1] if tn else A[r0:r1]
        P, S = og.products(Ar.to(out.device), W.to(out.device), tn)
        m = og.model_rows(spec, P, S, r0)
        o = out[r0:r1].double()
        st["outside"] += int(((o < m["lo"]) | (o > m["hi"]) | torch.isnan(o)).sum())
        if "aux_lo" in m:
            x = aux[r0:r1].double()
            st["aux_outside"] += int(((x < m["aux_lo"]) | (x > m["aux_hi"]) | torch.isnan(x)).sum())
        pt = m["pt"]
        if spec.out_bf16:
            st["n"] += o.numel()
            st["diff"] += int((o != pt).sum())
            nz = pt != 0
            ulp = og.bf16_ulp(pt)
            st["ulp_n"] += int(nz.sum())
            st["ulp_sum"] += float((torch.sign(pt) * (o - pt) / torch.where(nz, ulp, torch.ones_like(ulp)))[nz].sum())
        else:
            sq_err += float(((o - pt) ** 2).sum())
            sq_ref += float((pt ** 2).sum())
        if (c.epi == 3 and spec.bias is None) or tn:
            base = math.sqrt(c.K) * og.U32 * S
            pos = base > 0
            if bool(pos.any()):
                kappa = max(kappa, float(((o - P).abs()[pos] / base[pos]).max()))
            del base
        del P, S, m
    res = dict(outside=st["outside"], aux_outside=st["aux_outside"])
    if spec.out_bf16:
        res["diff_frac"] = st["diff"] / max(1, st["n"])
        res["mean_ulp"] = st["ulp_sum"] / max(1, st["ulp_n"])
    else:
        res["rel32"] = math.sqrt(sq_err / max(sq_ref, 1e-300))
    if (c.epi == 3 and spec.bias is None) or tn:
        res["kappa"] = kappa
    return res


def stat_failures(c, res):
    """The checks a result fails, by name."""
    key = c.epi
    bad = []
    if res["outside"]:
        bad.append("hard")
    if res.get("aux_outside"):
        bad.append("aux")
    if "diff_frac" in res and res["diff_frac"] > DIFF_FRAC[key]:
        bad.append("diff_frac")
    if "mean_ulp" in res and abs(res["mean_ulp"]) > MEAN_ULP[key]:
        bad.append("mean_ulp")
    if "rel32" in res and res["rel32"] > REL32[key]:
        bad.append("rel32")
    return bad


# ---------------------------------------------------------------------------------------------------------------
# running a case on the GPU
# ---------------------------------------------------------------------------------------------------------------
def _lib():
    from dgs_b200 import _lib as L
    return L


def _ptr(t):
    return None if t is None else t.data_ptr()


def launch(c, inp, ldc, mis):
    """One call of case c with output row stride ldc: (out Buf, aux Buf or None, resid or None)."""
    L = _lib()
    lib = L.lib()
    M, N, K = c.M, c.N, c.K
    f32 = c.epi in (2, 3, "tn")
    out = Buf(M, ldc, torch.float32 if f32 else torch.bfloat16, mis, DEV)
    if c.epi == 2 and not c.resid:
        out.rows()[:M, :N] = inp["x"]
    aux = resid = None
    if c.aux or c.epi == 4:
        aux = Buf(M, ldc, torch.bfloat16, False, DEV)
        if c.epi == 4:
            aux.rows()[:M, :N] = inp["u"]
    if c.resid:
        resid = torch.full((M, ldc), float("nan"), device=DEV)
        resid[:, :N] = inp["x"]
    before = (out.bits().clone(), None if aux is None else aux.bits().clone())
    A, W = inp["A"], inp["W"]
    if c.epi == "tn":
        L.check(lib.dgs_gemm_bf16_tn(_ptr(A), _ptr(W), out.ptr(), M, N, K, A.shape[1], W.shape[1], ldc, L.stream(None)))
    else:
        gate = inp.get("gate")
        lda = A.shape[1] if c.kpad else 0
        L.check(lib.dgs_gemm_bf16_ex(_ptr(A), _ptr(W), _ptr(inp["bias"]), None if gate is None else gate[:, N:].data_ptr(),
                                     out.ptr(), None if aux is None else aux.ptr(), _ptr(resid), M, N, K, lda, lda, c.epi,
                                     ldc, 0 if gate is None else gate.stride(0), c.rps, L.stream(None)))
    return out, aux, resid, before


def run_case(c, seed, sms):
    """Run case c and return (path, result dict) with every check's value."""
    path = case_path(c, sms)
    inp = make_inputs(c, seed)
    keep = {k: v.clone() for k, v in inp.items() if v is not None}
    ldc = c.N + c.ldc_pad
    out, aux, resid, before = launch(c, inp, ldc, c.mis)
    torch.cuda.synchronize()
    A, W = logical(c, inp)
    spec = spec_of(c, inp, path)
    o = out.rows()[:c.M, :c.N]
    res = check_outputs(c, spec, A, W, o, None if aux is None else aux.rows()[:c.M, :c.N])
    # guard bands and unchanged inputs
    res["guard"] = guard_changes(out, _Bits(out, before[0]), c.M, c.N)
    if aux is not None:
        res["guard"] += guard_changes(aux, _Bits(aux, before[1]), c.M, 0 if c.epi == 4 else c.N)
    res["inputs_changed"] = [k for k, v in keep.items() if not torch.equal(v, inp[k])]
    if resid is not None and not torch.equal(resid[:, :c.N], inp["x"]):
        res["inputs_changed"].append("resid")
    # determinism, and the register epilogue against the TMA store
    if path.splits == 1:
        out2 = launch(c, inp, ldc, c.mis)[0]
        res["rerun_differs"] = int((out2.rows()[:c.M, :c.N].contiguous().view(-1).view(torch.int8)
                                    != o.contiguous().view(-1).view(torch.int8)).sum())
    if path.tma and c.twin:
        reg = launch(c, inp, c.N + c.ldc_pad + 2, c.mis)[0]
        assert not case_path(c._replace(ldc_pad=c.ldc_pad + 2), sms).tma
        res["tma_vs_reg"] = int((reg.rows()[:c.M, :c.N].contiguous().view(-1).view(torch.int8)
                                 != o.contiguous().view(-1).view(torch.int8)).sum())
    torch.cuda.synchronize()
    return path, res


class _Bits:
    """A Buf-like view of saved bits."""

    def __init__(self, buf, bits):
        self.off, self.M, self.ldc, self._b = buf.off, buf.M, buf.ldc, bits

    def bits(self):
        return self._b


SMS = device_sms()
CASES = gemm_cases(SMS)


def _check_case(c, seed):
    path, res = run_case(c, seed, SMS)
    print(f"{c.name} seed {seed}: {c.M}x{c.N}x{c.K} epi {c.epi} path {instantiation(path, c.epi)} splits {path.splits}: "
          + " ".join(f"{k}={v:.3g}" if isinstance(v, float) else f"{k}={v}" for k, v in res.items()))
    assert res["outside"] == 0, res
    assert res["aux_outside"] == 0, res
    assert res["guard"] == 0, res
    assert res["inputs_changed"] == [], res
    assert res.get("rerun_differs", 0) == 0, res
    assert res.get("tma_vs_reg", 0) == 0, res
    assert stat_failures(c, res) == [], res


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=[c.name for c in CASES])
def test_gemm_case(c):
    _check_case(c, 0)


# three samples of 1370 tokens, the gate vectors read from column N of each sample's wider adaLN row: the sample
# boundaries (rows 1370 and 2740) fall inside 128-row tiles and inside 64-row warpgroup slices
GATE_ADALN_CASE = Case("gate_3x1370", 3 * 1370, 1024, 512, 2, rps=1370)


@pytest.mark.gpu
def test_gate_residual_epilogue():
    """The in-place gate + residual epilogue over three samples with the gate inside a wider adaLN row, every check of
    test_gemm_case, at each seed its bounds were measured at."""
    for seed in (0, 1, 2):
        _check_case(GATE_ADALN_CASE, seed)


@pytest.mark.gpu
def test_table_reaches_every_instantiation_on_this_device():
    reached = {instantiation(case_path(c, SMS), c.epi) for c in CASES}
    assert set(REACHABLE) <= reached, set(REACHABLE) - reached


@pytest.mark.gpu
@pytest.mark.parametrize("M,Cc,layers", [(1024, 3072, 3), (4096, 1024, 2), (64, 64, 1), (1024, 1024, 24)])
@pytest.mark.parametrize("with_rm", [False, True])
def test_cast_transpose_f32(M, Cc, layers, with_rm):
    """dgs_cast_transpose_f32 as the trainer calls it after every optimizer step: `layers` fp32 [M, C] matrices at a
    layer stride of the master arena (larger than M C) -> bf16 copies [layers, M, C] (optional) and transposed bf16
    copies [layers, C, M], bit for bit, with the guard bands around both outputs and the arena gaps untouched."""
    L = _lib()
    g = torch.Generator(DEV).manual_seed(M + Cc + layers)
    stride = M * Cc + 4096 + 64
    arena = torch.randn(layers * stride, device=DEV, generator=g) * 3
    arena_keep = arena.clone()
    mats = torch.stack([arena[i * stride:i * stride + M * Cc].view(M, Cc) for i in range(layers)])
    n = layers * M * Cc
    rm = torch.full((n + 2 * PRE,), SENT16, dtype=torch.int16, device=DEV)
    tr = torch.full((n + 2 * PRE,), SENT16, dtype=torch.int16, device=DEV)
    L.check(L.lib().dgs_cast_transpose_f32(arena.data_ptr(), stride, layers, M, Cc,
                                           rm.data_ptr() + 2 * PRE if with_rm else None, tr.data_ptr() + 2 * PRE,
                                           L.stream(None)))
    torch.cuda.synchronize()
    ref = mats.to(torch.bfloat16)
    assert torch.equal(tr[PRE:PRE + n].view(torch.bfloat16).view(layers, Cc, M), ref.transpose(1, 2))
    assert bool((tr[:PRE] == SENT16).all()) and bool((tr[PRE + n:] == SENT16).all())
    if with_rm:
        assert torch.equal(rm[PRE:PRE + n].view(torch.bfloat16).view(layers, M, Cc), ref)
        assert bool((rm[:PRE] == SENT16).all()) and bool((rm[PRE + n:] == SENT16).all())
    else:
        assert bool((rm == SENT16).all())
    assert torch.equal(arena, arena_keep)
