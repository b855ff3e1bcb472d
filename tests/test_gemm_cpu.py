"""CPU checks of the bf16 GEMM model (oracle/gemm.py) and of the case table that tests/test_gemm_gpu.py holds the kernel
to:

* with rounding off the model is the plain fp64 epilogue of A W^T;
* gemm_path, the table's restatement of the launcher, reaches every reachable gemm_kernel instantiation at 132 SMs
  (H100 SXM) and at 114 (H100 PCIe), each with M tails, a K tail, K = 8, a partial last wave and, where the
  instantiation allows, an N tail and fewer tiles than SMs;
* power: a stand-in kernel (fp32 accumulation on the CPU, the epilogue in fp32 operations) passes every check of the
  GPU test, and each planted defect (GEMM_DEFECTS) fails the check it targets, at a case of the GPU table;
* the stride checks of dgs_gemm_bf16 / _ex / _tn return DGS_ERR_INVALID_ARGUMENT and name the argument, with no
  device.
"""
import ctypes

import pytest
import torch

from oracle import gemm as og
from test_gemm_gpu import (DIFF_FRAC, MEAN_ULP, REACHABLE, REL32, TAILS, check_outputs, gemm_cases, gemm_path,
                           instantiation, case_path, logical, make_inputs, spec_of, stat_failures)

CPU = "cpu"


def _plain(spec, A, W):
    tn = spec.epi == "tn"
    a, w = (A.double().t(), W.double().t()) if tn else (A.double(), W.double())
    acc = a @ w.t()
    if tn:
        return acc, None
    v = acc + (0 if spec.bias is None else spec.bias.double())
    aux = v if spec.aux else None
    if spec.epi in (0, 3):
        return v, aux
    if spec.epi == 5:
        return v.clamp(min=0), aux
    if spec.epi == 1:
        return torch.nn.functional.gelu(v, approximate="tanh"), aux
    if spec.epi == 4:
        u = spec.u.double().requires_grad_(True)
        torch.nn.functional.gelu(u, approximate="tanh").sum().backward()
        return v * u.grad, aux
    g = spec.gate.double()[torch.arange(spec.M) // spec.rps]
    return spec.x.double() + g * v, aux


CASES = {c.name: c for c in gemm_cases(132)}


def _small(c):
    return c.M * c.N * c.K <= 3e8


@pytest.mark.parametrize("name", ["e0tma128_1", "e1reg128_0", "e5reg128_4", "e2reg128_0", "e2tma128_2", "e3reg128_1",
                                  "e4reg128_1", "tn128s_1", "tn128_0"])
def test_unrounded_model_is_the_fp64_epilogue(name):
    c = CASES[name]
    inp = make_inputs(c, 0, CPU)
    A, W = logical(c, inp)
    spec = spec_of(c, inp, case_path(c, 132))
    P, S = og.products(A, W, c.epi == "tn")
    m = og.model_rows(spec, P, S, 0, rounding=False)
    ref, aux = _plain(spec, A, W)
    scale = float(ref.abs().max()) + 1e-300
    assert float((m["pt"] - ref).abs().max()) <= 1e-12 * scale
    assert torch.equal(m["lo"], m["pt"]) and torch.equal(m["hi"], m["pt"])
    if aux is not None:
        assert float((m["aux_pt"] - aux).abs().max()) <= 1e-12 * float(aux.abs().max())


@pytest.mark.parametrize("sms", [132, 114])
def test_table_reaches_every_instantiation(sms):
    by_inst = {}
    for c in gemm_cases(sms):
        by_inst.setdefault(instantiation(case_path(c, sms), c.epi), []).append((c, case_path(c, sms)))
    assert set(REACHABLE) <= set(by_inst), set(REACHABLE) - set(by_inst)
    # the instantiations the launcher can reach are exactly these (epi 3 with a TMA store stays at 128 columns, epi 4
    # writes from registers, and the tn GEMM at 256 columns never splits K)
    assert set(by_inst) == set(REACHABLE), set(by_inst) - set(REACHABLE)
    for inst in REACHABLE:
        cs = by_inst[inst]
        assert {c.M % 128 for c, _ in cs} >= set(TAILS), inst
        assert any(c.K % 64 for c, _ in cs) and any(c.K == 8 for c, _ in cs) or inst[0] == "tn", inst
        assert any(p.tiles * p.splits > sms and (p.tiles * p.splits) % sms for c, p in cs) or inst == ("tn", 128, True), inst
        if inst[-1] == 128 or inst[0] == "tn" and inst[1] == 128:
            assert any(c.N % 128 for c, _ in cs), inst
        few_ok = not (inst[0] in (0, 1, 3, 4, 5) and inst[-1] == 256) and not (inst[0] == 2 and inst[1:] == ("reg", 256)) \
            and inst != ("tn", 256, False)
        if few_ok:
            assert any(p.tiles < sms for c, p in cs), inst
    tn = [c for inst in REACHABLE if inst[0] == "tn" for c, _ in by_inst[inst]]
    assert any(c.K % 64 for c in tn) and any(c.K == 8 for c in tn)


def test_gemm_path_restates_the_launcher():
    # the obj-256 linears at 132 SMs: qkv and fc1 on 128 x 256 tiles, the in-place gate on 128 x 256 at any M,
    # the tokenizer's fp32 TMA store on 128 x 128, fc1 with aux from registers
    assert gemm_path(4098, 3072, 1024, 0, 3072) == (256, True, 1, 33 * 12)
    assert gemm_path(4098, 1024, 1024, 2, 1024) == (256, True, 1, 33 * 4)
    assert gemm_path(4096, 1024, 1728, 3, 1024).bn == 128
    assert gemm_path(4098, 4096, 1024, 1, 4096, aux=True) == (256, False, 1, 33 * 16)
    assert gemm_path(4098, 1024, 512, 0, 1026).tma is False
    # the weight gradient of attn.proj: 64 tiles, split K into 3 units per tile (65 k-blocks, at least 8 per unit)
    p = gemm_path(1024, 1024, 4098, "tn", 1024)
    assert p.bn == 128 and p.tiles == 64 and p.splits == 3


def _standin(c, spec, A, W):
    """fp32 accumulation on the CPU and the epilogue in fp32 operations."""
    tn = c.epi == "tn"
    a, w = (A.float().t(), W.float().t()) if tn else (A.float(), W.float())
    acc = a @ w.t()
    if tn:
        return acc, None
    v = acc + (0 if spec.bias is None else spec.bias.float())
    aux = v.to(torch.bfloat16) if spec.aux else None
    k0, k1 = torch.tensor(og.K0, dtype=torch.float32), torch.tensor(og.K1, dtype=torch.float32)
    if c.epi == 0:
        return v.to(torch.bfloat16), aux
    if c.epi == 5:
        return v.clamp(min=0).to(torch.bfloat16), aux
    if c.epi == 3:
        return v, aux
    if c.epi == 1:
        t = torch.tanh(k0 * (v + k1 * v * v * v))
        return (0.5 * v * (1 + t)).to(torch.bfloat16), aux
    if c.epi == 4:
        x = spec.u.float()
        x2 = x * x
        t = torch.tanh(k0 * (x + k1 * x * x2))
        d = 0.5 * (1 + t) + 0.5 * x * (1 - t * t) * (k0 * (1 + 3 * k1 * x2))
        return (v * d).to(torch.bfloat16), aux
    g = spec.gate.float()[torch.arange(c.M) // spec.rps]
    return spec.x.float() + g * v, aux


# defect -> (a case of the GPU table where it shows, the check that must fail)
POWER = {
    "bias_pair_last_tile": ("e0tma128_1", "hard"),
    "gate_row_tile_first": ("e2tma128_1", "hard"),
    "gelu_erf": ("e1tma128_2", "diff_frac"),
    "bf16_round_to_zero": ("e0tma128_1", "diff_frac"),
    "last_kblock_dropped": ("e3tma128_1", "hard"),
    "rows_past_m_stored": ("e0reg128_1", "guard"),
    "splitk_partial_twice": ("tn128s_1", "hard"),
    "aux_post_activation": ("e1reg128_0", "aux"),
    "dgelu_no_x2_term": ("e4reg128_1", "hard"),
    "staged_chunk_swapped": ("e5tma128_1", "hard"),
}


def _setup(name):
    c = CASES[name]
    assert _small(c), name
    inp = make_inputs(c, 0, CPU)
    A, W = logical(c, inp)
    return c, A, W, spec_of(c, inp, case_path(c, 132))


def test_every_defect_has_a_power_case():
    assert set(POWER) == set(og.GEMM_DEFECTS)


@pytest.mark.parametrize("name", sorted({v[0] for v in POWER.values()}))
def test_standin_kernel_passes_every_check(name):
    c, A, W, spec = _setup(name)
    out, aux = _standin(c, spec, A, W)
    res = check_outputs(c, spec, A, W, out, aux)
    print(name, res)
    assert stat_failures(c, res) == [], res


def _margin(c, res, check):
    """How many times the bound a statistic is."""
    if check == "diff_frac":
        return res["diff_frac"] / DIFF_FRAC[c.epi]
    if check == "mean_ulp":
        return abs(res["mean_ulp"]) / MEAN_ULP[c.epi]
    return res["rel32"] / REL32[c.epi]


@pytest.mark.parametrize("defect", list(og.GEMM_DEFECTS))
def test_planted_defect_fails_its_check(defect):
    name, check = POWER[defect]
    c, A, W, spec = _setup(name)
    out, aux, guard = og.model_output(spec, A, W, defects=(defect,))
    res = check_outputs(c, spec, A, W, out, aux)
    res["guard"] = int((~torch.isnan(guard)).sum())
    failed = stat_failures(c, res) + (["guard"] if res["guard"] else [])
    print(defect, name, res, failed)
    assert check in failed, (defect, res)
    if check in ("diff_frac", "mean_ulp", "rel32"):
        assert _margin(c, res, check) >= 2, (defect, res)
    # and the same model without the defect passes
    out, aux, guard = og.model_output(spec, A, W)
    res = check_outputs(c, spec, A, W, out, aux)
    assert stat_failures(c, res) == [] and bool(torch.isnan(guard).all()), res


def test_stride_checks_without_gpu():
    from dgs_b200 import _lib
    L = _lib.lib()
    fake = ctypes.c_void_p(256)

    def ex(M, N, K, lda, ldb, ldc, epi=0):
        return L.dgs_gemm_bf16_ex(fake, fake, None, None, fake, None, None, M, N, K, lda, ldb, epi, ldc, 0, 1, None)

    assert L.dgs_gemm_bf16(fake, fake, None, None, fake, 256, 128, 64, 0, 96, 0, 1, None) == 1
    assert b"ldc=96" in L.dgs_last_error() and b"N=128" in L.dgs_last_error()
    assert ex(256, 128, 64, 0, 0, 96, epi=3) == 1 and b"ldc=96" in L.dgs_last_error()
    assert ex(256, 128, 64, 56, 0, 128) == 1 and b"lda=56" in L.dgs_last_error()
    assert ex(256, 128, 64, 0, 32, 128) == 1 and b"ldb=32" in L.dgs_last_error()

    def tn(M, N, K, lda, ldb, ldc):
        return L.dgs_gemm_bf16_tn(fake, fake, fake, M, N, K, lda, ldb, ldc, None)

    assert tn(256, 128, 64, 248, 0, 0) == 1 and b"lda=248" in L.dgs_last_error()
    assert tn(256, 128, 64, 0, 96, 0) == 1 and b"ldb=96" in L.dgs_last_error()
    assert tn(256, 128, 64, 0, 0, 96) == 1 and b"ldc=96" in L.dgs_last_error()
