"""The C-ABI library loads and exports every symbol include/dgs_b200.h declares (no compute calls)."""
import ctypes
import os
import re
import subprocess

import pytest

from dgs_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    txt = open(os.path.join(ROOT, "include", "dgs_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(dgs_[a-z0-9_]+)\s*\(", txt)) - {"dgs_alloc_fn"})


def _ensure_built():
    if not os.path.exists(_lib.LIB_PATH):
        import importlib.util
        spec = importlib.util.spec_from_file_location(
            "dgs_build", os.path.join(ROOT, "open-diffusiongs_b200", "csrc", "build.py"))
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
        m.build()


def test_library_exports_every_declared_symbol():
    _ensure_built()
    L = ctypes.CDLL(_lib.LIB_PATH)
    names = _declared()
    assert len(names) >= 10
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/dgs_b200.h but not exported"
    assert sorted(_lib.EXPORTED) == names


def _struct_fields(name):
    """Field names of the typedef struct `name` in include/dgs_b200.h, in declaration order."""
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "dgs_b200.h")).read(), flags=re.S)
    body = re.search(r"typedef struct \{([^{}]*)\}\s*" + name + r"\s*;", txt).group(1)
    return [m.group(1) for decl in body.split(";") if (m := re.search(r"(\w+)\s*$", decl.strip()))]


def test_backward_trace_structs_mirror_the_header():
    """dgs_b200._lib's ctypes mirrors of dgs_dit_bwd_trace / dgs_dit_bwd_opts: same fields, same order, all pointers."""
    assert _struct_fields("dgs_dit_bwd_trace") == [n for n, _ in _lib.DitBwdTrace._fields_] == list(_lib.BWD_TRACE_FIELDS)
    assert _struct_fields("dgs_dit_bwd_opts") == [n for n, _ in _lib.DitBwdOpts._fields_] == ["block_done", "trace"]
    assert ctypes.sizeof(_lib.DitBwdTrace) == len(_lib.BWD_TRACE_FIELDS) * ctypes.sizeof(ctypes.c_void_p)
    assert _lib.DitBwdOpts.trace.offset == ctypes.sizeof(ctypes.c_void_p)
    assert not _lib.DitBwdOpts().trace  # zero-filled: no trace unless one is attached


def test_abi_version_101_and_error_string():
    _ensure_built()
    L = _lib.lib()
    assert L.dgs_version() == _lib.DGS_VERSION == 101
    assert isinstance(L.dgs_last_error(), bytes)


def test_library_of_another_version_is_refused(tmp_path, monkeypatch):
    """lib() reads dgs_version() before it sets any argtypes: a library of another ABI version raises DgsError instead of
    being called with the wrong arguments."""
    src = tmp_path / "stub.c"
    src.write_text("int dgs_version(void) { return 100; }\n")
    so = tmp_path / "libdgs_b200.so"
    subprocess.check_call(["gcc", "-shared", "-fPIC", "-o", str(so), str(src)])
    monkeypatch.setattr(_lib, "LIB_PATH", str(so))
    monkeypatch.setattr(_lib, "_lib", None)
    with pytest.raises(_lib.DgsError, match=r"version 100.*version 101.*build\.py"):
        _lib.lib()
    assert _lib._lib is None


def test_argument_validation_without_gpu():
    """Error convention of the boundary: invalid arguments -> status code + message, no exception, no GPU."""
    _ensure_built()
    L = _lib.lib()
    a = _lib.RasterArgs(P=10, D=5, M=1, W=16, H=16)
    rc = L.dgs_raster_backward(ctypes.byref(a), 0, *([None] * 15))
    assert rc == 1 and b"degree" in L.dgs_last_error()
    assert L.dgs_raster_geom_bytes(1, 1000) > 1000 * 56
    assert L.dgs_raster_image_bytes(1, 256, 256) >= 256 * 256 * 8
    # DiT train-state read-out: every case fails its argument checks before any copy, so the pointers are never read
    w = _lib.DitWeights(width=1024, heads=16, layers=2, patch=8, n_gaussians=2, mlp_hidden=4096)
    fake = ctypes.c_void_p(256)

    def export(mode, layer, state=fake, **bufs):
        return L.dgs_dit_export_state(ctypes.byref(w), 1, 4, 32, 32, mode, state, layer,
                                      *[bufs.get(k) for k in ("x", "x_mid", "h1", "qkv", "attn", "lse", "proj_out", "h2",
                                                              "u_pre", "u", "fc2_out")], None)
    STORE, RECOMPUTE = _lib.TRAIN_STORE, _lib.TRAIN_RECOMPUTE
    assert export(STORE, 3, x=fake) == 1 and b"out of range" in L.dgs_last_error()
    assert export(RECOMPUTE, -1, x=fake) == 1 and b"out of range" in L.dgs_last_error()
    assert export(RECOMPUTE, 0, h1=fake) == 1 and b"STORE" in L.dgs_last_error()
    assert export(RECOMPUTE, 1, lse=fake) == 1 and b"STORE" in L.dgs_last_error()
    assert export(STORE, 2, u=fake) == 1 and b"layers [0, 2)" in L.dgs_last_error()
    assert export(STORE, 0, state=None, x=fake) == 1 and b"train_state is NULL" in L.dgs_last_error()
    assert export(7, 0, x=fake) == 1 and b"train_mode" in L.dgs_last_error()
    # end-stage read-out: likewise rejected before any copy
    ws_bytes = L.dgs_dit_workspace_bytes(ctypes.byref(w), 1, 4, 32, 32)
    assert ws_bytes > 0

    def ends(mode=STORE, state=fake, ws=fake, nbytes=ws_bytes, **bufs):
        return L.dgs_dit_export_ends(ctypes.byref(w), 1, 4, 32, 32, mode, state, ws, nbytes,
                                     *[bufs.get(k) for k in ("x_pre", "c", "mod", "gs_tok", "img_gs", "dx0", "dx_pre",
                                                             "dmod", "dc", "d_gs_tok")], None)
    assert ends(state=None, c=fake) == 1 and b"train_state is NULL" in L.dgs_last_error()
    assert ends(nbytes=ws_bytes - 1, mod=fake) == 1 and b"workspace too small" in L.dgs_last_error()
    assert ends(ws=None, dx0=fake) == 1 and b"workspace too small" in L.dgs_last_error()
    assert ends(mode=7, dmod=fake) == 1 and b"train_mode" in L.dgs_last_error()
    # a backward with the trace armed still rejects bad arguments before any device work (the trace is never read)
    trace = _lib.DitBwdTrace(**{k: 256 for k in _lib.BWD_TRACE_FIELDS})
    opts = _lib.DitBwdOpts(trace=ctypes.pointer(trace))
    io = _lib.DitIO(B=9, V=4, H=32, W=32, train_state=256, train_mode=STORE)
    wT = _lib.DitWeightsT(**{n: 256 for n, _ in _lib.DitWeightsT._fields_})
    dout = _lib.DitOutGrads(*([256] * 5))
    grads = _lib.DitGrads()

    def backward(io):
        return L.dgs_dit_backward_ex(ctypes.byref(w), ctypes.byref(wT), ctypes.byref(io), ctypes.byref(dout),
                                     ctypes.byref(grads), ctypes.byref(opts), fake, 1 << 40, None)
    assert backward(io) == 1 and b"batch 9 > 8" in L.dgs_last_error()
    io.B, io.train_state = 1, None
    assert backward(io) == 1 and b"train_state is NULL" in L.dgs_last_error()
    w.width = 512
    assert export(STORE, 0, x=fake) == 1 and b"width" in L.dgs_last_error()
    assert ends(x_pre=fake) == 1 and b"width" in L.dgs_last_error()
