"""Mesh cleaning on the H100 (dgs_mesh_clean through dgs_b200.mesh.clean): bit-for-bit equality with the serial oracle
(vertices, faces and the face count after each stage) on the hand-worked cases, on marching-cubes spheres and tori with
floating blobs and on the obj-256 extract_mesh pipeline with floaters; the properties of the cleaned mesh; the
clean-then-decimate postprocess; determinism, numpy / CUDA-tensor agreement and the edge cases."""
import numpy as np
import pytest
import torch

from mesh_clean_cases import cases
from mesh_shapes import cuda_grid, directed, mc, shell_model
from oracle import mesh_clean as oc

pytestmark = pytest.mark.gpu


def _native(v, f, **kw):
    from dgs_b200 import mesh
    stats = {}
    ov, of = mesh.clean(v, f, stats=stats, **kw)
    return ov, of, stats


def _same_as_oracle(v, f, **kw):
    ov, of, st = _native(v, f, **kw)
    rv, rf, counts = oc.clean(v, f, **kw)
    assert st["stage_faces"] == counts, f"stage face counts {st['stage_faces']} != oracle {counts}"
    assert ov.dtype == np.float32 and of.dtype == np.int64
    assert ov.tobytes() == rv.tobytes() and np.array_equal(of, rf)
    return ov, of, st


@pytest.mark.parametrize("case", cases(), ids=lambda c: c[0])
def test_hand_cases_equal_oracle(case):
    _, v, f, kw, ev, ef, counts = case
    ov, of, st = _same_as_oracle(v, f, **kw)
    assert np.array_equal(ov, ev.reshape(-1, 3)) and np.array_equal(of, ef.reshape(-1, 3)) and st["stage_faces"] == counts


def _blobs(X, Y, Z, centres, r):
    return torch.stack([r - torch.sqrt((X - a) ** 2 + (Y - b) ** 2 + (Z - c) ** 2) for a, b, c in centres]).amax(0)


@pytest.mark.parametrize("shape", ["sphere", "torus"])
@pytest.mark.parametrize("kw", [{}, dict(v_pct=0.3), dict(v_pct=2, min_f=200, min_d=10), dict(repair=False)],
                         ids=["defaults", "v_pct0.3", "v_pct2", "no_repair"])
def test_surfaces_with_blobs_equal_oracle(shape, kw):
    n = 96
    X, Y, Z = cuda_grid(n)
    if shape == "sphere":
        body = 30 - torch.sqrt(X * X + Y * Y + Z * Z)
    else:
        body = 9 - torch.sqrt((torch.sqrt(X * X + Y * Y) - 26) ** 2 + Z * Z)
    blobs = _blobs(X, Y, Z, [(40, 40, 40), (-40, 38, -36), (36, -40, 30)], 2.5)
    v, f = mc(torch.maximum(body, blobs))
    ov, of, st = _same_as_oracle(v, f, **kw)
    print(f"{shape} {kw}: {len(v)} -> {len(ov)} vertices, stage faces {st['stage_faces']}, "
          f"{st['merge_rounds']} merge rounds")
    assert st["stage_faces"][5] < st["stage_faces"][3]  # the blobs go


def _check_clean(v, f, min_f=64, min_d=20):
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    assert (f[:, 0] != f[:, 1]).all() and (f[:, 1] != f[:, 2]).all() and (f[:, 0] != f[:, 2]).all()
    assert len(np.unique(np.sort(f, axis=1), axis=0)) == len(f), "a duplicate face"
    assert (oc.doubled_area(v, f) > 0).all(), "a null face"
    e = np.sort(directed(f), axis=1)
    _, cnt = np.unique(e, axis=0, return_counts=True)
    assert cnt.max() <= 2, "an edge of more than 2 faces"
    # one fan per vertex: corners of a vertex joined through its edges form a single component
    fid = np.tile(np.arange(len(f)), 3)
    key = e[:, 0].astype(np.int64) * len(v) + e[:, 1]
    order = np.lexsort((fid, key))
    same = np.flatnonzero(key[order][1:] == key[order][:-1]) + 1
    a, b = fid[order][same], fid[order][same - 1]  # faces sharing an edge
    n_fans = 0
    vf = {}
    for i, t in enumerate(f.tolist()):
        for x in t:
            vf.setdefault(x, []).append(i)
    adj = {}
    for x, y in zip(a.tolist(), b.tolist()):
        adj.setdefault(x, set()).add(y)
        adj.setdefault(y, set()).add(x)
    for x, fs in vf.items():
        fs_set, seen, stack = set(fs), {fs[0]}, [fs[0]]
        while stack:
            g = stack.pop()
            for h in adj.get(g, ()):
                if h in fs_set and h not in seen and x in f[h] and len(set(f[g]) & set(f[h]) - {x}) == 1:
                    seen.add(h)
                    stack.append(h)
        n_fans += len(seen) != len(fs_set)
    assert n_fans == 0, f"{n_fans} vertices with more than one fan"
    _, lab = connected_components(coo_matrix((np.ones(len(a)), (a, b)), shape=(len(f), len(f))), directed=False)
    d = np.ptp(v, axis=0).astype(np.float64)
    diag = np.sqrt((d * d).sum())
    for c in np.unique(lab):
        fc = f[lab == c]
        dc = np.ptp(v[np.unique(fc)], axis=0).astype(np.float64)
        assert len(fc) >= min_f and np.sqrt((dc * dc).sum()) >= min_d / 100 * diag
    return lab


def test_obj256_pipeline_equals_oracle():
    import time
    from dgs_b200 import mesh
    m = shell_model(262146, 11)
    raw = m.extract_mesh()
    v, f = raw.vertices, raw.faces
    ov, of, st = _native(v, f)
    t0 = time.perf_counter()
    rv, rf, counts = oc.clean(v, f)
    oracle_s = time.perf_counter() - t0
    print(f"obj-256 + floaters: {len(v)} vertices / {len(f)} faces -> {len(ov)} / {len(of)}; stage faces "
          f"{st['stage_faces']}; {st['merge_rounds']} merge rounds; oracle {oracle_s:.1f} s")
    assert st["stage_faces"] == counts
    assert ov.tobytes() == rv.tobytes() and np.array_equal(of, rf)
    assert counts[4] < counts[3]  # the floaters are removed by diameter
    lab = _check_clean(ov, of)
    print(f"  {len(np.unique(lab))} components")
    # determinism and CUDA-tensor input: repeated calls, since a race in the component labelling once lost a face in
    # about one call in ten
    for _ in range(10):
        ov2, of2 = mesh.clean(v, f)
        assert ov2.tobytes() == ov.tobytes() and np.array_equal(of2, of)
    tv, tf = mesh.clean(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda())
    assert tv.is_cuda and tv.dtype == torch.float32 and tf.dtype == torch.int64
    assert tv.cpu().numpy().tobytes() == ov.tobytes() and np.array_equal(tf.cpu().numpy(), of)


def test_clean_then_decimate_postprocess():
    from dgs_b200 import mesh
    m = shell_model(262146, 11)
    out = m.extract_mesh(postprocess=mesh.clean_then_decimate)
    raw = m.extract_mesh()
    cv, cf = mesh.clean(raw.vertices, raw.faces)
    print(f"clean_then_decimate: {len(raw.faces)} -> {len(cf)} cleaned -> {len(out.faces)} faces")
    if len(cf) > 1e5:
        assert len(out.faces) <= 1e5
        dv, df = mesh.decimate(cv, cf, 1e5)
        assert np.array_equal(out.vertices, dv) and np.array_equal(out.faces, df)
    else:
        assert np.array_equal(out.vertices, cv) and np.array_equal(out.faces, cf)
    # a target above the cleaned face count: the cleaned mesh unchanged
    big = m.extract_mesh(postprocess=mesh.clean_then_decimate, decimate_target=len(cf) + 1)
    assert np.array_equal(big.vertices, cv) and np.array_equal(big.faces, cf)
    small = m.extract_mesh(postprocess=mesh.clean_then_decimate, decimate_target=len(cf) // 2)
    assert len(small.faces) <= len(cf) // 2


def test_edge_cases():
    from dgs_b200 import _lib, mesh
    X, Y, Z = cuda_grid(24)
    v, f = mc(8 - torch.sqrt(X * X + Y * Y + Z * Z))
    bad = f.copy()
    bad[7, 1] = len(v)
    with pytest.raises(_lib.DgsError, match="face 7 .* outside"):
        mesh.clean(v, bad)
    bad[7, 1] = -1
    with pytest.raises(_lib.DgsError, match="face 7 .* outside"):
        mesh.clean(v, bad)
    # V > 2^21: the sphere's indices moved above 2^21 by unreferenced padding, plus a duplicate in reverse winding
    pad = (1 << 21) + 5
    vp = np.concatenate([np.full((pad, 3), 100.0, np.float32), v])
    fp = np.concatenate([f + pad, f[:3, ::-1] + pad])
    pv, pf, _ = _same_as_oracle(vp, fp, v_pct=0.5)
    sv, sf, _ = _same_as_oracle(v, f, v_pct=0.5)
    assert pv.tobytes() == sv.tobytes() and np.array_equal(pf, sf)
    # faces that repeat an index are legal input and go as null faces without a merge
    rep = np.concatenate([f, [[0, 0, 1]]])
    _same_as_oracle(v, rep, v_pct=0)
