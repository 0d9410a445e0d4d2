"""CPU tests (no GPU) of the map-element refresh (include/sslpl_map.h): the new header's functions are exported and bound with their
prototypes and called with their arity from mapping.py; the rounding rules of tests/map_update_model.py against cv2 4.13; its medoid
against the reference's own MapPoint::ComputeDistinctiveDescriptors; and its entry rules on hand-made elements."""
import ast
import ctypes as C
import os
import re
import subprocess
import numpy as np
import pytest

import map_update_model as mu
import probe_cv_matexpr as probe

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG_DIR = os.path.join(ROOT, "structure-slam-pointline_b200")
f32 = np.float32


def _arity(header):
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", header)).read(), flags=re.S)
    return {name: params.count(",") + 1 for name, params in re.findall(r"\b(sslpl_[a-z0-9_]+)\s*\(([^)]*)\)", hdr)}


def test_map_header_functions_are_bound_and_complete_the_exports(pkg):
    arity = _arity("sslpl_map.h")
    assert set(arity) == {"sslpl_update_map_points_batch_device", "sslpl_update_map_lines_batch_device"}
    # the two headers together declare exactly what the library exports, and no function twice
    so = os.path.join(PKG_DIR, "libsslpl_b200.so")
    nm = subprocess.run(["nm", "-D", "--defined-only", so], capture_output=True, text=True, check=True).stdout
    exported = {ln.split()[-1] for ln in nm.splitlines() if ln.split() and ln.split()[-1].startswith("sslpl_")}
    main = set(_arity("sslpl.h"))
    assert not main & set(arity) and main | set(arity) == exported
    lib = pkg.lib()
    for name, n in arity.items():
        fn = getattr(lib, name)
        assert fn.restype is C.c_int and len(fn.argtypes) == n, name
    pts = lib.sslpl_update_map_points_batch_device.argtypes
    assert [i for i, t in enumerate(pts) if t is C.c_int] == [4, 5, 8, 11, 17, 18]
    lns = lib.sslpl_update_map_lines_batch_device.argtypes
    assert [i for i, t in enumerate(lns) if t is C.c_int] == [4, 5, 8, 13, 19, 20]


def test_mapping_call_sites_pass_the_header_arity():
    arity = _arity("sslpl_map.h")
    tree = ast.parse(open(os.path.join(PKG_DIR, "mapping.py")).read())
    seen = set()
    for node in ast.walk(tree):
        if (isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr.startswith("sslpl_")
                and isinstance(node.func.value, ast.Call) and getattr(node.func.value.func, "id", None) == "lib"):
            assert not node.keywords and len(node.args) == arity[node.func.attr], node.func.attr
            seen.add(node.func.attr)
    assert seen == set(arity)


def test_scale_add_rule_against_cv2():
    """cv2.scaleAdd on CV_32F is fma(a, (float)alpha, b): every random row, and the midpoint row at every length; the two-rounding rule
    misses both."""
    cnt, mid = probe.probe_scale_add()
    assert cnt == dict(fused=20000, two_roundings=11392)
    assert all(fused and not two for fused, two in mid.values())


def test_scale_add_model_edges():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(11)
    a = np.concatenate([rng.standard_normal((2000, 3)) * 1e-38, rng.standard_normal((2000, 3)) * 1e30]).astype(f32)
    b = np.concatenate([rng.standard_normal((2000, 3)) * 1e-38, -a[2000:] * f32(0.999)]).astype(f32)
    for k in range(len(a)):
        alpha = float(rng.uniform(0.5, 2.0))
        assert np.array_equal(cv2.scaleAdd(a[k:k + 1], alpha, b[k:k + 1]).view(np.uint32), mu.scale_add(a[k:k + 1], alpha, b[k:k + 1]).view(np.uint32)), k


def _groups(rng, ngroups=300):
    """Descriptor groups of 1 to 40 rows, with ties: repeated rows and rows at equal distances."""
    out = []
    for g in range(ngroups):
        n = int(rng.integers(1, 41))
        base = rng.integers(0, 256, 32, dtype=np.uint8)
        d = np.repeat(base[None], n, 0)
        flips = rng.random((n, 256)) < rng.choice([0.02, 0.1, 0.3])
        d ^= np.packbits(flips, axis=1, bitorder="little")
        if g % 3 == 0 and n > 2:
            d[rng.integers(0, n, n // 2)] = d[0]
        out.append(d)
    return out


def test_medoid_equals_reference(oracle):
    from oracle import ref as R
    rng = np.random.default_rng(3)
    G = _groups(rng)
    desc = np.concatenate(G); off = np.concatenate([[0], np.cumsum([len(g) for g in G])]).astype(np.int32)
    mine = [mu.medoid(g) for g in G]
    bi_o, _ = oracle.descriptor_medoid(desc, off)
    assert [G[i][m].tobytes() for i, m in enumerate(mine)] == [G[i][b].tobytes() for i, b in enumerate(bi_o)]
    if not R.available():
        pytest.skip("the reference's library is not built")
    bi_r = R.descriptor_medoid(desc, off)
    assert [G[i][m].tobytes() for i, m in enumerate(mine)] == [G[i][b].tobytes() for i, b in enumerate(bi_r)]


def _kf_set(rng, nkf=6, cap=8):
    kps = np.zeros((nkf, cap), [("octave", np.int32)])
    kps["octave"] = rng.integers(0, 8, (nkf, cap))
    desc = rng.integers(0, 256, (nkf, cap, 32), dtype=np.uint8)
    n = np.full(nkf, cap, np.int32); n[5] = 0
    pose = np.zeros((nkf, 15), f32); pose[:, 12:] = rng.standard_normal((nkf, 3)).astype(f32)
    return kps, desc, n, pose


def test_entry_rules():
    """Statuses and what each entry writes, on hand-made elements."""
    rng = np.random.default_rng(9)
    kps, desc, n, pose = _kf_set(rng)
    kps["octave"][2, 3] = 8
    sf = (f32(1.2) ** np.arange(8)).astype(f32)
    mp = rng.standard_normal((8, 9)).astype(f32); mp[:, :3] += f32(5)
    mpdesc = rng.integers(0, 256, (8, 32), dtype=np.uint8)
    bad = np.array([0, 1, 0, 0, 0, 0], np.uint8)
    E = [(0, 0, [(0, 1), (2, 2), (3, 0)]),      # OK
         (1, 4, [(1, 0)]),                       # only bad keyframes; refkf outside the list: feature 0 of KF 4
         (2, 2, [(0, 0), (2, 3)]),               # reference octave 8
         (3, 0, []),                             # no observations
         (0, 0, [(0, 2)]),                       # element 0 again
         (4, 0, [(0, 0), (0, 1)]),               # keyframe twice
         (5, 0, [(6, 0)]),                       # keyframe out of range
         (6, 0, [(0, 8)]),                       # feature out of range
         (7, 5, [(0, 0)]),                       # refkf without features, not in the list
         (8, 0, [(0, 0)])]                       # element out of range
    out, od, st = mu.update_points(kps, desc, n, pose, bad, mp, mpdesc, E, sf, mu.DESC | mu.GEOM)
    assert st.tolist() == [mu.OK, mu.NO_GOOD_KF, mu.REF_OCTAVE, mu.NO_OBS, mu.BAD, mu.BAD, mu.BAD, mu.BAD, mu.BAD, mu.BAD]
    assert np.array_equal(out[:, :3], mp[:, :3])
    assert np.array_equal(out[3:], mp[3:]) and np.array_equal(od[1], mpdesc[1]) and np.array_equal(od[3:], mpdesc[3:])
    assert not np.array_equal(od[0], mpdesc[0]) and np.array_equal(out[2, 6:], mp[2, 6:]) and not np.array_equal(out[2, 3:6], mp[2, 3:6])
    assert np.array_equal(out[1, 8], (f32(np.sqrt(np.sum((mp[1, :3].astype(np.float64) - pose[4, 12:]) ** 2))) * sf[kps["octave"][4, 0]]))
    _, _, st = mu.update_points(kps, desc, n, pose, bad, mp, mpdesc, E, sf, mu.DESC)
    assert st.tolist()[:4] == [mu.OK, mu.NO_GOOD_KF, mu.OK, mu.NO_OBS] and st[8] == mu.OK


def test_normal_is_the_mean_ray():
    """The rounding rules change only the last bits: the normal is the mean of the unit rays, the line normal in double."""
    rng = np.random.default_rng(2)
    kps, desc, n, pose = _kf_set(rng)
    sf = (f32(1.2) ** np.arange(8)).astype(f32)
    mp = np.zeros((1, 9), f32); mp[0, :3] = (1, 2, 3)
    E = [(0, 0, [(k, 0) for k in range(5)])]
    out, _, _ = mu.update_points(kps, desc, n, pose, None, mp, np.zeros((1, 32), np.uint8), E, sf, mu.GEOM)
    r = mp[0, :3].astype(np.float64) - pose[:5, 12:]
    assert np.allclose(out[0, 3:6], (r / np.linalg.norm(r, axis=1)[:, None]).mean(0), atol=1e-6)
    pos = np.array([[1, 2, 3, 2, 3, 4]], np.float64)
    ml, _, nrm, _ = mu.update_lines(kps, desc, n, pose, None, pos, np.zeros((1, 12), f32), np.zeros((1, 32), np.uint8), np.zeros((1, 3)),
                                   E, sf, mu.GEOM)
    r = 0.5 * (pos[0, :3] + pos[0, 3:]) - pose[:5, 12:].astype(np.float64)
    assert np.allclose(nrm[0], (r / np.linalg.norm(r, axis=1)[:, None]).mean(0), rtol=0, atol=1e-14)
    assert np.array_equal(ml[0, 6:9], nrm[0].astype(f32))
