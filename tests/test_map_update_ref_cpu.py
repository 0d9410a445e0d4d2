"""CPU tests (no GPU): tests/map_update_model.py with the stand-in's rounding equals the reference's own MapPoint::
ComputeDistinctiveDescriptors / UpdateNormalAndDepth and MapLine::ComputeDistinctiveDescriptors / UpdateAverageDir, bit for bit, on random
elements: 1 to 40 observations, bad keyframes, a reference keyframe outside the list, ties in the medoid and octaves at the pyramid's
edges.  The entry points are tests/ref_map_update.cpp, compiled here (into a temporary directory) against the reference's headers and
linked with oracle/_ref/libref.so, the reference's sources as oracle/ref_build.sh compiles them.  Skipped when the reference is absent."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import map_update_model as mu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle")
REF = os.environ.get("SSLPL_REFERENCE_DIR", "/root/reference")
f32 = np.float32
NKF, CAP, NLEV = 41, 12, 8
SF = np.ones(NLEV, f32)
for _l in range(1, NLEV):
    SF[_l] = SF[_l - 1] * f32(1.2)                     # ORBextractor's mvScaleFactor


@pytest.fixture(scope="module")
def lib():
    libref = os.path.join(ORACLE, "_ref", "libref.so")
    if not (os.path.isdir(os.path.join(REF, "include")) and os.path.exists(libref)):
        pytest.skip("the reference's sources or oracle/_ref/libref.so are not present")
    out = os.path.join(tempfile.mkdtemp(prefix="sslpl_ref_map_"), "libref_map_update.so")
    # the flags of oracle/ref_build.sh
    cmd = [os.environ.get("SSLPL_REF_CXX", "/usr/bin/g++"), "-std=c++14", "-O2", "-ffp-contract=off", "-fno-fast-math", "-march=x86-64-v3",
           "-fPIC", "-w", f"-I{ORACLE}/refshim", f"-I{REF}/include", f"-I{REF}", f"-I{ORACLE}", "-shared", "-o", out,
           os.path.join(ROOT, "tests", "ref_map_update.cpp"), f"-L{ORACLE}/_ref", "-lref", f"-Wl,-rpath,{ORACLE}/_ref", f"-L{ORACLE}", "-loracle",
           f"-Wl,-rpath,{ORACLE}", "-Wl,--no-undefined", "-lpthread"]
    subprocess.run(cmd, check=True)
    L = C.CDLL(out)
    L.ref_update_map_points.restype = None; L.ref_update_map_lines.restype = None
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _case(rng, nel=400):
    """Keyframes (octaves mostly at the pyramid's edges 0 and NLEV - 1, descriptors with repeated rows for medoid ties) and elements."""
    n = rng.integers(4, CAP + 1, NKF).astype(np.int32)
    octave = np.where(rng.random((NKF, CAP)) < 0.5, rng.choice([0, NLEV - 1], (NKF, CAP)), rng.integers(0, NLEV, (NKF, CAP))).astype(np.int32)
    base = rng.integers(0, 256, (6, 32), dtype=np.uint8)
    desc = base[rng.integers(0, 6, (NKF, CAP))] ^ np.packbits(rng.random((NKF, CAP, 256)) < 0.03, axis=-1, bitorder="little")
    desc[rng.random((NKF, CAP)) < 0.3] = base[0]                            # exact repeats: medoid ties
    pose = np.zeros((NKF, 15), f32)
    pose[:, 0] = pose[:, 5] = pose[:, 10] = 1
    pose[:, 12:] = rng.normal(0, 0.5, (NKF, 3)).astype(f32); pose[:, 3:12:4] = -pose[:, 12:]
    bad = (rng.random(NKF) < 0.25).astype(np.uint8)
    bad[[1, 2, 3]] = 1
    E = []
    for e in range(nel):
        m = int(rng.integers(1, 41)) if e % 4 else int(rng.integers(1, 4))
        ks = sorted(rng.choice(NKF, m, replace=False).tolist()) if e != 5 else [1, 2, 3]     # element 5: only bad keyframes
        obs = [(k, int(rng.integers(0, n[k]))) for k in ks]
        rk = int(rng.choice(ks)) if rng.random() < 0.8 else int(rng.integers(0, NKF))       # sometimes outside the list: feature 0
        E.append((e, rk, obs))
    X = (rng.normal(0, 2, (nel, 3)) + [0, 0, 4]).astype(f32)
    return n, octave, desc, pose, bad, E, X


def _kf(octave):
    return np.rec.fromarrays([octave], names="octave")


@pytest.mark.parametrize("what", [mu.DESC, mu.GEOM, mu.DESC | mu.GEOM])
def test_points_equal_reference(lib, what):
    rng = np.random.default_rng(20 + what)
    n, octave, desc, pose, bad, E, X = _case(rng)
    nel = len(E)
    elem, refkf, off, obs = mu.csr(E)
    od = np.zeros((nel, 32), np.uint8); has = np.zeros(nel, np.uint8); geom = np.zeros((nel, 6), f32)
    lib.ref_update_map_points(NKF, CAP, _p(n), _p(octave), _p(desc), _p(pose), _p(bad), _p(SF), NLEV, nel, _p(X), _p(refkf), _p(off), _p(obs),
                              what, _p(od), _p(has), _p(geom))
    mp0 = np.zeros((nel, 9), f32); mp0[:, :3] = X                          # a new MapPoint: zero normal and distances, no descriptor
    mp, md, st = mu.update_points(_kf(octave), desc, n, pose, bad, mp0, np.zeros((nel, 32), np.uint8), E, SF, what, rounding="minicv")
    assert set(st.tolist()) <= {mu.OK, mu.NO_GOOD_KF}
    if what & mu.DESC:
        assert (st == mu.NO_GOOD_KF).sum() >= 1
        assert np.array_equal(has == 1, st == mu.OK)
        assert np.array_equal(od[has == 1], md[has == 1])
    assert np.array_equal(geom.view(np.uint32), mp[:, 3:].view(np.uint32)), np.nonzero((geom != mp[:, 3:]).any(1))[0][:5]
    if what & mu.GEOM:
        cv2_rule = mu.update_points(_kf(octave), desc, n, pose, bad, mp0, np.zeros((nel, 32), np.uint8), E, SF, what)[0]
        assert (cv2_rule[:, 3:6] != mp[:, 3:6]).any(1).sum() > 0                # the rounding option is not idle


@pytest.mark.parametrize("what", [mu.DESC, mu.GEOM, mu.DESC | mu.GEOM])
def test_lines_equal_reference(lib, what):
    rng = np.random.default_rng(30 + what)
    n, octave, desc, pose, bad, E, X = _case(rng)
    nel = len(E)
    pos = np.concatenate([X, X + rng.normal(0, 0.5, (nel, 3))], 1).astype(np.float64) * (1 + rng.uniform(-1e-7, 1e-7, (nel, 6)))
    elem, refkf, off, obs = mu.csr(E)
    od = np.zeros((nel, 32), np.uint8); has = np.zeros(nel, np.uint8); geom = np.zeros((nel, 6), f32); nrm = np.zeros((nel, 3))
    lib.ref_update_map_lines(NKF, CAP, _p(n), _p(octave), _p(desc), _p(pose), _p(bad), _p(SF), NLEV, nel, _p(pos), _p(refkf), _p(off), _p(obs),
                             what, _p(od), _p(has), _p(geom), _p(nrm))
    ml, md, nrm_m, st = mu.update_lines(_kf(octave), desc, n, pose, bad, pos, np.zeros((nel, 12), f32), np.zeros((nel, 32), np.uint8),
                                        np.zeros((nel, 3)), E, SF, what, rounding="minicv")
    if what & mu.DESC:
        assert np.array_equal(has == 1, st == mu.OK) and (st == mu.NO_GOOD_KF).sum() >= 1
        assert np.array_equal(od[has == 1], md[has == 1])
    if what & mu.GEOM:                                                     # a new MapLine leaves its distances uninitialised
        assert np.array_equal(nrm.view(np.uint64), nrm_m.view(np.uint64))
        assert np.array_equal(geom.view(np.uint32), ml[:, 6:].view(np.uint32)), np.nonzero((geom != ml[:, 6:]).any(1))[0][:5]
