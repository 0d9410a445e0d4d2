"""CPU: the keyframe neighbourhood of tests/test_kf_triangulation_gpu.py, run on the oracle alone, exercises every gate of
ORBmatcher::SearchForTriangulation (ORBmatcher.cc:660-826) and LSDmatcher::SearchForTriangulation (LSDmatcher.cpp:382-415): each one
changes some pair's result, lineDescriptorMAD's nn12_mad is positive and rejects rows, and the flat keyframe matches nothing.  So the
GPU comparisons against the oracle are not vacuous."""
import numpy as np
import pytest

from test_kf_triangulation_gpu import (FLAT, NKF, feature_vectors, keyframe_frames, masks, neighbourhood_pairs, oracle_lines,
                                       oracle_points, pair_geometry, vocabulary_arrays)


@pytest.fixture(scope="module")
def kfs(pkg, oracle, synth):
    frames = keyframe_frames(synth)
    orc = oracle.OrbOracle(1000, 1.2, 8, 20, 7); lo = oracle.LineOracle(40)
    ex = [orc.extract(f) for f in frames]
    lx = [lo.extract(f) for f in frames]
    n = np.array([len(k) for k, _ in ex], np.int32); nl = np.array([len(l[1]) for l in lx], np.int32)
    cap, capl = int(n.max()), 40
    kps = np.zeros((NKF, cap), ex[0][0].dtype); desc = np.zeros((NKF, cap, 32), np.uint8); ldesc = np.zeros((NKF, capl, 32), np.uint8)
    for f in range(NKF):
        kps[f, :n[f]] = ex[f][0]; desc[f, :n[f]] = ex[f][1]; ldesc[f, :nl[f]] = lx[f][1]
    has_mp, has_ml = masks(np.random.default_rng(7), NKF, cap, capl)
    tb = orc.tables()
    K = dict(kps=kps, desc=desc, n=n, ldesc=ldesc, nl=nl, has_mp=has_mp, has_ml=has_ml, scale=tb["scale"], sigma2=tb["sigma2"],
             fv=feature_vectors(pkg, oracle, vocabulary_arrays(pkg), desc, n), group=NKF, W=640, H=480)
    assert n[FLAT] == 0 and nl[FLAT] == 0 and (np.delete(n, FLAT) > 500).all() and (np.delete(nl, FLAT) >= 20).all()
    return K


def _points(oracle, K, pairs, geom, check_ori=True, has_mp=None):
    return [oracle_points(oracle, K, pr, geom[p], check_ori, has_mp) for p, pr in enumerate(pairs)]


def _differs(a, b):
    return [p for p, ((na, pa), (nb, pb)) in enumerate(zip(a, b)) if na != nb or not np.array_equal(pa, pb)]


def test_every_point_gate_changes_some_pair(oracle, kfs):
    K = kfs
    pairs, _ = neighbourhood_pairs()
    geom = pair_geometry(np.random.default_rng(len(pairs)), pairs, K["kps"], K["n"], K["group"], K["W"], K["H"])
    base = _points(oracle, K, pairs, geom)
    counts = np.array([n for n, _ in base])
    live = [p for p, pr in enumerate(pairs) if FLAT not in pr]
    assert counts[pairs.index((0, FLAT))] == 0 and (counts[live] > 30).all(), counts
    # has_mp (ORBmatcher.cc:702-706, :725-729)
    assert len(_differs(base, _points(oracle, K, pairs, geom, has_mp=np.zeros_like(K["has_mp"])))) >= len(live) // 2
    # the epipole radius (:749-751): move every inside epipole far away
    inside = [p for p in range(len(pairs)) if 0 <= geom[p, 9] < 640 and 0 <= geom[p, 10] < 480]
    far = geom.copy(); far[inside, 9:] = 1e5
    assert inside and _differs(base, _points(oracle, K, pairs, far))
    # the epipolar distance (CheckDistEpipolarLine :140-157): the same epipoles with F from a motion 2 px off
    off = pair_geometry(np.random.default_rng(len(pairs)), pairs, K["kps"], K["n"], K["group"], K["W"], K["H"], shift=2.0)
    assert np.array_equal(off[:, 9:], geom[:, 9:]) and len(_differs(base, _points(oracle, K, pairs, off))) >= len(live) // 2
    # checkOrientation (:793-817)
    assert _differs(base, _points(oracle, K, pairs, geom, check_ori=False))


def test_every_line_gate_changes_some_pair(oracle, kfs):
    K = kfs
    _, pairs = neighbourhood_pairs()
    base = [oracle_lines(oracle, K, pr) for pr in pairs]
    assert all(n > 0 for n, _ in base)
    # has_ml (LSDmatcher.cpp:398-401)
    free = [oracle_lines(oracle, K, pr, has_ml=np.zeros_like(K["has_ml"])) for pr in pairs]
    assert len(_differs(base, free)) == len(pairs)
    # lineDescriptorMAD: nn12_mad > 0, and the 0.1 nn12_mad test (:406) rejects rows on most pairs even with no MapLines
    rejecting = 0
    for (i, j), (n, _) in zip(pairs, free):
        l1, l2 = K["ldesc"][i, :K["nl"][i]], K["ldesc"][j, :K["nl"][j]]
        _, nn12_mad = oracle.line_mad(oracle.knn2(l1, l2))
        assert nn12_mad > 0
        rejecting += n < len(l1)
    assert rejecting > len(pairs) // 2


def test_flat_keyframe(oracle, kfs):
    """No keypoints and no lines: 0 matches in both roles for points, and as KF1 for lines (as KF2 the batched call reports -1)."""
    K = kfs
    pairs = [(FLAT, 3), (3, FLAT)]
    geom = pair_geometry(np.random.default_rng(0), pairs, K["kps"], K["n"], K["group"], K["W"], K["H"])
    assert [n for n, _ in _points(oracle, K, pairs, geom)] == [0, 0]
    assert oracle_lines(oracle, K, (FLAT, 3))[0] == 0 and oracle_lines(oracle, K, (3, FLAT))[0] == -1
    assert oracle.line_match(3, K["ldesc"][FLAT, :0], K["ldesc"][3, :K["nl"][3]])[0] == 0
