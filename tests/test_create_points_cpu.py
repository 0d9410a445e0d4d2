"""CPU checks of tests/create_points_model.py, the restatement the batched CreateNewMapPoints is compared with on the GPU
(tests/test_kf_create_points_gpu.py): its SVD against cv2.SVDecomp, its hypot against libm, the MatExpr rounding rules against cv2, its
chain semantics against the reference's own ORBmatcher::SearchForTriangulation, and, on the GPU test's scenes, that the gates, the
masking between neighbours and created rows sharing an idx2 all occur, so that the GPU comparisons are not vacuous."""
import os
import sys

import cv2
import numpy as np
import pytest

import create_points_model as M
from test_kf_create_points_gpu import FLAT, geometry, glibc_version, neighbour_pairs, oracle_chain, scene, svd_tables

f32 = np.float32


@pytest.fixture(scope="module")
def small(pkg, oracle):
    return scene(pkg, oracle)


def test_svd_equals_cv2():
    rng = np.random.default_rng(4)
    A = svd_tables(rng, 120000)
    W, Vt = M.svd4(A)
    for k in range(len(A)):
        w, _, vt = cv2.SVDecomp(A[k].copy(), flags=cv2.SVD_MODIFY_A | cv2.SVD_FULL_UV)
        assert np.array_equal(w.ravel().view(np.uint32), W[k].view(np.uint32)) and np.array_equal(vt.view(np.uint32), Vt[k].view(np.uint32)), k
    assert (Vt[:, 3, 3] == 0).any()


@pytest.mark.skipif(glibc_version() < (2, 35), reason="libm hypot is glibc's corrected algorithm only from glibc 2.35")
def test_hypot_equals_libm(pkg, oracle, small):
    rng = np.random.default_rng(8)
    n = 10 ** 7
    x = rng.standard_normal(n) * np.exp2(rng.integers(-1074, 1023, n)); y = rng.standard_normal(n) * np.exp2(rng.integers(-1074, 1023, n))
    y[: n // 2] = x[: n // 2] * rng.standard_normal(n // 2) * np.exp2(rng.integers(-60, 60, n // 2))
    x[:8] = [0.0, -0.0, np.inf, -np.inf, np.nan, 1e-320, 1e308, 3.0]; y[:8] = [0.0, 5.0, np.nan, 1.0, np.inf, 1e-310, 1e308, 4.0]
    assert np.array_equal(M.hypot(x, y).view(np.uint64), np.hypot(x, y).view(np.uint64))
    # every (p, beta) the SVD meets in the triangulations of the test scene's neighbour loop
    trace = []
    pairs = neighbour_pairs()
    oracle_chain(oracle, small, pairs, geometry(small, pairs), trace)
    p = np.concatenate([t[0] for t in trace if not isinstance(t[0], str)]); b = np.concatenate([t[1] for t in trace if not isinstance(t[0], str)])
    assert len(p) > 10000
    assert np.array_equal(M.hypot(p, b).view(np.uint64), np.hypot(p, b).view(np.uint64))


def test_matexpr_probe_rules():
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import probe_cv_matexpr as P
    n, out = P.probe(n=4000, seed=9)
    for length in (3, 4):
        assert out[("addWeighted(s, -1)", length)]["double"] == n and out[("addWeighted(0.5, 0.5)", length)]["double"] == n
        assert out[("addWeighted midpoint", length)] == dict(double=1, fused=0)
        assert out[("convertTo", length)]["float"] == n and out[("subtract", length)]["float"] == n
    # and the model's helpers are those rules
    rng = np.random.default_rng(1)
    a, b = rng.standard_normal((2000, 4)).astype(f32), rng.standard_normal((2000, 4)).astype(f32)
    s = rng.standard_normal(2000).astype(f32)
    for k in range(2000):
        got = cv2.addWeighted(a[k:k + 1], float(s[k]), b[k:k + 1], -1.0, 0.0)
        assert np.array_equal(got.view(np.uint32), M.add_weighted(a[k:k + 1], float(s[k]), b[k:k + 1], -1.0).view(np.uint32))
        x = a[k:k + 1, :3].copy(); x[0, 0] = f32(np.abs(x).max() * 2)
        got = cv2.normalize(x, None, 1.0, 0.0, cv2.NORM_INF)
        assert np.array_equal(got.view(np.uint32), M.convert_scale(x, 1.0 / float(x[0, 0])).view(np.uint32))


def test_chain_rows_equal_reference_matcher(pkg, oracle, small):
    """The rows of every pair equal the reference's own ORBmatcher::SearchForTriangulation called with the masks the chain has at that
    neighbour (KF1's has_mp plus the created rows of the earlier pairs)."""
    from oracle import ref
    if not ref.available():
        pytest.skip("the reference's libref is not built here")
    K = dict(small)
    pairs = neighbour_pairs()
    geom = geometry(K, pairs)
    fx, fy, cx, cy = [float(v) for v in K["cam"][:4]]
    camv = ref.cam(fx, fy, cx, cy, 0, K["W"], 0, K["H"])
    call = lambda i, j, hm: ref.search_for_triangulation(K["desc"][i, :K["n"][i]], K["kps"][i, :K["n"][i]], K["desc"][j, :K["n"][j]],
                                                        K["kps"][j, :K["n"][j]], K["fv"][i], K["fv"][j], hm[i, :K["n"][i]], hm[j, :K["n"][j]],
                                                        camv, K["pose"][i, :12], K["pose"][j, :12], geom[pairs.index((i, j)), :9], False)
    for p, (i, j) in enumerate(pairs):            # the reference's own epipole (from the poses, in its float arithmetic)
        geom[p, 9:11] = call(i, j, K["has_mp"])[2]
    E = oracle_chain(oracle, K, pairs, geom)
    hm = K["has_mp"].copy()
    for p, (i, j) in enumerate(pairs):
        n, rows, _ = call(i, j, hm)
        assert n == E[p]["n"] and np.array_equal(rows, E[p]["rows"]), p
        hm[i, E[p]["rows"][E[p]["status"] == M.CREATED, 0]] = 1


def test_scene_is_not_vacuous(pkg, oracle, small):
    K = dict(small)
    pairs = neighbour_pairs()
    geom = geometry(K, pairs)
    trace = []
    E = oracle_chain(oracle, K, pairs, geom, trace)
    # no triangulation meets a matrix whose two smallest singular values are subnormal (where the SVD may differ from cv2)
    w = np.concatenate([t[1] for t in trace if isinstance(t[0], str)])
    assert len(w) > 1000 and w[:, 2].min() > 1e-6, w[:, 2].min()
    st = np.concatenate([e["status"] for e in E])
    seen = set(np.unique(st).tolist())
    # Every gate but two: w == 0 needs a zero column of A (test_svd_equals_cv2 shows the SVD gives vt(3, 3) = 0 there), and dist == 0
    # is a point at a camera centre, whose depth 0 the z tests reject first
    want = set(range(10)) - {M.W_ZERO, M.DIST0}
    assert want <= seen, (sorted(want - seen), np.bincount(st, minlength=10))
    assert E[FLAT - 1]["n"] == 0
    # masking: some later pair's rows differ from the matcher on the unmasked has_mp
    plain = M.create_points(lambda p, pr, hm: oracle.search_for_triangulation(
        K["desc"][pr[0], :K["n"][pr[0]]], K["desc"][pr[1], :K["n"][pr[1]]], K["fv"][pr[0]], K["fv"][pr[1]], K["has_mp"][pr[0], :K["n"][pr[0]]],
        K["has_mp"][pr[1], :K["n"][pr[1]]], K["kps"][pr[0], :K["n"][pr[0]]], K["kps"][pr[1], :K["n"][pr[1]]], geom[p, :9].reshape(3, 3),
        float(geom[p, 9]), float(geom[p, 10]), K["scale"], K["sigma2"], False), K, pairs, K["pose"], K["cam"], K["scale"], K["sigma2"],
        K["scale_factor"])
    assert sum(e["n"] != q["n"] for e, q in zip(E[1:], plain[1:])) > 0
    # created rows of one pair that share an idx2
    assert any(len(np.unique(e["rows"][e["status"] == 0, 1])) < (e["status"] == 0).sum() for e in E)
