"""CPU checks of tests/create_lines_model.py, the restatement the batched CreateNewMapLines2 is compared with on the GPU
(tests/test_kf_create_lines_gpu.py): the cv::gemm / addWeighted rules it rests on against cv2, its SVD against cv2.SVDecomp on
line-shaped matrices, its chain semantics against the reference's own LSDmatcher::SearchForTriangulation, and, on the GPU test's scene,
that the gates, the masking between neighbours and created rows sharing a tdx all occur, so that the GPU comparisons are not vacuous."""
import cv2
import numpy as np
import pytest

import create_lines_model as M
import create_points_model as MP
from test_kf_create_lines_gpu import EMPTY, SINGLE, line_svd_tables, neighbour_pairs, oracle_chain, scene

f32 = np.float32


@pytest.fixture(scope="module")
def small(pkg):
    return scene(pkg)


def chains():
    return neighbour_pairs() + [(10, k) for k in (1, 2, 3, 4, 5, 6, 7, 0)] + [(3, k) for k in (2, 4, 5, 0, 7, 10)]


def test_gemm_and_midpoint_rules():
    """K * Tcw takes cv::gemm's float path and klF.t() * M its double one, with and without GEMM_1_T (tools/probe_cv_gemm.py); the
    model's helpers are those rules; (S + E) / 2 is addWeighted(S, 0.5, E, 0.5, 0) in double."""
    import probe_cv_gemm as P
    out = P.probe_lines(n=2000, seed=5)
    assert out["K*Tcw (3,3,4)"]["float"] == 2000 and out["K*Tcw (3,3,4)"]["double"] < 2000
    for key in ("klF.t()*M GEMM_1_T (1,3,4)", "klF.t()*M (1,3,4)"):
        assert out[key]["double"] == 2000 and out[key]["float"] < 2000, (key, out[key])
    rng = np.random.default_rng(3)
    for _ in range(500):
        cam = np.array([rng.uniform(300, 1200), rng.uniform(300, 1200), rng.uniform(200, 700), rng.uniform(150, 500), 0, 0], f32)
        T = np.concatenate([rng.standard_normal((3, 3)), rng.uniform(-3, 3, (3, 1))], 1).astype(f32)
        K = np.array([[cam[0], 0, cam[2]], [0, cam[1], cam[3]], [0, 0, 1]], f32)
        Mm = cv2.gemm(K, T, 1.0, None, 0.0)
        assert np.array_equal(Mm.view(np.uint32), M.proj_mat(cam, T).view(np.uint32))
        l = (rng.standard_normal(3) * [1, 1, 400]).astype(f32)
        got = cv2.gemm(l.reshape(3, 1), Mm, 1.0, None, 0.0, flags=cv2.GEMM_1_T)
        assert np.array_equal(got.view(np.uint32), M.plane_rows(l[None], Mm).view(np.uint32))
    # midpoints: random ones, and constructed ones where halving the float sum would round differently (subnormal halves)
    a = rng.standard_normal((4000, 3)).astype(f32); b = rng.standard_normal((4000, 3)).astype(f32)
    tiny = np.finfo(f32).tiny
    a[:1000] = (rng.integers(1, 1 << 23, (1000, 3)) * 2 + 1).astype(f32) * f32(2.0 ** -149) * f32(1)
    b[:1000] = f32(tiny) * rng.integers(-3, 4, (1000, 3)).astype(f32)
    for k in range(len(a)):
        got = cv2.addWeighted(a[k:k + 1], 0.5, b[k:k + 1], 0.5, 0.0)
        assert np.array_equal(got.view(np.uint32), MP.add_weighted(a[k:k + 1], 0.5, b[k:k + 1], 0.5).view(np.uint32)), k


def test_svd_equals_cv2_on_line_matrices(pkg, oracle, small):
    """The model's SVD equals cv2.SVDecomp bit for bit on line-shaped matrices: the scene's, random lines and near-epipolar lines."""
    A = line_svd_tables(np.random.default_rng(6), 120000, small, oracle)
    assert len(A) == 120000
    W, Vt = M.svd4(A)
    diff = []
    for k in range(len(A)):
        w, _, vt = cv2.SVDecomp(A[k].copy(), flags=cv2.SVD_MODIFY_A | cv2.SVD_FULL_UV)
        if not (np.array_equal(w.ravel().view(np.uint32), W[k].view(np.uint32)) and np.array_equal(vt.view(np.uint32), Vt[k].view(np.uint32))):
            diff.append(k)
    assert not diff, (len(diff), W[diff[:4]])
    # A has rank 3 by construction (its smallest singular value is at rounding level), and the near-epipolar lines push the third one
    # towards rank 2, though not to the subnormal range where the SVD may leave cv2 for points
    assert (W[:, 3] / W[:, 0] < 1e-6).mean() > 0.9
    assert (W[:, 2] / W[:, 0]).min() < 1e-8 and W[:, 2].min() > np.finfo(f32).tiny


def test_chain_rows_equal_reference_matcher(pkg, oracle, small):
    """The rows of every pair equal the reference's own LSDmatcher::SearchForTriangulation called with the masks the chain has at that
    neighbour (KF1's has_ml plus the created rows of the earlier pairs)."""
    from oracle import ref
    if not ref.available():
        pytest.skip("the reference's libref is not built here")
    K = small
    pairs = [pr for pr in chains() if K["nl"][pr[1]] >= 2]
    E = oracle_chain(oracle, K, pairs)
    hm = None
    for p, (i, j) in enumerate(pairs):
        if p == 0 or pairs[p - 1][0] != i:
            hm = K["has_ml"].copy()
        n, rows, _ = ref.line_match(3, K["ldesc"][i, :K["nl"][i]], K["ldesc"][j, :K["nl"][j]], hm[i, :K["nl"][i]], hm[j, :K["nl"][j]])
        assert n == E[p]["n"] and np.array_equal(rows, E[p]["rows"]), p
        hm[i, E[p]["rows"][E[p]["status"] == M.CREATED, 0]] = 1


def test_scene_is_not_vacuous(pkg, oracle, small):
    K = small
    pairs = chains()
    E = oracle_chain(oracle, K, pairs)
    st = np.concatenate([e["status"] for e in E])
    seen = set(np.unique(st).tolist())
    # Every gate but four.  w == 0 needs a zero column of A (tests/test_create_points_cpu.py shows the SVD gives vt(3, 3) = 0 there).
    # The end point behind a camera while the start point passes every test (ZE1, ZE2) is not reached on this scene: both ends lie on
    # KF1's rays and within 0.61 depths of each other, so it takes a KF2 plane that crosses KF1's end ray behind the camera and its
    # start ray at least 0.3 depths in front of both; the device path of those two tests is the same as that of ZS1 / ZS2.
    want = set(range(13)) - {M.W_ZERO_S, M.W_ZERO_E, M.ZE1, M.ZE2}
    assert want <= seen, (sorted(want - seen), np.bincount(st, minlength=13))
    assert E[EMPTY - 1]["n"] == -1 and E[SINGLE - 1]["n"] == -1
    # masking: some later pair's rows differ from the matcher on the unmasked has_ml
    plain = M.create_lines(lambda p, pr, hm: oracle.line_match(3, K["ldesc"][pr[0], :K["nl"][pr[0]]], K["ldesc"][pr[1], :K["nl"][pr[1]]],
                                                                K["has_ml"][pr[0], :K["nl"][pr[0]]], K["has_ml"][pr[1], :K["nl"][pr[1]]]),
                           K, pairs)
    assert sum(e["n"] != q["n"] for e, q in zip(E, plain)) > 0
    # created rows of one pair that share a tdx
    assert any(len(np.unique(e["rows"][e["status"] == 0, 1])) < (e["status"] == 0).sum() for e in E)
    # near-epipolar lines reach the SVD: some matrix that a created row came from has a third singular value far below its first
    tr = []
    oracle_chain(oracle, K, pairs, tr)
    w = np.concatenate([t[1] for t in tr if isinstance(t[0], str) and t[0] == "w"])
    assert len(w) > 500 and (w[:, 2] / w[:, 0] < 1e-3).any()
