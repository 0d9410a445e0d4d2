"""GPU parity of LocalMapping's batched, device-resident triangulation matchers over keyframe pairs in HBM:
ORBmatcher::SearchForTriangulation(pKF1, pKF2, F12, pairs, false) (ORBmatcher.cc:660-826, LocalMapping::CreateNewMapPoints
LocalMapping.cc:371-440) and LSDmatcher::SearchForTriangulation(pKF1, pKF2, pairs) (LSDmatcher.cpp:382-415, CreateNewMapLines2 :911-988)
with KeyFrame::lineDescriptorMAD (KeyFrame.cc:820-846) on the device.  Every pair is compared with the oracle (pinned to the reference
in tests/test_ref_parity_cpu.py) and with the single-pair entry points.

The neighbourhood builder below is shared with tests/test_kf_triangulation_cpu.py, which checks on the oracle alone that every gate
of both matchers changes some pair's result, so that the comparisons here are not vacuous."""
import cv2
import numpy as np
import pytest

from test_motion_batch_gpu import _download, device_batch

pytestmark = pytest.mark.gpu

NKF = 21                       # KF 0 and its neighbours: 20 point neighbours (LocalMapping.cc:376, monocular nn = 20), 10 line neighbours
FLAT = 15                      # a flat keyframe (no keypoints, no lines): a point neighbour of KF 0, not a line neighbour
NPT, NLN = 20, 10
SSLPL_MAX_LEVELS = 16          # include/sslpl.h
LEVELSUP = 1                   # k = 10, L = 3 tree: FeatureVector nodes at level 2 (ORBvoc's levelsup 4 of L = 6 gives level 2 too)
VOCAB = dict(k=10, L=3, seed=21, stop_fraction=0.05, early_leaf_fraction=0.1)


def keyframe_frames(synth, W=640, H=480, nkf=NKF, flat=FLAT):
    """nkf frames of one synthetic scene (synth.batch with group = nkf), frame `flat` replaced by a flat grey image."""
    frames = synth.batch(W, H, nkf, group=nkf)
    if flat is not None:
        frames[flat] = 128
    return frames


def warp(k, group, W, H):
    """The image motion tools/synth.py applies to frame k of a group (a rotation about the image centre and a translation), 3x3."""
    t = (k % group) / (group - 1)
    M = cv2.getRotationMatrix2D((W / 2.0, H / 2.0), 1.0 * t, 1.0)
    M[0, 2] += 4.0 * t
    M[1, 2] += -3.0 * t
    return np.vstack([M, [0.0, 0.0, 1.0]])


def pair_geometry(rng, pairs, kps, n, group, W, H, p_inside=0.35, shift=0.0):
    """Per pair (kf1, kf2): F12 (x1' F12 x2 = 0, the convention of CheckDistEpipolarLine ORBmatcher.cc:140-157) and the epipole (ex, ey) of
    KF1's camera in KF2's image.  F21 = [e]x H21, with H21 the synthetic image motion from kf1 to kf2: every true correspondence lies on
    its epipolar line and e is F21's left null vector, as the epipole of a camera pair is.  With probability p_inside e sits on one of
    KF2's keypoints inside the image (the epipole-radius gate then drops it); else it is far outside.  `shift` moves H21 by that many
    pixels, which makes the epipolar-distance gate reject true matches.  Returns geom [npairs, 11] f32 = F12 row-major, ex, ey."""
    geom = np.zeros((len(pairs), 11), np.float32)
    for p, (i, j) in enumerate(pairs):
        H21 = warp(j, group, W, H) @ np.linalg.inv(warp(i, group, W, H))
        H21[0, 2] += shift
        if rng.random() < p_inside and n[j] > 0:
            kp = kps[j, int(rng.integers(0, n[j]))]
            e = np.array([kp["x"], kp["y"], 1.0])
        else:
            a = rng.uniform(0, 2 * np.pi)
            e = np.array([W / 2 + 4000 * np.cos(a), H / 2 + 4000 * np.sin(a), 1.0])
        ex = np.array([[0, -e[2], e[1]], [e[2], 0, -e[0]], [-e[1], e[0], 0]])
        F12 = (ex @ H21).T
        geom[p, :9] = (F12 / np.abs(F12).max()).reshape(-1)
        geom[p, 9:] = e[:2]
    return geom


def masks(rng, nkf, cap, capl, p_mp=0.3, p_ml=0.2):
    """has_mp [nkf, cap] (KeyFrame::GetMapPoint(i) != NULL) and has_ml [nkf, capl] (GetMapLine(i) != NULL)."""
    return (rng.random((nkf, cap)) < p_mp).astype(np.uint8), (rng.random((nkf, capl)) < p_ml).astype(np.uint8)


def vocabulary_arrays(pkg):
    return pkg.Vocabulary.random_arrays(VOCAB["k"], VOCAB["L"], seed=VOCAB["seed"], stop_fraction=VOCAB["stop_fraction"],
                                        early_leaf_fraction=VOCAB["early_leaf_fraction"])


def feature_vectors(pkg, oracle, voc_arrays, desc, n):
    """KeyFrame::ComputeBoW's FeatureVector of every keyframe on the oracle: (node ids, offsets, feature indices)."""
    parent, nd, w, leaf = voc_arrays
    out = []
    for f in range(len(n)):
        _, node, wt = oracle.vocab_transform(VOCAB["L"], parent, nd, w, leaf, desc[f, :n[f]], LEVELSUP)
        out.append(pkg.Vocabulary.feature_vector(node, wt))
    return out


def oracle_points(oracle, K, pair, geom_p, check_ori, has_mp=None):
    i, j = pair
    n1, n2 = int(K["n"][i]), int(K["n"][j])
    hm = K["has_mp"] if has_mp is None else has_mp
    return oracle.search_for_triangulation(K["desc"][i, :n1], K["desc"][j, :n2], K["fv"][i], K["fv"][j], hm[i, :n1], hm[j, :n2],
                                           K["kps"][i, :n1], K["kps"][j, :n2], geom_p[:9].reshape(3, 3), float(geom_p[9]), float(geom_p[10]),
                                           K["scale"], K["sigma2"], check_ori)


def oracle_lines(oracle, K, pair, has_ml=None):
    """(count, pairs) of LSDmatcher::SearchForTriangulation, with the batched call's -1 where KF1 has lines and KF2 fewer than 2."""
    i, j = pair
    n1, n2 = int(K["nl"][i]), int(K["nl"][j])
    hm = K["has_ml"] if has_ml is None else has_ml
    if n1 == 0:
        return 0, np.zeros((0, 2), np.int32)
    if n2 < 2:
        return -1, np.zeros((0, 2), np.int32)
    return oracle.line_match(3, K["ldesc"][i, :n1], K["ldesc"][j, :n2], hm[i, :n1], hm[j, :n2])


def neighbourhood_pairs():
    """KF 0 against its 20 point neighbours and 10 line neighbours (FLAT is among the point neighbours only)."""
    return [(0, k) for k in range(1, NPT + 1)], [(0, k) for k in range(1, NLN + 1) if k != FLAT]


# ------------------------------------------------------------------------------------------------------------------ GPU helpers
@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


def device_lines(pkg, torch, dfr, B, W, H, nlines=40):
    seg = pkg.LineSegment(nlines, max_width=W, max_height=H, max_batch=B)
    seg.extract_batch_device(dfr.data_ptr(), B, W, H, W, W * H)
    seg.sync()
    _, d_ld, _, d_nl, capl = seg.device_results()
    ld = _download(torch, d_ld, (B, capl, 32), "|u1")
    nl = _download(torch, d_nl, (B,), "<i4")
    return dict(seg=seg, d_ldesc=d_ld, d_nl=d_nl, capl=capl, ldesc=ld, nl=nl)


def keyframe_set(pkg, oracle, torch, frames, nfeatures=1000, nlines=40, seed=7, group=NKF):
    B, H, W = frames.shape
    D = device_batch(pkg, torch, frames, nfeatures)
    L = device_lines(pkg, torch, D["dfr"], B, W, H, nlines)
    rng = np.random.default_rng(seed)
    has_mp, has_ml = masks(rng, B, D["cap"], L["capl"])
    va = vocabulary_arrays(pkg)
    tb = oracle.OrbOracle(nfeatures, 1.2, 8, 20, 7).tables()
    K = dict(D, **L, has_mp=has_mp, has_ml=has_ml, voc_arrays=va, fv=feature_vectors(pkg, oracle, va, D["desc"], D["n"]),
             scale=tb["scale"], sigma2=tb["sigma2"], W=W, H=H, group=group)
    K["d_has_mp"] = torch.from_numpy(has_mp).cuda(); K["d_has_ml"] = torch.from_numpy(has_ml).cuda()
    K["voc"] = pkg.Vocabulary(VOCAB["k"], VOCAB["L"], *va)
    return K


def matcher(pkg, K, max_batch=32):
    return pkg.Matcher(max_features=K["cap"], max_lines=K["capl"], max_nodes=K["voc"].level_nodes(LEVELSUP), max_batch=max_batch)


def run_points(mt, torch, K, pairs, geom, check_ori, nlevels=8, d_has_mp=None):
    P = len(pairs)
    d_pair = torch.tensor(np.array(pairs, np.int32).reshape(-1, 2), device="cuda"); d_geom = torch.from_numpy(geom).cuda()
    d_pairs = torch.full((P, K["cap"], 2), 7, dtype=torch.int32, device="cuda"); d_nm = torch.full((P,), -7, dtype=torch.int32, device="cuda")
    mt.search_for_triangulation_batch_device(K["d_kps"], K["d_desc"], K["d_n"], len(K["n"]), K["cap"],
                                             (d_has_mp if d_has_mp is not None else K["d_has_mp"]).data_ptr(), K["voc"], LEVELSUP, P,
                                             d_pair.data_ptr(), d_geom.data_ptr(), K["scale"][:nlevels], K["sigma2"][:nlevels], check_ori,
                                             d_pairs.data_ptr(), d_nm.data_ptr())
    mt.sync()
    return d_pairs.cpu().numpy(), d_nm.cpu().numpy()


def run_lines(mt, torch, K, pairs, d_nl=None):
    P = len(pairs)
    d_pair = torch.tensor(np.array(pairs, np.int32).reshape(-1, 2), device="cuda")
    d_lp = torch.full((P, K["capl"], 2), 7, dtype=torch.int32, device="cuda"); d_nm = torch.full((P,), -7, dtype=torch.int32, device="cuda")
    mt.line_search_for_triangulation_batch_device(K["d_ldesc"], d_nl.data_ptr() if d_nl is not None else K["d_nl"], len(K["nl"]), K["capl"],
                                                  K["d_has_ml"].data_ptr(), P, d_pair.data_ptr(), d_lp.data_ptr(), d_nm.data_ptr())
    mt.sync()
    return d_lp.cpu().numpy(), d_nm.cpu().numpy()


def check_rows(got_rows, got_n, p, n, exp):
    assert got_n[p] == n, (p, int(got_n[p]), n)
    k = max(n, 0)
    assert np.array_equal(got_rows[p, :k], exp.reshape(-1, 2)), p
    assert (got_rows[p, k:] == -1).all(), p


@pytest.fixture(scope="module")
def kfs(pkg, oracle, synth, torch):
    K = keyframe_set(pkg, oracle, torch, keyframe_frames(synth))
    assert K["n"][FLAT] == 0 and K["nl"][FLAT] == 0
    assert (np.delete(K["n"], FLAT) > 500).all() and (np.delete(K["nl"], FLAT) >= 20).all()
    return K


def mixed_pairs():
    """Two neighbourhoods in one call (KF 0 and KF 12), a repeated pair, the flat keyframe in both roles."""
    return [(0, k) for k in (1, 4, 7, 9)] + [(12, k) for k in (11, 13, 14, 16, 20, 3)] + [(0, 4), (FLAT, 2), (2, FLAT), (5, 5)]


@pytest.mark.parametrize("check_ori", [True, False])
def test_points_equal_oracle(pkg, oracle, torch, kfs, check_ori):
    K = kfs
    mt = matcher(pkg, K)
    pts, _ = neighbourhood_pairs()
    for pairs in (pts, mixed_pairs()):
        geom = pair_geometry(np.random.default_rng(len(pairs)), pairs, K["kps"], K["n"], K["group"], K["W"], K["H"])
        rows, nm = run_points(mt, torch, K, pairs, geom, check_ori)
        for p, pr in enumerate(pairs):
            n, exp = oracle_points(oracle, K, pr, geom[p], check_ori)
            check_rows(rows, nm, p, n, exp)
        live = [p for p, pr in enumerate(pairs) if FLAT not in pr]
        assert (nm[[p for p in range(len(pairs)) if p not in live]] == 0).all() and (nm[live] > 30).all(), nm


def test_lines_equal_oracle(pkg, oracle, torch, kfs):
    K = kfs
    mt = matcher(pkg, K)
    _, lns = neighbourhood_pairs()
    for pairs in (lns, mixed_pairs()):
        rows, nm = run_lines(mt, torch, K, pairs)
        for p, pr in enumerate(pairs):
            n, exp = oracle_lines(oracle, K, pr)
            check_rows(rows, nm, p, n, exp)
        for p, (i, j) in enumerate(pairs):
            assert nm[p] == (0 if i == FLAT else -1 if j == FLAT else nm[p])
        assert (nm[[p for p, pr in enumerate(pairs) if FLAT not in pr]] > 0).all(), nm


@pytest.mark.parametrize("check_ori", [True, False])
def test_equal_single_pair_entry_points(pkg, torch, kfs, check_ori):
    """Every pair equals sslpl_search_for_triangulation / sslpl_line_match(mode 3) on the same handle."""
    K = kfs
    mt = matcher(pkg, K)
    pairs = mixed_pairs()
    geom = pair_geometry(np.random.default_rng(3), pairs, K["kps"], K["n"], K["group"], K["W"], K["H"])
    rows, nm = run_points(mt, torch, K, pairs, geom, check_ori)
    lrows, lnm = run_lines(mt, torch, K, pairs)
    om = pkg.ORBmatcher(0.6, check_ori, mt); lm = pkg.LSDmatcher(mt)
    for p, (i, j) in enumerate(pairs):
        n1, n2 = int(K["n"][i]), int(K["n"][j])
        n, exp = om.SearchForTriangulation(K["desc"][i, :n1], K["fv"][i], K["has_mp"][i, :n1], K["kps"][i, :n1], K["desc"][j, :n2], K["fv"][j],
                                           K["has_mp"][j, :n2], K["kps"][j, :n2], geom[p, :9], float(geom[p, 9]), float(geom[p, 10]),
                                           K["scale"], K["sigma2"])
        check_rows(rows, nm, p, n, exp)
        m1, m2 = int(K["nl"][i]), int(K["nl"][j])
        args = (K["ldesc"][i, :m1], K["has_ml"][i, :m1], K["ldesc"][j, :m2], K["has_ml"][j, :m2])
        if m1 > 0 and m2 < 2:
            with pytest.raises(pkg.SslplError, match="error -1:"):
                lm.SearchForTriangulation(*args)
            assert lnm[p] == -1 and (lrows[p] == -1).all()
        else:
            n, exp = lm.SearchForTriangulation(*args)
            check_rows(lrows, lnm, p, n, exp)


def test_defined_edge_cases(pkg, oracle, torch, kfs):
    K = kfs
    mt = matcher(pkg, K)
    # KF2 with exactly one line (and KF1 with lines): -1; KF1 with one line against KF2 with many: a normal pair
    nl1 = K["nl"].copy(); nl1[3] = 1
    d_nl1 = torch.from_numpy(nl1).cuda()
    pairs = [(0, 3), (3, 0), (0, 1)]
    rows, nm = run_lines(mt, torch, K, pairs, d_nl1)
    assert nm[0] == -1 and (rows[0] == -1).all()
    K1 = dict(K, nl=nl1)
    for p in (1, 2):
        check_rows(rows, nm, p, *oracle_lines(oracle, K1, pairs[p]))
    # out-of-range pair indices, on both entry points: -1 and no rows; the in-range pairs of the same call are unaffected
    bad = [(0, 1), (-1, 2), (0, NKF), (NKF, 0), (2, 3), (1 << 30, -5)]
    geom = pair_geometry(np.random.default_rng(9), [(0, 1), (0, 2), (0, 1), (0, 1), (2, 3), (0, 1)], K["kps"], K["n"], K["group"], K["W"], K["H"])
    rows, nm = run_points(mt, torch, K, bad, geom, True)
    lrows, lnm = run_lines(mt, torch, K, bad)
    for p, pr in enumerate(bad):
        if 0 <= min(pr) and max(pr) < NKF:
            check_rows(rows, nm, p, *oracle_points(oracle, K, pr, geom[p], True))
            check_rows(lrows, lnm, p, *oracle_lines(oracle, K, pr))
        else:
            assert nm[p] == -1 and (rows[p] == -1).all() and lnm[p] == -1 and (lrows[p] == -1).all(), p
    # nlevels smaller than some KF2 octaves: those features are never candidates == the oracle with has_mp2 = 1 for exactly them
    pairs, _ = neighbourhood_pairs()
    geom = pair_geometry(np.random.default_rng(5), pairs, K["kps"], K["n"], K["group"], K["W"], K["H"])
    nlev = 3
    rows, nm = run_points(mt, torch, K, pairs, geom, True, nlevels=nlev)
    full_rows, full_nm = run_points(mt, torch, K, pairs, geom, True)
    changed = 0
    for p, (i, j) in enumerate(pairs):
        hm = K["has_mp"].copy()
        hm[j] |= (K["kps"][j]["octave"] >= nlev).astype(np.uint8)
        check_rows(rows, nm, p, *oracle_points(oracle, K, (i, j), geom[p], True, has_mp=hm))
        changed += nm[p] != full_nm[p]
    assert changed > 0 and (K["kps"][1, :K["n"][1]]["octave"] >= nlev).any()


def test_large_frames(pkg, oracle, synth, torch):
    """1280x960, 4000 features, 500 lines."""
    frames = keyframe_frames(synth, 1280, 960, 4, None)
    K = keyframe_set(pkg, oracle, torch, frames, nfeatures=4000, nlines=500, seed=3, group=4)
    assert K["cap"] > 4000 and (K["n"] > 2000).all() and (K["nl"] > 100).all()
    mt = matcher(pkg, K, max_batch=4)
    pairs = [(0, 1), (0, 2), (0, 3), (2, 1)]
    geom = pair_geometry(np.random.default_rng(1), pairs, K["kps"], K["n"], 4, 1280, 960)
    rows, nm = run_points(mt, torch, K, pairs, geom, True)
    lrows, lnm = run_lines(mt, torch, K, pairs)
    for p, pr in enumerate(pairs):
        check_rows(rows, nm, p, *oracle_points(oracle, K, pr, geom[p], True))
        check_rows(lrows, lnm, p, *oracle_lines(oracle, K, pr))
    assert nm.min() > 300 and lnm.min() > 20, (nm, lnm)


def test_frame_handle_with_distortion(pkg, oracle, synth, torch):
    """Colour frames with k1 != 0 through pkg.Frame: the batched matcher reads device_keypoints_un(), the oracle the host keysUn."""
    B = 5
    gray = keyframe_frames(synth, nkf=B, flat=None)
    rng = np.random.default_rng(2)
    bgr = np.stack([np.clip(gray.astype(int) + rng.integers(-30, 30, gray.shape), 0, 255).astype(np.uint8) for _ in range(3)], 3)
    fr = pkg.Frame(1000, 1.2, 8, 20, 7, 40, max_width=640, max_height=480, max_batch=B)
    fr.set_camera(517.3, 516.5, 318.6, 255.3, [0.2624, -0.9531, -0.0054, 0.0026, 1.1633])
    r = fr.extract_batch(bgr)
    d_un, cap = fr.device_keypoints_un()
    _, d_desc, d_n, _ = fr.orb.device_results()
    has_mp = (rng.random((B, cap)) < 0.3).astype(np.uint8)
    va = vocabulary_arrays(pkg)
    tb = oracle.OrbOracle(1000, 1.2, 8, 20, 7).tables()
    K = dict(kps=r["keysUn"], desc=r["desc"], n=r["n"], cap=cap, d_kps=d_un, d_desc=d_desc, d_n=d_n, has_mp=has_mp,
             d_has_mp=torch.from_numpy(has_mp).cuda(), fv=feature_vectors(pkg, oracle, va, r["desc"], r["n"]),
             voc=pkg.Vocabulary(VOCAB["k"], VOCAB["L"], *va), scale=tb["scale"], sigma2=tb["sigma2"], capl=64)
    assert K["kps"].shape[1] == cap
    mt = matcher(pkg, K, max_batch=4)
    pairs = [(0, 1), (0, 2), (0, 3), (0, 4)]
    geom = pair_geometry(np.random.default_rng(4), pairs, K["kps"], K["n"], B, 640, 480, shift=0.0)
    rows, nm = run_points(mt, torch, K, pairs, geom, True)
    for p, pr in enumerate(pairs):
        check_rows(rows, nm, p, *oracle_points(oracle, K, pr, geom[p], True))
    assert nm.max() > 0


def test_caller_stream(pkg, oracle, torch, kfs):
    """On a caller-set stream the results are ready once that stream is synchronised; no sslpl_matcher_sync."""
    K = kfs
    mt = matcher(pkg, K)
    pts, lns = neighbourhood_pairs()
    geom = pair_geometry(np.random.default_rng(8), pts, K["kps"], K["n"], K["group"], K["W"], K["H"])
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        mt.set_stream(s.cuda_stream)
        d_pair = torch.tensor(np.array(pts, np.int32), device="cuda"); d_lpair = torch.tensor(np.array(lns, np.int32), device="cuda")
        d_geom = torch.from_numpy(geom).cuda()
        d_pairs = torch.full((len(pts), K["cap"], 2), 7, dtype=torch.int32, device="cuda"); d_nm = torch.full((len(pts),), -7, dtype=torch.int32, device="cuda")
        d_lp = torch.full((len(lns), K["capl"], 2), 7, dtype=torch.int32, device="cuda"); d_lnm = torch.full((len(lns),), -7, dtype=torch.int32, device="cuda")
        mt.search_for_triangulation_batch_device(K["d_kps"], K["d_desc"], K["d_n"], NKF, K["cap"], K["d_has_mp"].data_ptr(), K["voc"], LEVELSUP,
                                                 len(pts), d_pair.data_ptr(), d_geom.data_ptr(), K["scale"], K["sigma2"], True,
                                                 d_pairs.data_ptr(), d_nm.data_ptr())
        mt.line_search_for_triangulation_batch_device(K["d_ldesc"], K["d_nl"], NKF, K["capl"], K["d_has_ml"].data_ptr(), len(lns),
                                                      d_lpair.data_ptr(), d_lp.data_ptr(), d_lnm.data_ptr())
    s.synchronize()
    rows, nm, lrows, lnm = d_pairs.cpu().numpy(), d_nm.cpu().numpy(), d_lp.cpu().numpy(), d_lnm.cpu().numpy()
    for p, pr in enumerate(pts):
        check_rows(rows, nm, p, *oracle_points(oracle, K, pr, geom[p], True))
    for p, pr in enumerate(lns):
        check_rows(lrows, lnm, p, *oracle_lines(oracle, K, pr))
    mt.set_stream(0)


def test_argument_errors_enqueue_nothing(pkg, torch, kfs):
    K = kfs
    cap, capl = K["cap"], 64                    # the lines padded to max_lines + 64 = 64 rows per keyframe
    mb = 8
    mt = pkg.Matcher(max_features=cap - 64, max_lines=0, max_nodes=K["voc"].level_nodes(LEVELSUP), max_batch=mb)
    ld64 = torch.zeros((NKF, capl, 32), dtype=torch.uint8, device="cuda"); ld64[:, :K["capl"]] = torch.from_numpy(K["ldesc"]).cuda()
    hm64 = torch.zeros((NKF, capl), dtype=torch.uint8, device="cuda"); hm64[:, :K["capl"]] = K["d_has_ml"]
    pairs = np.array([(0, k) for k in range(1, mb + 1)], np.int32)
    geom = pair_geometry(np.random.default_rng(6), [tuple(pr) for pr in pairs], K["kps"], K["n"], K["group"], K["W"], K["H"])
    d_pair = torch.tensor(pairs, device="cuda"); d_geom = torch.from_numpy(geom).cuda()
    d_g0 = torch.from_numpy(pair_geometry(np.random.default_rng(6), [(0, 0)], K["kps"], K["n"], K["group"], K["W"], K["H"], p_inside=0)).cuda()
    d_pairs = torch.full((mb + 1, cap + 1, 2), 7, dtype=torch.int32, device="cuda"); d_nm = torch.full((mb + 1,), -7, dtype=torch.int32, device="cuda")
    d_lp = torch.full((mb + 1, capl + 1, 2), 7, dtype=torch.int32, device="cuda"); d_lnm = torch.full((mb + 1,), -7, dtype=torch.int32, device="cuda")
    good = dict(d_kps=K["d_kps"], d_desc=K["d_desc"], d_n=K["d_n"], nkf=mb + 1, cap=cap, d_has_mp=K["d_has_mp"].data_ptr(), vocab=K["voc"],
                levelsup=LEVELSUP, npairs=mb, d_pair=d_pair.data_ptr(), d_geom=d_geom.data_ptr(), scale=K["scale"], sigma2=K["sigma2"],
                check_ori=True, d_pairs=d_pairs.data_ptr(), d_nmatch=d_nm.data_ptr())
    lgood = dict(d_ldesc=ld64.data_ptr(), d_nl=K["d_nl"], nkf=mb + 1, capl=capl, d_has_ml=hm64.data_ptr(), npairs=mb,
                 d_pair=d_pair.data_ptr(), d_lpairs=d_lp.data_ptr(), d_nlmatch=d_lnm.data_ptr())
    one = np.ones(SSLPL_MAX_LEVELS + 1, np.float32)
    bad = [dict(d_kps=0), dict(d_desc=0), dict(d_n=0), dict(d_has_mp=0), dict(d_pair=0), dict(d_geom=0), dict(d_pairs=0), dict(d_nmatch=0),
           dict(nkf=0), dict(nkf=mb + 2), dict(npairs=0), dict(npairs=mb + 1), dict(cap=0), dict(cap=cap + 1),
           dict(scale=one[:0], sigma2=one[:0]), dict(scale=one, sigma2=one), dict(levelsup=0)]
    lbad = [dict(d_ldesc=0), dict(d_nl=0), dict(d_has_ml=0), dict(d_pair=0), dict(d_lpairs=0), dict(d_nlmatch=0), dict(nkf=0), dict(nkf=mb + 2),
            dict(npairs=0), dict(npairs=mb + 1), dict(capl=0), dict(capl=capl + 1)]
    assert K["voc"].level_nodes(0) > K["voc"].level_nodes(LEVELSUP)
    before = mt.launch_count
    for b in bad:
        with pytest.raises(pkg.SslplError, match="error -1:"):
            mt.search_for_triangulation_batch_device(**{**good, **b})
    for b in lbad:
        with pytest.raises(pkg.SslplError, match="error -1:"):
            mt.line_search_for_triangulation_batch_device(**{**lgood, **b})
    mt.sync()
    assert mt.launch_count == before
    assert (d_pairs == 7).all().item() and (d_nm == -7).all().item() and (d_lp == 7).all().item() and (d_lnm == -7).all().item()
    # the boundary values are accepted: nkf = max_batch + 1, npairs = max_batch, cap = max_features + 64, capl = max_lines + 64,
    # SSLPL_MAX_LEVELS levels, a vocabulary level of exactly max_nodes nodes; nkf = 1 with the pair (0, 0)
    mt.search_for_triangulation_batch_device(**{**good, "scale": np.resize(K["scale"], SSLPL_MAX_LEVELS), "sigma2": np.resize(K["sigma2"], SSLPL_MAX_LEVELS)})
    mt.line_search_for_triangulation_batch_device(**lgood)
    d_p0 = torch.zeros((1, 2), dtype=torch.int32, device="cuda")
    mt.search_for_triangulation_batch_device(**{**good, "nkf": 1, "npairs": 1, "d_pair": d_p0.data_ptr(), "d_geom": d_g0.data_ptr()})
    mt.line_search_for_triangulation_batch_device(**{**lgood, "nkf": 1, "npairs": 1, "d_pair": d_p0.data_ptr()})
    mt.sync()
    assert mt.launch_count == before + 7 * 2 + 2 * 2
    assert (d_nm[:mb] > 0).all().item() and (d_lnm[:mb] > 0).all().item() and (d_nm[mb:] == -7).all().item()

