"""CPU tests (no GPU): tests/kf_frame_match_model.py's keyframe-to-frame matchers against the reference's own bodies through oracle/ref.py:
ORBmatcher::SearchByBoW(KeyFrame*, Frame&) with the keyframe's MapPoints NULL / good / bad as an element map gives them, and
LSDmatcher::SearchByProjection(KeyFrame*, Frame&) with NULL MapLines.  The scenes are relocalisation-shaped: one frame against many
candidate keyframes whose MapPoints come from one shared pool, with bad elements and one MapPoint at two keyframe indices.  Skipped
when the reference library is absent."""
import numpy as np
import pytest

import kf_frame_match_model as km

NKF = 8                        # candidate keyframes: rows 0..7; the frame is row 8


@pytest.fixture(scope="module")
def ref():
    from oracle import ref as R
    if not R.available():
        pytest.skip("the reference library (oracle/_ref/libref.so) is not present")
    return R


def scene(pkg, oracle, synth, seed, W=640, H=480, nfeatures=1000, nlines=40):
    """A host row set: NKF keyframes and one frame of one synthetic scene, 1000 features and 40 lines each, element maps drawn from
    pools of 1500 MapPoints (8 % bad) and 150 MapLines."""
    rng = np.random.default_rng(seed)
    frames = synth.batch(W, H, NKF + 1, start=seed * (NKF + 1), group=NKF + 1)
    orb = oracle.OrbOracle(nfeatures, 1.2, 8, 20, 7); lo = oracle.LineOracle(nlines)
    pts = [orb.extract(f) for f in frames]; lns = [lo.extract(f) for f in frames]
    cap, capl = nfeatures + 64, nlines + 64
    nrows = len(frames)
    kps = np.zeros((nrows, cap), pkg.KEYPOINT_DTYPE); desc = np.zeros((nrows, cap, 32), np.uint8); ldesc = np.zeros((nrows, capl, 32), np.uint8)
    n = np.array([len(k) for k, _ in pts], np.int32); nl = np.array([len(d) for _, d, _ in lns], np.int32)
    for r in range(nrows):
        kps[r, :n[r]] = pts[r][0]; desc[r, :n[r]] = pts[r][1]; ldesc[r, :nl[r]] = lns[r][1]
    nmp, nml = 1500, 150
    R = dict(kps=kps, desc=desc, n=n, ldesc=ldesc, nl=nl, nmp=nmp, nml=nml,
             kfmp=km.element_maps(rng, n, cap, nmp), bad=(rng.random(nmp) < 0.08).astype(np.uint8),
             kfml=km.element_maps(rng, nl, capl, nml, p_null=0.3, twice=False))
    va = km.vocabulary_arrays(pkg)
    fvs = {}
    R["fv"] = lambda r: fvs.setdefault(r, km.feature_vector(oracle, va, desc[r, :km.clamp(n[r], cap)]))
    return R


@pytest.fixture(scope="module")
def scenes(pkg, oracle, synth):
    return [scene(pkg, oracle, synth, s) for s in range(2)]


@pytest.mark.parametrize("nnratio", [0.75, 0.9])                   # Tracking.cc:1979 (Relocalization), :1013 (TrackReferenceKeyFrame)
@pytest.mark.parametrize("check_ori", [True, False])
def test_points_model_equals_reference(oracle, ref, scenes, nnratio, check_ori):
    total = 0
    for R in scenes:
        for kr in range(NKF):
            n_m, m_m = km.search_by_bow(oracle, R, R["fv"], (kr, NKF), nnratio, check_ori)
            n1, n2 = int(R["n"][kr]), int(R["n"][NKF])
            state = km.element_state(R["kfmp"][kr, :n1], R["nmp"], R["bad"])
            n_r, m_r = ref.search_by_bow(R["desc"][kr, :n1], R["kps"][kr, :n1], R["desc"][NKF, :n2], R["kps"][NKF, :n2], R["fv"](kr),
                                         R["fv"](NKF), state, nnratio, check_ori)
            assert n_m == n_r, (kr, n_m, n_r)
            assert np.array_equal(m_m[:n2], m_r) and (m_m[n2:] == -1).all(), kr
            total += n_m
    assert total > 100


def test_points_element_semantics_matter(oracle, scenes):
    """Bad elements, out-of-range indices and NULLs each change some pair's result, so the parity above is not vacuous; the element shared
    by two keyframe indices and elements shared between keyframes are present."""
    R = scenes[0]
    changed = {"bad": 0, "out": 0, "null": 0}
    for kr in range(NKF):
        want = km.search_by_bow(oracle, R, R["fv"], (kr, NKF), 0.75, True)
        alt = dict(R, bad=None)
        changed["bad"] += not np.array_equal(km.search_by_bow(oracle, alt, R["fv"], (kr, NKF), 0.75, True)[1], want[1])
        alt = dict(R, kfmp=np.where(R["kfmp"] >= R["nmp"], 0, R["kfmp"]), bad=None)
        alt_null = dict(alt, kfmp=np.where(alt["kfmp"] < 0, 0, alt["kfmp"]))
        changed["out"] += not np.array_equal(km.search_by_bow(oracle, alt, R["fv"], (kr, NKF), 0.75, True)[1],
                                             km.search_by_bow(oracle, dict(R, bad=None), R["fv"], (kr, NKF), 0.75, True)[1])
        changed["null"] += not np.array_equal(km.search_by_bow(oracle, alt_null, R["fv"], (kr, NKF), 0.75, True)[1],
                                              km.search_by_bow(oracle, alt, R["fv"], (kr, NKF), 0.75, True)[1])
    assert min(changed.values()) > 0, changed
    assert (R["kfmp"][:, 3] == R["kfmp"][:, 7]).all()
    used = [set(R["kfmp"][r, :R["n"][r]][(R["kfmp"][r, :R["n"][r]] >= 0) & (R["kfmp"][r, :R["n"][r]] < R["nmp"])]) for r in range(NKF)]
    assert len(used[0] & used[1]) > 0


def test_lines_model_equals_reference(oracle, ref, scenes):
    total = 0
    for R in scenes:
        for kr in range(NKF):
            n_m, m_m = km.line_match(oracle, R, (kr, NKF))
            n1, n2 = int(R["nl"][kr]), int(R["nl"][NKF])
            has = km.element_state(R["kfml"][kr, :n1], R["nml"]) != 0
            n_r, m_r, _ = ref.line_match(0, R["ldesc"][kr, :n1], R["ldesc"][NKF, :n2], has.astype(np.uint8))
            assert n_m == n_r, (kr, n_m, n_r)
            assert np.array_equal(m_m[:n2], m_r) and (m_m[n2:] == -1).all(), kr
            total += n_m
        # all MapLines NULL: no match
        n_m, m_m = km.line_match(oracle, dict(R, kfml=np.full_like(R["kfml"], -1)), (0, NKF))
        assert n_m == 0 and (m_m == -1).all()
    assert total > 10


def test_conventions_outside_the_reference(oracle, scenes):
    """The -1 conventions of the batched calls: a row outside the set, and a keyframe with lines against a frame with fewer than 2."""
    R = scenes[0]
    for pair in ((-1, -1), (0, len(R["n"])), (len(R["n"]), 0)):
        n, m = km.search_by_bow(oracle, R, R["fv"], pair, 0.75, True)
        assert n == -1 and (m == -1).all()
        n, m = km.line_match(oracle, R, pair)
        assert n == -1 and (m == -1).all()
    for nlf, want in ((0, -1), (1, -1), (2, None)):
        nl = R["nl"].copy(); nl[NKF] = nlf
        n, m = km.line_match(oracle, dict(R, nl=nl), (0, NKF))
        assert (n == want) if want is not None else n >= 0
    nl = R["nl"].copy(); nl[0] = 0; nl[NKF] = 1
    assert km.line_match(oracle, dict(R, nl=nl), (0, NKF))[0] == 0
