"""CPU tests (no GPU): tests/init_match_model.py's chains of SearchForInitialization calls on the oracle against the same chains of the
reference's own ORBmatcher::SearchForInitialization (ORBmatcher.cc:408-523) through oracle/ref.py, vbPrevMatched carried from pair to pair
in both; and LSDmatcher::SerachForInitialize (LSDmatcher.cpp:257-284) pair by pair.  Frames come from the 2 x nFeatures extractor
(Tracking.cc:120, :163) at 640x480.  Skipped when the reference library is absent."""
import numpy as np
import pytest

import init_match_model as im

W, H, NF, NL = 640, 480, 2000, 40
BOUNDS = (0.0, float(W), 0.0, float(H))


@pytest.fixture(scope="module")
def ref():
    from oracle import ref as R
    if not R.available():
        pytest.skip("the reference library (oracle/_ref/libref.so) is not present")
    return R


def ref_call(ref):
    return lambda d1, k1, d2, k2, prev, bounds, nnratio, ori, window: ref.search_for_initialization(
        d1, k1, d2, k2, prev, ref.cam(500, 500, W / 2, H / 2, *bounds), 8, 1.2, nnratio, ori, window)


def row_set(pkg, oracle, frames):
    orb = oracle.OrbOracle(NF, 1.2, 8, 20, 7); lo = oracle.LineOracle(NL)
    pts = [orb.extract(f) for f in frames]; lns = [lo.extract(f) for f in frames]
    cap, capl = max(len(k) for k, _ in pts) + 8, NL + 64
    nrows = len(frames)
    R = dict(kps=np.zeros((nrows, cap), pkg.KEYPOINT_DTYPE), desc=np.zeros((nrows, cap, 32), np.uint8), n=np.array([len(k) for k, _ in pts]),
             ldesc=np.zeros((nrows, capl, 32), np.uint8), nl=np.array([len(d) for _, d, _ in lns]))
    for r in range(nrows):
        R["kps"][r, :R["n"][r]] = pts[r][0]; R["desc"][r, :R["n"][r]] = pts[r][1]; R["ldesc"][r, :R["nl"][r]] = lns[r][1]
    return R


def pan(img, nframes, step):
    """The image moved left by step px per frame (edge-padded): the matches, and the carried windows, walk towards the left border."""
    return np.stack([np.pad(img[:, step * k:], ((0, 0), (0, step * k)), mode="edge") for k in range(nframes)])


@pytest.fixture(scope="module")
def scenes(pkg, oracle, synth):
    seq = row_set(pkg, oracle, synth.batch(W, H, 9, start=32, group=16))
    panned = row_set(pkg, oracle, pan(synth.frame(W, H, 3), 9, 14))
    return seq, panned


def chains_1_to_8(nrows):
    """Chains of length 1 .. 8, each on its own init row, current rows the following rows (cyclically)."""
    pairs = []
    for L in range(1, 9):
        r1 = (L - 1) % nrows
        pairs += [(r1, (r1 + k) % nrows) for k in range(1, L + 1)]
    return pairs


def assert_same_chains(a, b):
    assert len(a) == len(b)
    for p, ((na, ma, pa), (nb, mb, pb)) in enumerate(zip(a, b)):
        assert na == nb, (p, na, nb)
        assert (ma is None) == (mb is None) and (ma is None or (np.array_equal(ma, mb) and np.array_equal(pa, pb))), p


@pytest.mark.parametrize("window", [50, 100])
@pytest.mark.parametrize("nnratio", [0.9, 0.7])
@pytest.mark.parametrize("check_ori", [True, False])
def test_point_chains_equal_reference(oracle, ref, scenes, window, nnratio, check_ori):
    R = scenes[0]
    pairs = chains_1_to_8(len(R["n"]))
    got = im.points(oracle.search_for_initialization, R, pairs, BOUNDS, nnratio, check_ori, window)
    want = im.points(ref_call(ref), R, pairs, BOUNDS, nnratio, check_ori, window)
    assert_same_chains(got, want)
    assert sum(n for n, _, _ in got) > 100 * len(pairs)


def test_carried_state_matters(oracle, scenes):
    """Carrying vbPrevMatched changes later pairs of a chain (here the panning one, which moves 14 px a frame), so the parities above
    cover the carried state."""
    R = scenes[1]
    pairs = [(0, k) for k in range(1, 9)]
    carried = im.points(oracle.search_for_initialization, R, pairs, BOUNDS)
    fresh = [im.points(oracle.search_for_initialization, R, [pr], BOUNDS)[0] for pr in pairs]
    assert carried[0][0] == fresh[0][0] and np.array_equal(carried[0][1], fresh[0][1])
    assert any(not np.array_equal(c[1], f[1]) for c, f in zip(carried[1:], fresh[1:]))


@pytest.mark.parametrize("window", [50, 100])
@pytest.mark.parametrize("shift", [(0.0, 0.0), (-130.0, 60.0), (700.0, -500.0)])
def test_windows_across_the_border(oracle, ref, scenes, window, shift):
    """A panning chain carries its windows to the left border; prev0 moved by `shift` starts windows partly or wholly outside the image."""
    R = scenes[1]
    pairs = [(0, k) for k in range(1, 9)] + [(1, 0), (1, 2)]
    cap = R["desc"].shape[1]
    prev0 = np.zeros((len(pairs), cap, 2), np.float32)
    for p in im.chain_starts(pairs):
        r1 = pairs[p][0]
        prev0[p, :, 0] = R["kps"][r1]["x"] + shift[0]; prev0[p, :, 1] = R["kps"][r1]["y"] + shift[1]
    got = im.points(oracle.search_for_initialization, R, pairs, BOUNDS, 0.9, True, window, prev0)
    want = im.points(ref_call(ref), R, pairs, BOUNDS, 0.9, True, window, prev0)
    assert_same_chains(got, want)
    last = got[7][2]
    assert (last[:, 0] < window).sum() > 50 or shift[0] > 600             # windows that cross x = 0 in the last pair of the pan


def test_lines_equal_reference(oracle, ref, scenes):
    for R in scenes:
        nrows = len(R["nl"])
        total = 0
        for pair in chains_1_to_8(nrows):
            n, rows = im.lines(oracle, R, pair)
            r1, r2 = pair
            n_r, m_r, _ = ref.line_match(1, R["ldesc"][r1, :R["nl"][r1]], R["ldesc"][r2, :R["nl"][r2]])
            assert n == n_r and np.array_equal(rows[:n], m_r) and (rows[n:] == -1).all(), pair
            total += n
        assert total > 10


def test_line_conventions_outside_the_reference(oracle, scenes):
    R = scenes[0]
    for pair in ((-1, 0), (0, len(R["nl"])), (len(R["nl"]), 0)):
        n, rows = im.lines(oracle, R, pair)
        assert n == -1 and (rows == -1).all()
    for nl1, nl2, want in ((5, 1, -1), (5, 0, -1), (0, 0, 0), (0, 1, 0)):
        nl = R["nl"].copy(); nl[0] = nl1; nl[1] = nl2
        n, rows = im.lines(oracle, dict(R, nl=nl), (0, 1))
        assert n == want and (rows == -1).all()
