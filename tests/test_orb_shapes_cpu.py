"""ORB extraction over frame shapes and extractor parameters (tests/orb_shapes.py): wide strips, portrait frames, the smallest
legal frames, sizes either side of the 30-px cells and the 64x32 blur tiles, 1 to 16 levels, scale factors 1.05 to 2.0, FAST
thresholds at the ends of the byte range, and saturated, binary and corner-pair contents.

- The oracle's restatement (oracle/orb_oracle.cpp) against the reference's own ORBextractor (oracle/_ref/libref.so, built where the
  reference's sources are present): keypoint bytes, descriptors and per-level counts bit for bit, wherever the reference is defined.
- Every level's keypoint count against max(N + 2, 4 nIni), the bound the device sizes its per-level capacities from."""
import os

import numpy as np
import pytest

import orb_shapes as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_ref = pytest.mark.skipif(not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libref.so")),
                               reason="the reference's ORBextractor (oracle/_ref/libref.so) is not built here")


def _run(oracle, c):
    orc = oracle.OrbOracle(c.nf, c.sf, c.nl, c.ini, c.mn)
    img = S.frame(c.kind, c.W, c.H)
    k, d = orc.extract(img)
    lv = S.levels(orc.tables(), c.W, c.H)
    counts = [len(orc.level_keypoints(l)[0]) for l in range(c.nl)]
    return orc, img, k, d, lv, counts


def _assert_within_bound(c, lv, counts):
    for v, n in zip(lv, counts):
        assert n <= v["bound"], f"{c.id}: level {v['l']} keeps {n} keypoints > max(N + 2, 4 nIni) = {v['bound']} ({v})"


@pytest.mark.parametrize("c", S.GRID, ids=[c.id for c in S.GRID])
def test_level_counts_within_bound(oracle, c):
    """The restated level geometry is the oracle's, and no level keeps more than max(N + 2, 4 nIni) keypoints."""
    orc, img, k, d, lv, counts = _run(oracle, c)
    for v in lv:
        assert orc.level_size(v["l"]) == (v["w"], v["h"]), (c.id, v)
        if not v["cells"] or v["nIni"] == 0:
            assert counts[v["l"]] == 0, (c.id, v)
    _assert_within_bound(c, lv, counts)
    assert len(k) == sum(counts) and list(np.bincount(k["octave"], minlength=c.nl)) == counts


def test_first_split_exceeds_the_level_budget(oracle):
    """What the bound is for: on wide frames and small budgets the first split alone leaves 4 nIni nodes, far past N + 16."""
    c = next(c for c in S.STRIPS if c.id == "4095x120-noise")
    _, _, _, _, lv, counts = _run(oracle, c)
    assert lv[3]["nIni"] == 63 and lv[3]["N"] == 126 and counts[3] == 252 == lv[3]["bound"]
    c = next(c for c in S.STRIPS if c.id == "1280x62-noise-8x1")
    _, _, _, _, lv, counts = _run(oracle, c)
    assert (lv[0]["N"], lv[0]["nIni"], counts[0]) == (8, 42, 168)
    over = [c.id for c in S.STRIPS if any(n > v["N"] + 16 for v, n in zip(*_run(oracle, c)[4:]))]
    assert len(over) == len(S.STRIPS), sorted(set(c.id for c in S.STRIPS) - set(over))


def test_grid_covers_the_edges(oracle):
    """The sweep reaches what it is meant to: levels with N = 0 and N = 1, levels without a cell or with nIni = 0 next to
    ones with keypoints, frames the reference is not defined on, and widths that are not multiples of 16."""
    seen = dict(N0=0, N1=0, nocell=0, nini0=0, undefined=0, odd_width=0)
    for c in S.GRID:
        lv = S.levels(oracle.OrbOracle(c.nf, c.sf, c.nl, c.ini, c.mn).tables(), c.W, c.H)
        seen["N0"] += any(v["N"] == 0 and v["cells"] for v in lv)
        seen["N1"] += any(v["N"] == 1 and v["cells"] for v in lv)
        seen["nocell"] += any(not v["cells"] for v in lv)
        seen["nini0"] += any(v["cells"] and v["nIni"] == 0 for v in lv)
        seen["undefined"] += not S.reference_defined(lv)
        seen["odd_width"] += c.W % 16 != 0
    assert all(seen.values()), seen


@needs_ref
@pytest.mark.parametrize("c", S.GRID, ids=[c.id for c in S.GRID])
def test_oracle_equals_reference(oracle, c):
    """Keypoints (all seven cv::KeyPoint fields), descriptors and per-level counts of the oracle equal the reference's own
    ORBextractor::operator() bit for bit; entries outside S.reference_defined run against the oracle only."""
    from oracle import ref as R
    orc, img, k, d, lv, counts = _run(oracle, c)
    if not S.reference_defined(lv):
        pytest.skip("the reference's ORBextractor has no defined result on this frame (see orb_shapes.reference_defined)")
    rk, rd, rc = R.orb_extract(img, c.nf, c.sf, c.nl, c.ini, c.mn)
    assert len(rk) == len(k), (c.id, len(rk), len(k))
    assert rk.tobytes() == k.tobytes(), f"{c.id}: keypoints differ"
    assert np.array_equal(rd, d), f"{c.id}: descriptors differ in {int((rd != d).any(1).sum())} rows"
    assert list(rc) == counts, (c.id, list(rc), counts)
    _assert_within_bound(c, lv, list(rc))
