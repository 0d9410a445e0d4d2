"""The CUDA ORB path against the CPU oracle over frame shapes and extractor parameters (tests/orb_shapes.py), stage by stage with
test_orb_gpu._compare_all: pyramid levels and the bordered level, FAST candidates, octree selection, blurred planes, keypoints with
exact angles and coordinates, and descriptors.  Every case also checks that the handle reports no device-side error and that no
frame keeps more keypoints than sslpl_orb_max_keypoints() (the per-level capacities cover the octree's first split, up to 4 nIni
keypoints on a level of a wide frame)."""
import numpy as np
import pytest

import orb_shapes as S
from test_orb_gpu import _compare_all

pytestmark = pytest.mark.gpu

BY_ID = {c.id: c for c in S.GRID}
FORM_STRIPS = ["4095x120-noise", "1920x240-noise-300", "4000x300-noise-500", "1280x62-noise-8x8"]


def _extractor(pkg, c, max_batch=1):
    return pkg.ORBextractor(c.nf, c.sf, c.nl, c.ini, c.mn, max_width=c.W, max_height=c.H, max_batch=max_batch)


def _check_caps(ext, orc, c, counts_by_frame):
    """Every frame within ext.cap, and ext.cap covering the bound of the largest frame the handle accepts (c.W x c.H)."""
    lv_max = S.levels(orc.tables(), c.W, c.H)
    assert ext.cap >= sum(max(v["N"] + 2, 4 * v["nIni"]) for v in lv_max), (c.id, ext.cap)
    for counts in counts_by_frame:
        assert sum(counts) <= ext.cap, (c.id, sum(counts), ext.cap)


def _level_counts(ext, nl, frame=0):
    return [len(ext.level_keypoints(l, frame)[0]) for l in range(nl)]


@pytest.mark.parametrize("c", S.GRID, ids=[c.id for c in S.GRID])
def test_shape_sweep(pkg, oracle, c):
    ext = _extractor(pkg, c)
    orc = oracle.OrbOracle(c.nf, c.sf, c.nl, c.ini, c.mn)
    img = S.frame(c.kind, c.W, c.H)
    _compare_all(ext, orc, img, c.id)
    ext.sync()                                             # raises on any device-side flag (pool, keys, sort, keypoints)
    counts = _level_counts(ext, c.nl)
    for v, n in zip(S.levels(orc.tables(), c.W, c.H), counts):
        assert n <= v["bound"], (c.id, v, n)
    _check_caps(ext, orc, c, [counts])


def test_max_keypoints_of_the_benchmark_configurations(pkg):
    """640x480 / 1000 features and 1280x960 / 4000 features keep their capacity: 4 nIni stays below N + 16 on every level."""
    assert pkg.ORBextractor(1000, 1.2, 8, 20, 7, max_width=640, max_height=480).cap == 1128
    assert pkg.ORBextractor(4000, 1.2, 8, 20, 7, max_width=1280, max_height=960).cap == 4128
    # a wide handle is sized for its widest frame: 4095 px at 1000 features, 8 levels
    assert pkg.ORBextractor(1000, 1.2, 8, 20, 7, max_width=4095, max_height=480).cap == 2484


@pytest.mark.parametrize("cid", FORM_STRIPS)
def test_batch_equals_single(pkg, oracle, cid):
    """extract_batch over 3 different frames equals one call per frame and the oracle."""
    c = BY_ID[cid]
    frames = np.stack([S.frame(kind, c.W, c.H, seed) for seed, kind in enumerate(["noise", "synth", "pairs"])])
    ext = _extractor(pkg, c, max_batch=3)
    kps, desc, n = ext.extract_batch(frames)
    ext.sync()
    single = _extractor(pkg, c)
    orc = oracle.OrbOracle(c.nf, c.sf, c.nl, c.ini, c.mn)
    for f in range(3):
        k1, d1 = single(frames[f])
        ok, od = orc.extract(frames[f])
        assert n[f] == len(k1) == len(ok), (cid, f, n[f], len(k1), len(ok))
        assert kps[f, :n[f]].tobytes() == k1.tobytes() == ok.tobytes(), (cid, f)
        assert np.array_equal(desc[f, :n[f]], d1) and np.array_equal(d1, od), (cid, f)
    _check_caps(ext, orc, c, [_level_counts(ext, c.nl, f) for f in range(3)])


@pytest.mark.parametrize("cid", FORM_STRIPS)
def test_async_begin_with_cap_equal_to_max_keypoints(pkg, oracle, cid):
    """extract_batch_begin into pinned buffers of exactly ext.cap keypoints per frame, then sync()."""
    c = BY_ID[cid]
    frames = np.stack([S.frame(kind, c.W, c.H, seed + 5) for seed, kind in enumerate(["noise", "pairs", "noise"])])
    ext = _extractor(pkg, c, max_batch=3)
    hp = pkg.host_alloc(frames.shape, np.uint8); hp[...] = frames
    out = (pkg.host_alloc((3, ext.cap), pkg.KEYPOINT_DTYPE), pkg.host_alloc((3, ext.cap, 32), np.uint8), pkg.host_alloc((3,), np.int32))
    ext.extract_batch_begin(hp, out)
    ext.sync()
    orc = oracle.OrbOracle(c.nf, c.sf, c.nl, c.ini, c.mn)
    for f in range(3):
        ok, od = orc.extract(frames[f])
        n = int(out[2][f])
        assert n == len(ok) <= ext.cap, (cid, f, n, len(ok), ext.cap)
        assert out[0][f, :n].tobytes() == ok.tobytes() and np.array_equal(out[1][f, :n], od), (cid, f)


def test_reconfigure_narrow_wide_narrow(pkg, oracle):
    """One handle sized for 4095 px goes 640x480 -> 4095x120 -> 640x480: capacities set at create time hold for every size."""
    ext = pkg.ORBextractor(1000, 1.2, 8, 20, 7, max_width=4095, max_height=480)
    orc = oracle.OrbOracle(1000, 1.2, 8, 20, 7)
    narrow = S.frame("noise", 640, 480, 1)
    for tag, img in [("640x480", narrow), ("4095x120", S.frame("noise", 4095, 120)), ("640x480-again", narrow)]:
        n = _compare_all(ext, orc, img, tag)
        ext.sync()
        assert n <= ext.cap, (tag, n, ext.cap)
    ext2 = pkg.ORBextractor(1000, 1.2, 8, 20, 7, max_width=640, max_height=480)
    assert _compare_all(ext2, orc, narrow, "640x480-own-handle") == n


@pytest.mark.parametrize("cid", FORM_STRIPS + ["4095x240-pairs-1000", "1921x240-noise-300"])
def test_strips_without_tma(pkg, oracle, monkeypatch, cid):
    """SSLPL_NO_TMA=1: the stencil kernels stage their boxes with ordinary loads."""
    c = BY_ID[cid]
    monkeypatch.setenv("SSLPL_NO_TMA", "1")
    ext = _extractor(pkg, c)
    monkeypatch.delenv("SSLPL_NO_TMA")
    orc = oracle.OrbOracle(c.nf, c.sf, c.nl, c.ini, c.mn)
    _compare_all(ext, orc, S.frame(c.kind, c.W, c.H), f"{cid}-no-tma")
    ext.sync()
    _check_caps(ext, orc, c, [_level_counts(ext, c.nl)])


def test_frame_handle_on_a_wide_strip(pkg, oracle):
    """The Frame handle takes its keypoint capacity from sslpl_orb_max_keypoints(): a wide strip must extract, equal to the oracle."""
    c = BY_ID["4095x120-noise"]
    fr = pkg.Frame(c.nf, c.sf, c.nl, c.ini, c.mn, 40, max_width=c.W, max_height=c.H, max_batch=1)
    img = S.frame("noise", c.W, c.H, 2)
    g = fr.extract(img)
    ok, od = oracle.OrbOracle(c.nf, c.sf, c.nl, c.ini, c.mn).extract(img)
    assert len(g["keys"]) == len(ok) > 0
    for fld in ("x", "y", "size", "angle", "response", "octave", "class_id"):
        assert np.array_equal(g["keys"][fld], ok[fld]), fld
    assert np.array_equal(g["desc"], od)
    assert fr.cap == pkg.ORBextractor(c.nf, c.sf, c.nl, c.ini, c.mn, max_width=c.W, max_height=c.H).cap
