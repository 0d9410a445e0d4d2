"""k_fast's cell strips (one warp per 30-px cell, four horizontally adjacent cells of one level per CTA, one staged box per strip) and
k_blur's 64x128 tiles, checked through the handle's read-outs: every level's per-cell candidate lists (cell rows, cell columns, raster
order inside a cell) and every blurred plane, bit for bit, against the CPU oracle or against one call per frame.  The shapes put the
end of a cell row inside a strip (cell columns not a multiple of 4), levels of one cell column, cells taller than 32 rows (the strip's
second box), tile rows cut by the level's height, SSLPL_NO_TMA=1 and a device view whose pitch breaks TMA's alignment rules."""
import numpy as np
import pytest

import orb_shapes as S

pytestmark = pytest.mark.gpu

EDGE = 19


def _cells(ext, l):
    """(nCols, nRows, hCell) of level l, as ORBextractor.cc:786-789 computes them."""
    w, h = ext.level_size(l)
    width, height = np.float32(w - 2 * EDGE + 6), np.float32(h - 2 * EDGE + 6)
    nc, nr = int(width / np.float32(30)), int(height / np.float32(30))
    if nc <= 0 or nr <= 0:
        return 0, 0, 0
    return nc, nr, int(np.ceil(height / np.float32(nr)))


def _same_candidates(a, b, tag):
    assert len(a[0]) == len(b[0]), f"{tag}: {len(a[0])} vs {len(b[0])} candidates"
    for u, v in zip(a, b):
        assert np.array_equal(u, v), f"{tag}: candidates differ"


def _against_oracle(ext, orc, img, tag, frame=0):
    """Candidates of every level and the blurred planes of the levels that keep keypoints (the oracle blurs only those)."""
    orc.extract(img)
    for l in range(ext.nlevels):
        _same_candidates(ext.candidates(l, frame), orc.candidates(l)[:3], f"{tag} level {l}")
        if len(orc.level_keypoints(l)[0]):
            assert np.array_equal(ext.blurred(l, frame), orc.blurred(l)), f"{tag}: blurred level {l}"


def _against_single(ext, single, frames, idx, tag):
    """Every level's candidates and blurred plane of the batch's frame f equal a one-frame call on frame f."""
    for f in idx:
        single(frames[f])
        for l in range(ext.nlevels):
            _same_candidates(ext.candidates(l, f), single.candidates(l), f"{tag} frame {f} level {l}")
            assert np.array_equal(ext.blurred(l, f), single.blurred(l)), f"{tag} frame {f}: blurred level {l}"


def test_batch_513_frames_640x480(pkg, oracle, synth):
    """The benchmark's shape: 513 frames of 640x480, 1000 features; every frame equal to a one-frame call, three to the oracle."""
    B = 513
    frames = synth.batch(640, 480, B)
    ext = pkg.ORBextractor(1000, 1.2, 8, 20, 7, max_width=640, max_height=480, max_batch=B)
    ext.extract_batch(frames)
    ext.sync()
    geo = [_cells(ext, l) for l in range(8)]
    assert any(nc % 4 for nc, _, _ in geo) and any(hc > 32 for _, _, hc in geo), geo
    _against_single(ext, pkg.ORBextractor(1000, 1.2, 8, 20, 7, max_width=640, max_height=480), frames, range(B), "batch640")
    orc = oracle.OrbOracle(1000, 1.2, 8, 20, 7)
    for f in (0, 256, B - 1):
        _against_oracle(ext, orc, frames[f], f"batch640 frame {f}", frame=f)


def test_1280x960_4000(pkg, oracle, synth):
    ext = pkg.ORBextractor(4000, 1.2, 8, 20, 7, max_width=1280, max_height=960)
    img = synth.frame(1280, 960, 3)
    ext(img)
    ext.sync()
    _against_oracle(ext, oracle.OrbOracle(4000, 1.2, 8, 20, 7), img, "1280x960")


# (W, H): 4095x120 and 1921x240 have cell rows of every length modulo 4 and cells taller than 32 rows; 517x333 and 613x480 end
# their cell rows inside a strip; 300x700 and 200x4000 shrink to one cell column; 129x63 and 62x62 hold a single cell
SHAPES = [(4095, 120), (1921, 240), (517, 333), (613, 480), (300, 700), (200, 4000), (129, 63), (62, 62), (38, 38)]


@pytest.mark.parametrize("tma", [True, False], ids=["tma", "no-tma"])
@pytest.mark.parametrize("W,H", SHAPES, ids=[f"{w}x{h}" for w, h in SHAPES])
def test_shapes(pkg, oracle, monkeypatch, W, H, tma):
    if not tma:
        monkeypatch.setenv("SSLPL_NO_TMA", "1")
    ext = pkg.ORBextractor(1000, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2)
    monkeypatch.delenv("SSLPL_NO_TMA", raising=False)
    frames = np.stack([S.frame("noise", W, H, 11), S.frame("synth", W, H, 12)])
    ext.extract_batch(frames)
    ext.sync()
    orc = oracle.OrbOracle(1000, 1.2, 8, 20, 7)
    for f in range(2):
        _against_oracle(ext, orc, frames[f], f"{W}x{H} frame {f}", frame=f)
    single = pkg.ORBextractor(1000, 1.2, 8, 20, 7, max_width=W, max_height=H)
    _against_single(ext, single, frames, range(2), f"{W}x{H}")


def test_shapes_cover_the_strip_cases(pkg):
    """SHAPES holds cell rows ending inside a strip, single-column levels and tall cells."""
    seen = set()
    for W, H in SHAPES:
        ext = pkg.ORBextractor(1000, 1.2, 8, 20, 7, max_width=W, max_height=H)
        ext(S.frame("noise", W, H))
        for l in range(8):
            nc, _, hc = _cells(ext, l)
            if nc:
                seen |= {f"cols%4={nc % 4}"} | ({"one column"} if nc == 1 else set()) | ({"tall"} if hc > 32 else set())
    assert seen >= {"cols%4=0", "cols%4=1", "cols%4=2", "cols%4=3", "one column", "tall"}, seen


def test_odd_pitch_device_view(pkg, oracle):
    """Frames in HBM at an odd pitch and an odd offset: level 0 is staged with byte loads, the pyramid levels with TMA."""
    torch = pytest.importorskip("torch")
    W, H, pitch, off = 640, 480, 653, 5
    frames = np.stack([S.frame("noise", W, H, 21), S.frame("synth", W, H, 22)])
    host = np.zeros((2 * H * pitch + off,), np.uint8)
    for f in range(2):
        host[off + f * H * pitch: off + (f + 1) * H * pitch].reshape(H, pitch)[:, :W] = frames[f]
    buf = torch.from_numpy(host).cuda()
    ext = pkg.ORBextractor(1000, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2)
    ext.extract_batch_device(buf.data_ptr() + off, 2, W, H, pitch, H * pitch)
    ext.sync()
    orc = oracle.OrbOracle(1000, 1.2, 8, 20, 7)
    for f in range(2):
        _against_oracle(ext, orc, frames[f], f"odd pitch frame {f}", frame=f)
