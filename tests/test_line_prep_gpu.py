"""The LSD / LBD per-pixel pre-pass (k_lsd_prep, k_lsd_seeds in csrc/line.cu) plane by plane, against a plain reference built from
OpenCV's own calls, numpy and glibc's cos / sin, with no tolerance: Sobel dx / dy, level-line angles, both cos / sin pairs, gradient
norms, the largest norm and the seed order.  Also every way a frame can reach the line path (host frames, host batches, device views
whose base, pitch or frame stride is not word aligned, padding full of junk) and handles that saw a larger frame before.

Reference (lsd.cpp and BinaryDescriptor calls):
  detection image  cv2.resize(cv2.GaussianBlur(img, (7, 7), 0.75), None, fx=0.8, fy=0.8, interpolation=cv2.INTER_LINEAR_EXACT)
  dx, dy           cv2.Sobel(cv2.GaussianBlur(img, (5, 5), 1), cv2.CV_16S, ..., ksize=3)
  ll_angle         2x2 differences in integers; norm = sqrt((gx^2 + gy^2) / 4); defined where norm > rho = 2 / sin(22.5 deg); the last
                   row and column are NOTDEF (-1024) with norm 0; angle = cv2.fastAtan2(gx, -gy) (the oracle's copy, pinned to cv2);
                   ad = angle * pi / 180 in double; cs = float(cos / sin(float(ad))); cs0 = float(cos / sin(ad))
  seeds            defined pixels in raster order, stably sorted by 1023 - int(norm * (1023 / maxgrad))
The CPU test at the end proves the image part of the reference against the oracle before any GPU runs."""
import math
import numpy as np
import cv2
import pytest

torch = pytest.importorskip("torch")
RHO = 2.0 / math.sin(math.pi * 22.5 / 180)
NOTDEF = np.float32(-1024.0)
SPAN = 511                                   # DA, BC in [-255, 255]
IN_TILE, DET_TILE = (160, 40), (128, 32)     # k_lsd_prep's tile at input resolution and at detection scale

# frame sizes: the 16 x 16 minimum (the staged box is larger than the frame), one tile exactly and one pixel over, last tiles 1, 2, 3 and
# 5 pixels wide or high, W % 4 and sw % 4 independent (644 -> 515, 645 -> 516), tall / narrow and short / wide, exact and ragged tilings
SHAPES = [(16, 16), (160, 40), (161, 41), (321, 122), (482, 83), (165, 45), (803, 203), (644, 97), (645, 100), (24, 640), (1000, 18),
          (333, 251), (640, 480), (1280, 960), (1920, 1080), (1918, 1078)]

_TABLE = {}


def ref_table(oracle):
    """ll_angle of every (DA, BC) pair: dict of [511, 511] (angdeg, modgrad) and [511, 511, 2] (cs, cs0) arrays."""
    if not _TABLE:
        da, bc = np.meshgrid(np.arange(-255, 256), np.arange(-255, 256), indexing="ij")
        gx, gy = da + bc, da - bc
        mod = np.sqrt((gx * gx + gy * gy) / 4.0)
        ang = np.full(mod.shape, NOTDEF, np.float32)
        cs = np.zeros(mod.shape + (2,), np.float32); cs0 = np.zeros(mod.shape + (2,), np.float32)
        ii, jj = np.nonzero(mod > RHO)
        deg = np.array([oracle.fast_atan2(float(gx[i, j]), float(-gy[i, j])) for i, j in zip(ii.tolist(), jj.tolist())], np.float32)
        ad = deg.astype(np.float64) * (math.pi / 180)
        a = ad.astype(np.float32).astype(np.float64)
        ang[ii, jj] = deg
        cs[ii, jj, 0] = [math.cos(v) for v in a.tolist()]; cs[ii, jj, 1] = [math.sin(v) for v in a.tolist()]
        cs0[ii, jj, 0] = [math.cos(v) for v in ad.tolist()]; cs0[ii, jj, 1] = [math.sin(v) for v in ad.tolist()]
        _TABLE.update(angdeg=ang, cs=cs, cs0=cs0, modgrad=mod)
    return _TABLE


def ref_small(img):
    return cv2.resize(cv2.GaussianBlur(img, (7, 7), 0.75), None, fx=0.8, fy=0.8, interpolation=cv2.INTER_LINEAR_EXACT)


def ref_sobel(img):
    b5 = cv2.GaussianBlur(img, (5, 5), 1)
    return cv2.Sobel(b5, cv2.CV_16S, 1, 0, ksize=3), cv2.Sobel(b5, cv2.CV_16S, 0, 1, ksize=3)


def ref_planes(oracle, img):
    t = ref_table(oracle)
    dx, dy = ref_sobel(img)
    s = ref_small(img).astype(np.int64)
    SH, SW = s.shape
    idx = (s[1:, 1:] - s[:-1, :-1] + 255) * SPAN + (s[:-1, 1:] - s[1:, :-1] + 255)     # (D - A, B - C) of each 2x2 window
    ang = np.full((SH, SW), NOTDEF, np.float32); mod = np.zeros((SH, SW)); cs = np.zeros((SH, SW, 2), np.float32); cs0 = cs.copy()
    ang[:-1, :-1] = t["angdeg"].reshape(-1)[idx]; mod[:-1, :-1] = t["modgrad"].reshape(-1)[idx]
    cs[:-1, :-1] = t["cs"].reshape(-1, 2)[idx]; cs0[:-1, :-1] = t["cs0"].reshape(-1, 2)[idx]
    defined = np.flatnonzero(mod.reshape(-1) > RHO)
    maxgrad = float(mod.reshape(-1)[defined].max()) if len(defined) else 0.0
    seeds = defined
    if len(defined):
        key = 1023 - (mod.reshape(-1)[defined] * (1023.0 / maxgrad)).astype(np.int64)
        seeds = defined[np.argsort(key, kind="stable")]
    return dict(dx=dx, dy=dy, angdeg=ang, cs=cs, cs0=cs0, modgrad=mod, maxgrad=maxgrad, seeds=seeds.astype(np.uint32))


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({2: np.uint16, 4: np.uint32, 8: np.uint64}[a.itemsize]) if a.dtype.kind == "f" else a


def assert_plane(tag, name, got, want, tile):
    """Bit-exact comparison of one per-pixel plane; the message names the first differing pixel, its tile and both values."""
    assert got.shape == want.shape, f"{tag}: {name} shape {got.shape} != {want.shape}"
    bad = _bits(got) != _bits(want)
    if bad.ndim == 3:
        bad = bad.any(2)
    if bad.any():
        y, x = (int(v) for v in np.argwhere(bad)[0])
        raise AssertionError(f"{tag}: {name} differs at {int(bad.sum())} pixels; first at (x={x}, y={y}), tile ({x // tile[0]}, {y // tile[1]}): "
                             f"got {got[y, x]!r}, want {want[y, x]!r}")


def assert_prep(tag, got, want):
    for name in ("dx", "dy"):
        assert_plane(tag, name, got[name], want[name], IN_TILE)
    for name in ("angdeg", "cs", "cs0", "modgrad"):
        assert_plane(tag, name, got[name], want[name], DET_TILE)
    assert _bits(np.float64(got["maxgrad"])) == _bits(np.float64(want["maxgrad"])), f"{tag}: maxgrad {got['maxgrad']!r} != {want['maxgrad']!r}"
    gs, ws = got["seeds"], want["seeds"]
    if not np.array_equal(gs, ws):
        k = int(np.argmax(gs[:min(len(gs), len(ws))] != ws[:min(len(gs), len(ws))])) if min(len(gs), len(ws)) else 0
        raise AssertionError(f"{tag}: seeds differ ({len(gs)} vs {len(ws)}); first at rank {k}: got {gs[k:k + 3]}, want {ws[k:k + 3]}")


def contents(icl, synth, W, H):
    """The inputs of the shape grid: synthetic scene, ICL frame (tiled / cropped), uniform noise, 0/255 rectangle (edges at 0, 90, 180
    and 270 degrees crossing tile seams), flat, and flat frames whose only gradient is in the last row or the last column."""
    rng = np.random.default_rng(W * 7919 + H)
    yy, xx = np.mgrid[0:H, 0:W]
    x0 = 160 if W > 320 else W // 4
    y0 = 40 if H > 80 else H // 4
    rect = np.where((xx >= x0) & (xx < W - x0 + 1) & (yy >= y0) & (yy < H - y0 + 1), 255, 0).astype(np.uint8)
    last_row = np.full((H, W), 100, np.uint8); last_row[-1, :] = 180
    last_col = np.full((H, W), 100, np.uint8); last_col[:, -1] = 20
    return [("synthetic", synth.frame(W, H, (W + H) % 9)),
            ("icl", np.ascontiguousarray(np.tile(icl, (-(-H // 480), -(-W // 640)))[:H, :W])),
            ("noise", rng.integers(0, 256, (H, W), dtype=np.uint8)),
            ("steps", rect), ("flat", np.full((H, W), 77, np.uint8)), ("last row", last_row), ("last column", last_col)]


def _line_outputs(ls, kl, ld, eq, frame=0):
    return dict(prep=ls.prep_planes(frame), raw=ls.raw_segments(frame), kl=kl.tobytes(), ld=np.asarray(ld).copy(), eq=np.asarray(eq).copy())


def _assert_same_outputs(tag, got, want):
    assert_prep(tag, got["prep"], want["prep"])
    assert np.array_equal(got["raw"], want["raw"]), f"{tag}: raw segments differ ({len(got['raw'])} vs {len(want['raw'])})"
    assert got["kl"] == want["kl"], f"{tag}: KeyLines differ"
    assert np.array_equal(got["ld"], want["ld"]), f"{tag}: LBD descriptors differ"
    assert np.array_equal(got["eq"], want["eq"]), f"{tag}: line equations differ"


def _assert_oracle(tag, oracle, img, out, nfeat=40):
    lo = oracle.LineOracle(nfeat)
    okl, old, oeq = lo.extract(img)
    oraw = lo.raw_segments()
    assert out["raw"].shape == oraw.shape and np.max(np.abs(out["raw"] - oraw), initial=0) <= 1e-4, f"{tag}: raw segments differ from the oracle"
    assert len(out["ld"]) == len(old) and np.array_equal(out["ld"], old), f"{tag}: LBD descriptors differ from the oracle"
    assert np.allclose(out["eq"], oeq, rtol=1e-9, atol=1e-9), f"{tag}: line equations differ from the oracle"


# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_ll_table_covers_the_whole_angle_domain(pkg, oracle):
    """Every 2x2 difference pair through the kernel's own per-pixel function: NOTDEF exactly where norm <= rho, and every angle, norm and
    cos / sin pair bit-equal to the reference (261121 inputs)."""
    got = pkg.LineSegment(40, max_width=64, max_height=64).ll_table()
    want = ref_table(oracle)
    report = []
    for name in ("angdeg", "modgrad", "cs", "cs0"):
        bad = _bits(got[name]) != _bits(want[name])
        if bad.ndim == 3:
            bad = bad.any(2)
        if bad.any():
            ii, jj = np.nonzero(bad)
            first = [(int(i) - 255, int(j) - 255, got[name][i, j].tolist(), want[name][i, j].tolist()) for i, j in zip(ii[:4], jj[:4])]
            report.append(f"{name}: {int(bad.sum())} of {SPAN * SPAN} entries differ, first (DA, BC, got, want): {first}")
    assert not report, "; ".join(report)
    assert np.array_equal(got["angdeg"] == NOTDEF, want["modgrad"] <= RHO)


@pytest.mark.gpu
@pytest.mark.parametrize("W,H", SHAPES, ids=[f"{w}x{h}" for w, h in SHAPES])
def test_prep_planes_and_seeds_equal_the_reference(pkg, oracle, icl_gray, synth, W, H):
    ls = pkg.LineSegment(40, max_width=W, max_height=H)
    for name, img in contents(icl_gray, synth, W, H):
        ls.ExtractLineSegment(img)
        got = ls.prep_planes()
        want = ref_planes(oracle, img)
        assert_prep(f"{W}x{H} {name}", got, want)
        if name == "flat":
            assert got["maxgrad"] == 0.0 and len(got["seeds"]) == 0


class _DevArray:
    """A raw device pointer as a __cuda_array_interface__ object, for torch.as_tensor."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = dict(shape=(nbytes,), typestr="|u1", data=(ptr, False), version=3, strides=None)


def _download(ptr, nbytes, dtype):
    t = torch.as_tensor(_DevArray(ptr, nbytes), device="cuda")
    return t.cpu().numpy().view(dtype)


VIEWS = [  # (name, base offset, pitch(W), frame stride(pitch, H), padding fill)
    ("base +1, odd pitch", 1, lambda w: (w + 2) | 1, lambda p, h: p * h, "random"),
    ("base +2, odd pitch", 2, lambda w: (w + 4) | 1, lambda p, h: p * h, "0xA5"),
    ("base +3, odd pitch", 3, lambda w: (w + 6) | 1, lambda p, h: p * h, "random"),
    ("word pitch, 0xA5 padding", 0, lambda w: (w + 8 + 3) // 4 * 4, lambda p, h: p * h, "0xA5"),
    ("word pitch, random padding", 0, lambda w: (w + 64 + 15) // 16 * 16, lambda p, h: p * h, "random"),
    ("frame stride pitch*H+5", 0, lambda w: (w + 4 + 3) // 4 * 4, lambda p, h: p * h + 5, "random"),
]


def place_frames(frames, offset, pitch, stride, fill, seed=0):
    """Host image of a device buffer: frames at offset + f * stride, rows `pitch` bytes apart, everything else junk."""
    B, H, W = frames.shape
    n = offset + stride * (B - 1) + pitch * (H - 1) + W + 64
    buf = np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8) if fill == "random" else np.full(n, 0xA5, np.uint8)
    for f in range(B):
        view = np.lib.stride_tricks.as_strided(buf[offset + f * stride:], shape=(H, W), strides=(pitch, 1))
        view[...] = frames[f]
    return buf


@pytest.mark.gpu
@pytest.mark.parametrize("W,H", [(640, 480), (333, 251)])
def test_every_entry_path_gives_the_same_planes(pkg, oracle, synth, icl_gray, W, H):
    """Host single frame, host batch, and device views that take the byte-load staging (base or pitch not word aligned), word-aligned
    views with junk padding, and a frame stride that leaves junk between frames: the same planes, seeds, segments, KeyLines, LBD
    bytes and line equations, all equal to the reference and the oracle."""
    B, cap = 5, 40
    frames = np.stack([np.ascontiguousarray(icl_gray[:H, :W])] + [synth.frame(W, H, f) for f in (1, 3, 8, 17)])
    ls = pkg.LineSegment(cap, max_width=W, max_height=H, max_batch=B)
    single = []
    for f in range(B):
        kl, ld, eq = ls.ExtractLineSegment(frames[f])
        out = _line_outputs(ls, kl, ld, eq)
        assert_prep(f"single {f}", out["prep"], ref_planes(oracle, frames[f]))
        _assert_oracle(f"single {f}", oracle, frames[f], out, cap)
        single.append(out)
    kl, ld, eq, n = ls.extract_batch(frames)
    for f in range(B):
        _assert_same_outputs(f"host batch, frame {f}", _line_outputs(ls, kl[f, :n[f]], ld[f, :n[f]], eq[f, :n[f]], f), single[f])
    for name, off, pitch_of, stride_of, fill in VIEWS:
        pitch = pitch_of(W); stride = stride_of(pitch, H)
        buf = torch.from_numpy(place_frames(frames, off, pitch, stride, fill)).cuda()
        ls.extract_batch_device(buf.data_ptr() + off, B, W, H, pitch, stride)
        ls.sync()
        d_kl, d_ld, d_eq, d_n, dcap = ls.device_results()
        n = _download(d_n, 4 * B, np.int32)
        kl = _download(d_kl, B * dcap * pkg.KEYLINE_DTYPE.itemsize, pkg.KEYLINE_DTYPE).reshape(B, dcap)
        ld = _download(d_ld, B * dcap * 32, np.uint8).reshape(B, dcap, 32)
        eq = _download(d_eq, B * dcap * 24, np.float64).reshape(B, dcap, 3)
        for f in range(B):
            _assert_same_outputs(f"{name}, frame {f}", _line_outputs(ls, kl[f, :n[f]], ld[f, :n[f]], eq[f, :n[f]], f), single[f])
        del buf


@pytest.mark.gpu
def test_results_do_not_depend_on_an_earlier_larger_frame(pkg, oracle, synth):
    """A handle that processed a 640x480 frame and then a 613x437 crop gives what a fresh handle gives on the crop.  The line handle's
    staging rows are 624 bytes apart for the crop, the Frame handle's grey plane 640: stale columns of the big frame lie past the crop."""
    big = synth.frame(640, 480, 2)
    crop = np.ascontiguousarray(synth.frame(640, 480, 5)[:437, :613])
    used = pkg.LineSegment(40, max_width=640, max_height=480)
    used.ExtractLineSegment(big)
    got = _line_outputs(used, *used.ExtractLineSegment(crop))
    fresh = pkg.LineSegment(40, max_width=640, max_height=480)
    want = _line_outputs(fresh, *fresh.ExtractLineSegment(crop))
    _assert_same_outputs("line handle after 640x480", got, want)
    assert_prep("crop vs reference", want["prep"], ref_planes(oracle, crop))
    fr = pkg.Frame(1000, 1.2, 8, 20, 7, 40, max_width=640, max_height=480)
    fr.extract(big)
    got = fr.extract(crop); got_prep = fr.line.prep_planes()
    fr2 = pkg.Frame(1000, 1.2, 8, 20, 7, 40, max_width=640, max_height=480)
    want = fr2.extract(crop); want_prep = fr2.line.prep_planes()
    for k in want:
        assert got[k].tobytes() == want[k].tobytes(), f"Frame handle after 640x480: {k} differs"
    assert_prep("Frame handle after 640x480", got_prep, want_prep)


def test_reference_matches_the_oracle_images(oracle, icl_gray, synth):
    """CPU: the reference's detection-scale image and Sobel planes equal the oracle's (the restatement pinned to cv2) over the whole
    shape grid, so a GPU failure of the plane tests points at the kernel, not at the reference."""
    for W, H in SHAPES:
        for name, img in contents(icl_gray, synth, W, H):
            if name not in ("synthetic", "noise", "last row"):
                continue
            lo = oracle.LineOracle(40)
            lo.extract(img)
            small = ref_small(img)
            assert small.shape == (int(round(H * 0.8)), int(round(W * 0.8)))
            assert np.array_equal(small, lo.scaled()), f"{W}x{H} {name}: detection-scale image differs from the oracle"
            dx, dy = ref_sobel(img)
            odx, ody = oracle.lbd_prep(img)
            assert np.array_equal(dx, odx) and np.array_equal(dy, ody), f"{W}x{H} {name}: Sobel planes differ from the oracle"
