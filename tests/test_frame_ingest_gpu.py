"""GPU: frame ingest held to cv2 bit for bit.  The keypoint undistortion (k_undistort: mvKeysUn, Frame.cc:483-513) and the image bounds
(Frame.cc:515-543) against cv2.undistortPoints of OpenCV 4.13 and tests/undistort_model.py for every camera of the model, including
wide-angle ones whose distortion factor turns negative inside the image; the k1 gate and camera changes on a live handle; and the
device grey plane (k_cvt_gray) against cv2.cvtColor for BGR / RGB, 3 and 4 channels, awkward widths, padded rows and batches."""
import ctypes as C

import cv2
import numpy as np
import pytest

import undistort_model as M

pytestmark = pytest.mark.gpu

NAMES = [c[0] for c in M.CAMERAS]
SIZES = [(640, 480), (1280, 960), (752, 480), (320, 240), (1241, 376), (38, 38)]


def _cv2(xy, K, D):
    Km, Dm = M.cv2_args(K, D)
    return cv2.undistortPoints(np.asarray(xy, np.float32).reshape(-1, 1, 2), Km, Dm, None, Km).reshape(-1, 2)


def _mismatch(got, want):
    """Rows whose float32 bits differ.  A NaN (only on the ring where the distortion factor is exactly 1 / 0) only has to meet a NaN:
    x86 and the GPU encode a NaN made from inf * 0 with different sign bits."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    both_nan = np.isnan(got) & np.isnan(want)
    return np.flatnonzero(((got.view(np.uint32) != want.view(np.uint32)) & ~both_nan).any(1))


def _xy(k):
    return np.stack([k["x"], k["y"]], 1)


def _check_keys_un(keys, un, K, D):
    """keysUn x / y equal cv2 on keys (bits); every other field is keys' own."""
    assert len(keys) == len(un) and len(keys) > 100
    want = _cv2(_xy(keys), K, D) if M.distorted(D) else _xy(keys)
    bad = _mismatch(_xy(un), want)
    assert bad.size == 0, (bad.size, len(keys), _xy(keys)[bad[:3]], _xy(un)[bad[:3]], want[bad[:3]])
    rest = un.copy()
    rest["x"], rest["y"] = keys["x"], keys["y"]
    assert rest.tobytes() == keys.tobytes()


@pytest.fixture(scope="module")
def small(pkg):
    fr = pkg.Frame(500, 1.2, 8, 20, 7, 40, max_width=1280, max_height=960, max_batch=4)
    yield fr
    fr.close()


@pytest.mark.parametrize("name", NAMES)
def test_device_undistortion_equals_model_and_cv2(small, name):
    K, D = M.camera(name)
    small.set_camera(*K, D)
    pts = M.test_points(K, D, n_random=1 << 20)
    got = small.debug_undistort(pts)
    model, exits = M.undistort_points(pts, K, D, exits=True)
    for want in (model, _cv2(pts, K, D)):
        bad = _mismatch(got, want)
        assert bad.size == 0, (name, bad.size, exits[bad].mean(), pts[bad[:3]], got[bad[:3]], want[bad[:3]])
    if name in M.NEGATIVE_FACTOR:
        assert exits[:1 << 20].mean() > 0.05


@pytest.mark.parametrize("name", NAMES)
def test_image_bounds_equal_model_and_cv2(small, name):
    K, D = M.camera(name)
    small.set_camera(*K, D)
    for cols, rows in SIZES:
        got = small.image_bounds(cols, rows)
        c = _cv2(np.array([[0, 0], [cols, 0], [0, rows], [cols, rows]], np.float32), K, D)
        via_cv2 = np.array([min(c[0, 0], c[2, 0]), max(c[1, 0], c[3, 0]), min(c[0, 1], c[1, 1]), max(c[2, 1], c[3, 1])], np.float32)
        for want in (M.image_bounds(cols, rows, K, D), via_cv2):
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (name, cols, rows, got, want)


@pytest.mark.parametrize("W, H, nfeatures, B", [(640, 480, 1000, 6), (1280, 960, 4000, 4)])
def test_keypoints_un_equal_cv2_end_to_end(pkg, synth, W, H, nfeatures, B):
    """Frame.extract and extract_batch under every camera, one handle: keysUn is cv2.undistortPoints of keys."""
    frames = synth.batch(W, H, B, start=3)
    fr = pkg.Frame(nfeatures, 1.2, 8, 20, 7, 40, max_width=W, max_height=H, max_batch=B)
    for name, K, D in M.CAMERAS:
        fr.set_camera(*K, D)
        r = fr.extract(frames[0])
        _check_keys_un(r["keys"], r["keysUn"], K, D)
        b = fr.extract_batch(frames)
        for f in range(B):
            n = int(b["n"][f])
            _check_keys_un(b["keys"][f, :n], b["keysUn"][f, :n], K, D)
        assert b["keys"][0, :int(b["n"][0])].tobytes() == r["keys"].tobytes()
    fr.close()


@pytest.mark.parametrize("k1", [0.0, -0.0])
def test_k1_gate(pkg, synth, k1):
    """k1 == 0 (either sign) with every other coefficient nonzero: mvKeysUn is mvKeys and the bounds are the image (Frame.cc:485, :517)."""
    fr = pkg.Frame(1000, 1.2, 8, 20, 7, 40, max_width=640, max_height=480, max_batch=2)
    fr.set_camera(500.0, 500.0, 320.0, 240.0, [k1, -0.3, 0.01, -0.02, 0.5])
    r = fr.extract(synth.frame(640, 480, 1))
    assert len(r["keys"]) > 100 and r["keysUn"].tobytes() == r["keys"].tobytes()
    b = fr.extract_batch(synth.batch(640, 480, 2))
    for f in range(2):                                     # entries past a frame's count are unspecified
        n = int(b["n"][f])
        assert n > 100 and b["keysUn"][f, :n].tobytes() == b["keys"][f, :n].tobytes()
    assert fr.device_keypoints_un()[0] == fr.orb.device_results()[0]
    for cols, rows in SIZES:
        assert list(fr.image_bounds(cols, rows)) == [0, cols, 0, rows]
    fr.close()


def test_camera_changes_on_one_handle(pkg, synth):
    """distorted -> k1 = 0 -> distorted: keysUn and what device_keypoints_un() points at follow the camera of each call."""
    fr = pkg.Frame(1000, 1.2, 8, 20, 7, 40, max_width=640, max_height=480, max_batch=1)
    img = synth.frame(640, 480, 2)
    for name in ("wide_k1", "zero", "tum1", "zero", "wide_k3"):
        K, D = M.camera(name) if name != "zero" else ((500.0, 500.0, 320.0, 240.0), (0.0, 0.1, 0.001, 0.001))
        fr.set_camera(*K, D)
        r = fr.extract(img)
        _check_keys_un(r["keys"], r["keysUn"], K, D)
        d_un, cap = fr.device_keypoints_un()
        orb_kps, _, _, orb_cap = fr.orb.device_results()
        assert cap == orb_cap and (d_un == orb_kps) == (not M.distorted(D)), name
        assert np.array_equal(fr.image_bounds(640, 480).view(np.uint32), M.image_bounds(640, 480, K, D).view(np.uint32)), name
    fr.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# the grey plane: k_cvt_gray against cv2.cvtColor, read back through the ORB handle's level 0 (which is the frame's own grey buffer)
# ---------------------------------------------------------------------------------------------------------------------------------
CODES = {(3, False): cv2.COLOR_BGR2GRAY, (3, True): cv2.COLOR_RGB2GRAY, (4, False): cv2.COLOR_BGRA2GRAY, (4, True): cv2.COLOR_RGBA2GRAY}
# k_cvt_gray runs 256-thread rows; 38 x 38 is the smallest frame the ORB pyramid accepts (2 x its 19-pixel border)
WIDTHS = [38, 39, 255, 256, 257, 333, 1280]
HEIGHTS = [38, 41]


def _colour(rng, h, w, cn):
    """Independent full-range channels, with rows of every 0 / 255 combination of the channels."""
    img = rng.integers(0, 256, (h, w, cn), dtype=np.uint8)
    combos = np.array([[(m >> c) & 1 for c in range(cn)] for m in range(1 << cn)], np.uint8) * 255
    img[:2] = np.resize(combos, (2 * w, cn)).reshape(2, w, cn)
    img[-1] = 255
    return img


@pytest.fixture(scope="module")
def grey_handle(pkg):
    fr = pkg.Frame(200, 1.2, 8, 20, 7, 40, max_width=1280, max_height=960, max_batch=3)
    yield fr
    fr.close()


def _extract_raw(pkg, fr, buf, B, w, h, pitch, stride, cn, rgb):
    """sslpl_frame_extract_batch on a raw host buffer (any pitch and frame stride); counts only."""
    n = np.zeros(B, np.int32); nl = np.zeros(B, np.int32)
    rc = pkg.lib().sslpl_frame_extract_batch(fr._h, buf.ctypes.data_as(C.c_void_p), B, w, h, pitch, stride, cn, int(rgb),
                                             None, None, None, fr.cap, n.ctypes.data_as(C.c_void_p),
                                             None, None, None, fr.lcap, nl.ctypes.data_as(C.c_void_p))
    assert rc == 0, pkg.lib().sslpl_last_error()


@pytest.mark.parametrize("cn, rgb", [(3, False), (3, True), (4, False), (4, True)])
def test_grey_plane_equals_cvtcolor(grey_handle, cn, rgb):
    fr = grey_handle
    rng = np.random.default_rng(cn * 2 + rgb)
    for w in WIDTHS:
        for h in HEIGHTS + ([480] if w == 1280 else []):
            img = _colour(rng, h, w, cn)
            fr.extract(img, rgb_order=rgb)
            got = fr.orb.level(0)
            assert got.shape == (h, w) and np.array_equal(got, cv2.cvtColor(img, CODES[cn, rgb])), (w, h)


@pytest.mark.parametrize("cn, rgb", [(1, False), (3, False), (3, True), (4, False), (4, True)])
def test_grey_plane_of_padded_batches(pkg, grey_handle, cn, rgb):
    """Rows with padding (pitch > width * channels) and frames apart by more than height * pitch, the padding filled with bytes a
    misplaced read would pick up."""
    fr = grey_handle
    rng = np.random.default_rng(10 + cn * 2 + rgb)
    for w, h, B in [(257, 41, 3), (333, 64, 2), (1280, 38, 3), (38, 38, 1)]:
        pitch = w * cn + 13
        stride = h * pitch + 77
        buf = np.full(B * stride, 0xA5, np.uint8)
        imgs = [_colour(rng, h, w, cn) if cn > 1 else rng.integers(0, 256, (h, w), dtype=np.uint8) for _ in range(B)]
        for f, img in enumerate(imgs):
            rows = buf[f * stride:f * stride + h * pitch].reshape(h, pitch)
            rows[:, :w * cn] = img.reshape(h, w * cn)
        _extract_raw(pkg, fr, buf, B, w, h, pitch, stride, cn, rgb)
        for f, img in enumerate(imgs):
            want = img if cn == 1 else cv2.cvtColor(img, CODES[cn, rgb])
            assert np.array_equal(fr.orb.level(0, frame=f), want), (w, h, f)


@pytest.mark.parametrize("cn, rgb", [(3, True), (4, False)])
def test_grey_plane_of_contiguous_colour_batches(grey_handle, cn, rgb):
    fr = grey_handle
    rng = np.random.default_rng(20 + cn)
    frames = np.stack([_colour(rng, 96, 257, cn) for _ in range(3)])
    fr.extract_batch(frames, rgb_order=rgb)
    for f in range(3):
        assert np.array_equal(fr.orb.level(0, frame=f), cv2.cvtColor(frames[f], CODES[cn, rgb])), f
