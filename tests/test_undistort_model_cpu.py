"""CPU tests (no GPU): tests/undistort_model.py, the restatement the device's mvKeysUn and image bounds are held to, equals
cv2.undistortPoints(pts, K, D, None, K) of OpenCV 4.13 bit for bit (float32 bits, so NaN and -0 count) for every camera of the
ingest tests, at random points, on a dense grid with the principal point and the corners, and on rings around the radius where the
distortion factor changes sign; and Frame::ComputeImageBounds' corner min / max at several image sizes."""
import cv2
import numpy as np
import pytest

import undistort_model as M

SIZES = [(640, 480), (1280, 960), (752, 480), (320, 240), (1241, 376), (16, 16)]


def _cv2(xy, K, D):
    Km, Dm = M.cv2_args(K, D)
    return cv2.undistortPoints(np.asarray(xy, np.float32).reshape(-1, 1, 2), Km, Dm, None, Km).reshape(-1, 2)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("name", [c[0] for c in M.CAMERAS])
def test_model_equals_cv2_undistort_points(name):
    K, D = M.camera(name)
    pts = M.test_points(K, D)
    assert len(pts) >= 1 << 18
    got, exits = M.undistort_points(pts, K, D, exits=True)
    want = _cv2(pts, K, D)
    bad = np.flatnonzero((_bits(got) != _bits(want)).any(1))
    assert bad.size == 0, (name, bad.size, pts[bad[:4]], got[bad[:4]], want[bad[:4]])
    if name in M.NEGATIVE_FACTOR:                # the exit is exercised, and inside the image
        assert exits[:1 << 18].mean() > 0.05, exits.mean()
    elif M.zero_factor_r2(D) is None:
        assert not exits.any()


@pytest.mark.parametrize("name", [c[0] for c in M.CAMERAS])
def test_model_image_bounds_equal_cv2(name):
    K, D = M.camera(name)
    for cols, rows in SIZES:
        c = _cv2(np.array([[0, 0], [cols, 0], [0, rows], [cols, rows]], np.float32), K, D)
        want = np.array([min(c[0, 0], c[2, 0]), max(c[1, 0], c[3, 0]), min(c[0, 1], c[1, 1]), max(c[2, 1], c[3, 1])], np.float32)
        got = M.image_bounds(cols, rows, K, D)
        assert np.array_equal(_bits(got), _bits(want)), (name, cols, rows, got, want)


def test_negative_factor_corners_stay_where_they_are():
    """Every corner of a 640x480 image under the first wide-angle camera takes the exit, so the bounds are the image itself."""
    K, D = M.camera("wide_k1")
    corners = np.array([[0, 0], [640, 0], [0, 480], [640, 480]], np.float32)
    out, exits = M.undistort_points(corners, K, D, exits=True)
    assert exits.all() and np.array_equal(out, corners)
    assert list(M.image_bounds(640, 480, K, D)) == [0, 640, 0, 480]


@pytest.mark.parametrize("k1", [0.0, -0.0])
def test_k1_gate(k1):
    """Frame.cc:485 / :517: k1 == 0 (either sign) skips undistortion whatever the other coefficients are."""
    K = (500.0, 500.0, 320.0, 240.0)
    D = (k1, -0.3, 0.01, -0.02, 0.5)
    assert not M.distorted(D) and M.distorted((1e-30, 0, 0, 0))
    pts = M.test_points(K, D, n_random=1 << 10)
    assert np.array_equal(_bits(M.undistort_keypoints(pts, K, D)), _bits(pts))
    for cols, rows in SIZES:
        assert np.array_equal(_bits(M.image_bounds(cols, rows, K, D)), _bits(np.array([0, cols, 0, rows], np.float32)))
