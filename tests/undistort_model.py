"""Plain float64 NumPy restatement of Frame::UndistortKeyPoints and Frame::ComputeImageBounds (reference src/Frame.cc:483-543) as
cv2.undistortPoints(pts, K, D, None, K) of OpenCV 4.13 computes them, in the operation order of csrc/frame.cu's undistort_pt.

Every step is one IEEE-rounded float64 add or multiply (no libm, no fused multiply-add), so its results are bit-equal to cv2 and to the
device.  The camera is what sslpl_frame_set_camera receives: float32 intrinsics and coefficients, widened to double.  The fixed-point
loop runs five iterations; on the first iteration whose distortion factor icdist = 1 / (1 + ((k3 r2 + k2) r2 + k1) r2) is negative it
puts the point back at its normalised start (x0, y0) and stops, as cv2 4.x does (its regression test undistortPoints.regression_14583).
"""
import numpy as np

# (name, (fx, fy, cx, cy), (k1, k2, p1, p2[, k3])): the cameras the ingest tests run under.  The first two are real calibrations, the
# wide-angle ones have a radius where the distortion factor changes sign inside or near a 640x480 image.
CAMERAS = [
    ("tum1", (517.3, 516.5, 318.6, 255.3), (0.2624, -0.9531, -0.0054, 0.0026, 1.1633)),
    ("euroc", (458.654, 457.296, 367.215, 248.375), (-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05)),
    ("wide_k1", (250.0, 250.0, 320.0, 240.0), (-0.5, 0.0, 0.0, 0.0)),
    ("wide_k1k2k3", (200.0, 200.0, 320.0, 240.0), (-0.35, 0.1, 0.0, 0.0, -0.01)),
    ("wide_k3", (400.0, 400.0, 320.0, 240.0), (-0.2, 0.0, 0.0, 0.0, -0.3)),
    ("wide_tangential", (260.0, 260.0, 320.0, 240.0), (-0.45, 0.05, 0.001, 0.002, 0.0)),
    ("tum2", (520.908620, 521.007327, 325.141442, 249.701764), (0.231222, -0.784899, -0.003257, -0.000105, 0.917205)),
    ("tum3_like", (535.4, 539.2, 320.1, 247.6), (0.0412, -0.1036, 0.0007, -0.0011)),
    ("tangential_only", (500.0, 500.0, 320.0, 240.0), (1e-7, 0.0, 0.01, -0.008)),
    ("k3_dominant", (450.0, 450.0, 320.0, 240.0), (0.02, 0.0, 0.0, 0.0, -0.8)),
    ("fx_ne_fy", (610.0, 480.0, 330.0, 250.0), (-0.3, 0.09, 0.0005, -0.0007)),
    ("off_centre", (500.0, 500.0, 120.0, 400.0), (-0.25, 0.05, 0.0, 0.0, 0.0)),
]
NEGATIVE_FACTOR = ("wide_k1", "wide_k1k2k3", "wide_k3", "wide_tangential")   # take the exit inside a 640x480 image


def camera(name):
    for n, K, D in CAMERAS:
        if n == name:
            return K, D
    raise KeyError(name)


def cv2_args(K, D):
    """(K, D) as the float32 matrices the reference passes to cv::undistortPoints (Tracking.cc:58-72)."""
    fx, fy, cx, cy = K
    return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32), np.array(D, np.float32)


def distorted(D):
    """Frame.cc:485 and :517: only k1 decides, compared as a float (so -0.0 counts as zero)."""
    return len(D) > 0 and np.float32(D[0]) != 0


def undistort_points(xy, K, D, exits=False):
    """cv2.undistortPoints(xy, K, D, None, K) for float32 points [N, 2] -> float32 [N, 2] (no k1 gate: see undistort_keypoints);
    with exits=True also a bool [N], True where the loop took the exit."""
    xy = np.asarray(xy, np.float32).reshape(-1, 2)
    fx, fy, cx, cy = (np.float64(np.float32(v)) for v in K)
    k = np.zeros(5)
    k[:len(D)] = np.asarray(D, np.float32)
    with np.errstate(all="ignore"):
        x0 = (xy[:, 0].astype(np.float64) - cx) * (1.0 / fx)
        y0 = (xy[:, 1].astype(np.float64) - cy) * (1.0 / fy)
        x, y = x0.copy(), y0.copy()
        live = np.ones(len(xy), bool)
        for _ in range(5):
            r2 = x * x + y * y
            icdist = 1.0 / (1.0 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2)
            stop = live & (icdist < 0)
            x[stop], y[stop] = x0[stop], y0[stop]
            live &= ~stop
            dx = 2.0 * k[2] * x * y + k[3] * (r2 + 2.0 * x * x)
            dy = k[2] * (r2 + 2.0 * y * y) + 2.0 * k[3] * x * y
            x = np.where(live, (x0 - dx) * icdist, x)
            y = np.where(live, (y0 - dy) * icdist, y)
        out = np.stack([(fx * x + cx).astype(np.float32), (fy * y + cy).astype(np.float32)], 1)
    return (out, ~live) if exits else out


def undistort_keypoints(xy, K, D):
    """Frame::UndistortKeyPoints on keypoint coordinates: unchanged when k1 == 0."""
    xy = np.asarray(xy, np.float32).reshape(-1, 2)
    return undistort_points(xy, K, D) if distorted(D) else xy.copy()


def _min(a, b):                     # std::min / std::max on floats
    return b if b < a else a


def _max(a, b):
    return b if a < b else a


def image_bounds(cols, rows, K, D):
    """Frame::ComputeImageBounds: float32 [mnMinX, mnMaxX, mnMinY, mnMaxY]."""
    if not distorted(D):
        return np.array([0, cols, 0, rows], np.float32)
    c = undistort_points(np.array([[0, 0], [cols, 0], [0, rows], [cols, rows]], np.float32), K, D)
    return np.array([_min(c[0, 0], c[2, 0]), _max(c[1, 0], c[3, 0]), _min(c[0, 1], c[1, 1]), _max(c[2, 1], c[3, 1])], np.float32)


def zero_factor_r2(D):
    """Smallest positive r2 (normalised) at which 1 + k1 r2 + k2 r2^2 + k3 r2^3 vanishes, or None."""
    k = np.zeros(5)
    k[:len(D)] = np.asarray(D, np.float32)
    roots = np.roots([k[4], k[1], k[0], 1.0][next(i for i, c in enumerate([k[4], k[1], k[0], 1.0]) if c != 0):])
    pos = [r.real for r in roots if abs(r.imag) < 1e-12 and r.real > 0]
    return min(pos) if pos else None


def test_points(K, D, n_random=1 << 18, cols=640, rows=480, seed=0):
    """float32 points [N, 2]: uniform random over the image, a dense grid with the principal point, the corners and the image
    edges in it, and rings just inside and just outside the radius where the distortion factor vanishes."""
    rng = np.random.default_rng(seed)
    fx, fy, cx, cy = (np.float32(v) for v in K)
    rnd = np.stack([rng.uniform(0, cols, n_random), rng.uniform(0, rows, n_random)], 1).astype(np.float32)
    gx, gy = np.meshgrid(np.linspace(0, cols, 513, dtype=np.float32), np.linspace(0, rows, 385, dtype=np.float32))
    grid = np.stack([gx.ravel(), gy.ravel()], 1)
    special = np.array([[cx, cy], [0, 0], [cols, 0], [0, rows], [cols, rows], [cols / 2, rows / 2], [cx, 0], [0, cy]], np.float32)
    parts = [rnd, grid, special]
    s = zero_factor_r2(D)
    if s is not None:
        r = np.sqrt(s)
        th = rng.uniform(0, 2 * np.pi, 1 << 14)
        for f in (1 - 1e-3, 1 - 1e-6, 1 - 1e-9, 1.0, 1 + 1e-9, 1 + 1e-6, 1 + 1e-3):
            parts.append(np.stack([cx + np.float64(fx) * r * f * np.cos(th), cy + np.float64(fy) * r * f * np.sin(th)], 1).astype(np.float32))
    return np.concatenate(parts)
