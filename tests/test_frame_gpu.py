"""GPU: the frame-level entry point (sslpl_frame_*): one upload feeding ORB and LSD+LBD on two streams (Frame.cc:69-131), colour
conversion on the device (Tracking.cc:148-161, bit-exact cv2.cvtColor) and keypoint undistortion (Frame.cc:483-543, vs cv2.undistortPoints)."""
import numpy as np
import cv2
import pytest

pytestmark = pytest.mark.gpu


def test_frame_equals_the_two_extractors_and_the_reference_fixtures(pkg, oracle, icl_gray, synth):
    from test_ref_golden_cpu import load
    fr = pkg.Frame(1000, 1.2, 8, 20, 7, 40, max_width=640, max_height=480)
    for img in (icl_gray, synth.frame(640, 480, 3)):
        r = fr.extract(img)
        k, d = pkg.ORBextractor(1000, 1.2, 8, 20, 7, max_width=640, max_height=480)(img)
        kl, ld, eq = pkg.LineSegment(40, max_width=640, max_height=480).ExtractLineSegment(img)
        assert r["keys"].tobytes() == k.tobytes() and np.array_equal(r["desc"], d) and r["keysUn"].tobytes() == k.tobytes()
        assert r["keylines"].tobytes() == kl.tobytes() and np.array_equal(r["ldesc"], ld) and np.array_equal(r["lineeq"], eq)
    g = load("ref_orb.npz")                                # the reference's own Frame constructor output (tools/make_ref_golden.py)
    r = fr.extract(icl_gray)
    assert r["keys"].tobytes() == g["orb_icl1000_kps"].tobytes() and np.array_equal(r["desc"], g["orb_icl1000_desc"])
    assert np.array_equal(r["ldesc"], load("ref_frame.npz")["ldesc"])


def test_colour_input_equals_cvtcolor(pkg, synth):
    rng = np.random.default_rng(3)
    base = synth.frame(640, 480, 5)
    bgr = np.stack([np.clip(base.astype(int) + rng.integers(-40, 40, base.shape), 0, 255).astype(np.uint8) for _ in range(3)], 2)
    fr = pkg.Frame(1000, 1.2, 8, 20, 7, 40, max_width=640, max_height=480)
    for cn, code_bgr, code_rgb in [(3, cv2.COLOR_BGR2GRAY, cv2.COLOR_RGB2GRAY), (4, cv2.COLOR_BGRA2GRAY, cv2.COLOR_RGBA2GRAY)]:
        img = bgr if cn == 3 else np.concatenate([bgr, np.full(base.shape + (1,), 255, np.uint8)], 2)
        for rgb in (False, True):
            gray = cv2.cvtColor(img, code_rgb if rgb else code_bgr)
            a = fr.extract(img, rgb_order=rgb); b = fr.extract(gray)
            assert a["keys"].tobytes() == b["keys"].tobytes() and np.array_equal(a["desc"], b["desc"]) and np.array_equal(a["ldesc"], b["ldesc"]), (cn, rgb)


def test_undistort_keypoints_and_bounds_equal_cv2(pkg, icl_gray):
    fr = pkg.Frame(1000, 1.2, 8, 20, 7, 40, max_width=640, max_height=480)
    K = np.array([[517.3, 0, 318.6], [0, 516.5, 255.3], [0, 0, 1]], np.float32)       # TUM1.yaml-like
    D = np.array([0.2624, -0.9531, -0.0054, 0.0026, 1.1633], np.float32)
    fr.set_camera(K[0, 0], K[1, 1], K[0, 2], K[1, 2], D)
    r = fr.extract(icl_gray)
    pts = np.stack([r["keys"]["x"], r["keys"]["y"]], 1).reshape(-1, 1, 2)
    ref = cv2.undistortPoints(pts, K, D, None, K).reshape(-1, 2)
    got = np.stack([r["keysUn"]["x"], r["keysUn"]["y"]], 1)
    assert len(got) > 500 and np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    for f in ("size", "angle", "response", "octave", "class_id"):
        assert np.array_equal(r["keysUn"][f], r["keys"][f])
    corners = np.array([[0, 0], [640, 0], [0, 480], [640, 480]], np.float32).reshape(-1, 1, 2)
    c = cv2.undistortPoints(corners, K, D, None, K).reshape(-1, 2)
    exp = [min(c[0, 0], c[2, 0]), max(c[1, 0], c[3, 0]), min(c[0, 1], c[1, 1]), max(c[2, 1], c[3, 1])]
    assert np.array_equal(fr.image_bounds(640, 480).view(np.uint32), np.array(exp, np.float32).view(np.uint32))
    fr.set_camera(500, 500, 320, 240, [0, 0, 0, 0])                                    # k1 == 0: mvKeysUn = mvKeys (Frame.cc:485)
    r = fr.extract(icl_gray)
    assert r["keysUn"].tobytes() == r["keys"].tobytes() and list(fr.image_bounds(640, 480)) == [0, 640, 0, 480]


def test_frame_batch(pkg, synth):
    frames = synth.batch(640, 480, 5)
    fr = pkg.Frame(1000, 1.2, 8, 20, 7, 40, max_width=640, max_height=480, max_batch=5)
    b = fr.extract_batch(frames)
    one = pkg.Frame(1000, 1.2, 8, 20, 7, 40, max_width=640, max_height=480)
    for f in range(5):
        r = one.extract(frames[f])
        n, nl = int(b["n"][f]), int(b["nl"][f])
        assert n == len(r["keys"]) and b["keys"][f, :n].tobytes() == r["keys"].tobytes() and np.array_equal(b["desc"][f, :n], r["desc"])
        assert nl == len(r["keylines"]) and np.array_equal(b["ldesc"][f, :nl], r["ldesc"])
