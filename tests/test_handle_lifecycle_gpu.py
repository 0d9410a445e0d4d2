"""The lifecycle the ORB, line, matcher and frame handles share (StreamHandle in csrc/common.cuh): sync on a handle that has not run,
the stream round trip, the kernels each call counts and the stage names of a profiled call."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

W, H, NLEVELS = 320, 240, 8


def _handle(pkg, kind):
    if kind == "orb":
        return pkg.ORBextractor(500, 1.2, NLEVELS, 20, 7, max_width=W, max_height=H)
    if kind == "line":
        return pkg.LineSegment(40, max_width=W, max_height=H)
    if kind == "matcher":
        return pkg.Matcher(max_features=256, max_lines=64, max_nodes=64)
    return pkg.Frame(500, 1.2, NLEVELS, 20, 7, 40, max_width=W, max_height=H)


def _run(h, kind, img):
    """One call of the handle's work, its results as a list of arrays."""
    if kind == "orb":
        return list(h(img))
    if kind == "line":
        return list(h.ExtractLineSegment(img))
    rows = img[:64, :256].reshape(-1, 32)
    return [h.knn2(rows[:200], rows[200:])]


@pytest.mark.parametrize("kind", ["orb", "line", "matcher", "frame"])
def test_sync_before_the_first_call(pkg, kind):
    h = _handle(pkg, kind)
    h.sync()
    h.close()


@pytest.mark.parametrize("kind", ["orb", "line", "matcher"])
def test_stream_round_trip(pkg, synth, kind):
    h = _handle(pkg, kind)
    img = synth.frame(W, H, 1)
    own = h.stream
    assert own
    want = _run(h, kind, img)
    s = torch.cuda.Stream()
    h.set_stream(s.cuda_stream)
    assert h.stream == s.cuda_stream
    got = _run(h, kind, img)
    h.set_stream(0)
    assert h.stream == own
    again = _run(h, kind, img)
    assert len(want) == len(got) == len(again) and len(want[0]) > 0
    for a, b, c in zip(want, got, again):
        assert np.array_equal(a, b) and np.array_equal(a, c)
    h.close()


def _delta(h, fn):
    before = h.launch_count
    fn()
    return h.launch_count - before


def test_extractor_launch_counts(pkg, synth):
    img = synth.frame(W, H, 0)
    orb, line = _handle(pkg, "orb"), _handle(pkg, "line")
    assert _delta(orb, lambda: orb(img)) == NLEVELS + 3          # nlevels - 1 resizes, FAST, octree, blur, orientation + descriptors
    assert _delta(line, lambda: line.ExtractLineSegment(img)) == 8


def test_line_debug_calls_count_their_kernel(pkg):
    line = _handle(pkg, "line")
    x = np.linspace(-3, 3, 300)
    calls = [line.ll_table,
             lambda: line.debug_nfa(W, H, [10, 40], [5, 30], [0.125, 0.125]),
             lambda: line.debug_sincos(x),
             lambda: line.debug_atan2(x.astype(np.float32), np.ones(300, np.float32))]
    for call in calls:
        assert _delta(line, call) == 1


def test_frame_launch_counts(pkg, synth):
    fr = _handle(pkg, "frame")
    gray = synth.frame(W, H, 0)
    base = NLEVELS + 3 + 8
    assert _delta(fr, lambda: fr.extract(gray)) == base + 1                        # k_undistort: extract() asks for mvKeysUn
    for cn in (3, 4):
        colour = np.repeat(gray[:, :, None], cn, axis=2)
        assert _delta(fr, lambda: fr.extract(colour)) == base + 2                  # + k_cvt_gray
    frames = pkg.host_alloc((1, H, W)); frames[0] = gray
    out = dict(keys=pkg.host_alloc((1, fr.cap), pkg.KEYPOINT_DTYPE), desc=pkg.host_alloc((1, fr.cap, 32)), n=pkg.host_alloc(1, np.int32),
               keylines=pkg.host_alloc((1, fr.lcap), pkg.KEYLINE_DTYPE), ldesc=pkg.host_alloc((1, fr.lcap, 32)),
               lineeq=pkg.host_alloc((1, fr.lcap, 3), np.float64), nl=pkg.host_alloc(1, np.int32))

    def begin():
        fr.extract_batch_begin(frames, out)
        fr.sync()
    assert _delta(fr, begin) == base                                                 # no mvKeysUn asked for, k1 == 0
    fr.set_camera(300.0, 300.0, W / 2, H / 2, (0.1, 0.0, 0.0, 0.0, 0.0))
    assert _delta(fr, begin) == base + 1                                             # k1 != 0: mvKeysUn is always computed


def test_frame_debug_calls_count_their_kernel(pkg):
    fr = _handle(pkg, "frame")
    pts = np.stack([np.linspace(0, W, 300), np.linspace(0, H, 300)], 1).astype(np.float32)
    assert _delta(fr, lambda: fr.image_bounds(W, H)) == 0                          # k1 == 0: the image itself, nothing launched
    fr.set_camera(300.0, 300.0, W / 2, H / 2, (0.1, 0.0, 0.0, 0.0))
    assert _delta(fr, lambda: fr.debug_undistort(pts)) == 1
    assert _delta(fr, lambda: fr.image_bounds(W, H)) == 1                          # the four corners through the same k_undistort


@pytest.mark.parametrize("kind, names", [("orb", ["pyramid", "fast", "octree", "blur", "orient_desc"]),
                                         ("line", ["lsd_prep", "lsd_seeds", "lsd_regions", "lsd_nfa", "keylines_lbd"])])
def test_profiled_stage_names(pkg, synth, kind, names):
    h = _handle(pkg, kind)
    h.set_profiling(True)
    _run(h, kind, synth.frame(W, H, 0))
    ms = h.stage_ms()
    assert list(ms) == names and all(t >= 0 for t in ms.values())
