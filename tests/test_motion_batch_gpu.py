"""GPU parity of the batched, device-resident motion-model matcher: ORBmatcher::SearchByProjection(CurrentFrame, LastFrame, th,
bMono = true) (ORBmatcher.cc:1331-1473) over consecutive frames in HBM, with Tracking::TrackWithMotionModel's wide-window retry
(Tracking.cc:1204-1244).  Every pair is compared with the oracle (pinned to the reference in tests/test_ref_parity_cpu.py) and with
the single-pair entry point sslpl_search_by_projection_frame.

The sequence builder below is shared with tests/test_motion_batch_cpu.py, which checks on the oracle alone that it yields pairs on
both sides of the retry threshold."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CAM = (481.2, 480.0, 319.5, 239.5)                 # Examples/ICL.yaml (|fy|)
BOUNDS = (0.0, 640.0, 0.0, 480.0)
SF = (np.float32(1.2) ** np.arange(8)).astype(np.float32)
RETRY = 20                                         # Tracking.cc:1240


def _rot(ang):
    Rx = np.array([[1, 0, 0], [0, np.cos(ang[0]), -np.sin(ang[0])], [0, np.sin(ang[0]), np.cos(ang[0])]])
    Ry = np.array([[np.cos(ang[1]), 0, np.sin(ang[1])], [0, 1, 0], [-np.sin(ang[1]), 0, np.cos(ang[1])]])
    Rz = np.array([[np.cos(ang[2]), -np.sin(ang[2]), 0], [np.sin(ang[2]), np.cos(ang[2]), 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def motion_sequence(kps, desc, n, seed, cam=CAM, bounds=BOUNDS, bad_every=3, bad_yaw=1.1, p_valid=0.85, p_obs=0.9, p_flip=0.02):
    """MapPoints and poses for a batch of frames whose keypoints (mvKeysUn, [F, cap] KEYPOINT_DTYPE), descriptors [F, cap, 32] and
    counts n[F] are given.  Frame f's keypoints get seeded random depths and become world points through frame f's pose; the pose
    of frame f + 1 is frame f's moved by a small rigid motion, except that every `bad_every`-th pair gets a large pose error, a yaw of about `bad_yaw`
    (the first pass of the matcher then finds few matches).  A few points lie behind the camera or project outside the bounds; a
    fraction of the flags are invalid or have no observations; MapPoint descriptors have a few flipped bits.
    Returns dict(Xw [F, cap, 3] f32, flag [F, cap] u8 (bit0 valid, bit1 obs), dmp [F, cap, 32] u8, Tcw [F, 12] f32)."""
    rng = np.random.default_rng(seed)
    F, cap = kps.shape
    fx, fy, cx, cy = cam
    T = np.eye(4)
    Tcw = np.zeros((F, 12), np.float32); Xw = np.zeros((F, cap, 3), np.float32)
    flag = np.zeros((F, cap), np.uint8); dmp = np.array(desc, np.uint8, copy=True)
    for f in range(F):
        if f > 0:
            dT = np.eye(4); dT[:3, :3] = _rot(rng.normal(0, 0.01, 3)); dT[:3, 3] = rng.normal(0, 0.03, 3)
            if (f - 1) % bad_every == bad_every - 1:                              # pose error: a yaw that moves most projections out of view
                dT[:3, :3] = _rot((0.0, bad_yaw + rng.normal(0, 0.02), 0.0)) @ dT[:3, :3]
            T = dT @ T
        Tf = T.astype(np.float32)
        Tcw[f] = Tf[:3, :4].reshape(-1)
        m = int(n[f])
        z = rng.uniform(1.0, 6.0, m)
        Xc = np.stack([(kps[f, :m]["x"] - cx) / fx * z, (kps[f, :m]["y"] - cy) / fy * z, z], 1)
        Xc[rng.random(m) < 0.03, 2] *= -1                                       # behind the camera
        Xc[rng.random(m) < 0.03, :2] *= 6.0                                     # outside the image bounds
        R, t = Tf[:3, :3].astype(np.float64), Tf[:3, 3].astype(np.float64)
        Xw[f, :m] = ((Xc - t) @ R).astype(np.float32)                           # Rcw^T (Xc - tcw)
        flag[f, :m] = (rng.random(m) < p_valid).astype(np.uint8) | ((rng.random(m) < p_obs).astype(np.uint8) << 1)
        flip = rng.random((m, 32)) < p_flip
        dmp[f, :m][flip] ^= (1 << rng.integers(0, 8, int(flip.sum()))).astype(np.uint8)
    return dict(Xw=Xw, flag=flag, dmp=dmp, Tcw=Tcw)


def pair_inputs(kps, desc, n, seq, p, own_desc=False):
    """Pair p (LastFrame = frame p, CurrentFrame = frame p + 1) in the form of oracle.search_by_projection_frame."""
    n1, n2 = int(n[p]), int(n[p + 1])
    fl = seq["flag"][p, :n1]
    last = dict(valid=fl & 1, obs=(fl >> 1) & 1, Xw=seq["Xw"][p, :n1], dmp=(desc if own_desc else seq["dmp"])[p, :n1],
                oct=kps[p, :n1]["octave"].astype(np.int32), angle=kps[p, :n1]["angle"])
    k2 = kps[p + 1, :n2]
    cur = dict(desc=desc[p + 1, :n2], x=k2["x"], y=k2["y"], oct=k2["octave"].astype(np.int32), angle=k2["angle"], uright=None, claimed=None)
    return last, cur, seq["Tcw"][p + 1]


def oracle_motion_model(oracle, kps, desc, n, seq, p, th, check_ori, retry_below, own_desc=False, cam=CAM, bounds=BOUNDS):
    """TrackWithMotionModel's matching for pair p on the oracle: th, then 2 * th when that gave fewer than retry_below.
    Returns (nmatches, assign2 with -1 for "no MapPoint", first-pass count)."""
    last, cur, T = pair_inputs(kps, desc, n, seq, p, own_desc)
    cam6 = tuple(cam) + (0.0, 0.0)
    n0, a = oracle.search_by_projection_frame(last, cur, T, None, cam6, bounds, SF, th, True, check_ori)
    nm = n0
    if retry_below > 0 and n0 < retry_below:
        nm, a = oracle.search_by_projection_frame(last, cur, T, None, cam6, bounds, SF, 2 * th, True, check_ori)
    return nm, a, n0


def sequence_frames(synth):
    """Nine 640x480 frames: synthetic frames 0-8 (a new scene from frame 8 on) with frame 4 flat, i.e. without keypoints."""
    frames = synth.batch(640, 480, 9)
    frames[4] = 128
    return frames


# ------------------------------------------------------------------------------------------------------------------ GPU helpers
class _DevView:
    """A raw device buffer as a torch tensor (__cuda_array_interface__), to read the library's device results back."""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = dict(shape=tuple(shape), typestr=typestr, data=(int(ptr), False), version=2, strides=None)


def _download(torch, ptr, shape, typestr):
    return torch.as_tensor(_DevView(ptr, shape, typestr), device="cuda").cpu().numpy()


def device_batch(pkg, torch, frames, nfeatures=1000):
    """ORB device path over the frames: returns the extractor, its raw device results and their host copies."""
    B, H, W = frames.shape
    ext = pkg.ORBextractor(nfeatures, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=B)
    dfr = torch.from_numpy(np.ascontiguousarray(frames)).cuda()
    ext.extract_batch_device(dfr.data_ptr(), B, W, H, W, W * H)
    ext.sync()
    d_kps, d_desc, d_n, cap = ext.device_results()
    kps = _download(torch, d_kps, (B, cap * pkg.KEYPOINT_DTYPE.itemsize), "|u1").view(pkg.KEYPOINT_DTYPE).reshape(B, cap)
    desc = _download(torch, d_desc, (B, cap, 32), "|u1")
    n = _download(torch, d_n, (B,), "<i4")
    return dict(ext=ext, dfr=dfr, d_kps=d_kps, d_desc=d_desc, d_n=d_n, cap=cap, kps=kps, desc=desc, n=n)


def upload_sequence(torch, seq):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in seq.items()}


def run_batch(mt, torch, D, dseq, nframes, th, check_ori, retry_below, own_desc=False, cam=CAM, bounds=BOUNDS, d_kps=None):
    cap = D["cap"]
    d_assign = torch.full((nframes - 1, cap), 7, dtype=torch.int32, device="cuda")
    d_nmatch = torch.full((nframes - 1,), -7, dtype=torch.int32, device="cuda")
    mt.search_by_projection_frame_batch_device(d_kps or D["d_kps"], D["d_desc"], D["d_n"], nframes, cap, dseq["Xw"].data_ptr(),
                                               dseq["flag"].data_ptr(), 0 if own_desc else dseq["dmp"].data_ptr(), dseq["Tcw"].data_ptr(),
                                               cam, bounds, SF, th, check_ori, retry_below, d_assign.data_ptr(), d_nmatch.data_ptr())
    mt.sync()
    return d_assign.cpu().numpy(), d_nmatch.cpu().numpy()


def check_against_oracle(oracle, kps, desc, n, seq, got_a, got_n, th, check_ori, retry_below, own_desc=False, cam=CAM, bounds=BOUNDS):
    firsts = []
    for p in range(len(got_n)):
        nm, a, n0 = oracle_motion_model(oracle, kps, desc, n, seq, p, th, check_ori, retry_below, own_desc, cam, bounds)
        n2 = int(n[p + 1])
        row = got_a[p]
        assert got_n[p] == nm and np.array_equal(np.where(row[:n2] == -2, -1, row[:n2]), a), (p, int(got_n[p]), nm)
        assert (row[n2:] == -1).all(), p
        firsts.append(n0)
    return np.array(firsts)


@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


@pytest.fixture(scope="module")
def seq9(pkg, synth, torch):
    """Nine 640x480 frames (frame 4 flat: zero keypoints) through the ORB device path, with their MapPoints and poses."""
    frames = sequence_frames(synth)
    D = device_batch(pkg, torch, frames)
    assert D["n"][4] == 0 and (np.delete(D["n"], 4) > 500).all()
    seq = motion_sequence(D["kps"], D["desc"], D["n"], seed=11)
    return D, seq, upload_sequence(torch, seq)


@pytest.mark.parametrize("check_ori", [True, False])
@pytest.mark.parametrize("retry_below", [0, RETRY])
@pytest.mark.parametrize("own_desc", [False, True])
def test_batch_equals_oracle(pkg, oracle, torch, seq9, check_ori, retry_below, own_desc):
    D, seq, dseq = seq9
    B = len(D["n"])
    mt = pkg.Matcher(max_features=D["cap"], max_lines=64, max_nodes=64, max_batch=B - 1)         # nframes = max_batch + 1
    got_a, got_n = run_batch(mt, torch, D, dseq, B, 15.0, check_ori, retry_below, own_desc)
    firsts = check_against_oracle(oracle, D["kps"], D["desc"], D["n"], seq, got_a, got_n, 15.0, check_ori, retry_below, own_desc)
    live = [p for p in range(B - 1) if p not in (3, 4)]                                           # pairs 3 and 4 touch the flat frame
    assert (got_n[[3, 4]] == 0).all() and (firsts[live] < RETRY).any() and (firsts[live] >= RETRY).any()
    # nframes = 2 on the same handle: pair 0 alone
    a2, n2 = run_batch(mt, torch, D, dseq, 2, 15.0, check_ori, retry_below, own_desc)
    assert n2[0] == got_n[0] and np.array_equal(a2[0], got_a[0])


@pytest.mark.parametrize("check_ori", [True, False])
def test_batch_equals_single_pair_entry_point(pkg, torch, seq9, check_ori):
    """Raw tables (-2 included) of every pair equal sslpl_search_by_projection_frame on the same pair, th or 2 * th as retried."""
    D, seq, dseq = seq9
    B = len(D["n"])
    mt = pkg.Matcher(max_features=D["cap"], max_lines=64, max_nodes=3072, max_batch=B - 1)
    got_a, got_n = run_batch(mt, torch, D, dseq, B, 15.0, check_ori, RETRY)
    retried = 0
    for p in range(B - 1):
        last, cur, T = pair_inputs(D["kps"], D["desc"], D["n"], seq, p)
        cam6 = CAM + (0.0, 0.0)
        nm, a = mt.search_by_projection_frame(last, cur, T, None, cam6, BOUNDS, SF, 15.0, True, check_ori, raw=True)
        if nm < RETRY:
            nm, a = mt.search_by_projection_frame(last, cur, T, None, cam6, BOUNDS, SF, 30.0, True, check_ori, raw=True)
            retried += 1
        n2 = int(D["n"][p + 1])
        assert got_n[p] == nm and np.array_equal(got_a[p, :n2], a), p
    assert 0 < retried < B - 1


def test_large_frames(pkg, oracle, synth, torch):
    """1280x960, 4000 features: a larger cap and denser grid cells."""
    frames = synth.batch(1280, 960, 4, start=0)
    D = device_batch(pkg, torch, frames, nfeatures=4000)
    assert D["cap"] > 4000 and (D["n"] > 2000).all()
    bounds = (0.0, 1280.0, 0.0, 960.0); cam = (962.4, 960.0, 639.5, 479.5)
    seq = motion_sequence(D["kps"], D["desc"], D["n"], seed=5, cam=cam, bounds=bounds, bad_every=2)
    mt = pkg.Matcher(max_features=D["cap"], max_lines=64, max_nodes=64, max_batch=3)
    got_a, got_n = run_batch(mt, torch, D, upload_sequence(torch, seq), 4, 15.0, True, RETRY, cam=cam, bounds=bounds)
    check_against_oracle(oracle, D["kps"], D["desc"], D["n"], seq, got_a, got_n, 15.0, True, RETRY, cam=cam, bounds=bounds)
    assert got_n.max() > 500


def test_frame_handle_with_distortion(pkg, oracle, synth, torch):
    """Colour frames with k1 != 0 through pkg.Frame: the batched matcher reads device_keypoints_un(), the oracle the host keysUn of
    the same call (and the image bounds of the distorted camera)."""
    B = 5
    gray = synth.batch(640, 480, B, start=9)
    rng = np.random.default_rng(2)
    bgr = np.stack([np.clip(gray.astype(int) + rng.integers(-30, 30, gray.shape), 0, 255).astype(np.uint8) for _ in range(3)], 3)
    fr = pkg.Frame(1000, 1.2, 8, 20, 7, 40, max_width=640, max_height=480, max_batch=B)
    K = (517.3, 516.5, 318.6, 255.3)
    fr.set_camera(*K, [0.2624, -0.9531, -0.0054, 0.0026, 1.1633])
    r = fr.extract_batch(bgr)
    bounds = tuple(float(v) for v in fr.image_bounds(640, 480))
    d_un, cap = fr.device_keypoints_un()
    d_kps, d_desc, d_n, cap2 = fr.orb.device_results()
    assert cap == cap2 and d_un != d_kps
    un = _download(torch, d_un, (B, cap * 28), "|u1").view(pkg.KEYPOINT_DTYPE).reshape(B, cap)
    for f in range(B):
        assert un[f, :r["n"][f]].tobytes() == r["keysUn"][f, :r["n"][f]].tobytes()
    assert not np.array_equal(r["keysUn"][0, :r["n"][0]]["x"], r["keys"][0, :r["n"][0]]["x"])
    seq = motion_sequence(r["keysUn"], r["desc"], r["n"], seed=3, cam=K, bounds=bounds)
    D = dict(d_kps=d_un, d_desc=d_desc, d_n=d_n, cap=cap)
    mt = pkg.Matcher(max_features=cap, max_lines=64, max_nodes=64, max_batch=B - 1)
    got_a, got_n = run_batch(mt, torch, D, upload_sequence(torch, seq), B, 15.0, True, RETRY, cam=K, bounds=bounds)
    check_against_oracle(oracle, r["keysUn"], r["desc"], r["n"], seq, got_a, got_n, 15.0, True, RETRY, cam=K, bounds=bounds)
    assert got_n.max() > 100
    fr.set_camera(*K, [0.0, 0.1])                                    # k1 == 0: mvKeysUn is the ORB handle's keypoints (Frame.cc:485)
    fr.extract_batch(bgr)
    assert fr.device_keypoints_un()[0] == fr.orb.device_results()[0]


def test_caller_stream(pkg, oracle, torch, seq9):
    """On a caller-set stream the results are ready once that stream is synchronised; no sslpl_matcher_sync."""
    D, seq, dseq = seq9
    B = len(D["n"])
    mt = pkg.Matcher(max_features=D["cap"], max_lines=64, max_nodes=64, max_batch=B - 1)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        mt.set_stream(s.cuda_stream)
        d_assign = torch.full((B - 1, D["cap"]), 7, dtype=torch.int32, device="cuda")
        d_nmatch = torch.full((B - 1,), -7, dtype=torch.int32, device="cuda")
        mt.search_by_projection_frame_batch_device(D["d_kps"], D["d_desc"], D["d_n"], B, D["cap"], dseq["Xw"].data_ptr(), dseq["flag"].data_ptr(),
                                                   dseq["dmp"].data_ptr(), dseq["Tcw"].data_ptr(), CAM, BOUNDS, SF, 15.0, True, RETRY,
                                                   d_assign.data_ptr(), d_nmatch.data_ptr())
    s.synchronize()
    got_a, got_n = d_assign.cpu().numpy(), d_nmatch.cpu().numpy()
    check_against_oracle(oracle, D["kps"], D["desc"], D["n"], seq, got_a, got_n, 15.0, True, RETRY)
    mt.set_stream(0)


def test_argument_errors_enqueue_nothing(pkg, torch, seq9):
    D, seq, dseq = seq9
    B = len(D["n"])
    cap = D["cap"]
    mt = pkg.Matcher(max_features=cap - 64, max_lines=64, max_nodes=64, max_batch=B - 1)
    d_assign = torch.full((B, cap + 1), 7, dtype=torch.int32, device="cuda")
    d_nmatch = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    good = dict(d_kps=D["d_kps"], d_desc=D["d_desc"], d_n=D["d_n"], nframes=B, cap=cap, d_Xw=dseq["Xw"].data_ptr(), d_mpflag=dseq["flag"].data_ptr(),
                d_dmp=0, d_Tcw=dseq["Tcw"].data_ptr(), cam=CAM, bounds=BOUNDS, scale_factors=SF, th=15.0, check_ori=True, retry_below=RETRY,
                d_assign=d_assign.data_ptr(), d_nmatch=d_nmatch.data_ptr())
    bad = [dict(d_kps=0), dict(d_desc=0), dict(d_n=0), dict(d_Xw=0), dict(d_mpflag=0), dict(d_Tcw=0), dict(d_assign=0), dict(d_nmatch=0),
           dict(nframes=1), dict(nframes=B + 1), dict(cap=0), dict(cap=cap + 1), dict(scale_factors=np.zeros(0, np.float32)),
           dict(scale_factors=np.ones(33, np.float32)), dict(th=0.0), dict(th=-15.0), dict(th=float("nan")),
           dict(bounds=(0.0, 0.0, 0.0, 480.0)), dict(bounds=(0.0, 640.0, 480.0, 0.0))]
    before = mt.launch_count
    for b in bad:
        with pytest.raises(pkg.SslplError, match="error -1:"):
            mt.search_by_projection_frame_batch_device(**{**good, **b})
    mt.sync()
    assert mt.launch_count == before and (d_assign == 7).all().item() and (d_nmatch == -7).all().item()
    mt.search_by_projection_frame_batch_device(**good)                                           # the boundary values are accepted
    mt.sync()
    assert mt.launch_count == before + 3 and (d_nmatch[:B - 1] >= 0).all().item()
