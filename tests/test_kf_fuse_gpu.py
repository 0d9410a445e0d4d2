"""GPU parity of LocalMapping::SearchInNeighbors' batched, device-resident Fuse calls (LocalMapping.cc:1178-1279): ORBmatcher::Fuse
(ORBmatcher.cc:828-973) and LSDmatcher::Fuse (LSDmatcher.cpp:417-548) over (keyframe, element) entries of keyframes the extractors left in
HBM, with MapPoint / MapLine::PredictScale on the device.  Every entry is compared bit for bit with the oracle's projection and search
stages (pinned to the reference in tests/test_ref_parity_cpu.py) and with the single-call search entry points fed the oracle's projection;
the device PredictScale with the oracle's (int)ceil(logf(ratio) / logScaleFactor) around every threshold; and a SearchInNeighbors replay
with the re-test / re-submit rule of include/sslpl.h with the sequential reference order.  tests/test_kf_fuse_cpu.py shows on the oracle
alone that every gate decides some entry here."""
import numpy as np
import pytest

import fuse_model as fm
from test_kf_fuse_cpu import _sources, check_replay, point_entries, replay_lines, replay_points
from test_kf_triangulation_gpu import FLAT, NKF, keyframe_frames
from test_motion_batch_gpu import _download, device_batch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


def device_keyframes(pkg, torch, frames, nfeatures=1000, nlines=40):
    """ORB and line device paths over the frames: raw device results, their host copies, poses (fuse_model.poses) and camera."""
    B, H, W = frames.shape
    D = device_batch(pkg, torch, frames, nfeatures)
    seg = pkg.LineSegment(nlines, max_width=W, max_height=H, max_batch=B)
    seg.extract_batch_device(D["dfr"].data_ptr(), B, W, H, W, W * H)
    seg.sync()
    d_kl, d_ld, _, d_nl, capl = seg.device_results()
    kl = _download(torch, d_kl, (B, capl * pkg.KEYLINE_DTYPE.itemsize), "|u1").view(pkg.KEYLINE_DTYPE).reshape(B, capl)
    cam, bounds = fm.camera(W, H)
    pose = fm.poses(B, B, W, H)
    return dict(D, seg=seg, d_kl=d_kl, d_ldesc=d_ld, d_nl=d_nl, capl=capl, kl=kl, ldesc=_download(torch, d_ld, (B, capl, 32), "|u1"),
                nl=_download(torch, d_nl, (B,), "<i4"), pose=pose, d_pose=torch.from_numpy(pose).cuda(), cam=cam, bounds=bounds, W=W, H=H)


def matcher(pkg, K, max_batch=None):
    return pkg.Matcher(max_features=K["cap"], max_lines=K["capl"], max_nodes=3072, max_batch=max_batch or len(K["n"]) - 1)


def _dev(torch, a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


def enqueue_points(mt, torch, K, table, desc, E, skip, d_pose=None, th=fm.TH):
    """Enqueue one batched point call; returns the output tensors (sentinels 7 / -7 where nothing is written)."""
    T = dict(mp=_dev(torch, table, np.float32), d=_dev(torch, np.asarray(desc).reshape(-1, 32), np.uint8),
             E=_dev(torch, np.asarray(E).reshape(-1, 2), np.int32), s=_dev(torch, skip, np.uint8))
    T["bi"] = torch.full((max(len(E), 1),), 7, dtype=torch.int32, device="cuda"); T["bd"] = torch.full((max(len(E), 1),), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    mt.fuse_points_batch_device(K["d_kps"], K["d_desc"], K["d_n"], len(K["n"]), K["cap"], (d_pose if d_pose is not None else K["d_pose"]).data_ptr(),
                                len(table), T["mp"].data_ptr(), T["d"].data_ptr(), len(E), T["E"].data_ptr(), T["s"].data_ptr(), K["cam"], K["bounds"],
                                fm.SF, fm.INV_SIGMA2, fm.LOGS, th, T["bi"].data_ptr(), T["bd"].data_ptr())
    return T


def enqueue_lines(mt, torch, K, table, desc, E, skip, d_pose=None, th=fm.TH):
    T = dict(ml=_dev(torch, table, np.float32), d=_dev(torch, np.asarray(desc).reshape(-1, 32), np.uint8),
             E=_dev(torch, np.asarray(E).reshape(-1, 2), np.int32), s=_dev(torch, skip, np.uint8))
    T["bi"] = torch.full((max(len(E), 1),), 7, dtype=torch.int32, device="cuda"); T["bd"] = torch.full((max(len(E), 1),), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    mt.fuse_lines_batch_device(K["d_kl"], K["d_ldesc"], K["d_nl"], len(K["nl"]), K["capl"], (d_pose if d_pose is not None else K["d_pose"]).data_ptr(),
                               len(table), T["ml"].data_ptr(), T["d"].data_ptr(), len(E), T["E"].data_ptr(), T["s"].data_ptr(), K["cam"], K["bounds"],
                               fm.SF, fm.LOGS, th, T["bi"].data_ptr(), T["bd"].data_ptr())
    return T


def results(T, n):
    return T["bi"].cpu().numpy()[:n], T["bd"].cpu().numpy()[:n]


def run_points(mt, torch, K, table, desc, E, skip, d_pose=None):
    T = enqueue_points(mt, torch, K, table, desc, E, skip, d_pose)
    mt.sync()
    return results(T, len(E))


def run_lines(mt, torch, K, table, desc, E, skip, d_pose=None):
    T = enqueue_lines(mt, torch, K, table, desc, E, skip, d_pose)
    mt.sync()
    return results(T, len(E))


def check_points(mt, oracle, K, table, desc, E, skip, got, pose=None):
    """Every entry equals the oracle, and (in range) the single-call search fed the oracle's projection."""
    pose = K["pose"] if pose is None else pose
    bi, bd, per_kf = fm.oracle_points(oracle, K, pose, table, desc, E, skip)
    bad = np.nonzero((got[0] != bi) | (got[1] != bd))[0]
    assert len(bad) == 0, (len(bad), [(tuple(E[j]), int(got[0][j]), int(got[1][j]), int(bi[j]), int(bd[j])) for j in bad[:5]])
    for k, (sel, args) in per_kf.items():
        sbi, sbd = mt.fuse_points_search(*args)
        assert np.array_equal(sbi, got[0][sel]) and np.array_equal(sbd, got[1][sel]), k
    return bi, bd


def check_lines(mt, oracle, K, table, desc, E, skip, got, pose=None):
    pose = K["pose"] if pose is None else pose
    bi, bd, per_kf = fm.oracle_lines(oracle, K, pose, table, desc, E, skip)
    bad = np.nonzero((got[0] != bi) | (got[1] != bd))[0]
    assert len(bad) == 0, (len(bad), [(tuple(E[j]), int(got[0][j]), int(got[1][j]), int(bi[j]), int(bd[j])) for j in bad[:5]])
    for k, (sel, args) in per_kf.items():
        sbi, sbd = mt.fuse_lines_search(*args)
        assert np.array_equal(sbi, got[0][sel]) and np.array_equal(sbd, got[1][sel]), k
    return bi, bd


def with_specials(rng, E, skip, nel, nkf):
    """Repeated entries, NULL entries, skipped entries and out-of-range indices appended to an entry list."""
    rep = E[rng.integers(0, len(E), 200)]
    null = np.stack([rng.integers(0, nkf, 20), np.full(20, -1)], 1)
    out = np.array([(nkf, 0), (-1, 0), (0, nel), (1, -2), (1 << 30, 3), (2, -(1 << 30))])
    forced = E[rng.integers(0, len(E), 50)]
    E2 = np.concatenate([E, rep, null, out, forced]).astype(np.int32)
    s2 = np.concatenate([skip, skip[rng.integers(0, len(E), 200)] * 0, np.zeros(20 + len(out), np.uint8), np.ones(50, np.uint8)]).astype(np.uint8)
    return E2, s2, len(E) + 200 + 20


@pytest.fixture(scope="module")
def kfs(pkg, synth, torch):
    K = device_keyframes(pkg, torch, keyframe_frames(synth))
    assert K["n"][FLAT] == 0 and K["nl"][FLAT] == 0 and (np.delete(K["n"], FLAT) > 500).all() and (np.delete(K["nl"], FLAT) >= 20).all()
    return K


def point_case(K, seed=3):
    rng = np.random.default_rng(seed)
    src = _sources(rng, K["n"], len(K["n"]), 0.05)
    T = fm.point_table(rng, src, K["kps"], K["desc"], K["pose"], len(K["n"]), K["W"], K["H"])
    E, skip = point_entries(rng, K, src, int(K["n"][0]))
    E, skip, nout = with_specials(rng, E, skip, len(T["mp"]), len(K["n"]))
    return T, E, skip, nout


def line_case(K, seed=4):
    rng = np.random.default_rng(seed)
    nkf = len(K["nl"])
    src = [(k, i) for k in range(nkf) for i in range(int(K["nl"][k])) if k == 0 or rng.random() < 0.3]
    T = fm.line_table(rng, src, K["kl"], K["ldesc"], K["pose"], nkf, K["W"], K["H"], p_gate=0.06)
    n0 = int(K["nl"][0])
    E = np.array([(k, e) for k in range(1, nkf) for e in range(n0)] + [(0, e) for e in range(n0, len(src))], np.int32)
    skip = (rng.random(len(E)) < 0.03).astype(np.uint8)
    E, skip, nout = with_specials(rng, E, skip, len(T["ml"]), nkf)
    return T, E, skip, nout


def test_points_equal_oracle(pkg, oracle, torch, kfs):
    """Phase A (KF 0's MapPoints into its 20 neighbours, the flat keyframe among them) and phase B (the neighbours' candidates into
    KF 0) in one call, nkf = max_batch + 1, with repeated, NULL, skipped and out-of-range entries."""
    K = kfs
    mt = matcher(pkg, K)
    T, E, skip, nout = point_case(K)
    got = run_points(mt, torch, K, T["mp"], T["desc"], E, skip)
    bi, bd = check_points(mt, oracle, K, T["mp"], T["desc"], E, skip, got)
    out = np.arange(nout, nout + 6)
    assert (bi[out] == -1).all() and (bd[out] == -1).all()
    assert (bd[E[:, 0] == FLAT] == 256).all() and ((bd <= fm.TH_LOW) & (bi >= 0)).sum() > 2000


def test_lines_equal_oracle(pkg, oracle, torch, kfs):
    K = kfs
    mt = matcher(pkg, K)
    T, E, skip, nout = line_case(K)
    got = run_lines(mt, torch, K, T["ml"], T["desc"], E, skip)
    bi, bd = check_lines(mt, oracle, K, T["ml"], T["desc"], E, skip, got)
    out = np.arange(nout, nout + 6)
    assert (bi[out] == -1).all() and (bd[out] == -1).all()
    assert (bd[E[:, 0] == FLAT] == fm.INT_MAX).all() and ((bd <= fm.TH_LOW) & (bi >= 0)).sum() > 150
    pyr = (T["gate"][np.clip(E[:, 1], 0, len(T["gate"]) - 1)] == fm.LINE_GATES.index("pyramid")) & (E[:, 1] >= 0) & (E[:, 1] < len(T["gate"]))
    assert pyr.sum() > 0 and (bd[pyr] == fm.INT_MAX).all()


def test_zero_distance_and_zero_max_distance(pkg, oracle, torch, kfs):
    """dist = 0 with minInv = 0 (ratio +inf, or NaN with maxRaw = 0) and maxRaw = 0 (ratio 0): level 0 for a MapPoint, dropped for a
    MapLine.  Keyframe 2's camera centre is moved onto chosen elements (the pose table's Ow is an input like any other)."""
    K = kfs
    mt = matcher(pkg, K)
    rng = np.random.default_rng(5)
    src = [(2, int(i)) for i in range(0, int(K["n"][2]), 5)]
    T = fm.point_table(rng, src, K["kps"], K["desc"], K["pose"], len(K["n"]), K["W"], K["H"], p_gate=0)
    mp = T["mp"].copy()
    pose = K["pose"].copy(); pose[2, 12:] = mp[0, :3]
    mp[1, :3] = mp[0, :3]; mp[:4, 6] = 0                          # rows 0, 1 at dist 0 with minInv = 0: ratio +inf, and NaN with maxRaw = 0
    mp[1:4, 8] = 0; mp[2:4, 7] = 1e6                              # rows 2, 3: maxRaw = 0 at dist > 0, ratio 0
    po = mp[2:4, :3].astype(np.float64) - pose[2, 12:]; mp[2:4, 3:6] = po / np.linalg.norm(po, axis=1)[:, None]   # seen from the moved centre
    E = np.array([(2, e) for e in range(len(mp))], np.int32); skip = np.zeros(len(E), np.uint8)
    got = run_points(mt, torch, K, mp, T["desc"], E, skip, torch.from_numpy(pose).cuda())
    check_points(mt, oracle, K, mp, T["desc"], E, skip, got, pose)
    q = oracle.fuse_project_points(skip[:4], mp[:4, :3], mp[:4, 3:6], mp[:4, 6], mp[:4, 7], mp[:4, 8], pose[2, :12].reshape(3, 4), pose[2, 12:],
                                   np.append(K["cam"], 0.0), K["bounds"], fm.NLEV, fm.LOGS)
    assert q["active"].all() and (q["level"] == 0).all()
    # lines: the mid-point of row 0 as Ow
    lsrc = [(2, i) for i in range(int(K["nl"][2]))]
    L = fm.line_table(rng, lsrc, K["kl"], K["ldesc"], K["pose"], len(K["nl"]), K["W"], K["H"], p_gate=0)
    ml = L["ml"].copy()
    lpose = K["pose"].copy(); lpose[2, 12:] = np.float32(0.5) * (ml[0, :3] + ml[0, 3:6])
    ml[1, :6] = ml[0, :6]; ml[:4, 9] = 0; ml[1:4, 11] = 0; ml[2:4, 10] = 1e6
    E = np.array([(2, e) for e in range(len(ml))], np.int32); skip = np.zeros(len(E), np.uint8)
    got = run_lines(mt, torch, K, ml, L["desc"], E, skip, torch.from_numpy(lpose).cuda())
    check_lines(mt, oracle, K, ml, L["desc"], E, skip, got, lpose)
    assert (got[1][:4] == fm.INT_MAX).all()


def test_large_frames(pkg, oracle, synth, torch):
    """1280x960, 4000 features, 500 lines: larger caps, denser grid cells."""
    frames = keyframe_frames(synth, 1280, 960, nkf=5, flat=None)
    K = device_keyframes(pkg, torch, frames, nfeatures=4000, nlines=500)
    mt = matcher(pkg, K)
    T, E, skip, _ = point_case(K, seed=6)
    got = run_points(mt, torch, K, T["mp"], T["desc"], E, skip)
    bi, bd = check_points(mt, oracle, K, T["mp"], T["desc"], E, skip, got)
    assert ((bd <= fm.TH_LOW) & (bi >= 0)).sum() > 2000
    T, E, skip, _ = line_case(K, seed=7)
    got = run_lines(mt, torch, K, T["ml"], T["desc"], E, skip)
    bi, bd = check_lines(mt, oracle, K, T["ml"], T["desc"], E, skip, got)
    assert ((bd <= fm.TH_LOW) & (bi >= 0)).sum() > 200


def test_caller_stream_back_to_back(pkg, oracle, torch, kfs):
    """Two point calls and a line call enqueued back to back on a caller-set stream, no wait between them: each equals its own result
    on the handle's stream once that caller stream is synchronised."""
    K = kfs
    mt = matcher(pkg, K)
    Tp, Ep, sp, _ = point_case(K, seed=8)
    Tl, El, sl, _ = line_case(K, seed=9)
    want_a = run_points(mt, torch, K, Tp["mp"], Tp["desc"], Ep, sp)
    want_b = run_points(mt, torch, K, Tp["mp"], Tp["desc"], Ep[::-1].copy(), sp[::-1].copy())
    want_l = run_lines(mt, torch, K, Tl["ml"], Tl["desc"], El, sl)
    s = torch.cuda.Stream()
    mt.set_stream(s.cuda_stream)
    try:
        a = enqueue_points(mt, torch, K, Tp["mp"], Tp["desc"], Ep, sp)
        b = enqueue_points(mt, torch, K, Tp["mp"], Tp["desc"], Ep[::-1].copy(), sp[::-1].copy())
        c = enqueue_lines(mt, torch, K, Tl["ml"], Tl["desc"], El, sl)
        s.synchronize()
        for got, want, n in ((a, want_a, len(Ep)), (b, want_b, len(Ep)), (c, want_l, len(El))):
            r = results(got, n)
            assert np.array_equal(r[0], want[0]) and np.array_equal(r[1], want[1])
    finally:
        mt.set_stream(0)
    assert np.array_equal(want_b[0], want_a[0][::-1]) and np.array_equal(want_b[1], want_a[1][::-1])


def test_argument_errors_enqueue_nothing(pkg, torch, kfs):
    K = kfs
    mt = matcher(pkg, K)
    T, E, skip, _ = point_case(K)
    L, El, sl, _ = line_case(K)
    n0 = mt.launch_count
    d = dict(mp=_dev(torch, T["mp"], np.float32), d=_dev(torch, T["desc"], np.uint8), E=_dev(torch, E, np.int32),
             ml=_dev(torch, L["ml"], np.float32), ld=_dev(torch, L["desc"], np.uint8), El=_dev(torch, El, np.int32))
    bi = torch.full((len(E),), 7, dtype=torch.int32, device="cuda"); bd = torch.full((len(E),), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    nkf = len(K["n"])

    def pts(**kw):
        a = dict(d_kps=K["d_kps"], d_desc=K["d_desc"], d_n=K["d_n"], nkf=nkf, cap=K["cap"], d_kfpose=K["d_pose"].data_ptr(), nmp=len(T["mp"]),
                 d_mp=d["mp"].data_ptr(), d_mpdesc=d["d"].data_ptr(), nentries=len(E), d_entry=d["E"].data_ptr(), d_skip=0, cam=K["cam"],
                 bounds=K["bounds"], scale_factors=fm.SF, inv_level_sigma2=fm.INV_SIGMA2, log_scale_factor=fm.LOGS, th=fm.TH,
                 d_best_idx=bi.data_ptr(), d_best_dist=bd.data_ptr())
        a.update(kw)
        mt.fuse_points_batch_device(**a)

    def lns(**kw):
        a = dict(d_kl=K["d_kl"], d_ldesc=K["d_ldesc"], d_nl=K["d_nl"], nkf=nkf, capl=K["capl"], d_kfpose=K["d_pose"].data_ptr(), nml=len(L["ml"]),
                 d_ml=d["ml"].data_ptr(), d_mldesc=d["ld"].data_ptr(), nentries=len(El), d_entry=d["El"].data_ptr(), d_skip=0, cam=K["cam"],
                 bounds=K["bounds"], scale_factors=fm.SF, log_scale_factor=fm.LOGS, th=fm.TH, d_best_idx=bi.data_ptr(), d_best_dist=bd.data_ptr())
        a.update(kw)
        mt.fuse_lines_batch_device(**a)

    for fn, bads in ((pts, [dict(nkf=0), dict(nkf=nkf + 1), dict(cap=0), dict(cap=K["cap"] + 65), dict(nmp=-1), dict(nentries=-1), dict(d_entry=0),
                            dict(d_kfpose=0), dict(d_mp=0), dict(d_kps=0), dict(d_best_idx=0), dict(scale_factors=fm.SF[:0]),
                            dict(scale_factors=np.ones(17, np.float32), inv_level_sigma2=np.ones(17, np.float32)),
                            dict(log_scale_factor=0.0), dict(log_scale_factor=float("nan")), dict(bounds=np.array([0, 0, 0, 480], np.float32))]),
                     (lns, [dict(nkf=0), dict(nkf=nkf + 1), dict(capl=0), dict(capl=K["capl"] + 65), dict(nml=-1), dict(d_ml=0), dict(d_kl=0),
                            dict(d_entry=0), dict(log_scale_factor=-1.0), dict(scale_factors=fm.SF[:0])])):
        for kw in bads:
            with pytest.raises(pkg.SslplError):
                fn(**kw)
    pts(nentries=0); lns(nentries=0)
    mt.sync()
    assert mt.launch_count == n0
    assert (bi.cpu() == 7).all() and (bd.cpu() == -7).all()


# ------------------------------------------------------------------------------------------------------------------ PredictScale
def _ulps(t, k):
    b = np.asarray(t, np.float32).view(np.int32).astype(np.int64)
    r = (b[:, None] + np.arange(-k, k + 1)[None, :]).reshape(-1)
    return r[(r >= 0) & (r <= 0x7f800000)].astype(np.int32).view(np.float32)


def _check_levels(mt, oracle, ratio, s, nlevels):
    raw = fm.oracle_levels(oracle, ratio, s, nlevels)
    for clamp in (True, False):
        got = mt.debug_predict_scale(ratio, s, nlevels, clamp)
        want = fm.window_levels(raw, nlevels, clamp)
        bad = np.nonzero(got != want)[0]
        assert len(bad) == 0, (s, nlevels, clamp, [(float(ratio[j]), int(got[j]), int(want[j])) for j in bad[:5]])


def test_predict_scale_at_thresholds(pkg, oracle):
    """Every float within 256 ulp of every threshold, scale factors 1.2, 1.5 and 2.0, 4 to 16 levels, clamp on and off."""
    mt = pkg.Matcher(max_features=64, max_lines=8, max_nodes=8)
    for sf in (1.2, 1.5, 2.0):
        s = np.float32(np.log(np.float32(sf)))
        for nlevels in range(4, 17):
            thr = pkg.predict_scale_table(s, nlevels)
            finite = thr[np.isfinite(thr)]
            _check_levels(mt, oracle, _ulps(finite, 256), s, nlevels)


def test_predict_scale_random_and_special(pkg, oracle):
    mt = pkg.Matcher(max_features=64, max_lines=8, max_nodes=8)
    rng = np.random.default_rng(17)
    r = rng.integers(0, 1 << 32, 1 << 24, dtype=np.uint64).astype(np.uint32).view(np.float32)
    f32 = np.finfo(np.float32)
    special = np.array([0.0, -0.0, -1.0, -f32.max, f32.smallest_subnormal, -f32.smallest_subnormal, f32.smallest_normal, 1e-40, 3e-39,
                        f32.max, np.inf, -np.inf, np.nan, -np.nan, 1.0, 0.8333333, 1.2], np.float32)
    s = fm.LOGS
    _check_levels(mt, oracle, np.concatenate([r, special, np.abs(r[:1 << 20])]), s, fm.NLEV)
    got = mt.debug_predict_scale(special, s, fm.NLEV, False)
    assert list(got[[0, 1, 2, 10, 11, 12]]) == [fm.INT_MIN] * 6 and got[4] == -1 and got[9] == fm.NLEV
    assert (mt.debug_predict_scale(special, s, fm.NLEV, True)[[0, 1, 2, 10, 11, 12]] == 0).all()


# ------------------------------------------------------------------------------------------------------------------ replay
def test_replay_search_in_neighbors(pkg, oracle, torch, kfs):
    """SearchInNeighbors on a small map model, sequentially on the oracle and as two batched device calls per element type with the
    re-test / re-submit rule: the same keyframe slots, bad flags, observations, descriptors and per-call fused counts."""
    K = kfs
    mt = matcher(pkg, K)
    pts = lambda E, sk, tab, d: run_points(mt, torch, K, tab, d, np.array(E, np.int32).reshape(-1, 2), sk)
    check_replay(replay_points(oracle, K, pts))
    lns = lambda E, sk, tab, d: run_lines(mt, torch, K, tab, d, np.array(E, np.int32).reshape(-1, 2), sk)
    check_replay(replay_lines(oracle, K, lns))
