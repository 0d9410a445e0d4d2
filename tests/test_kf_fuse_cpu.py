"""CPU: MapPoint / MapLine::PredictScale's threshold table against the host's own logf for every float, and the inputs of
tests/test_kf_fuse_gpu.py run on the oracle alone: every gate of the Fuse projection and search stages (ORBmatcher.cc:828-950,
LSDmatcher.cpp:417-523) and the TH_LOW test of the caller change some entry's result, and the SearchInNeighbors replay does Replace in
both directions and re-submits entries.  So the GPU comparisons are not vacuous."""
import os
import threading

import numpy as np
import pytest

import fuse_model as fm
from test_kf_triangulation_gpu import FLAT, NKF, keyframe_frames


def test_predict_scale_table_every_float(pkg, oracle):
    """Scale factor 1.2, 8 levels: for all 2^32 bit patterns the lookup over sslpl_predict_scale_table (count of thresholds <= ratio,
    INT_MIN for a ratio that is not finite and positive) equals the oracle's (int)ceil(logf(ratio) / logScaleFactor), mapped to
    [-1, nlevels] outside the pyramid, INT_MIN included."""
    thr = pkg.predict_scale_table(fm.LOGS, fm.NLEV)
    assert thr.dtype == np.float32 and (np.diff(thr) > 0).all() and thr[1] == np.nextafter(np.float32(1), np.float32(2))
    chunk, nchunks = 1 << 22, 1 << 10
    nthreads = max(1, min(16, os.cpu_count() or 1))
    bad, lock, it = [], threading.Lock(), iter(range(nchunks))

    def work():
        while True:
            with lock:
                c = next(it, None)
            if c is None:
                return
            r = (np.arange(chunk, dtype=np.uint64) + c * chunk).astype(np.uint32).view(np.float32)
            got = fm.table_levels(thr, r, clamp=False)
            want = fm.window_levels(fm.oracle_levels(oracle, r, fm.LOGS, fm.NLEV, chunk=chunk), fm.NLEV, clamp=False)
            if not np.array_equal(got, want):
                with lock:
                    bad.append((c, int((got != want).sum())))

    ts = [threading.Thread(target=work) for _ in range(nthreads)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not bad, bad[:5]


def test_predict_scale_table_arguments(pkg):
    for s, n in ((0.0, 8), (-0.18, 8), (float("inf"), 8), (float("nan"), 8), (0.18, 0), (0.18, 17)):
        with pytest.raises(pkg.SslplError):
            pkg.predict_scale_table(s, n)
    thr = pkg.predict_scale_table(np.log(np.float32(2.0)), 16)
    assert len(thr) == 17 and thr[0] == np.float32(0.5) * np.nextafter(np.float32(1), np.float32(2))


# ------------------------------------------------------------------------------------------------------------------ the keyframe set
def host_keyframes(oracle, frames, nfeatures=1000, nlines=40):
    """The keyframe set of the GPU test from the oracle's extractors (bit-identical to the device's, tests/test_orb_gpu.py,
    tests/test_line_gpu.py): dict(kps, desc, n, kl, ldesc, nl, pose, cam, bounds)."""
    B, H, W = frames.shape
    orc = oracle.OrbOracle(nfeatures, 1.2, 8, 20, 7); lo = oracle.LineOracle(nlines)
    ex = [orc.extract(f) for f in frames]; lx = [lo.extract(f) for f in frames]
    n = np.array([len(k) for k, _ in ex], np.int32); nl = np.array([len(l[1]) for l in lx], np.int32)
    cap, capl = max(int(n.max()), 1), max(int(nl.max()), 1)
    kps = np.zeros((B, cap), ex[0][0].dtype); desc = np.zeros((B, cap, 32), np.uint8)
    kl = np.zeros((B, capl), lx[0][0].dtype); ldesc = np.zeros((B, capl, 32), np.uint8)
    for f in range(B):
        kps[f, :n[f]] = ex[f][0]; desc[f, :n[f]] = ex[f][1]; kl[f, :nl[f]] = lx[f][0]; ldesc[f, :nl[f]] = lx[f][1]
    cam, bounds = fm.camera(W, H)
    return dict(kps=kps, desc=desc, n=n, kl=kl, ldesc=ldesc, nl=nl, pose=fm.poses(B, B, W, H), cam=cam, bounds=bounds, W=W, H=H)


def point_entries(rng, K, table_src, n0):
    """Phase A: KF 0's MapPoints (table rows 0 .. n0-1) into every other keyframe (FLAT among them); phase B: the other rows into KF 0."""
    A = [(k, e) for k in range(1, len(K["n"])) for e in range(n0)]
    B = [(0, e) for e in range(n0, len(table_src))]
    E = np.array(A + B, np.int32)
    return E, (rng.random(len(E)) < 0.03).astype(np.uint8)


@pytest.fixture(scope="module")
def kfs(oracle, synth):
    K = host_keyframes(oracle, keyframe_frames(synth))
    assert K["n"][FLAT] == 0 and K["nl"][FLAT] == 0 and (np.delete(K["n"], FLAT) > 500).all()
    return K


def _sources(rng, n, nkf, p_other):
    src = [(0, i) for i in range(int(n[0]))]
    for k in range(1, nkf):
        src += [(k, int(i)) for i in np.nonzero(rng.random(int(n[k])) < p_other)[0]]
    return src


def _changed(a, b):
    return int(((a[0] != b[0]) | (a[1] != b[1])).sum())


def test_every_point_gate_changes_some_entry(oracle, kfs):
    K = kfs
    rng = np.random.default_rng(3)
    src = _sources(rng, K["n"], NKF, 0.05)
    T = fm.point_table(rng, src, K["kps"], K["desc"], K["pose"], NKF, K["W"], K["H"])
    E, skip = point_entries(rng, K, src, int(K["n"][0]))
    base = fm.oracle_points(oracle, K, K["pose"], T["mp"], T["desc"], E, skip)[:2]
    fused = (base[1] <= fm.TH_LOW) & (base[0] >= 0)
    assert fused.sum() > 2000, fused.sum()
    assert _changed(base, fm.oracle_points(oracle, K, K["pose"], T["mp"], T["desc"], E, np.zeros_like(skip))[:2]) > 100      # skip
    for g, name in enumerate(fm.POINT_GATES):
        mp, d = T["mp"].copy(), T["desc"].copy()
        s = T["gate"] == g
        mp[s], d[s] = T["base"][s], T["base_desc"][s]
        assert s.sum() > 10 and _changed(base, fm.oracle_points(oracle, K, K["pose"], mp, d, E, skip)[:2]) > 10, name
    rows = T["gate"][E[:, 1]] == fm.POINT_GATES.index("desc")
    assert ((base[0] >= 0) & (base[1] > fm.TH_LOW) & rows).sum() > 10            # TH_LOW: a nearest candidate that is not fused


def test_every_line_gate_changes_some_entry(oracle, kfs):
    K = kfs
    rng = np.random.default_rng(4)
    src = [(k, i) for k in range(NKF) for i in range(int(K["nl"][k])) if k == 0 or rng.random() < 0.3]
    T = fm.line_table(rng, src, K["kl"], K["ldesc"], K["pose"], NKF, K["W"], K["H"], p_gate=0.06)
    n0 = int(K["nl"][0])
    E = np.array([(k, e) for k in range(1, NKF) for e in range(n0)] + [(0, e) for e in range(n0, len(src))], np.int32)
    skip = (rng.random(len(E)) < 0.03).astype(np.uint8)
    base = fm.oracle_lines(oracle, K, K["pose"], T["ml"], T["desc"], E, skip)[:2]
    assert ((base[1] <= fm.TH_LOW) & (base[0] >= 0)).sum() > 150
    assert _changed(base, fm.oracle_lines(oracle, K, K["pose"], T["ml"], T["desc"], E, np.zeros_like(skip))[:2]) > 5
    for g, name in enumerate(fm.LINE_GATES):
        ml, d = T["ml"].copy(), T["desc"].copy()
        s = T["gate"] == g
        ml[s], d[s] = T["base"][s], T["base_desc"][s]
        assert s.sum() > 0 and _changed(base, fm.oracle_lines(oracle, K, K["pose"], ml, d, E, skip)[:2]) > 0, name
    # the out-of-pyramid rows reach PredictScale with level nlevels (MapLine::PredictScale is not clamped) and are dropped
    pyr = np.nonzero(T["gate"] == fm.LINE_GATES.index("pyramid"))[0]
    q = oracle.fuse_project_lines(np.zeros(len(pyr), np.uint8), T["ml"][pyr, :6], T["ml"][pyr, 6:9], T["ml"][pyr, 9], T["ml"][pyr, 10], T["ml"][pyr, 11],
                                  K["pose"][0, :12].reshape(3, 4), K["pose"][0, 12:], np.append(K["cam"], 0.0), K["bounds"], fm.NLEV, fm.LOGS)
    assert (q["level"] >= fm.NLEV).any() and not q["active"][q["level"] >= fm.NLEV].any()


# ------------------------------------------------------------------------------------------------------------------ replay
REPLAY_CUR, REPLAY_TARGETS = 0, [1, 2, 3, 4, 5, 6, FLAT]


def replay_points(oracle, K, batch, seed=11):
    """SearchInNeighbors' point phases run twice on one map: sequentially on the oracle and with batch(entries, skip, table, desc).
    Returns (sequential (state, counts), batched (state, counts, stats), both maps)."""
    kf = [REPLAY_CUR] + REPLAY_TARGETS
    out = []
    for mode in ("seq", "batch"):
        rng = np.random.default_rng(seed)
        M, src = fm.replay_map(rng, [K["desc"][k] for k in range(len(K["n"]))], K["n"], kf)
        T = fm.point_table(rng, src, K["kps"], K["desc"], K["pose"], len(K["n"]), K["W"], K["H"], p_gate=0.02)
        if mode == "seq":
            one = lambda k, e, M: tuple(int(v[0]) for v in fm.oracle_points(oracle, K, K["pose"], T["mp"], np.array(M.desc), [(k, e)], [0])[:2])
            counts = fm.search_in_neighbors(M, REPLAY_CUR, REPLAY_TARGETS, fm.run_sequential(one), points=True)
            out.append((M.state(), counts, None, M))
        else:
            stats = dict(calls=0, resubmitted=0)
            run = fm.run_batched(lambda E, sk, M: batch(E, sk, T["mp"], np.array(M.desc)), stats)
            counts = fm.search_in_neighbors(M, REPLAY_CUR, REPLAY_TARGETS, run, points=True)
            out.append((M.state(), counts, stats, M))
    return out


def replay_lines(oracle, K, batch, seed=12):
    kf = [REPLAY_CUR] + REPLAY_TARGETS
    out = []
    for mode in ("seq", "batch"):
        rng = np.random.default_rng(seed)
        M, src = fm.replay_map(rng, [K["ldesc"][k] for k in range(len(K["nl"]))], K["nl"], kf, p_own=0.8)
        T = fm.line_table(rng, src, K["kl"], K["ldesc"], K["pose"], len(K["nl"]), K["W"], K["H"], p_gate=0.02)
        if mode == "seq":
            one = lambda k, e, M: tuple(int(v[0]) for v in fm.oracle_lines(oracle, K, K["pose"], T["ml"], np.array(M.desc), [(k, e)], [0])[:2])
            counts = fm.search_in_neighbors(M, REPLAY_CUR, REPLAY_TARGETS, fm.run_sequential(one), points=False)
            out.append((M.state(), counts, None, M))
        else:
            stats = dict(calls=0, resubmitted=0)
            run = fm.run_batched(lambda E, sk, M: batch(E, sk, T["ml"], np.array(M.desc)), stats)
            counts = fm.search_in_neighbors(M, REPLAY_CUR, REPLAY_TARGETS, run, points=False)
            out.append((M.state(), counts, stats, M))
    return out


def check_replay(out, min_resubmitted=1):
    (s_seq, c_seq, _, M_seq), (s_bat, c_bat, stats, M_bat) = out
    assert c_seq == c_bat, (c_seq, c_bat)
    assert s_seq == s_bat
    assert stats["calls"] == 2 and stats["resubmitted"] >= min_resubmitted, stats
    assert M_seq.replaced["into_existing"] > 0 and M_seq.replaced["into_incoming"] > 0, M_seq.replaced
    assert sum(c_seq) > 0


def test_replay_is_exercised_on_the_oracle(oracle, kfs):
    """The batched driver with the oracle standing in for the device: the re-test / re-submit rule reproduces the sequential run, and
    the scenario does Replace in both directions and re-submits entries (points and lines)."""
    K = kfs
    pts = lambda E, sk, tab, d: fm.oracle_points(oracle, K, K["pose"], tab, d, E, sk)[:2]
    check_replay(replay_points(oracle, K, pts))
    lns = lambda E, sk, tab, d: fm.oracle_lines(oracle, K, K["pose"], tab, d, E, sk)[:2]
    check_replay(replay_lines(oracle, K, lns))
