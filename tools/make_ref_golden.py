#!/usr/bin/env python3
"""Freeze outputs of THE REFERENCE ITSELF (oracle/_ref/libref.so = the reference's sources compiled unmodified, see
oracle/ref_build.sh) into small fixtures under tests/golden/ref_*.npz, so that machines without the reference's sources
can still hold the oracle and the CUDA path against the reference.  Run where oracle/ref_build.sh can build the reference:

    python tools/make_ref_golden.py

Inputs are the committed ICL frame and the deterministic synthetic frames of tools/synth.py; every array the tests need
to rebuild the call is stored next to the reference's output.  tests/golden/ref_parity.npz holds the reference's answers to
every call of tests/test_ref_parity_cpu.py (tests/ref_replay.py), recorded by running that module."""
import os
import sys
import hashlib
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tools")); sys.path.insert(0, os.path.join(ROOT, "tests"))
import cv2
import synth
from oracle import oracle as O, ref as R
from scenarios import projection_scenario, line_scenario, local_lines_scenario, fuse_points_scenario, fuse_lines_scenario

G = os.path.join(ROOT, "tests", "golden")


def main():
    icl = cv2.imread(os.path.join(G, "icl_office_gray.png"), 0)
    out = {}
    # ---- ORBextractor::operator() on the ICL frame (1000 and 2000 features) and on synthetic frames
    for tag, img, nf in [("icl1000", icl, 1000), ("icl2000", icl, 2000), ("syn0", synth.frame(640, 480, 0), 1000), ("syn13", synth.frame(640, 480, 13), 1000)]:
        k, d, lc = R.orb_extract(img, nf)
        out[f"orb_{tag}_kps"] = k; out[f"orb_{tag}_desc"] = d; out[f"orb_{tag}_levels"] = lc
    np.savez_compressed(os.path.join(G, "ref_orb.npz"), **out)

    # ---- matchers on the synthetic pair (0, 1) and on ICL + 2-px shift
    m = {}
    orc = O.OrbOracle(1000, 1.2, 8, 20, 7)
    k1, d1 = orc.extract(synth.frame(640, 480, 0)); k2, d2 = orc.extract(synth.frame(640, 480, 1))
    voc = synth.vocabulary(100)
    fv1 = O.feature_vector_csr(O.bow_assign(d1, voc)); fv2 = O.feature_vector_csr(O.bow_assign(d2, voc))
    rng = np.random.default_rng(99)
    valid1 = (rng.random(len(d1)) < 0.7).astype(np.uint8); valid2 = (rng.random(len(d2)) < 0.8).astype(np.uint8)
    m["valid1"] = valid1; m["valid2"] = valid2
    for ratio, ori in [(0.7, True), (0.9, False)]:
        n, mm = R.search_by_bow(d1, k1, d2, k2, fv1, fv2, valid1, ratio, ori)
        m[f"bow_{ratio}_{int(ori)}"] = mm; m[f"bow_{ratio}_{int(ori)}_n"] = np.int32(n)
        n, mm = R.search_by_bow_kf(d1, k1, d2, k2, fv1, fv2, valid1, valid2, ratio, ori)
        m[f"bowkf_{ratio}_{int(ori)}"] = mm; m[f"bowkf_{ratio}_{int(ori)}_n"] = np.int32(n)
    # triangulation: fixed poses
    T1 = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)
    a = 0.03; R2 = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    for tag, t2 in [("in", np.array([0.02, 0.01, -0.5])), ("out", np.array([-0.4, 0.05, 0.02]))]:
        T2 = np.hstack([R2, t2[:, None]]).astype(np.float32)
        K = np.array([[500, 0, 320], [0, 500, 240], [0, 0, 1.0]])
        R12 = R2.T; t12 = -R2.T @ t2
        tx = np.array([[0, -t12[2], t12[1]], [t12[2], 0, -t12[0]], [-t12[1], t12[0], 0]])
        F12 = (np.linalg.inv(K).T @ tx @ R12 @ np.linalg.inv(K)).astype(np.float32)
        has1 = 1 - valid1; has2 = 1 - valid2
        n, pairs, (ex, ey) = R.search_for_triangulation(d1, k1, d2, k2, fv1, fv2, has1, has2, R.CAM640, T1, T2, F12, True)
        m[f"tri_{tag}_pairs"] = pairs; m[f"tri_{tag}_F12"] = F12; m[f"tri_{tag}_epi"] = np.array([ex, ey], np.float32)
    # lines: knn-based matchers on LBD descriptors of the two frames
    lo = O.LineOracle(40)
    _, l1, _ = lo.extract(synth.frame(640, 480, 0)); _, l2, _ = lo.extract(synth.frame(640, 480, 1))
    h1 = (rng.random(len(l1)) < 0.6).astype(np.uint8); h2 = (rng.random(len(l2)) < 0.6).astype(np.uint8)
    m["line_h1"] = h1; m["line_h2"] = h2; m["line_d1"] = l1; m["line_d2"] = l2
    for mode in range(4):
        n, mm, mad = R.line_match(mode, l1, l2, h1, h2)
        m[f"line_mode{mode}"] = mm; m[f"line_mode{mode}_n"] = np.int32(n); m["line_mad"] = np.array(mad)
    # projection matcher (TrackWithMotionModel), mono and stereo
    for seed, th, mono in [(1, 15.0, True), (4, 15.0, False)]:
        last, cur, Tcw, Tlw, cam, bounds, sf = projection_scenario(O, synth, seed, n_claimed=0.05, stereo=not mono, f0=seed)
        camv = R.cam(cam[0], cam[1], cam[2], cam[3], *bounds)
        n, a2 = R.search_by_projection_frame(last, cur, Tcw, Tlw, camv, 8, 1.2, th, mono, True, mbf=cam[4])
        m[f"proj_{seed}"] = np.where(a2 == -2, -1, a2); m[f"proj_{seed}_n"] = np.int32(n)
    np.savez_compressed(os.path.join(G, "ref_match.npz"), **m)

    # ---- Frame::Frame on the ICL frame: lines (40), grid
    fr = R.frame_from_image(icl)
    np.savez_compressed(os.path.join(G, "ref_frame.npz"), keylines=fr["keylines"], ldesc=fr["ldesc"], lineeq=fr["lineeq"],
                        grid_off=fr["grid_off"], grid_idx=fr["grid_idx"])
    row3()
    import subprocess
    subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.join(ROOT, "tests", "test_ref_parity_cpu.py")],
                   check=True, cwd=ROOT, env=dict(os.environ, SSLPL_REF_RECORD="1"))
    for f in ("ref_orb.npz", "ref_match.npz", "ref_frame.npz", "ref_row3.npz", "ref_parity.npz"):
        p = os.path.join(G, f)
        print(f, os.path.getsize(p), hashlib.sha1(open(p, "rb").read()).hexdigest()[:12])


def row3():
    """SURVEY.md 8(f) row 3: the reference's line projection matchers and Fuse on the deterministic scenarios of tests/scenarios.py"""
    r = {}
    sc = line_scenario(O, synth, 2, f0=2, stereo_sign=1)
    cam = R.cam(*sc["cam5"][:4], *sc["bounds"])
    n, a = R.line_projection_frame(sc["last"], sc["cur"], sc["Tcw"], sc["Tlw"], cam, sc["cam5"][4], 8, 1.2, 0.8, 20.0, False)
    r["lpf_n"] = np.int32(n); r["lpf_assign"] = np.where(a == -2, -1, a)
    ml, cur, sf = local_lines_scenario(O, synth, 2, f0=2)
    n, a = R.line_projection_mls(ml, cur, R.cam(500, 500, 320, 240, 0, 640, 0, 480), 8, 1.2, 0.8, 3.0)
    r["lpm_n"] = np.int32(n); r["lpm_assign"] = np.where(a == -2, -1, a)
    for tag, stereo in (("mono", False), ("stereo", True)):
        sc = fuse_points_scenario(O, synth, 2, f0=2, stereo=stereo)
        n, f, acc = R.fuse_points(sc["mp"], sc["kf"], sc["Tcw"], R.cam(*sc["cam5"][:4], *sc["bounds"]), sc["cam5"][4], 8, 1.2, 3.0)
        r[f"fp_{tag}_n"] = np.int32(n); r[f"fp_{tag}_idx"] = f
        r[f"fp_{tag}_Ow"] = acc["Ow"]; r[f"fp_{tag}_min_inv"] = acc["min_inv"]; r[f"fp_{tag}_max_inv"] = acc["max_inv"]; r[f"fp_{tag}_log_scale"] = np.float32(acc["log_scale"])
    sc = fuse_lines_scenario(O, synth, 2, f0=2)
    ml = dict(sc["ml"])
    q0 = O.fuse_project_lines(ml["state"] != 1, ml["Pw"], ml["normal"], ml["min_raw"] * np.float32(0.8), ml["max_raw"] * np.float32(1.2), ml["max_raw"],
                              sc["Tcw"][:3], np.zeros(3), sc["cam5"], sc["bounds"], 8, np.log(np.float32(1.2)))
    ml["state"] = np.where((q0["level"] < 0) | (q0["level"] >= 8), 0, ml["state"]).astype(np.uint8)      # keep to levels inside the pyramid (see the test)
    n, f, acc = R.fuse_lines(ml, sc["kf"], sc["Tcw"], R.cam(*sc["cam5"][:4], *sc["bounds"]), 8, 1.2, 10.0)
    r["fl_state"] = ml["state"]; r["fl_n"] = np.int32(n); r["fl_idx"] = f
    r["fl_Ow"] = acc["Ow"]; r["fl_min_inv"] = acc["min_inv"]; r["fl_max_inv"] = acc["max_inv"]; r["fl_log_scale"] = np.float32(acc["log_scale"])
    np.savez_compressed(os.path.join(G, "ref_row3.npz"), **r)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "row3":
        row3()
    else:
        main()
