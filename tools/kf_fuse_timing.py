"""Time LocalMapping::SearchInNeighbors' Fuse work for one new keyframe (LocalMapping.cc:1178-1279, monocular): ORBmatcher::Fuse and
LSDmatcher::Fuse of the keyframe's elements into 20 neighbours (phase A), then of the neighbours' candidates into the keyframe (phase B).
Keyframes are extracted once on the device (21 synthetic frames of one scene); poses, MapPoints and MapLines come from
tests/fuse_model.py (about 1000 / 4000 MapPoints of the keyframe, 30 % of every neighbour's features as candidates, all lines).

Forms, alternated in the same run after a warm-up, each timed on the host clock around work that ends in a device synchronise:
  (a) batched: one sslpl_fuse_points_batch_device + one sslpl_fuse_lines_batch_device call per phase on data in HBM;
  (b) per target: the host projection stage (the oracle's restatement) and the single search calls sslpl_fuse_points_search /
      sslpl_fuse_lines_search per target keyframe, each of which uploads its inputs and synchronises;
  (c) cpu: the oracle's projection and search stages.
All three must give identical entries.  Sizes: 640x480 / 1000 features / 40 lines and 1280x960 / 4000 features / 500 lines.
Prints one JSON line with the card's name and power limit read in the same run.  Needs a GPU; writes nothing.

    python tools/kf_fuse_timing.py [--reps 10]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]


def _stats(xs):
    xs = sorted(xs)
    return {"median": round(float(np.median(xs)), 3), "min": round(xs[0], 3), "max": round(xs[-1], 3), "n": len(xs)}


def run_config(pkg, oracle, torch, W, H, nfeat, nlines, reps):
    import synth
    import fuse_model as fm
    from test_kf_fuse_gpu import device_keyframes, matcher
    from test_kf_triangulation_gpu import NKF, keyframe_frames
    K = device_keyframes(pkg, torch, keyframe_frames(synth, W, H, NKF, None), nfeat, nlines)
    rng = np.random.default_rng(1)
    n0, l0 = int(K["n"][0]), int(K["nl"][0])
    src = [(0, i) for i in range(n0)] + [(k, int(i)) for k in range(1, NKF) for i in np.nonzero(rng.random(int(K["n"][k])) < 0.3)[0]]
    lsrc = [(k, i) for k in range(NKF) for i in range(int(K["nl"][k]))]
    P = fm.point_table(rng, src, K["kps"], K["desc"], K["pose"], NKF, W, H)
    L = fm.line_table(rng, lsrc, K["kl"], K["ldesc"], K["pose"], NKF, W, H)
    phases_p = [np.array([(k, e) for k in range(1, NKF) for e in range(n0)], np.int32), np.array([(0, e) for e in range(n0, len(src))], np.int32)]
    phases_l = [np.array([(k, e) for k in range(1, NKF) for e in range(l0)], np.int32), np.array([(0, e) for e in range(l0, len(lsrc))], np.int32)]
    mt = matcher(pkg, K)
    dev = lambda a, t: torch.from_numpy(np.ascontiguousarray(a, t)).cuda()
    d_mp, d_md, d_ml, d_ld = dev(P["mp"], np.float32), dev(P["desc"], np.uint8), dev(L["ml"], np.float32), dev(L["desc"], np.uint8)
    d_ep = [dev(E, np.int32) for E in phases_p]; d_el = [dev(E, np.int32) for E in phases_l]
    o_p = [(torch.empty(len(E), dtype=torch.int32, device="cuda"), torch.empty(len(E), dtype=torch.int32, device="cuda")) for E in phases_p]
    o_l = [(torch.empty(len(E), dtype=torch.int32, device="cuda"), torch.empty(len(E), dtype=torch.int32, device="cuda")) for E in phases_l]
    torch.cuda.synchronize()

    def batched():
        t0 = time.perf_counter()
        for j in range(2):
            mt.fuse_points_batch_device(K["d_kps"], K["d_desc"], K["d_n"], NKF, K["cap"], K["d_pose"].data_ptr(), len(P["mp"]), d_mp.data_ptr(),
                                        d_md.data_ptr(), len(phases_p[j]), d_ep[j].data_ptr(), 0, K["cam"], K["bounds"], fm.SF, fm.INV_SIGMA2,
                                        fm.LOGS, fm.TH, o_p[j][0].data_ptr(), o_p[j][1].data_ptr())
            mt.fuse_lines_batch_device(K["d_kl"], K["d_ldesc"], K["d_nl"], NKF, K["capl"], K["d_pose"].data_ptr(), len(L["ml"]), d_ml.data_ptr(),
                                       d_ld.data_ptr(), len(phases_l[j]), d_el[j].data_ptr(), 0, K["cam"], K["bounds"], fm.SF, fm.LOGS, fm.TH,
                                       o_l[j][0].data_ptr(), o_l[j][1].data_ptr())
        mt.sync()
        return (time.perf_counter() - t0) * 1e3

    def per_target():
        out = []
        t0 = time.perf_counter()
        for Ep, El in zip(phases_p, phases_l):
            bi, bd = np.empty(len(Ep), np.int32), np.empty(len(Ep), np.int32)
            for k in np.unique(Ep[:, 0]):
                sel = Ep[:, 0] == k; e = Ep[sel, 1]; T = K["pose"][k]; n = int(K["n"][k]); kp = K["kps"][k, :n]; mp = P["mp"][e]
                q = oracle.fuse_project_points(np.zeros(len(e), np.uint8), mp[:, :3], mp[:, 3:6], mp[:, 6], mp[:, 7], mp[:, 8], T[:12].reshape(3, 4), T[12:],
                                               np.append(K["cam"], 0.0), K["bounds"], fm.NLEV, fm.LOGS)
                bi[sel], bd[sel] = mt.fuse_points_search(q, P["desc"][e], K["desc"][k, :n], kp["x"], kp["y"], kp["octave"].astype(np.int32), None,
                                                         K["bounds"], fm.SF, fm.INV_SIGMA2, fm.TH)
            lbi, lbd = np.empty(len(El), np.int32), np.empty(len(El), np.int32)
            for k in np.unique(El[:, 0]):
                sel = El[:, 0] == k; e = El[sel, 1]; T = K["pose"][k]; n = int(K["nl"][k]); kl = K["kl"][k, :n]; ml = L["ml"][e]
                q = oracle.fuse_project_lines(np.zeros(len(e), np.uint8), ml[:, :6], ml[:, 6:9], ml[:, 9], ml[:, 10], ml[:, 11], T[:12].reshape(3, 4), T[12:],
                                              np.append(K["cam"], 0.0), K["bounds"], fm.NLEV, fm.LOGS)
                lbi[sel], lbd[sel] = mt.fuse_lines_search(q, L["desc"][e], K["ldesc"][k, :n], fm.keyline_rows(kl), kl["octave"].astype(np.int32), fm.SF, fm.TH)
            out.append((bi, bd, lbi, lbd))
        return (time.perf_counter() - t0) * 1e3, out

    def cpu():
        out = []
        t0 = time.perf_counter()
        for Ep, El in zip(phases_p, phases_l):
            bi, bd, _ = fm.oracle_points(oracle, K, K["pose"], P["mp"], P["desc"], Ep, np.zeros(len(Ep), np.uint8))
            lbi, lbd, _ = fm.oracle_lines(oracle, K, K["pose"], L["ml"], L["desc"], El, np.zeros(len(El), np.uint8))
            out.append((bi, bd, lbi, lbd))
        return (time.perf_counter() - t0) * 1e3, out

    batched(); _, want = per_target(); _, want_cpu = cpu()               # warm-up, and the equality check
    got = [(o_p[j][0].cpu().numpy(), o_p[j][1].cpu().numpy(), o_l[j][0].cpu().numpy(), o_l[j][1].cpu().numpy()) for j in range(2)]
    same = all(np.array_equal(a, b) and np.array_equal(a, c) for g, w, wc in zip(got, want, want_cpu) for a, b, c in zip(g, w, wc))
    fused = sum(int(((g[1] <= fm.TH_LOW) & (g[0] >= 0)).sum()) for g in got)
    t = {"batched": [], "per_target": [], "cpu": []}
    for _ in range(reps):
        t["batched"].append(batched())
        t["per_target"].append(per_target()[0])
        t["cpu"].append(cpu()[0])
    return {"width": W, "height": H, "features": nfeat, "lines": nlines, "targets": NKF - 1,
            "point_entries": [len(E) for E in phases_p], "line_entries": [len(E) for E in phases_l], "point_fusions": fused,
            "ms": {k: _stats(v) for k, v in t.items()}, "identical": bool(same)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--reps", type=int, default=10, help="alternated samples of each form")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("kf_fuse_timing: no CUDA device (this measures the H100 path; there is nothing to time on the CPU)")
    import __graft_entry__ as g
    pkg = g.load_package(); oracle = g.load_oracle()
    card = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        power = "unknown"
    res = [run_config(pkg, oracle, torch, 640, 480, 1000, 40, args.reps), run_config(pkg, oracle, torch, 1280, 960, 4000, 500, args.reps)]
    print(json.dumps({"tool": "kf_fuse_timing", "card": card, "power_limit": power, "reps": args.reps, "configs": res}))


if __name__ == "__main__":
    main()
