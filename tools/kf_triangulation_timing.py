"""Time LocalMapping's triangulation matching for one new keyframe: ORBmatcher::SearchForTriangulation against 20 covisible neighbours
(LocalMapping::CreateNewMapPoints, LocalMapping.cc:371-440, monocular nn = 20) and LSDmatcher::SearchForTriangulation against 10
(CreateNewMapLines2, :911-988).  Keyframes are extracted once on the device (21 synthetic frames of one scene); F12 / epipoles, MapPoint
and MapLine masks and the vocabulary tree come from the builder of tests/test_kf_triangulation_gpu.py.

Forms, alternated in the same run after a warm-up, each timed on the host clock around work that ends in a device synchronise:
  (a) batched: sslpl_search_for_triangulation_batch_device + sslpl_line_search_for_triangulation_batch_device on data in HBM;
  (b) loop: the 20 + 10 single-pair calls LocalMapping makes today (sslpl_search_for_triangulation / sslpl_line_match mode 3 from host
      buffers, each of which synchronises), with the keyframes' FeatureVectors already on the host as KeyFrame::mFeatVec is.
(a) and (b) must give identical pairs.  Sizes: 640x480 / 1000 features / 40 lines and 1280x960 / 4000 features / 500 lines.
Prints one JSON line with the card's name and power limit read in the same run.  Needs a GPU; writes nothing.

    python tools/kf_triangulation_timing.py [--reps 20]
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
    return {"median": round(float(np.median(xs)), 4), "min": round(xs[0], 4), "max": round(xs[-1], 4), "n": len(xs)}


def run_config(pkg, torch, W, H, nfeat, nlines, reps):
    import synth
    from test_kf_triangulation_gpu import (FLAT, LEVELSUP, NKF, NLN, NPT, VOCAB, device_lines, keyframe_frames, masks, pair_geometry,
                                           vocabulary_arrays)
    from test_motion_batch_gpu import device_batch
    frames = keyframe_frames(synth, W, H, NKF, None)
    D = device_batch(pkg, torch, frames, nfeat)
    L = device_lines(pkg, torch, D["dfr"], NKF, W, H, nlines)
    cap, capl = D["cap"], L["capl"]
    tb = D["ext"]._tables()
    scale, sigma2 = tb["scale"], tb["sigma2"]
    has_mp, has_ml = masks(np.random.default_rng(7), NKF, cap, capl)
    va = vocabulary_arrays(pkg)
    voc = pkg.Vocabulary(VOCAB["k"], VOCAB["L"], *va)
    mt = pkg.Matcher(max_features=cap, max_lines=capl, max_nodes=voc.level_nodes(LEVELSUP), max_batch=NPT)
    fv = []
    for f in range(NKF):                                                  # KeyFrame::mFeatVec, on the host for the loop form
        _, node, wt = mt.bow_transform(voc, D["desc"][f, :D["n"][f]], LEVELSUP)
        fv.append(pkg.Vocabulary.feature_vector(node, wt))
    pts = [(0, k) for k in range(1, NPT + 1)]
    lns = [(0, k) for k in range(1, NLN + 1)]
    geom = pair_geometry(np.random.default_rng(NPT), pts, D["kps"], D["n"], NKF, W, H)
    d_pair = torch.tensor(np.array(pts, np.int32), device="cuda"); d_lpair = torch.tensor(np.array(lns, np.int32), device="cuda")
    d_geom = torch.from_numpy(geom).cuda(); d_has_mp = torch.from_numpy(has_mp).cuda(); d_has_ml = torch.from_numpy(has_ml).cuda()
    d_pairs = torch.empty((NPT, cap, 2), dtype=torch.int32, device="cuda"); d_nm = torch.empty((NPT,), dtype=torch.int32, device="cuda")
    d_lp = torch.empty((NLN, capl, 2), dtype=torch.int32, device="cuda"); d_lnm = torch.empty((NLN,), dtype=torch.int32, device="cuda")
    om = pkg.ORBmatcher(0.6, True, mt); lm = pkg.LSDmatcher(mt)

    def batched():
        t0 = time.perf_counter()
        mt.search_for_triangulation_batch_device(D["d_kps"], D["d_desc"], D["d_n"], NKF, cap, d_has_mp.data_ptr(), voc, LEVELSUP, NPT,
                                                 d_pair.data_ptr(), d_geom.data_ptr(), scale, sigma2, True, d_pairs.data_ptr(), d_nm.data_ptr())
        mt.line_search_for_triangulation_batch_device(L["d_ldesc"], L["d_nl"], NKF, capl, d_has_ml.data_ptr(), NLN, d_lpair.data_ptr(),
                                                      d_lp.data_ptr(), d_lnm.data_ptr())
        mt.sync()
        return (time.perf_counter() - t0) * 1e3

    def loop():
        out_p, out_l = [], []
        t0 = time.perf_counter()
        for p, (i, j) in enumerate(pts):
            n1, n2 = int(D["n"][i]), int(D["n"][j])
            out_p.append(om.SearchForTriangulation(D["desc"][i, :n1], fv[i], has_mp[i, :n1], D["kps"][i, :n1], D["desc"][j, :n2], fv[j],
                                                   has_mp[j, :n2], D["kps"][j, :n2], geom[p, :9], float(geom[p, 9]), float(geom[p, 10]),
                                                   scale, sigma2))
        for i, j in lns:
            m1, m2 = int(L["nl"][i]), int(L["nl"][j])
            out_l.append(lm.SearchForTriangulation(L["ldesc"][i, :m1], has_ml[i, :m1], L["ldesc"][j, :m2], has_ml[j, :m2]))
        return (time.perf_counter() - t0) * 1e3, out_p, out_l

    batched(); _, out_p, out_l = loop()                                   # warm-up, and the equality check
    rows, nm, lrows, lnm = d_pairs.cpu().numpy(), d_nm.cpu().numpy(), d_lp.cpu().numpy(), d_lnm.cpu().numpy()
    same = all(nm[p] == n and np.array_equal(rows[p, :n], e) and (rows[p, n:] == -1).all() for p, (n, e) in enumerate(out_p)) and \
        all(lnm[p] == n and np.array_equal(lrows[p, :n], e) and (lrows[p, n:] == -1).all() for p, (n, e) in enumerate(out_l))
    t = {"batched": [], "loop": []}
    for _ in range(reps):
        t["batched"].append(batched())
        t["loop"].append(loop()[0])
    return {"width": W, "height": H, "features": nfeat, "lines": nlines, "cap": cap, "capl": capl,
            "point_pairs": NPT, "line_pairs": NLN, "point_matches_mean": round(float(nm.mean()), 1), "line_matches_mean": round(float(lnm.mean()), 1),
            "ms": {k: _stats(v) for k, v in t.items()}, "identical_batched_vs_loop": bool(same)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--reps", type=int, default=20, help="alternated samples of each form")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("kf_triangulation_timing: no CUDA device (this measures the H100 path; there is nothing to time on the CPU)")
    import __graft_entry__ as g
    pkg = g.load_package()
    card = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        power = "unknown"
    res = [run_config(pkg, torch, 640, 480, 1000, 40, args.reps), run_config(pkg, torch, 1280, 960, 4000, 500, args.reps)]
    print(json.dumps({"tool": "kf_triangulation_timing", "card": card, "power_limit": power, "reps": args.reps, "configs": res}))


if __name__ == "__main__":
    main()
