"""Time the end of LocalMapping::SearchInNeighbors for one keyframe (LocalMapping.cc:1266-1276): ComputeDistinctiveDescriptors and
UpdateNormalAndDepth of every MapPoint of the keyframe, ComputeDistinctiveDescriptors and UpdateAverageDir of every MapLine.  Keyframes
are extracted once on the device (21 synthetic frames of one scene, poses from tests/fuse_model.py); every feature and line of keyframe 0
is an element, observed by keyframe 0 and a random half of the other 20 (the reference keyframe is keyframe 0).

Forms, alternated in the same run after a warm-up, each timed on the host clock around work that ends in a device synchronise:
  (a) batched: one sslpl_update_map_points_batch_device and one sslpl_update_map_lines_batch_device call on data in HBM;
  (b) host: download the element rows, take the medoids with the oracle's C++ (orc_descriptor_medoid, one call per kind over all
      elements), the geometry with tests/map_update_model.py (NumPy, one element at a time), and upload the rows again.
Both must give identical rows.  Sizes: 640x480 / 1000 features / 40 lines and 1280x960 / 4000 features / 500 lines.  Prints one JSON
line with the card's name and power limit read in the same run.  Needs a GPU; writes nothing.

    python tools/map_update_timing.py [--reps 5]
"""
import argparse
import importlib
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
    import map_update_model as mu
    from test_kf_fuse_gpu import device_keyframes, matcher
    from test_kf_triangulation_gpu import NKF, keyframe_frames
    mapping = importlib.import_module(pkg.__name__ + ".mapping")
    K = device_keyframes(pkg, torch, keyframe_frames(synth, W, H, NKF, None), nfeat, nlines)
    rng = np.random.default_rng(1)

    def entries(n):
        return [(e, 0, [(0, e)] + [(k, int(rng.integers(0, n[k]))) for k in range(1, NKF) if rng.random() < 0.5]) for e in range(int(n[0]))]

    Ep, El = entries(K["n"]), entries(K["nl"])
    P = fm.point_table(rng, [(0, e) for e, _, _ in Ep], K["kps"], K["desc"], K["pose"], NKF, W, H)
    L = fm.line_table(rng, [(0, e) for e, _, _ in El], K["kl"], K["ldesc"], K["pose"], NKF, W, H)
    pos = L["ml"][:, :6].astype(np.float64)
    mt = matcher(pkg, K)
    dev = lambda a, t: torch.from_numpy(np.ascontiguousarray(a, t)).cuda()
    d_mp, d_md, d_ml, d_ld, d_pos = dev(P["mp"], np.float32), dev(P["desc"], np.uint8), dev(L["ml"], np.float32), dev(L["desc"], np.uint8), dev(pos, np.float64)
    cp, cl = [dev(a, np.int32) for a in mu.csr(Ep)], [dev(a, np.int32) for a in mu.csr(El)]
    sp, sl = torch.empty(len(Ep), dtype=torch.int32, device="cuda"), torch.empty(len(El), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()

    def batched():
        t0 = time.perf_counter()
        mapping.update_map_points(mt, K["d_kps"], K["d_desc"], K["d_n"], NKF, K["cap"], K["d_pose"].data_ptr(), 0, len(Ep), d_mp.data_ptr(),
                                  d_md.data_ptr(), len(Ep), *(a.data_ptr() for a in cp), fm.SF, 3, sp.data_ptr())
        mapping.update_map_lines(mt, K["d_kl"], K["d_ldesc"], K["d_nl"], NKF, K["capl"], K["d_pose"].data_ptr(), 0, len(El), d_pos.data_ptr(),
                                 d_ml.data_ptr(), d_ld.data_ptr(), 0, len(El), *(a.data_ptr() for a in cl), fm.SF, 3, sl.data_ptr())
        mt.sync()
        return (time.perf_counter() - t0) * 1e3

    def host_kind(E, d_tab, d_desc, desc, lines):
        tab = d_tab.cpu().numpy()
        groups = [np.array([desc[k, i] for k, i in obs], np.uint8) for _, _, obs in E]
        off = np.concatenate([[0], np.cumsum([len(g) for g in groups])]).astype(np.int32)
        bi, _ = oracle.descriptor_medoid(np.concatenate(groups), off)
        tdesc = np.stack([g[b] for g, b in zip(groups, bi)])
        if lines:
            tab = mu.update_lines(K["kl"], K["ldesc"], K["nl"], K["pose"], None, pos, tab, tdesc, None, E, fm.SF, mu.GEOM)[0]
        else:
            tab = mu.update_points(K["kps"], K["desc"], K["n"], K["pose"], None, tab, tdesc, E, fm.SF, mu.GEOM)[0]
        d_tab.copy_(torch.from_numpy(tab)); d_desc.copy_(torch.from_numpy(tdesc))

    h_mp, h_md, h_ml, h_ld = (dev(a, t) for a, t in ((P["mp"], np.float32), (P["desc"], np.uint8), (L["ml"], np.float32), (L["desc"], np.uint8)))

    def host():
        t0 = time.perf_counter()
        host_kind(Ep, h_mp, h_md, K["desc"], False)
        host_kind(El, h_ml, h_ld, K["ldesc"], True)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    batched(); host()                                                   # warm-up, and the equality check
    same = all(torch.equal(a, b) for a, b in ((d_mp, h_mp), (d_md, h_md), (d_ml, h_ml), (d_ld, h_ld)))
    ok = bool((sp == 0).all() and (sl == 0).all())
    t = {"batched": [], "host": []}
    for _ in range(reps):
        t["batched"].append(batched())
        t["host"].append(host())
    return {"width": W, "height": H, "features": nfeat, "lines": nlines, "points": len(Ep), "mapl": len(El),
            "observations": [int(cp[2][-1]), int(cl[2][-1])], "ms": {k: _stats(v) for k, v in t.items()}, "identical": bool(same), "all_ok": ok}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--reps", type=int, default=5, help="alternated samples of each form")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("map_update_timing: no CUDA device (this measures the H100 path; there is nothing to time on the CPU)")
    import __graft_entry__ as g
    pkg = g.load_package(); oracle = g.load_oracle()
    card = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        power = "unknown"
    res = [run_config(pkg, oracle, torch, 640, 480, 1000, 40, args.reps), run_config(pkg, oracle, torch, 1280, 960, 4000, 500, args.reps)]
    print(json.dumps({"tool": "map_update_timing", "card": card, "power_limit": power, "reps": args.reps, "configs": res}))


if __name__ == "__main__":
    main()
