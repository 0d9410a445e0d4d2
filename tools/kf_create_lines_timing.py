#!/usr/bin/env python3
"""Time LocalMapping::CreateNewMapLines2 for one keyframe against 10 neighbours (LocalMapping.cc:911-1173, monocular) two ways:
  batched     sslpl_create_new_map_lines_batch_device: line matcher and triangulation of all 10 neighbours in one asynchronous call;
  match+host  the batched line matcher (sslpl_line_search_for_triangulation_batch_device) one neighbour at a time with the mask updated
              between them, its rows downloaded and both end points triangulated on the host by tests/create_lines_model.py.
Both forms must give identical rows, statuses and s3D / e3D bits.  Host clock around a device synchronise; after a warm-up the two are
sampled alternately; medians with min and max.  Scenes are tests/test_kf_create_lines_gpu.py's, at 640x480 / 40 lines and 1280x960 /
500 lines.  Prints the card and its power limit.
Usage: python tools/kf_create_lines_timing.py [--reps 10]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    import create_lines_model as M
    import test_kf_create_lines_gpu as T
    pkg = g.load_package()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip())
    for W, H, nl in ((640, 480, 40), (1280, 960, 500)):
        K = T.scene(pkg, W, H, nl, empty=None, single=None, seed=1)
        D = T.upload(torch, K)
        mt = T.matcher(pkg, D)
        pairs = T.neighbour_pairs()
        P, capl = len(pairs), D["capl"]
        d_pair = torch.tensor(np.array(pairs, np.int32), device="cuda")
        o = T.outputs(torch, P, capl)
        d_hm = torch.empty_like(D["d_has_ml_t"]); d_rows = torch.empty((1, capl, 2), dtype=torch.int32, device="cuda")
        d_n1 = torch.empty(1, dtype=torch.int32, device="cuda")

        def batched():
            mt.create_new_map_lines_batch_device(D["d_kl_t"].data_ptr(), D["d_ldesc_t"].data_ptr(), D["d_eq_t"].data_ptr(), D["d_nl_t"].data_ptr(),
                                                 len(D["nl"]), capl, D["d_has_ml_t"].data_ptr(), P, d_pair.data_ptr(), D["d_pose_t"].data_ptr(),
                                                 D["d_depth_t"].data_ptr(), D["cam"], *[o[k].data_ptr() for k in ("rows", "n", "status", "line3d", "nnew")])
            mt.sync()
            n = o["n"].cpu().numpy(); rows = o["rows"].cpu().numpy(); st = o["status"].cpu().numpy(); l3 = o["line3d"].cpu().numpy()
            return [(rows[p, :n[p]], st[p, :n[p]], l3[p, :n[p]][(st[p, :n[p]] == 0) | (st[p, :n[p]] >= 4)]) for p in range(P)]

        def match_host():
            hm = D["has_ml"].copy()
            out = []
            for p, (i, j) in enumerate(pairs):
                d_hm.copy_(torch.from_numpy(hm))
                mt.line_search_for_triangulation_batch_device(D["d_ldesc_t"].data_ptr(), D["d_nl_t"].data_ptr(), len(D["nl"]), capl, d_hm.data_ptr(),
                                                              1, d_pair[p:p + 1].data_ptr(), d_rows.data_ptr(), d_n1.data_ptr())
                mt.sync()
                n = int(d_n1.item())
                rows = d_rows[0, :max(n, 0)].cpu().numpy()
                st, l3, written = M.triangulate_lines(K["kl"][i], K["kl"][j], K["lineeq"][i], K["lineeq"][j], rows, K["pose"][i], K["pose"][j],
                                                      K["depth"][j], K["cam"])
                hm[i, rows[st == M.CREATED, 0]] = 1
                out.append((rows, st, l3[written]))
            return out

        forms = dict(batched=batched, match_host=match_host)
        res = {k: f() for k, f in forms.items()}                       # warm-up, and the two forms agree bit for bit
        for (ra, sa, la), (rb, sb, lb) in zip(res["batched"], res["match_host"]):
            assert np.array_equal(ra, rb) and np.array_equal(sa, sb) and np.array_equal(la.view(np.uint32), lb.view(np.uint32))
        created = sum(int((s == 0).sum()) for _, s, _ in res["batched"])
        times = {k: [] for k in forms}
        for _ in range(args.reps):
            for k, f in forms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter(); f(); times[k].append((time.perf_counter() - t0) * 1e3)
        print(f"{W}x{H} / {nl} lines, KF 0 + {P} neighbours, {created} lines created: " +
              "  ".join(f"{k} median {np.median(v):.3f} ms (min {min(v):.3f}, max {max(v):.3f})" for k, v in times.items()))


if __name__ == "__main__":
    main()
