#!/usr/bin/env python3
"""Time LocalMapping::CreateNewMapPoints for one keyframe against 20 neighbours (LocalMapping.cc:371-637, monocular) three ways:
  batched     sslpl_create_new_map_points_batch_device: matcher and triangulation of all 20 neighbours in one asynchronous call;
  match+host  the batched matcher (sslpl_search_for_triangulation_batch_device, checkOrientation false) one neighbour at a time with the
              mask updated between them, its rows downloaded and triangulated on the host by tests/create_points_model.py;
  oracle      the CPU restatement alone (the oracle's SearchForTriangulation and the model's triangulation).
Host clock around a device synchronise; after a warm-up the three are sampled alternately.  Scenes are tests/test_kf_create_points_gpu.py's,
at 640x480 / 1000 features and 1280x960 / 4000 features.  Prints the card and its power limit.
Usage: python tools/kf_create_points_timing.py [--reps 10]"""
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
    import create_points_model as M
    import test_kf_create_points_gpu as T
    pkg, oracle = g.load_package(), g.load_oracle()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip())
    for W, H, nf in ((640, 480, 1000), (1280, 960, 4000)):
        K = T.scene(pkg, oracle, W, H, nf, seed=1)
        D = T.upload(pkg, torch, K)
        mt = T.matcher(pkg, D)
        pairs = T.neighbour_pairs()
        geom = T.geometry(D, pairs)
        P, cap = len(pairs), D["cap"]
        d_pair = torch.tensor(np.array(pairs, np.int32), device="cuda"); d_geom = torch.from_numpy(geom).cuda()
        o = [torch.empty((P, cap, 2), dtype=torch.int32, device="cuda"), torch.empty(P, dtype=torch.int32, device="cuda"),
             torch.empty((P, cap), dtype=torch.int32, device="cuda"), torch.empty((P, cap, 3), dtype=torch.float32, device="cuda"),
             torch.empty(P, dtype=torch.int32, device="cuda")]
        d_hm = torch.empty_like(D["d_has_mp_t"]); d_rows = torch.empty((1, cap, 2), dtype=torch.int32, device="cuda")
        d_n1 = torch.empty(1, dtype=torch.int32, device="cuda")

        def batched():
            mt.create_new_map_points_batch_device(D["d_kps_t"].data_ptr(), D["d_desc_t"].data_ptr(), D["d_n_t"].data_ptr(), len(D["n"]), cap,
                                                  D["d_has_mp_t"].data_ptr(), D["voc"], T.LEVELSUP, P, d_pair.data_ptr(), d_geom.data_ptr(),
                                                  D["d_pose_t"].data_ptr(), D["cam"], D["scale"], D["sigma2"], D["scale_factor"],
                                                  *[t.data_ptr() for t in o])
            mt.sync()
            return int(o[4].sum().item())

        def match_host():
            hm = D["has_mp"].copy()
            nnew = 0
            for p, (i, j) in enumerate(pairs):
                d_hm.copy_(torch.from_numpy(hm))
                mt.search_for_triangulation_batch_device(D["d_kps_t"].data_ptr(), D["d_desc_t"].data_ptr(), D["d_n_t"].data_ptr(), len(D["n"]),
                                                         cap, d_hm.data_ptr(), D["voc"], T.LEVELSUP, 1, d_pair[p:p + 1].data_ptr(),
                                                         d_geom[p:p + 1].data_ptr(), D["scale"], D["sigma2"], False, d_rows.data_ptr(), d_n1.data_ptr())
                mt.sync()
                n = int(d_n1.item())
                rows = d_rows[0, :max(n, 0)].cpu().numpy()
                st, _, _ = M.triangulate_points(K["kps"][i], K["kps"][j], rows, K["pose"][i], K["pose"][j], K["cam"], K["scale"], K["sigma2"],
                                                K["scale_factor"])
                hm[i, rows[st == M.CREATED, 0]] = 1
                nnew += int((st == M.CREATED).sum())
            return nnew

        def cpu():
            return sum(e["nnew"] for e in T.oracle_chain(oracle, K, pairs, geom))

        forms = dict(batched=batched, match_host=match_host, oracle=cpu)
        counts = {k: f() for k, f in forms.items()}                    # warm-up, and the three agree on the created count
        assert len(set(counts.values())) == 1, counts
        times = {k: [] for k in forms}
        for _ in range(args.reps):
            for k, f in forms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter(); f(); times[k].append((time.perf_counter() - t0) * 1e3)
        print(f"{W}x{H} / {nf} features, KF 0 + {P} neighbours, {counts['batched']} points created: " +
              "  ".join(f"{k} median {np.median(v):.2f} ms (min {min(v):.2f}, max {max(v):.2f})" for k, v in times.items()))


if __name__ == "__main__":
    main()
