"""Times SearchByProjection(Frame &F, KeyFrame *pKF, sAlreadyFound, th, ORBdist) — the post-PnP matcher of Tracking::Relocalization — on
the GPU: the batched call over (keyframe, frame) pairs in HBM against one single-pair call per pair (host buffers in and out) and against
the reference's own matcher on the host CPUs.

Four synthetic keyframe / frame scenes at 640x480 and 1000 features (tests/reloc_model.py's reloc_scene), each pair with its own pose;
64 and 512 pairs, at (th, ORBdist) = (10, 100) and (3, 64) as Relocalization runs them.  The batched time is CUDA events around one call
(grid build and walk), after warm-up; the single-pair time is the wall time of the loop over the pairs; the reference time is the sum of
the wall times of its matcher calls alone (tests/ref_reloc.cpp, oracle/_ref/libref_reloc.so; reported as not measured without it).
Prints the card's name and power limit of this run, medians and min-max in ms, and one JSON line.

usage: python tools/reloc_timing.py [--reps 20] [--single-reps 3]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tools"))
SETTINGS = [(10, 100), (3, 64)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def stats(ms):
    ms = np.asarray(ms)
    return {"median_ms": round(float(np.median(ms)), 4), "min_ms": round(float(ms.min()), 4), "max_ms": round(float(ms.max()), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--single-reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    import __graft_entry__ as g
    import reloc_model as rm
    import synth
    if not torch.cuda.is_available():
        raise SystemExit("reloc_timing: no CUDA device: device times cannot be measured here")
    pkg = g.load_package(); O = g.load_oracle()
    gpu = card()
    print(f"card: {gpu}")
    scenes = [rm.reloc_scene(O, synth, s, f0=2 * s) for s in range(4)]
    cap = 1064
    mt = pkg.Matcher(max_features=1100, max_lines=64, max_nodes=1024, max_batch=512)
    R = rm.DeviceRows(torch, scenes, cap)
    rng = np.random.default_rng(5)
    result = {"card": gpu, "features": 1000, "runs": []}
    for npairs in (64, 512):
        sc = rng.integers(0, len(scenes), npairs)
        T = np.zeros((npairs, 12), np.float32)
        for p, s in enumerate(sc):
            Rt = rm._rot(rng.normal(0, 0.004, 3)).astype(np.float32); T0 = scenes[s]["Tcw"]
            T[p, :9] = (Rt @ T0[:, :3]).astype(np.float32).reshape(-1)
            T[p] = np.concatenate([T[p, :9].reshape(3, 3), (T0[:, 3] + rng.normal(0, 0.01, 3)).astype(np.float32)[:, None]], 1).reshape(-1)
        pair = np.stack([2 * sc, 2 * sc + 1], 1).astype(np.int32)
        found = np.zeros((npairs, cap), np.uint8); held = np.zeros((npairs, cap), np.uint8)
        for p, s in enumerate(sc):
            S = scenes[s]
            found[p, :len(S["kfmp"])] = np.where(S["kfmp"] >= 0, S["found_el"][np.maximum(S["kfmp"], 0)], 0)
            held[p, :len(S["held"])] = S["held"]
        dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
        d_pair, d_T, d_found, d_held = dev(pair), dev(T), dev(found), dev(held)
        d_assign = torch.empty((npairs, cap), dtype=torch.int32, device="cuda"); d_nm = torch.empty(npairs, dtype=torch.int32, device="cuda")
        for th, orb in SETTINGS:
            call = lambda: mt.search_by_projection_kf_batch_device(
                R.kps.data_ptr(), R.desc.data_ptr(), R.n.data_ptr(), R.nrows, cap, R.kfmp.data_ptr(), R.bad.data_ptr(), R.nel, R.el.data_ptr(),
                R.eldesc.data_ptr(), npairs, d_pair.data_ptr(), d_T.data_ptr(), d_found.data_ptr(), d_held.data_ptr(), rm.CAM, rm.BOUNDS, rm.SF,
                rm.LOG_SF, th, orb, True, d_assign.data_ptr(), d_nm.data_ptr())
            stream = torch.cuda.ExternalStream(mt.stream)
            for _ in range(3):
                call()
            mt.sync()
            batch = []
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream); call(); e1.record(stream); e1.synchronize()
                batch.append(e0.elapsed_time(e1))
            nm_batch = d_nm.cpu().numpy()
            # one single-pair call per pair, host buffers
            args = []
            for p, s in enumerate(sc):
                S = scenes[s]
                e = np.maximum(S["kfmp"], 0); el = rm.element_table(S["Xw"], S["mindist"], S["maxdist"])
                flag = ((S["kfmp"] >= 0) & (S["bad"][e] == 0) & (found[p, :len(e)] == 0)).astype(np.uint8)
                kf = dict(flag=flag, Xw=el[e, :3], dmp=S["eldesc"][e], dist3=el[e, 6:9], angle=S["kf_kps"]["angle"])
                k = S["kps"]
                cur = dict(desc=S["desc"], x=k["x"], y=k["y"], oct=k["octave"].astype(np.int32), angle=k["angle"], held=S["held"])
                args.append((kf, cur, T[p]))
            single = []
            nm_single = np.zeros(npairs, np.int32)
            for _ in range(a.single_reps):
                t0 = time.perf_counter()
                for p, (kf, cur, Tp) in enumerate(args):
                    nm_single[p] = mt.search_by_projection_kf(kf, cur, Tp, rm.CAM, rm.BOUNDS, rm.SF, rm.LOG_SF, th, orb)[0]
                single.append((time.perf_counter() - t0) * 1e3)
            assert np.array_equal(nm_single, nm_batch), "batched and single-pair counts differ"
            host = None
            if rm.ref_available():
                sec = C.c_double(); tot = 0.0
                for p, s in enumerate(sc):
                    S = scenes[s]
                    fe = np.zeros(len(S["Xw"]), np.uint8)
                    fe[S["kfmp"][(S["kfmp"] >= 0) & (found[p, :len(S["kfmp"])] != 0)]] = 1
                    rm.ref_search_by_projection_kf(S["kf_kps"], S["kfmp"], S["Xw"], S["mindist"], S["maxdist"], S["eldesc"], S["bad"], fe,
                                                   S["kps"], S["desc"], S["held"], T[p].reshape(3, 4), rm.CAM, rm.BOUNDS, len(rm.SF), 1.2, th,
                                                   orb, True, seconds=sec)
                    tot += sec.value
                host = round(tot * 1e3, 3)
            run = {"npairs": npairs, "th": th, "ORBdist": orb, "batched": stats(batch), "single_calls": stats(single),
                   "reference_cpu_ms": host if host is not None else "not measured", "mean_matches": round(float(nm_batch.mean()), 1)}
            result["runs"].append(run)
            print(f"{npairs:4d} pairs (th {th:2d}, ORBdist {orb:3d}): batched {run['batched']['median_ms']:.3f} ms "
                  f"[{run['batched']['min_ms']:.3f}-{run['batched']['max_ms']:.3f}], single calls {run['single_calls']['median_ms']:.1f} ms "
                  f"[{run['single_calls']['min_ms']:.1f}-{run['single_calls']['max_ms']:.1f}], reference {run['reference_cpu_ms']} ms, "
                  f"{run['mean_matches']} matches per pair")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
