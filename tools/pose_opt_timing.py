"""Times sslpl_pose_optimization_batch_device (Optimizer::PoseOptimization, Optimizer.cc:666-1022) on the GPU: one batched call over
512 frames, against 512 calls with nframes = 1 (the same device rows, one launch per frame, as a caller without batching would make
them) and against tests/pose_model.py, the CPU restatement the tests hold the device to.  g2o itself is not timed: it needs Eigen,
which is not available to build here, so no g2o figure exists.

Two shapes, synthetic scenes from a seed (tests/pose_model.make_scene, 20 % gross outliers, 2 deg / 5 cm initial error): 640x480 with
1000 points and 40 lines, and 1280x960 with 4000 points and 500 lines.  The batched time is CUDA events around one call after warm-up
(median and min-max over --reps samples); the per-frame time is CUDA events around the loop of 512 single-frame calls (median over
--single-reps); the model time is the median wall time per frame over --model-frames frames, times 512.  The batched and per-frame
results must be bitwise equal.  Prints the card's name and power limit of this run and one JSON line.

usage: python tools/pose_opt_timing.py [--reps 20] [--single-reps 3] [--model-frames 8]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
SHAPES = [("640x480", 640, 480, 1000, 40), ("1280x960", 1280, 960, 4000, 500)]
NFRAMES = 512


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def stats(ms):
    ms = np.asarray(ms)
    return {"median_ms": round(float(np.median(ms)), 4), "min_ms": round(float(ms.min()), 4), "max_ms": round(float(ms.max()), 4)}


def timed(torch, stream, call, reps):
    for _ in range(2):
        call()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream); call(); e1.record(stream); e1.synchronize()
        out.append(e0.elapsed_time(e1))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--single-reps", type=int, default=3)
    ap.add_argument("--model-frames", type=int, default=8)
    a = ap.parse_args()
    import torch
    import __graft_entry__ as g
    import pose_model as pm
    from test_pose_opt_gpu import model, pack, upload
    pkg = g.load_package()
    print(card())
    result = {"card": card(), "frames": NFRAMES, "shapes": {}}
    for name, W, H, npts, nlines in SHAPES:
        rng = np.random.default_rng(2024)
        S = [pm.make_scene(rng, W, H, npts, nlines, outlier_frac=0.2) for _ in range(NFRAMES)]
        P = pack(pkg, S)
        U = upload(torch, P)
        mt = pkg.Matcher(max_features=P["cap"], max_lines=P["capl"], max_nodes=16, max_batch=NFRAMES)
        cap, capl = P["cap"], P["capl"]
        To = torch.zeros((NFRAMES, 12), dtype=torch.float32, device="cuda")
        out = torch.zeros((NFRAMES, cap), dtype=torch.uint8, device="cuda")
        lout = torch.zeros((NFRAMES, capl), dtype=torch.uint8, device="cuda")
        ni = torch.zeros(NFRAMES, dtype=torch.int32, device="cuda")
        stream = torch.cuda.Stream()
        mt.set_stream(stream.cuda_stream)

        def call(f0=0, nf=NFRAMES, To=To, out=out, lout=lout, ni=ni):
            mt.pose_optimization_batch_device(U["kps"].data_ptr() + f0 * cap * 28, U["n"].data_ptr() + 4 * f0, nf, cap,
                                              U["fmp"].data_ptr() + 4 * f0 * cap, len(P["mp"]), U["mp"].data_ptr(),
                                              U["lineeq"].data_ptr() + 24 * f0 * capl, U["nl"].data_ptr() + 4 * f0, capl,
                                              U["fml"].data_ptr() + 4 * f0 * capl, len(P["mlpos"]), U["mlpos"].data_ptr(),
                                              U["T"].data_ptr() + 48 * f0, P["cam"], P["inv"], To.data_ptr() + 48 * f0,
                                              out.data_ptr() + f0 * cap, lout.data_ptr() + f0 * capl, ni.data_ptr() + 4 * f0)

        batched = timed(torch, stream, call, a.reps)
        ref = [x.cpu().numpy().copy() for x in (To, out, lout, ni)]
        for x in (To, out, lout, ni):
            x.zero_()
        torch.cuda.synchronize()
        single = timed(torch, stream, lambda: [call(f, 1) for f in range(NFRAMES)], a.single_reps)
        torch.cuda.synchronize()
        same = all(np.array_equal(r, x.cpu().numpy()) for r, x in zip(ref, (To, out, lout, ni)))
        if not same:
            raise SystemExit(f"{name}: the per-frame calls differ from the batched call")
        cpu = []
        for f in range(a.model_frames):
            t0 = time.perf_counter()
            model(P, f)
            cpu.append((time.perf_counter() - t0) * 1e3)
        mt.set_stream(0)
        del mt
        row = {"batched": stats(batched), "per_frame_calls": stats(single),
               "cpu_model_ms_per_frame": round(float(np.median(cpu)), 3),
               "cpu_model_ms_x512": round(float(np.median(cpu)) * NFRAMES, 1),
               "mean_inliers": round(float(ref[3].mean()), 1)}
        print(name, f"{npts} points / {nlines} lines:", json.dumps(row))
        result["shapes"][name] = row
    print(json.dumps(result))


if __name__ == "__main__":
    main()
