"""Time the motion-model matcher (ORBmatcher::SearchByProjection(CurrentFrame, LastFrame, th, bMono), ORBmatcher.cc:1331-1473, with
TrackWithMotionModel's 2 * th retry, Tracking.cc:1240-1244) over bench.py's batch640 shape: 513 frames of 640x480, 1000 features,
extracted once on the device, MapPoints and poses from the sequence builder of tests/test_motion_batch_gpu.py.

Forms, alternated in the same run after a warm-up:
  (a) sslpl_search_by_projection_frame_batch_device over the 512 pairs, without and with the retry (CUDA events);
  (b) 512 calls of sslpl_search_by_projection_frame from host buffers, the retry made by a second call (host clock: every call ends
      with a stream synchronisation);
and, once, the CPU oracle over the same pairs on a thread pool of all host cores.  (a) and (b) must give identical tables.
Prints one JSON line, with the card's name and power limit read in the same run.  Needs a GPU; writes nothing.

    python tools/motion_batch_timing.py [--frames 513] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]


def _stats(xs):
    xs = sorted(xs)
    return {"median": round(float(np.median(xs)), 4), "min": round(xs[0], 4), "max": round(xs[-1], 4), "n": len(xs)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--frames", type=int, default=513)
    ap.add_argument("--features", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=5, help="alternated samples of every form")
    ap.add_argument("--inner", type=int, default=10, help="batched calls per event-timed sample")
    ap.add_argument("--th", type=float, default=15.0)
    ap.add_argument("--retry-below", type=int, default=20)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("motion_batch_timing: no CUDA device (this measures the H100 path; there is nothing to time on the CPU)")
    import __graft_entry__ as g
    import synth
    from test_motion_batch_gpu import BOUNDS, CAM, SF, device_batch, motion_sequence, pair_inputs, upload_sequence
    pkg, O = g.load_package(), g.load_oracle()
    card = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        power = "unknown"

    F, th, rb = args.frames, args.th, args.retry_below
    frames = synth.batch(640, 480, F)
    D = device_batch(pkg, torch, frames, args.features)
    seq = motion_sequence(D["kps"], D["desc"], D["n"], seed=1)
    dseq = upload_sequence(torch, seq)
    cap, npairs = D["cap"], F - 1
    mt = pkg.Matcher(max_features=cap, max_lines=64, max_nodes=3072, max_batch=npairs)
    stream = torch.cuda.Stream()                            # not the legacy default stream: its handle 0 means "the matcher's own stream"
    torch.cuda.synchronize()
    mt.set_stream(stream.cuda_stream)
    d_assign = torch.empty((npairs, cap), dtype=torch.int32, device="cuda")
    d_nmatch = torch.empty((npairs,), dtype=torch.int32, device="cuda")
    cam6 = CAM + (0.0, 0.0)
    pairs = [pair_inputs(D["kps"], D["desc"], D["n"], seq, p) for p in range(npairs)]

    def batched(retry, inner):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(inner):
            mt.search_by_projection_frame_batch_device(D["d_kps"], D["d_desc"], D["d_n"], F, cap, dseq["Xw"].data_ptr(), dseq["flag"].data_ptr(),
                                                       dseq["dmp"].data_ptr(), dseq["Tcw"].data_ptr(), CAM, BOUNDS, SF, th, True, retry,
                                                       d_assign.data_ptr(), d_nmatch.data_ptr())
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / inner

    def per_pair(retry):
        out = []
        t0 = time.perf_counter()
        for last, cur, T in pairs:
            n, a = mt.search_by_projection_frame(last, cur, T, None, cam6, BOUNDS, SF, th, True, True, raw=True)
            if retry > 0 and n < retry:
                n, a = mt.search_by_projection_frame(last, cur, T, None, cam6, BOUNDS, SF, 2 * th, True, True, raw=True)
            out.append((n, a))
        return (time.perf_counter() - t0) * 1e3, out

    def identical(out):
        got_a, got_n = d_assign.cpu().numpy(), d_nmatch.cpu().numpy()
        return all(got_n[p] == n and np.array_equal(got_a[p, :len(a)], a) and (got_a[p, len(a):] == -1).all() for p, (n, a) in enumerate(out))

    # warm-up, and the equality check at the timed size
    same = {}
    for retry in (0, rb):
        batched(retry, 1)
        _, out = per_pair(retry)
        same[retry] = identical(out)
    retried = int((np.array([n for n, _ in per_pair(0)[1]]) < rb).sum())

    t = {"batched": [], "batched_retry": [], "per_pair_host": [], "per_pair_host_retry": []}
    for _ in range(args.reps):
        t["batched"].append(batched(0, args.inner))
        t["batched_retry"].append(batched(rb, args.inner))
        t["per_pair_host"].append(per_pair(0)[0])
        t["per_pair_host_retry"].append(per_pair(rb)[0])

    def oracle_pair(p):
        last, cur, T = pairs[p]
        n, a = O.search_by_projection_frame(last, cur, T, None, cam6, BOUNDS, SF, th, True, True)
        if rb > 0 and n < rb:
            n, a = O.search_by_projection_frame(last, cur, T, None, cam6, BOUNDS, SF, 2 * th, True, True)
        return n

    threads = os.cpu_count() or 1
    t0 = time.perf_counter()
    with ThreadPoolExecutor(threads) as ex:                 # the oracle's ctypes calls release the GIL
        on = list(ex.map(oracle_pair, range(npairs)))
    oracle_ms = (time.perf_counter() - t0) * 1e3
    got_n = d_nmatch.cpu().numpy()                          # the last batched call ran with the retry
    mt.set_stream(0)
    print(json.dumps({"tool": "motion_batch_timing", "card": card, "power_limit": power, "frames": F, "pairs": npairs, "width": 640,
                      "height": 480, "features": args.features, "cap": cap, "th": th, "retry_below": rb, "pairs_retried": retried,
                      "matches_mean": round(float(got_n.mean()), 1),
                      "ms": {k: _stats(v) for k, v in t.items()}, "oracle_ms_once": round(oracle_ms, 1), "oracle_threads": threads,
                      "identical_batched_vs_per_pair": bool(same[0] and same[rb]),
                      "oracle_counts_equal": bool(np.array_equal(np.array(on), got_n))}))


if __name__ == "__main__":
    main()
