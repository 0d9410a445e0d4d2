"""Times the batched initialisation matchers on the GPU: sslpl_search_for_initialization_batch_device (ORBmatcher::SearchForInitialization
over chains of pairs, vbPrevMatched carried) and sslpl_line_search_for_initialize_batch_device (LSDmatcher::SerachForInitialize), against
the single-pair calls (host buffers in and out, vbPrevMatched carried on the host, as a caller makes them today) and against the oracle on
the host CPUs.

Two shapes, each 64 chains of 8 pairs (one initial frame against its next 8 frames, 576 rows): 640x480 with 2000 features and 40 lines, and
1280x960 with 8000 features and 500 lines (the 2 x nFeatures extractor of Tracking.cc:120).  Rows are synthetic, generated from a seed: an
initial frame's keypoints spread over the image with ORB's level proportions, random angles and descriptors; frame k of its chain moves them
by k times a per-chain drift plus jitter, flips 3 % of the descriptor bits, replaces 10 % of the features and shuffles the order.  Lines are
descriptors only, built the same way.  The batched time is CUDA events around one call after warm-up (median and min-max over --reps
samples); the single-call time is the wall time of the loop over the pairs; the oracle time the wall time of its per-pair calls.  All three
forms must give identical tables.  Prints the card's name and power limit of this run and one JSON line.

usage: python tools/init_match_timing.py [--reps 20] [--single-reps 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tools"))
SHAPES = [("640x480", 640, 480, 2000, 40), ("1280x960", 1280, 960, 8000, 500)]
NCHAIN, LEN = 64, 8
LEVEL_SHARE = np.array([217, 181, 151, 126, 105, 87, 73, 60], np.float64)       # ORBextractor's per-level features at 1000 (1.2, 8 levels)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def stats(ms):
    ms = np.asarray(ms)
    return {"median_ms": round(float(np.median(ms)), 4), "min_ms": round(float(ms.min()), 4), "max_ms": round(float(ms.max()), 4)}


def timed(torch, stream, call, reps):
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream); call(); e1.record(stream); e1.synchronize()
        out.append(e0.elapsed_time(e1))
    return out


def noisy(rng, d):
    flip = np.zeros(d.shape, np.uint8)
    for b in range(8):
        flip |= ((rng.random(d.shape) < 0.03).astype(np.uint8) << b)
    return d ^ flip


def rows(pkg, rng, W, H, nfeat, nlines):
    """Row c * (LEN + 1) is chain c's initial frame, the next LEN rows its frames."""
    nrows = NCHAIN * (LEN + 1)
    cap, capl = nfeat + 64, nlines + 64
    kps = np.zeros((nrows, cap), pkg.KEYPOINT_DTYPE); desc = np.zeros((nrows, cap, 32), np.uint8); ldesc = np.zeros((nrows, capl, 32), np.uint8)
    for c in range(NCHAIN):
        r0 = c * (LEN + 1)
        x = rng.uniform(0, W, nfeat).astype(np.float32); y = rng.uniform(0, H, nfeat).astype(np.float32)
        octv = rng.choice(8, nfeat, p=LEVEL_SHARE / LEVEL_SHARE.sum()).astype(np.int32)
        ang = rng.uniform(0, 360, nfeat).astype(np.float32)
        d = rng.integers(0, 256, (nfeat, 32), dtype=np.uint8); ld = rng.integers(0, 256, (nlines, 32), dtype=np.uint8)
        drift = rng.uniform(-6, 6, 2)
        for k in range(LEN + 1):
            new = rng.random(nfeat) < (0.1 if k else 0.0)
            order = rng.permutation(nfeat) if k else np.arange(nfeat)
            r = kps[r0 + k, :nfeat]
            r["x"] = np.clip(x + k * drift[0] + rng.normal(0, 1.5, nfeat) * (k > 0), 0, W - 1)[order]
            r["y"] = np.clip(y + k * drift[1] + rng.normal(0, 1.5, nfeat) * (k > 0), 0, H - 1)[order]
            r["x"][new[order]] = rng.uniform(0, W, new.sum()); r["y"][new[order]] = rng.uniform(0, H, new.sum())
            r["octave"] = octv[order]; r["angle"] = ((ang + rng.normal(0, 3, nfeat) * (k > 0)) % 360)[order]
            dk = noisy(rng, d) if k else d
            dk[new] = rng.integers(0, 256, (new.sum(), 32), dtype=np.uint8)
            desc[r0 + k, :nfeat] = dk[order]
            ldesc[r0 + k, :nlines] = noisy(rng, ld) if k else ld
    pairs = np.array([(c * (LEN + 1), c * (LEN + 1) + k) for c in range(NCHAIN) for k in range(1, LEN + 1)], np.int32)
    return dict(kps=kps, desc=desc, n=np.full(nrows, nfeat, np.int32), ldesc=ldesc, nl=np.full(nrows, nlines, np.int32)), pairs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--single-reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    import __graft_entry__ as gr
    import init_match_model as im
    if not torch.cuda.is_available():
        raise SystemExit("init_match_timing: no CUDA device: device times cannot be measured here")
    pkg = gr.load_package(); O = gr.load_oracle()
    gpu = card()
    print(f"card: {gpu}")
    result = {"card": gpu, "runs": []}
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    for shape, W, H, nfeat, nlines in SHAPES:
        rng = np.random.default_rng(nfeat)
        R, pairs = rows(pkg, rng, W, H, nfeat, nlines)
        nrows, cap, capl, npairs = len(R["n"]), R["desc"].shape[1], R["ldesc"].shape[1], len(pairs)
        bounds = (0.0, float(W), 0.0, float(H))
        mt = pkg.Matcher(max_features=nfeat, max_lines=nlines, max_nodes=3072, max_batch=nrows)
        stream = torch.cuda.ExternalStream(mt.stream)
        d_kps, d_desc, d_n, d_pair = dev(R["kps"].view(np.uint8)), dev(R["desc"]), dev(R["n"]), dev(pairs)
        d_m12 = torch.empty((npairs, cap), dtype=torch.int32, device="cuda"); d_prev = torch.empty((npairs, cap, 2), dtype=torch.float32, device="cuda")
        d_nm = torch.empty(npairs, dtype=torch.int32, device="cuda")
        call = lambda: mt.search_for_initialization_batch_device(d_kps.data_ptr(), d_desc.data_ptr(), d_n.data_ptr(), nrows, cap, npairs,
                                                                 d_pair.data_ptr(), 0, bounds, 0.9, True, 100, d_m12.data_ptr(),
                                                                 d_prev.data_ptr(), d_nm.data_ptr())
        batch = timed(torch, stream, call, a.reps)
        got_m, got_p, got_n = d_m12.cpu().numpy(), d_prev.cpu().numpy(), d_nm.cpu().numpy()
        plist = [tuple(int(v) for v in p) for p in pairs]

        def check(want, what):
            for p, (n, row, state) in enumerate(want):
                assert n == got_n[p] and np.array_equal(row, got_m[p]) and np.array_equal(state, got_p[p, :len(state)]), (what, p)

        single = []
        for _ in range(a.single_reps):
            t0 = time.perf_counter()
            want = im.points(mt.search_for_initialization, R, plist, bounds, 0.9, True, 100)
            single.append((time.perf_counter() - t0) * 1e3)
            check(want, "single")
        t0 = time.perf_counter()
        want = im.points(O.search_for_initialization, R, plist, bounds, 0.9, True, 100)
        oracle_ms = (time.perf_counter() - t0) * 1e3
        check(want, "oracle")
        run = {"shape": shape, "features": nfeat, "lines": nlines, "chains": NCHAIN, "pairs": npairs,
               "points": {"batched": stats(batch), "single_calls": stats(single), "oracle_cpu_ms": round(oracle_ms, 1),
                          "mean_matches": round(float(got_n.mean()), 1)}}
        d_ldesc, d_nl = dev(R["ldesc"]), dev(R["nl"])
        d_lp = torch.empty((npairs, capl, 2), dtype=torch.int32, device="cuda"); d_lnm = torch.empty(npairs, dtype=torch.int32, device="cuda")
        lcall = lambda: mt.line_search_for_initialize_batch_device(d_ldesc.data_ptr(), d_nl.data_ptr(), nrows, capl, npairs, d_pair.data_ptr(),
                                                                   d_lp.data_ptr(), d_lnm.data_ptr())
        lbatch = timed(torch, stream, lcall, a.reps)
        lgot, lnm = d_lp.cpu().numpy(), d_lnm.cpu().numpy()
        lm = pkg.LSDmatcher(mt)
        lsingle = []
        for _ in range(a.single_reps):
            t0 = time.perf_counter()
            for p, (r1, r2) in enumerate(plist):
                ns, ms = lm.SerachForInitialize(R["ldesc"][r1, :nlines], R["ldesc"][r2, :nlines])
                assert ns == lnm[p] and np.array_equal(ms, lgot[p, :ns]), ("single lines", p)
            lsingle.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        for p, pr in enumerate(plist):
            no, rows_o = im.lines(O, R, pr)
            assert no == lnm[p] and np.array_equal(rows_o, lgot[p]), ("oracle lines", p)
        run["lines_match"] = {"batched": stats(lbatch), "single_calls": stats(lsingle),
                              "oracle_cpu_ms": round((time.perf_counter() - t0) * 1e3, 1), "mean_matches": round(float(lnm.mean()), 1)}
        result["runs"].append(run)
        pt, ln = run["points"], run["lines_match"]
        print(f"{shape} {nfeat} features / {nlines} lines, {NCHAIN} chains x {LEN} pairs: SearchForInitialization batched "
              f"{pt['batched']['median_ms']:.3f} ms [{pt['batched']['min_ms']:.3f}-{pt['batched']['max_ms']:.3f}], single calls "
              f"{pt['single_calls']['median_ms']:.1f} ms, oracle {pt['oracle_cpu_ms']:.1f} ms, {pt['mean_matches']} matches per pair; "
              f"SerachForInitialize batched {ln['batched']['median_ms']:.3f} ms [{ln['batched']['min_ms']:.3f}-{ln['batched']['max_ms']:.3f}], "
              f"single calls {ln['single_calls']['median_ms']:.1f} ms, oracle {ln['oracle_cpu_ms']:.1f} ms, {ln['mean_matches']} matches per pair",
              flush=True)
        del d_kps, d_desc, d_ldesc
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
