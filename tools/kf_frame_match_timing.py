"""Times the batched keyframe-to-frame matchers on the GPU: sslpl_search_by_bow_batch_device (ORBmatcher::SearchByBoW(KeyFrame*, Frame&))
and sslpl_match_lines_kf_batch_device (LSDmatcher::SearchByProjection(KeyFrame*, Frame&)), against one single-pair call per pair (host
buffers in and out, FeatureVectors already built on the host, as a caller makes them today) and against the oracle on the host CPUs.

Two shapes: 1000 features / 40 lines per row (a 640x480 frame) and 4000 / 500 (1280x960).  Rows are synthetic: descriptors drawn
from a few places with 3 % of the bits flipped, generated on the device from a seed; random angles; element maps from a shared pool with
8 % bad MapPoints.  The vocabulary is a random k = 10, L = 6 tree (the shape of ORBvoc) at levelsup 4, as Frame::ComputeBoW uses it.
- Relocalisation: 64 query frames against a database of 500 and of 5000 keyframes; the pairs are those of
  sslpl_detect_relocalization_candidates_batch_device -> sslpl_reloc_pairs_batch_device (up to 8 candidates per frame, 512 slots),
  matched at nnratio 0.75.
- Tracking: 512 frames, each paired with its reference keyframe (64 keyframes, 8 frames each), points at nnratio 0.9 and lines.
The batched time is CUDA events around one call after warm-up (median and min-max over --reps samples); the single-pair time is the wall
time of the loop over the pairs; the oracle time the wall time of its per-pair calls.  All three forms must give identical tables.
Prints the card's name and power limit of this run and one JSON line.

usage: python tools/kf_frame_match_timing.py [--reps 20] [--single-reps 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tools"))
SHAPES = [("640x480", 1000, 40), ("1280x960", 4000, 500)]
VOC_L, LEVELSUP = 6, 4


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def stats(ms):
    ms = np.asarray(ms)
    return {"median_ms": round(float(np.median(ms)), 4), "min_ms": round(float(ms.min()), 4), "max_ms": round(float(ms.max()), 4)}


def device_rows(torch, g, nrows, nfeat, cap, place, nplaces=8):
    """[nrows, cap, 32] descriptors on the device: row r draws nfeat of its place's 600 base descriptors, 3 % of the bits flipped."""
    base = torch.randint(0, 256, (nplaces, 600, 32), dtype=torch.uint8, device="cuda", generator=g)
    pick = torch.randint(0, 600, (nrows, cap), device="cuda", generator=g)
    d = base[torch.as_tensor(place, device="cuda")[:, None], pick]
    noise = torch.randint(0, 256, d.shape, dtype=torch.uint8, device="cuda", generator=g)
    for _ in range(4):
        noise &= torch.randint(0, 256, d.shape, dtype=torch.uint8, device="cuda", generator=g)
    d ^= noise
    d[:, nfeat:] = 0
    return d.contiguous()


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--single-reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    import __graft_entry__ as gr
    import kf_frame_match_model as km
    if not torch.cuda.is_available():
        raise SystemExit("kf_frame_match_timing: no CUDA device: device times cannot be measured here")
    pkg = gr.load_package(); O = gr.load_oracle()
    gpu = card()
    print(f"card: {gpu}")
    va = pkg.Vocabulary.random_arrays(10, VOC_L, seed=5, stop_fraction=0.01)
    voc = pkg.Vocabulary(10, VOC_L, *va)
    nc = voc.level_nodes(LEVELSUP)
    result = {"card": gpu, "runs": []}
    for shape, nfeat, nlines in SHAPES:
        cap, capl = nfeat + 64, nlines + 64
        mt = pkg.Matcher(max_features=nfeat, max_lines=nlines, max_nodes=nc, max_batch=512)
        stream = torch.cuda.ExternalStream(mt.stream)
        for kind, ndb in (("reloc", 500), ("reloc", 5000), ("tracking", 64)):
            rng = np.random.default_rng(ndb + nfeat)
            g = torch.Generator(device="cuda"); g.manual_seed(ndb + nfeat)
            nq = 64 if kind == "reloc" else 512
            nrows = ndb + nq
            place = rng.integers(0, 8, nrows)
            if kind == "tracking":
                place[ndb:] = place[np.arange(nq) // 8]                      # frame f tracks keyframe f // 8, of the same place
            n = np.full(nrows, nfeat, np.int32)
            d_desc = device_rows(torch, g, nrows, nfeat, cap, place)
            kps = np.zeros((nrows, cap), pkg.KEYPOINT_DTYPE)
            kps["angle"] = rng.uniform(0, 360, (nrows, cap)).astype(np.float32)
            nmp = 40 * nfeat
            kfmp = km.element_maps(rng, n, cap, nmp, twice=False)
            bad = (rng.random(nmp) < 0.08).astype(np.uint8)
            dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
            d_kps, d_n, d_kfmp, d_bad = dev(kps.view(np.uint8)), dev(n), dev(kfmp), dev(bad)
            if kind == "reloc":
                word = torch.empty((nrows, cap), dtype=torch.int32, device="cuda"); val = torch.empty((nrows, cap), dtype=torch.float64, device="cuda")
                bn = torch.empty(nrows, dtype=torch.int32, device="cuda")
                d_db, d_query = dev(np.arange(ndb, dtype=np.int32)), dev(np.arange(ndb, nrows, dtype=np.int32))
                d_covis = dev(np.full((nrows, 10), -1, np.int32)); rs = torch.zeros(nrows, dtype=torch.float32, device="cuda")
                cand = torch.empty((nq, ndb), dtype=torch.int32, device="cuda"); ncand = torch.empty(nq, dtype=torch.int32, device="cuda")
                words = torch.empty((nq, ndb), dtype=torch.int32, device="cuda"); score = torch.empty((nq, ndb), dtype=torch.float32, device="cuda")
                d_pair = torch.empty((512, 2), dtype=torch.int32, device="cuda")
                mt.bow_vectors_batch_device(voc, d_desc.data_ptr(), d_n.data_ptr(), nrows, cap, word.data_ptr(), val.data_ptr(), bn.data_ptr())
                mt.detect_relocalization_candidates_batch_device(word.data_ptr(), val.data_ptr(), bn.data_ptr(), nrows, cap, d_db.data_ptr(),
                                                                 ndb, d_query.data_ptr(), nq, d_covis.data_ptr(), rs.data_ptr(),
                                                                 cand.data_ptr(), ncand.data_ptr(), words.data_ptr(), score.data_ptr())
                mt.reloc_pairs_batch_device(d_query.data_ptr(), cand.data_ptr(), ncand.data_ptr(), nq, ndb, 8, d_pair.data_ptr())
                mt.sync()
                pairs, nnratio = d_pair.cpu().numpy(), 0.75
            else:
                pairs, nnratio = np.stack([np.arange(nq) // 8, ndb + np.arange(nq)], 1).astype(np.int32), 0.9
                d_pair = dev(pairs)
            npairs = len(pairs)
            d_match = torch.empty((npairs, cap), dtype=torch.int32, device="cuda"); d_nm = torch.empty(npairs, dtype=torch.int32, device="cuda")
            call = lambda: mt.search_by_bow_batch_device(d_kps.data_ptr(), d_desc.data_ptr(), d_n.data_ptr(), nrows, cap, d_kfmp.data_ptr(),
                                                         d_bad.data_ptr(), nmp, voc, LEVELSUP, npairs, d_pair.data_ptr(), nnratio, True,
                                                         d_match.data_ptr(), d_nm.data_ptr())
            batch = timed(torch, stream, call, a.reps)
            got, nm = d_match.cpu().numpy(), d_nm.cpu().numpy()
            # the host side of today's caller: rows named by the pairs, their FeatureVectors
            named = sorted({int(r) for r in pairs.reshape(-1) if r >= 0})
            desc = np.zeros((nrows, cap, 32), np.uint8)
            idx = torch.as_tensor(named, device="cuda")
            desc[named] = d_desc[idx].cpu().numpy()
            R = dict(kps=kps, desc=desc, n=n, kfmp=kfmp, bad=bad, nmp=nmp)
            fvs = {r: km.feature_vector(O, va, desc[r, :nfeat], LEVELSUP, VOC_L) for r in named}
            live = [p for p in range(npairs) if pairs[p, 0] >= 0]
            om = pkg.ORBmatcher(nnratio, True, mt)
            single = []
            for _ in range(a.single_reps):
                t0 = time.perf_counter()
                for p in live:
                    kr, fr = pairs[p]
                    valid = (km.element_state(kfmp[kr, :nfeat], nmp, bad) == 1).astype(np.uint8)
                    ns, ms = om.SearchByBoW(desc[kr, :nfeat], fvs[kr], valid, kps[kr, :nfeat]["angle"], desc[fr, :nfeat], fvs[fr],
                                            kps[fr, :nfeat]["angle"])
                    assert ns == nm[p] and np.array_equal(ms, got[p, :nfeat]), ("single", p)
                single.append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter()
            for p in range(npairs):
                no, mo = km.search_by_bow(O, R, fvs.get, tuple(pairs[p]), nnratio, True)
                assert no == nm[p] and np.array_equal(mo, got[p]), ("oracle", p)
            oracle_ms = (time.perf_counter() - t0) * 1e3
            run = {"shape": shape, "features": nfeat, "kind": kind, "keyframes": ndb, "pairs": npairs, "live_pairs": len(live),
                   "points": {"batched": stats(batch), "single_calls": stats(single), "oracle_cpu_ms": round(oracle_ms, 1)},
                   "mean_matches": round(float(nm[live].mean()), 1)}
            if kind == "tracking":
                nl = np.full(nrows, nlines, np.int32)
                d_ldesc = device_rows(torch, g, nrows, nlines, capl, place)
                kfml = km.element_maps(rng, nl, capl, 10 * nlines, p_null=0.3, twice=False)
                d_nl, d_kfml = dev(nl), dev(kfml)
                d_lm = torch.empty((npairs, capl), dtype=torch.int32, device="cuda"); d_lnm = torch.empty(npairs, dtype=torch.int32, device="cuda")
                lcall = lambda: mt.match_lines_kf_batch_device(d_ldesc.data_ptr(), d_nl.data_ptr(), nrows, capl, d_kfml.data_ptr(), 10 * nlines,
                                                               npairs, d_pair.data_ptr(), d_lm.data_ptr(), d_lnm.data_ptr())
                lbatch = timed(torch, stream, lcall, a.reps)
                lgot, lnm = d_lm.cpu().numpy(), d_lnm.cpu().numpy()
                ldesc = d_ldesc.cpu().numpy()
                L = dict(ldesc=ldesc, nl=nl, kfml=kfml, nml=10 * nlines)
                lm = pkg.LSDmatcher(mt)
                lsingle = []
                for _ in range(a.single_reps):
                    t0 = time.perf_counter()
                    for p in range(npairs):
                        kr, fr = pairs[p]
                        has = (km.element_state(kfml[kr, :nlines], 10 * nlines) != 0).astype(np.uint8)
                        ns, ms = lm.SearchByProjection(ldesc[kr, :nlines], has, ldesc[fr, :nlines])
                        assert ns == lnm[p] and np.array_equal(ms, lgot[p, :nlines]), ("single lines", p)
                    lsingle.append((time.perf_counter() - t0) * 1e3)
                t0 = time.perf_counter()
                for p in range(npairs):
                    no, mo = km.line_match(O, L, tuple(pairs[p]))
                    assert no == lnm[p] and np.array_equal(mo, lgot[p]), ("oracle lines", p)
                run["lines"] = {"lines": nlines, "batched": stats(lbatch), "single_calls": stats(lsingle),
                                "oracle_cpu_ms": round((time.perf_counter() - t0) * 1e3, 1), "mean_matches": round(float(lnm.mean()), 1)}
            result["runs"].append(run)
            pt = run["points"]
            line = (f"{shape} {nfeat:4d} features, {kind:8s} ({ndb} keyframes, {len(live)}/{npairs} pairs): SearchByBoW batched "
                    f"{pt['batched']['median_ms']:.3f} ms [{pt['batched']['min_ms']:.3f}-{pt['batched']['max_ms']:.3f}], single calls "
                    f"{pt['single_calls']['median_ms']:.1f} ms, oracle {pt['oracle_cpu_ms']:.1f} ms, {run['mean_matches']} matches per pair")
            if "lines" in run:
                ln = run["lines"]
                line += (f"; lines batched {ln['batched']['median_ms']:.3f} ms [{ln['batched']['min_ms']:.3f}-{ln['batched']['max_ms']:.3f}], "
                         f"single calls {ln['single_calls']['median_ms']:.1f} ms, oracle {ln['oracle_cpu_ms']:.1f} ms")
            print(line, flush=True)
            del d_desc
            torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
