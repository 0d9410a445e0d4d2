"""Times the batched keyframe database on the GPU against the reference's KeyFrameDatabase on the host CPUs.

A database of 500 and of 5000 keyframes at 1000 features, drawn from 20 places, with a random k = 10, L = 5 vocabulary tree (100,000
words); 1 and 64 queries, loop (DetectLoopCandidates) and reloc (DetectRelocalizationCandidates).  The device BowVector build of all rows
(sslpl_bow_vectors_batch_device) is timed on its own; the query calls start from BowVectors in HBM.  Device times are CUDA events around
one call, after warm-up; host times are the wall time of the reference's own queries (tests/ref_kfdb.cpp, linked with
oracle/_ref/libref.so into oracle/_ref/libref_kfdb.so by oracle/ref_kfdb_build.sh); without that library they are reported as not
measured.
Prints the card's name and power limit of this run, medians and min-max in ms, and one JSON line.

usage: python tools/kfdb_timing.py [--reps 20] [--host-reps 3]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
ORACLE = os.path.join(ROOT, "oracle")
NFEAT, NPLACES = 1000, 20


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def host_lib():
    """The reference's KeyFrameDatabase behind tests/ref_kfdb.cpp (oracle/_ref/libref_kfdb.so, which build() makes where the reference's
    sources are present and which travels with oracle/_ref), or None."""
    path = os.path.join(ORACLE, "_ref", "libref_kfdb.so")
    if not os.path.exists(path):
        return None
    L = C.CDLL(path)
    L.ref_kfdb_query.restype = None
    return L


def stats(ms):
    ms = np.asarray(ms)
    return {"median_ms": round(float(np.median(ms)), 4), "min_ms": round(float(ms.min()), 4), "max_ms": round(float(ms.max()), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    import __graft_entry__ as g
    pkg = g.load_package()
    if not torch.cuda.is_available():
        raise SystemExit("kfdb_timing: no CUDA device: device times cannot be measured here")
    gpu = card()
    print(f"card: {gpu}")
    parent, desc, weight, leaf = pkg.Vocabulary.random_arrays(10, 5, seed=1)
    voc = pkg.Vocabulary(10, 5, parent, desc, weight, leaf)
    mt = pkg.Matcher(max_features=NFEAT, max_lines=64, max_nodes=1024, max_batch=1)
    href = host_lib()
    hvoc = None
    if href is not None:
        from oracle import ref as R
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from test_ref_parity_cpu import write_vocab_text
        path = os.path.join("/tmp", f"kfdb_timing_voc_{os.getpid()}.txt")
        write_vocab_text(path, 10, 5, parent, desc, weight, leaf)
        hvoc = R.Vocabulary(path)
        os.unlink(path)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    st = torch.cuda.ExternalStream(mt.stream)

    def timed(fn):
        ev0.record(st); fn(); ev1.record(st); ev1.synchronize()
        return ev0.elapsed_time(ev1)

    results = []
    for ndb in (500, 5000):
        rng = np.random.default_rng(ndb)
        nrows, cap = ndb + 64, NFEAT + 64
        base = rng.integers(0, 256, (NPLACES, 2000, 32), dtype=np.uint8)
        place = rng.integers(0, NPLACES, nrows)
        d = np.zeros((nrows, cap, 32), np.uint8)
        for r in range(nrows):
            d[r, :NFEAT] = base[place[r], rng.integers(0, 2000, NFEAT)] ^ np.packbits(rng.random((NFEAT, 256)) < 0.03, axis=-1, bitorder="little")
        d_desc = torch.from_numpy(d).cuda(); d_n = torch.full((nrows,), NFEAT, dtype=torch.int32, device="cuda")
        word = torch.empty((nrows, cap), dtype=torch.int32, device="cuda"); val = torch.empty((nrows, cap), dtype=torch.float64, device="cuda")
        bn = torch.empty(nrows, dtype=torch.int32, device="cuda")
        build = lambda: mt.bow_vectors_batch_device(voc, d_desc.data_ptr(), d_n.data_ptr(), nrows, cap, word.data_ptr(), val.data_ptr(), bn.data_ptr())
        for _ in range(3):
            timed(build)
        results.append(dict(ndb=ndb, stage="bow_vectors", rows=nrows, **stats([timed(build) for _ in range(a.reps)])))
        covis = np.full((nrows, 10), -1, np.int32)
        for r in range(nrows):
            same = np.nonzero(place == place[r])[0]
            k = min(10, len(same))
            covis[r, :k] = rng.choice(same, k, replace=False)
        db = rng.permutation(ndb).astype(np.int32)
        tables = (word.data_ptr(), val.data_ptr(), bn.data_ptr(), nrows, cap)
        d_db, d_cov = torch.from_numpy(db).cuda(), torch.from_numpy(covis).cuda()
        for nq in (1, 64):
            query = (ndb + np.arange(nq)).astype(np.int32)
            d_q = torch.from_numpy(query).cuda()
            conn = np.zeros(nq + 1, np.int32)
            d_off, d_conn = torch.from_numpy(conn).cuda(), torch.zeros(1, dtype=torch.int32, device="cuda")
            d_ms = torch.full((nq,), 0.01, dtype=torch.float32, device="cuda")
            d_rs = torch.zeros(nrows, dtype=torch.float32, device="cuda")
            cand = torch.empty((nq, ndb), dtype=torch.int32, device="cuda"); ncand = torch.empty(nq, dtype=torch.int32, device="cuda")
            words = torch.empty((nq, ndb), dtype=torch.int32, device="cuda"); score = torch.empty((nq, ndb), dtype=torch.float32, device="cuda")
            out = (cand.data_ptr(), ncand.data_ptr(), words.data_ptr(), score.data_ptr())
            calls = {
                "loop": lambda: mt.detect_loop_candidates_batch_device(*tables, d_db.data_ptr(), ndb, d_q.data_ptr(), nq, d_cov.data_ptr(),
                                                                       d_off.data_ptr(), d_conn.data_ptr(), 0, d_ms.data_ptr(), *out),
                "reloc": lambda: mt.detect_relocalization_candidates_batch_device(*tables, d_db.data_ptr(), ndb, d_q.data_ptr(), nq,
                                                                                 d_cov.data_ptr(), d_rs.data_ptr(), *out)}
            for mode, fn in calls.items():
                for _ in range(3):
                    timed(fn)
                dev_ms = [timed(fn) for _ in range(a.reps)]
                nc = ncand.cpu().numpy()
                row = dict(ndb=ndb, stage=mode, nq=nq, mean_candidates=round(float(nc.mean()), 2), **stats(dev_ms))
                if href is not None:
                    host_ms = run_host(href, hvoc, word, val, bn, covis, db, query, mode == "loop", a.host_reps)
                    row["host_ref"] = stats(host_ms)
                else:
                    row["host_ref"] = "not measured (oracle/_ref/libref_kfdb.so absent)"
                results.append(row)
    for r in results:
        print(json.dumps(r))
    print(json.dumps({"tool": "kfdb_timing", "card": gpu, "vocabulary": "k=10 L=5 random (100000 words)", "features": NFEAT,
                      "results": results}))


def run_host(L, hvoc, word, val, bn, covis, db, query, loop, reps):
    """The reference's KeyFrameDatabase with the same rows, database and queries: ms of the queries (build and add not counted)."""
    w, v, n = word.cpu().numpy(), val.cpu().numpy(), bn.cpu().numpy()
    nrows, nq = len(n), len(query)
    off = np.zeros(nrows + 1, np.int32); off[1:] = np.cumsum(n)
    fw = np.concatenate([w[r, :n[r]] for r in range(nrows)]).astype(np.int32)
    fv = np.concatenate([v[r, :n[r]] for r in range(nrows)]).astype(np.float64)
    ncov = (covis >= 0).sum(1).astype(np.int32)
    coff = np.zeros(nrows + 1, np.int32); cflat = np.zeros(1, np.int32)
    rs = np.zeros(nrows, np.float32); ms = np.full(nq, 0.01, np.float32); none = np.zeros(1, np.int32)
    cand = np.zeros((nq, nrows), np.int32); ncand = np.zeros(nq, np.int32); words = np.zeros((nq, nrows), np.int32)
    score = np.zeros((nq, nrows), np.float32)
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    out = []
    for _ in range(reps):
        sec = C.c_double()
        L.ref_kfdb_query(C.c_void_p(hvoc.h), nrows, p(off), p(fw), p(fv), p(covis), p(ncov), p(coff), p(cflat), p(rs), len(db), p(db), 0,
                         p(none), int(loop), nq, p(query), p(ms), p(cand), p(ncand), p(words), p(score), C.byref(sec))
        out.append(sec.value * 1e3)
    return out


if __name__ == "__main__":
    main()
