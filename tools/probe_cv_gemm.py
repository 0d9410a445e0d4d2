#!/usr/bin/env python3
"""How cv::gemm rounds small CV_32F products (the `Rcw*x3Dw+tcw` of the reference's projection matchers, ORBmatcher.cc:1364).
Probed on cv2 4.13: for inner length 2..4 equal to the output width or height the products and the running sum are FLOAT
(left to right, addend last); every other shape accumulates in double and rounds once.  oracle/refshim/minicv.cpp
(gemm_eval) follows this table.
probe_lines() measures the two products of LocalMapping::CreateNewMapLines2 (LocalMapping.cc:1047-1058): M = K * Tcw (3x3 by 3x4, with
a camera-shaped K whose zeros take part in the sum) and klF.t() * M (1x3 by 3x4), the latter both as cv2.gemm of a 3x1 operand with
GEMM_1_T (the form the MatExpr runs) and of a 1x3 one without it.  Usage: python tools/probe_cv_gemm.py"""
import numpy as np
import cv2

rng = np.random.default_rng(2)


def f32mm(A, B, C=None):
    m, k = A.shape; n = B.shape[1]; out = np.zeros((m, n), np.float32)
    for i in range(m):
        for j in range(n):
            s = np.float32(A[i, 0] * B[0, j])
            for q in range(1, k):
                s = np.float32(s + np.float32(A[i, q] * B[q, j]))
            if C is not None:
                s = np.float32(s + C[i, j])
            out[i, j] = s
    return out


def f64mm(A, B, C=None):
    m, k = A.shape; n = B.shape[1]; out = np.zeros((m, n))
    for i in range(m):
        for j in range(n):
            s = 0.0
            for q in range(k):
                s += float(A[i, q]) * float(B[q, j])
            if C is not None:
                s += float(C[i, j])
            out[i, j] = s
    return out.astype(np.float32)


def probe_lines(n=2000, seed=5):
    """{shape: dict(float=matches of the float path, double=matches of the double path)} over n random inputs each."""
    g = np.random.default_rng(seed)
    out = {k: dict(float=0, double=0) for k in ("K*Tcw (3,3,4)", "klF.t()*M GEMM_1_T (1,3,4)", "klF.t()*M (1,3,4)")}
    for _ in range(n):
        K = np.array([[g.uniform(300, 1200), 0, g.uniform(200, 700)], [0, g.uniform(300, 1200), g.uniform(150, 500)], [0, 0, 1]], np.float32)
        T = np.concatenate([g.standard_normal((3, 3)), g.uniform(-3, 3, (3, 1))], 1).astype(np.float32)
        l = (g.standard_normal(3) * [1, 1, 400]).astype(np.float32)
        M = cv2.gemm(K, T, 1.0, None, 0.0)
        c = out["K*Tcw (3,3,4)"]; c["float"] += np.array_equal(M, f32mm(K, T)); c["double"] += np.array_equal(M, f64mm(K, T))
        for key, got in (("klF.t()*M GEMM_1_T (1,3,4)", cv2.gemm(l.reshape(3, 1), M, 1.0, None, 0.0, flags=cv2.GEMM_1_T)),
                         ("klF.t()*M (1,3,4)", cv2.gemm(l.reshape(1, 3), M, 1.0, None, 0.0))):
            c = out[key]; c["float"] += np.array_equal(got, f32mm(l.reshape(1, 3), M)); c["double"] += np.array_equal(got, f64mm(l.reshape(1, 3), M))
    return out


if __name__ == "__main__":
    for key, c in probe_lines().items():
        print(f"{key:28s} float-path {c['float']}/2000  double-path {c['double']}/2000")
    for (m, k, n) in [(3, 3, 1), (3, 3, 3), (4, 4, 4), (4, 4, 1), (2, 2, 2), (3, 4, 1), (5, 5, 5), (3, 3, 2), (1, 3, 1), (1, 3, 3), (3, 1, 3), (6, 6, 1)]:
        for useC in (False, True):
            c32 = c64 = 0; N = 1000
            for _ in range(N):
                A = rng.standard_normal((m, k)).astype(np.float32); B = rng.standard_normal((k, n)).astype(np.float32)
                Cm = rng.standard_normal((m, n)).astype(np.float32)
                out = cv2.gemm(A, B, 1.0, Cm if useC else None, 1.0 if useC else 0.0)
                c32 += np.array_equal(out, f32mm(A, B, Cm if useC else None)); c64 += np.array_equal(out, f64mm(A, B, Cm if useC else None))
            small = 2 <= k <= 4 and (k == n or k == m)
            print((m, k, n), "with C" if useC else "no C  ", f"float-path {c32}/{N}  double-path {c64}/{N}  -> model says {'float' if small else 'double'}")
