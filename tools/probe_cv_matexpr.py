#!/usr/bin/env python3
"""How cv::Mat expressions round the short CV_32F rows of LocalMapping::CreateNewMapPoints / CreateNewMapLines2 (LocalMapping.cc:475-616,
:1016-1148).  MatExpr evaluates them as:
  s*A - B      -> cv::addWeighted(A, s, B, -1, 0)        (the rows of the triangulation matrix, :501-504)
  (A + B) / 2  -> cv::addWeighted(A, 0.5, B, 0.5, 0)     (the line mid-points)
  A / s        -> A.convertTo(dst, CV_32F, 1. / s, 0)    (x3D = x3D.rowRange(0, 3) / x3D.at<float>(3), :515)
  A - B        -> cv::subtract(A, B)                     (normal1 = x3D - Ow1, :601)
cv2 reaches the same functions: addWeighted and subtract directly, convertTo through normalize(NORM_INF, alpha = 1), whose scale is
1.0 / max|x| in double.  Each candidate rounding rule is counted against cv2 on random rows of length 3 and 4.  On cv2 4.13 (x86-64):
  addWeighted  in double, rounded once to float: (float)((double)a*alpha + (double)b*beta + gamma).  Random rows do not tell this
               from a fused multiply-add; a constructed row whose exact value lies just past a float midpoint does (the double sum
               rounds onto the midpoint, then ties-to-even);
  convertTo    fl(fl(x * (float)scale) + 0): the double scale is narrowed to float first;
  subtract     fl(a - b);
  scaleAdd     normal + normali / cv::norm(normali) of MapPoint::UpdateNormalAndDepth (MapPoint.cc:359): Mat / double is an AddEx
               expression with alpha = 1.0 / norm, and Mat + that expression assigns through MatOp_AddEx::assign, which calls
               scaleAdd(normali, alpha, normal) when beta = 1 (an assumption from OpenCV's published matop.cpp: cv2's Python API has
               no MatExpr, so only scaleAdd itself is measured here).  On CV_32F that is one fused multiply-add with alpha narrowed to float,
               fma(a, (float)alpha, b) (the build's FMA3 dispatch: a canonical choice).  Random rows tell it from fl(fl(a * alpha) + b);
               a constructed row (a * alpha = 1 + 2^-11 + 2^-24, a float midpoint, plus b = 2^-80) does at every length.
tests/create_points_model.py and tests/map_update_model.py follow these rules; test_create_points_cpu.py and test_map_update_cpu.py
re-check them.  (oracle/refshim/minicv.cpp evaluates
Mat / double in double and rounds once; that stand-in is not used by this path.)  Usage: python tools/probe_cv_matexpr.py"""
import numpy as np
import cv2

f32 = np.float32


def aw_float(a, alpha, b, beta, gamma):
    return ((a * f32(alpha)) + (b * f32(beta))) + f32(gamma)


def aw_double(a, alpha, b, beta, gamma):
    return (a.astype(np.float64) * alpha + b.astype(np.float64) * beta + gamma).astype(f32)


def midpoint_case(length):
    """a*alpha = 1 + 2^-11 + 2^-24 (a float midpoint, even neighbour below) and b = -2^-80: the exact a*alpha - b lies just above
    the midpoint, so one rounding gives 1 + 2^-11 + 2^-23 and the double sum (which drops 2^-80) gives 1 + 2^-11."""
    a = np.full((1, length), 1 + 2.0 ** -12, f32)
    b = np.full((1, length), -2.0 ** -80, f32)
    got = cv2.addWeighted(a, float(a[0, 0]), b, -1.0, 0.0)
    return bool((got == f32(1 + 2.0 ** -11)).all()), bool((got == f32(1 + 2.0 ** -11 + 2.0 ** -23)).all())


def cvt_float(x, scale):
    return (x * f32(scale)) + f32(0)


def cvt_double(x, scale):
    return (x.astype(np.float64) * scale).astype(f32)


def scale_add_midpoint(length):
    """(fused, two roundings) of cv2.scaleAdd on a row whose exact a * alpha + b lies just above a float midpoint."""
    a = np.full((1, length), 1 + 2.0 ** -12, f32)
    b = np.full((1, length), 2.0 ** -80, f32)
    got = cv2.scaleAdd(a, float(a[0, 0]), b)
    return bool((got == f32(1 + 2.0 ** -11 + 2.0 ** -23)).all()), bool((got == f32(1 + 2.0 ** -11)).all())


def probe_scale_add(n=20000, seed=7, length=3):
    """Counts of random rows on which cv2.scaleAdd equals the fused rule and the two-rounding rule, and the midpoint row per length."""
    from map_update_model import scale_add, two_roundings
    rng = np.random.default_rng(seed)
    A, B = rows(rng, n, length), rows(rng, n, length)
    s = np.abs(rows(rng, n, 1)[:, 0]).astype(np.float64) + 0.1
    cnt = dict(fused=0, two_roundings=0)
    for k in range(n):
        got = cv2.scaleAdd(A[k:k + 1], float(1.0 / s[k]), B[k:k + 1]).view(np.uint32)
        cnt["fused"] += np.array_equal(got, scale_add(A[k:k + 1], 1.0 / s[k], B[k:k + 1]).view(np.uint32))
        cnt["two_roundings"] += np.array_equal(got, two_roundings(A[k:k + 1], 1.0 / s[k], B[k:k + 1]).view(np.uint32))
    mid = {L: scale_add_midpoint(L) for L in (1, 3, 4, 8)}
    return cnt, mid


def rows(rng, n, length):
    e = rng.integers(-8, 8, (n, length))
    return (rng.standard_normal((n, length)) * np.exp2(e)).astype(f32)


def probe(n=20000, seed=5):
    rng = np.random.default_rng(seed)
    out = {}
    for length in (3, 4):
        A, B = rows(rng, n, length), rows(rng, n, length)
        s = rows(rng, n, 1)[:, 0]
        cnt = dict(float=0, double=0)
        half = dict(float=0, double=0)
        for k in range(n):
            got = cv2.addWeighted(A[k:k + 1], float(s[k]), B[k:k + 1], -1.0, 0.0)
            cnt["float"] += np.array_equal(got.view(np.uint32), aw_float(A[k:k + 1], s[k], B[k:k + 1], -1.0, 0.0).view(np.uint32))
            cnt["double"] += np.array_equal(got.view(np.uint32), aw_double(A[k:k + 1], float(s[k]), B[k:k + 1], -1.0, 0.0).view(np.uint32))
            got = cv2.addWeighted(A[k:k + 1], 0.5, B[k:k + 1], 0.5, 0.0)
            half["float"] += np.array_equal(got.view(np.uint32), aw_float(A[k:k + 1], 0.5, B[k:k + 1], 0.5, 0.0).view(np.uint32))
            half["double"] += np.array_equal(got.view(np.uint32), aw_double(A[k:k + 1], 0.5, B[k:k + 1], 0.5, 0.0).view(np.uint32))
        out[("addWeighted(s, -1)", length)] = cnt
        out[("addWeighted(0.5, 0.5)", length)] = half
        dbl, fused = midpoint_case(length)
        out[("addWeighted midpoint", length)] = dict(double=int(dbl), fused=int(fused))
        cvt = dict(float=0, double=0)
        sub = 0
        for k in range(n):
            x = A[k:k + 1].copy()
            x[0, k % length] = f32(np.abs(x).max() * f32(1.5))       # the divisor is the largest magnitude, so the scale is 1 / it
            scale = 1.0 / float(np.abs(x).max())
            got = cv2.normalize(x, None, 1.0, 0.0, cv2.NORM_INF)
            cvt["float"] += np.array_equal(got.view(np.uint32), cvt_float(x, scale).view(np.uint32))
            cvt["double"] += np.array_equal(got.view(np.uint32), cvt_double(x, scale).view(np.uint32))
            sub += np.array_equal(cv2.subtract(A[k:k + 1], B[k:k + 1]).view(np.uint32), (A[k:k + 1] - B[k:k + 1]).view(np.uint32))
        out[("convertTo", length)] = cvt
        out[("subtract", length)] = dict(float=sub)
    return n, out


if __name__ == "__main__":
    n, out = probe()
    for (op, length), c in out.items():
        print(f"{op:22s} length {length}: " + "  ".join(f"{k} {v}/{1 if 'midpoint' in op else n}" for k, v in c.items()))
    import os, sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
    cnt, mid = probe_scale_add()
    print("scaleAdd               length 3: " + "  ".join(f"{k} {v}/20000" for k, v in cnt.items()))
    for L, (fused, two) in mid.items():
        print(f"scaleAdd midpoint      length {L}: fused {int(fused)}/1  two_roundings {int(two)}/1")
