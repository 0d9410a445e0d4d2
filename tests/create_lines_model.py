"""TEST INFRASTRUCTURE: a NumPy restatement of LocalMapping::CreateNewMapLines2's neighbour loop (LocalMapping.cc:911-1173, monocular),
bit for bit.  The primitives (OpenCV's 4x4 Jacobi SVD, glibc's hypot, the addWeighted / convertTo / Mat::dot / cv::norm rules and the
float gemm of a 3x3 by a 3-vector) are those of tests/create_points_model.py; the two gemm shapes only lines use are here:
  - M = K * Tcw (3x3 by 3x4): cv::gemm's float path (inner length 3 = output height), K's zeros taking part in the sum order;
  - klF.t() * M (1x3 by 3x4): accumulated in double and rounded once.
tools/probe_cv_gemm.py measures both on cv2; tests/test_create_lines_cpu.py pins the result.  No libm function is called.
The matcher rows come from the oracle's LSDmatcher::SearchForTriangulation under the mask the reference would see at each neighbour."""
import numpy as np

from create_points_model import add_weighted, chain_bad, convert_scale, dot3, gemm3, norm3, svd4

f32, f64 = np.float32, np.float64

# status codes of sslpl_create_new_map_lines_batch_device (include/sslpl.h), one per `continue` in reference order
CREATED, PARALLAX, W_ZERO_S, W_ZERO_E, NEAR_S1, NEAR_S2, LONG, NEAR_E1, NEAR_E2, ZS1, ZS2, ZE1, ZE2 = range(13)
STATUS_NAMES = ["created", "parallax", "w == 0 (start)", "w == 0 (end)", "start near KF1", "start near KF2", "too long", "end near KF1",
                "end near KF2", "start z1 <= 0", "start z2 <= 0", "end z1 <= 0", "end z2 <= 0"]


def proj_mat(cam, T):
    """K * Tcw of CV_32F (3x3 by 3x4): float products summed left to right, K's zeros included."""
    fx, fy, cx, cy = [f32(v) for v in cam[:4]]
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], f32)
    T = np.asarray(T, f32).reshape(3, 4)
    with np.errstate(all="ignore"):
        return np.stack([(K[i, 0] * T[0] + K[i, 1] * T[1]) + K[i, 2] * T[2] for i in range(3)])


def plane_rows(l, M):
    """klF.t() * M for float line functions l [n, 3] and M [3, 4]: double products summed from 0.0 in order, rounded once -> [n, 4]."""
    l = np.asarray(l, f32).astype(f64); M = np.asarray(M, f32).astype(f64)
    with np.errstate(all="ignore"):
        return (((0.0 + l[:, 0:1] * M[0]) + l[:, 1:2] * M[1]) + l[:, 2:3] * M[2]).astype(f32)


def _dehomogenise(vt):
    v = vt[:, 3]
    return v[:, 3] == 0, np.stack([convert_scale(v[:, k], (1.0 / v[:, 3].astype(f64))) for k in range(3)], 1)


def line_matrices(kl1, kl2, eq1, eq2, rows, pose1, pose2, cam):
    """The pieces of the per-match body up to the SVDs for one neighbour's rows (qdx, tdx): (cosParallaxRays [n] f32, A [n, 4, 4] of the
    start point, B [n, 4, 4] of the end point)."""
    fx, fy, cx, cy, invfx, invfy = [f32(v) for v in cam]
    T1 = np.asarray(pose1[:12], f32).reshape(3, 4); T2 = np.asarray(pose2[:12], f32).reshape(3, 4)
    i1, i2 = rows[:, 0], rows[:, 1]
    with np.errstate(all="ignore"):
        def norm_pts(kl, i, x, y):                                                               # :1025-1036 (KF1's cx / invfx for both)
            return (kl[x][i].astype(f32) - cx) * invfx, (kl[y][i].astype(f32) - cy) * invfy
        s1x, s1y = norm_pts(kl1, i1, "startPointX", "startPointY"); e1x, e1y = norm_pts(kl1, i1, "endPointX", "endPointY")
        s2x, s2y = norm_pts(kl2, i2, "startPointX", "startPointY"); e2x, e2y = norm_pts(kl2, i2, "endPointX", "endPointY")
        one = np.ones(len(rows), f32)
        mid1 = add_weighted(np.stack([s1x, s1y, one], 1), 0.5, np.stack([e1x, e1y, one], 1), 0.5)   # (S + E) / 2
        mid2 = add_weighted(np.stack([s2x, s2y, one], 1), 0.5, np.stack([e2x, e2y, one], 1), 0.5)
        ray1 = gemm3(T1[:, :3].T, mid1); ray2 = gemm3(T2[:, :3].T, mid2)                          # :1038-1039
        cosp = (dot3(ray1, ray2) / (norm3(ray1) * norm3(ray2))).astype(f32)                       # :1041
        P1 = plane_rows(np.asarray(eq1, f64)[i1].astype(f32), proj_mat(cam, T1))                 # :1047-1048, :1057-1058
        P2 = plane_rows(np.asarray(eq2, f64)[i2].astype(f32), proj_mat(cam, T2))

        def ends(x, y):                                                                           # :1059-1060, :1076-1077
            return np.stack([P1, P2, add_weighted(T1[2], x[:, None].astype(f64), T1[0], -1.0),
                             add_weighted(T1[2], y[:, None].astype(f64), T1[1], -1.0)], 1)
        return cosp, ends(s1x, s1y), ends(e1x, e1y)


def triangulate_lines(kl1, kl2, eq1, eq2, rows, pose1, pose2, depth2, cam, trace=None):
    """The per-match body of CreateNewMapLines2 (:1007-1169) for one neighbour's rows (qdx, tdx) -> (status [n] int32, line3d [n, 6]
    float32 = s3D, e3D, written [n] bool: both SVDs gave w != 0).  trace: a list that receives the SVD traces (svd4's) and ("A", A, live)
    with the matrices each SVD got and the rows whose result reaches a status."""
    n = len(rows)
    rows = np.asarray(rows, np.int64).reshape(-1, 2)
    T1 = np.asarray(pose1[:12], f32).reshape(3, 4); O1 = np.asarray(pose1[12:15], f32)
    T2 = np.asarray(pose2[:12], f32).reshape(3, 4); O2 = np.asarray(pose2[12:15], f32)
    d2 = f32(depth2)
    status = np.full(n, -1, np.int32)
    out = np.zeros((n, 6), f32)
    cosp, A, B = line_matrices(kl1, kl2, eq1, eq2, rows, pose1, pose2, cam)
    with np.errstate(all="ignore"):
        ok = (cosp < cosp + f32(1)) & (cosp > 0) & (cosp.astype(f64) < 0.98)                    # :1053, :1090
        status[~ok] = PARALLAX
        wzs, S = _dehomogenise(svd4(A, trace)[1])                                                # :1062-1070
        status[ok & wzs] = W_ZERO_S
        st = ok & ~wzs
        wze, E = _dehomogenise(svd4(B, trace)[1])                                                # :1079-1088
        status[st & wze] = W_ZERO_E
        if trace is not None:
            trace.append(("A", A, ok)); trace.append(("A", B, st))
        st &= ~wze
        written = st.copy()
        out[written] = np.concatenate([S, E], 1)[written]

        def ratio(a, b):                                                                          # (float)cv::norm(a - b) / depth2
            return norm3(a - b).astype(f32) / d2

        def cz(T, X):                                                                             # Rcw.row(2).dot(X) + tcw(2)
            return (dot3(np.broadcast_to(T[2, :3], X.shape), X) + f64(T[2, 3])).astype(f32)

        for bad, code in ((ratio(S, O1).astype(f64) < 0.3, NEAR_S1), (ratio(S, O2).astype(f64) < 0.3, NEAR_S2),
                          (ratio(E, S).astype(f64) > 0.61, LONG), (ratio(E, O1).astype(f64) < 0.3, NEAR_E1),
                          (ratio(E, O2).astype(f64) < 0.3, NEAR_E2), (cz(T1, S) <= 0, ZS1), (cz(T2, S) <= 0, ZS2),
                          (cz(T1, E) <= 0, ZE1), (cz(T2, E) <= 0, ZE2)):
            status[st & bad] = code; st &= ~bad
        status[st] = CREATED
    return status, out, written


def chain_bad_lines(pairs, nl):
    """The pairs the batched call gives count -1: those of chain_bad, and those whose KF1 has lines and KF2 fewer than 2."""
    nkf = len(nl)
    return [b or (nl[i] > 0 and nl[j] < 2) for b, (i, j) in zip(chain_bad(pairs, nkf), pairs)]


def create_lines(match, K, pairs, trace=None):
    """CreateNewMapLines2 over the chains of `pairs`.  match(pair_index, (kf1, kf2), has_ml) -> (count, rows [count, 2]) is the matcher
    (LSDmatcher::SearchForTriangulation); has_ml starts from K["has_ml"] for every chain and gains the KF1 lines of the created rows pair
    by pair.  K: kl [nkf, capl] KEYLINE_DTYPE, lineeq [nkf, capl, 3], nl, has_ml, pose [nkf, 15], depth [nkf], cam.
    -> list per pair of dict(n, rows, status, line3d, written, nnew); n = -1 for a bad pair."""
    nl = np.minimum(np.maximum(np.asarray(K["nl"]), 0), K["has_ml"].shape[1])
    bad = chain_bad_lines(pairs, nl)
    out = []
    hm = None
    for p, (i, j) in enumerate(pairs):
        if p == 0 or pairs[p - 1][0] != i:
            hm = K["has_ml"].copy()
        if bad[p]:
            out.append(dict(n=-1, rows=np.zeros((0, 2), np.int32), status=np.zeros(0, np.int32), line3d=np.zeros((0, 6), f32),
                            written=np.zeros(0, bool), nnew=0))
            continue
        n, rows = match(p, (i, j), hm) if nl[i] > 0 else (0, np.zeros((0, 2), np.int32))
        rows = np.asarray(rows, np.int32).reshape(-1, 2)
        status, l3, written = triangulate_lines(K["kl"][i], K["kl"][j], K["lineeq"][i], K["lineeq"][j], rows, K["pose"][i], K["pose"][j],
                                                K["depth"][j], K["cam"], trace)
        hm[i, rows[status == CREATED, 0]] = 1                   # mpCurrentKeyFrame->AddMapLine(pML, idx1), :1159
        out.append(dict(n=int(n), rows=rows, status=status, line3d=l3, written=written, nnew=int((status == CREATED).sum())))
    return out
