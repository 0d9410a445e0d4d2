"""TEST INFRASTRUCTURE: a NumPy restatement of LocalMapping::CreateNewMapPoints' neighbour loop (LocalMapping.cc:371-637, monocular),
bit for bit, with the primitives it rests on:
  - hypot: glibc >= 2.35's (sysdeps/ieee754/dbl-64/e_hypot.c, Borges' corrected algorithm, the kernel without FMA), from +, -, *, / and
    sqrt only, so it does not depend on the libm of the machine it runs on;
  - svd4: OpenCV 4.13's one-sided Jacobi JacobiSVDImpl_<float> (modules/core/src/lapack.cpp), which cv::SVD::compute runs for a 4x4
    CV_32F matrix;
  - the MatExpr rounding rules tools/probe_cv_matexpr.py measured on cv2 4.13 (addWeighted in double, convertTo with a float scale,
    subtract in float) and the Mat::dot / cv::norm double accumulations.
NumPy float32 array arithmetic rounds every operation (no contraction), float64 likewise, and sqrt is correctly rounded.
The matcher rows come from the oracle's SearchForTriangulation under the mask the reference would see at each neighbour."""
import numpy as np

f32, f64 = np.float32, np.float64

# status codes of sslpl_create_new_map_points_batch_device (include/sslpl.h), one per `continue` in reference order
CREATED, PARALLAX, W_ZERO, Z1, Z2, OCTAVE1, REPROJ1, REPROJ2, DIST0, SCALE = range(10)
STATUS_NAMES = ["created", "parallax", "w == 0", "z1 <= 0", "z2 <= 0", "kf1 octave", "reprojection 1", "reprojection 2", "dist == 0",
                "scale consistency"]

_SCALE, _LARGE, _TINY, _EPS = 2.0 ** -600, 2.0 ** 511, 2.0 ** -459, 2.0 ** -54


def _hypot_kernel(ax, ay):
    h = np.sqrt(ax * ax + ay * ay)
    d1 = h - ay                                            # h <= 2 ay
    t1a = ax * (2.0 * d1 - ax)
    t2a = (d1 - 2.0 * (ax - ay)) * d1
    d2 = h - ax                                            # else
    t1b = 2.0 * d2 * (ax - 2.0 * ay)
    t2b = (4.0 * d2 - ay) * ay + d2 * d2
    first = h <= 2.0 * ay
    t1 = np.where(first, t1a, t1b); t2 = np.where(first, t2a, t2b)
    return h - (t1 + t2) / (2.0 * h)


def hypot(x, y):
    """glibc >= 2.35 hypot (double), elementwise."""
    x = np.asarray(x, f64); y = np.asarray(y, f64)
    with np.errstate(all="ignore"):
        x0, y0 = np.broadcast_arrays(x, y)
        x, y = np.abs(x0), np.abs(y0)
        ax = np.where(x < y, y, x); ay = np.where(x < y, x, y)
        common = np.where(ay <= ax * _EPS, ax + ay, _hypot_kernel(ax, ay))
        large = np.where(ay <= ax * _EPS, ax + ay, _hypot_kernel(ax * _SCALE, ay * _SCALE) / _SCALE)
        tiny = np.where(ax >= ay / _EPS, ax + ay, _hypot_kernel(ax / _SCALE, ay / _SCALE) * _SCALE)
        out = np.where(ax > _LARGE, large, np.where(ay < _TINY, tiny, common))
        fin = np.isfinite(x) & np.isfinite(y)
        out = np.where(fin, out, np.where(np.isinf(x) | np.isinf(y), np.inf, x0 + y0))
    return out


def _sq(v):                                                 # sum over k of (double)t * t, in k order
    s = np.zeros(v.shape[0])
    for k in range(v.shape[1]):
        t = v[:, k].astype(f64)
        s = s + t * t
    return s


def svd4(A, trace=None):
    """cv::SVD::compute(A, w, u, vt, MODIFY_A | FULL_UV) of [N, 4, 4] float32 matrices -> (w [N, 4], vt [N, 4, 4]) float32.
    trace: a list that receives the (p, beta) arrays of every rotation's hypot call, and ("w", W) with the singular values."""
    A = np.asarray(A, f32).reshape(-1, 4, 4)
    N = len(A)
    At = np.ascontiguousarray(np.swapaxes(A, 1, 2))        # _SVDcompute transposes (m == n: no swap), At's rows are A's columns
    Vt = np.tile(np.eye(4, dtype=f32), (N, 1, 1))
    W = np.stack([_sq(At[:, i]) for i in range(4)], 1)
    eps = float(f32(2) * np.finfo(f32).eps)                 # JacobiSVD(float): eps = FLT_EPSILON * 2, minval = FLT_MIN
    active = np.ones(N, bool)
    with np.errstate(all="ignore"):
        for _ in range(30):                                 # max_iter = max(m, 30)
            changed = np.zeros(N, bool)
            for i in range(3):
                for j in range(i + 1, 4):
                    a, b = W[:, i], W[:, j]
                    p = np.zeros(N)
                    for k in range(4):
                        p = p + At[:, i, k].astype(f64) * At[:, j, k].astype(f64)
                    go = active & ~(np.abs(p) <= eps * np.sqrt(a * b))
                    if not go.any():
                        continue
                    p = p * 2
                    beta = a - b
                    gamma = hypot(p, beta)
                    if trace is not None:
                        trace.append((p[go], beta[go]))
                    neg = beta < 0
                    delta = (gamma - beta) * 0.5
                    s_n = np.sqrt(delta / gamma).astype(f32)
                    c_n = (p / (gamma * s_n.astype(f64) * 2)).astype(f32)
                    c_p = np.sqrt((gamma + beta) / (gamma * 2)).astype(f32)
                    s_p = (p / (gamma * c_p.astype(f64) * 2)).astype(f32)
                    c = np.where(neg, c_n, c_p)[:, None]; s = np.where(neg, s_n, s_p)[:, None]
                    Ai, Aj = At[:, i], At[:, j]
                    t0 = c * Ai + s * Aj
                    t1 = -s * Ai + c * Aj
                    g = go[:, None]
                    At[:, i] = np.where(g, t0, Ai); At[:, j] = np.where(g, t1, Aj)
                    W[:, i] = np.where(go, _sq(t0), a); W[:, j] = np.where(go, _sq(t1), b)
                    Vi, Vj = Vt[:, i], Vt[:, j]
                    v0 = c * Vi + s * Vj
                    v1 = -s * Vi + c * Vj
                    Vt[:, i] = np.where(g, v0, Vi); Vt[:, j] = np.where(g, v1, Vj)
                    changed |= go
            active &= changed
            if not active.any():
                break
    W = np.sqrt(np.stack([_sq(At[:, i]) for i in range(4)], 1))
    r = np.arange(N)
    for i in range(3):                                      # selection sort, strict <
        j = np.full(N, i)
        for k in range(i + 1, 4):
            j = np.where(W[r, j] < W[:, k], k, j)
        Wi, Wj = W[r, i].copy(), W[r, j].copy()
        W[r, i], W[r, j] = Wj, Wi
        Vi, Vj = Vt[r, i].copy(), Vt[r, j].copy()
        Vt[r, i], Vt[r, j] = Vj, Vi
    if trace is not None:
        trace.append(("w", W.copy()))
    return W.astype(f32), Vt


# ---------------------------------------------------------------------------------------------------- cv::Mat expression rules
def add_weighted(a, alpha, b, beta, gamma=0.0):
    """cv::addWeighted on CV_32F: (float)((double)a * alpha + (double)b * beta + gamma)."""
    return (np.asarray(a, f32).astype(f64) * alpha + np.asarray(b, f32).astype(f64) * beta + gamma).astype(f32)


def convert_scale(x, scale):
    """Mat::convertTo(CV_32F, scale, 0) on CV_32F: fl(fl(x * (float)scale) + 0)."""
    return (np.asarray(x, f32) * f32(scale)) + f32(0)


def dot3(a, b):
    """Mat::dot of float rows of 3 (double products, summed from 0.0 in order)."""
    a = np.asarray(a, f32).astype(f64); b = np.asarray(b, f32).astype(f64)
    return ((0.0 + a[..., 0] * b[..., 0]) + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def norm3(a):
    """cv::norm (NORM_L2) of a float row of 3, as the double it returns."""
    return np.sqrt(dot3(a, a))


def gemm3(R, x):
    """cv::gemm(R 3x3, x 3x1) on CV_32F: float products summed left to right (tools/probe_cv_gemm.py)."""
    R = np.asarray(R, f32); x = np.asarray(x, f32)
    return np.stack([(R[i, 0] * x[..., 0] + R[i, 1] * x[..., 1]) + R[i, 2] * x[..., 2] for i in range(3)], -1)


# ---------------------------------------------------------------------------------------------------- the triangulation of one pair
def triangulate_points(kp1, kp2, rows, pose1, pose2, cam, scale, sigma2, scale_factor, trace=None):
    """The per-match body of CreateNewMapPoints (LocalMapping.cc:459-634, monocular) for one neighbour's rows (idx1, idx2) ->
    (status [n] int32, x3d [n, 3] float32, written [n] bool: the row got past the w == 0 test)."""
    n = len(rows)
    fx, fy, cx, cy, invfx, invfy = [f32(v) for v in cam]
    T1 = np.asarray(pose1[:12], f32).reshape(3, 4); O1 = np.asarray(pose1[12:15], f32)
    T2 = np.asarray(pose2[:12], f32).reshape(3, 4); O2 = np.asarray(pose2[12:15], f32)
    scale = np.asarray(scale, f32); sigma2 = np.asarray(sigma2, f32); nlev = len(scale)
    i1, i2 = rows[:, 0], rows[:, 1]
    x1k, y1k, o1 = kp1["x"][i1].astype(f32), kp1["y"][i1].astype(f32), kp1["octave"][i1].astype(np.int64)
    x2k, y2k, o2 = kp2["x"][i2].astype(f32), kp2["y"][i2].astype(f32), kp2["octave"][i2].astype(np.int64)
    status = np.full(n, -1, np.int32)
    x3d = np.zeros((n, 3), f32)
    with np.errstate(all="ignore"):
        one = np.ones(n, f32)
        xn1 = np.stack([(x1k - cx) * invfx, (y1k - cy) * invfy, one], 1)                        # :475-476
        xn2 = np.stack([(x2k - cx) * invfx, (y2k - cy) * invfy, one], 1)
        ray1 = gemm3(T1[:, :3].T, xn1); ray2 = gemm3(T2[:, :3].T, xn2)                          # :479-480 (Rwc = Rcw.t())
        cosp = (dot3(ray1, ray2) / (norm3(ray1) * norm3(ray2))).astype(f32)                      # :482
        ok = (cosp < cosp + f32(1)) & (cosp > 0) & (cosp.astype(f64) < 0.9998)                  # :484-497, monocular
        status[~ok] = PARALLAX
        A = np.stack([add_weighted(T1[2], xn1[:, 0:1].astype(f64), T1[0], -1.0),                # :500-504
                      add_weighted(T1[2], xn1[:, 1:2].astype(f64), T1[1], -1.0),
                      add_weighted(T2[2], xn2[:, 0:1].astype(f64), T2[0], -1.0),
                      add_weighted(T2[2], xn2[:, 1:2].astype(f64), T2[1], -1.0)], 1)
        _, vt = svd4(A, trace)                                                                        # :506-509
        v = vt[:, 3]
        wz = ok & (v[:, 3] == 0)                                                                  # :511
        status[wz] = W_ZERO
        live = ok & ~wz
        X = np.stack([v[:, k] * (1.0 / v[:, 3].astype(f64)).astype(f32) + f32(0) for k in range(3)], 1)  # :515, convertTo
        x3d[live] = X[live]

        def cam_coord(T, r):                                                                      # float(Rcw.row(r).dot(x3Dt) + tcw(r))
            return (dot3(np.broadcast_to(T[r, :3], X.shape), X) + f64(T[r, 3])).astype(f32)

        z1 = cam_coord(T1, 2); z2 = cam_coord(T2, 2)                                              # :533-539
        st = live.copy()
        for bad, code in ((z1 <= 0, Z1), (z2 <= 0, Z2), ((o1 < 0) | (o1 >= nlev), OCTAVE1)):
            status[st & bad] = code; st &= ~bad
        oc1 = np.clip(o1, 0, nlev - 1); oc2 = np.clip(o2, 0, nlev - 1)

        def reproj(T, z, xk, yk, s2):                                                             # :543-558 / :574-585
            xx = cam_coord(T, 0); yy = cam_coord(T, 1)
            invz = (1.0 / z.astype(f64)).astype(f32)
            u = fx * xx * invz + cx; vv = fy * yy * invz + cy
            ex = u - xk; ey = vv - yk
            return (ex * ex + ey * ey).astype(f64) > 5.991 * s2.astype(f64)

        for bad, code in ((reproj(T1, z1, x1k, y1k, sigma2[oc1]), REPROJ1), (reproj(T2, z2, x2k, y2k, sigma2[oc2]), REPROJ2)):
            status[st & bad] = code; st &= ~bad
        dist1 = norm3(X - O1).astype(f32); dist2 = norm3(X - O2).astype(f32)                    # :601-605
        bad = (dist1 == 0) | (dist2 == 0)
        status[st & bad] = DIST0; st &= ~bad
        ratio_dist = dist2 / dist1                                                                # :610-616
        ratio_oct = scale[oc1] / scale[oc2]
        rf = f32(1.5) * f32(scale_factor)
        bad = (ratio_dist * rf < ratio_oct) | (ratio_dist > ratio_oct * rf)
        status[st & bad] = SCALE; st &= ~bad
        status[st] = CREATED
    return status, x3d, live


def chain_bad(pairs, nkf):
    """The pairs the batched call gives count -1: an index outside [0, nkf), kf2 == kf1, or a kf2 repeated within its chain (a maximal
    run of consecutive pairs with the same kf1)."""
    bad = []
    seen = set()
    for p, (i, j) in enumerate(pairs):
        if p == 0 or pairs[p - 1][0] != i:
            seen = set()
        b = not (0 <= i < nkf and 0 <= j < nkf) or i == j or j in seen
        if 0 <= i < nkf and 0 <= j < nkf and i != j:
            seen.add(j)
        bad.append(b)
    return bad


def create_points(match, K, pairs, pose, cam, scale, sigma2, scale_factor, trace=None):
    """CreateNewMapPoints over the chains of `pairs`.  match(pair_index, (kf1, kf2), has_mp) -> (count, rows [count, 2]) is the matcher
    (SearchForTriangulation, checkOrientation false); has_mp starts from K["has_mp"] for every chain and gains the KF1 features of the
    created rows pair by pair.  -> list per pair of dict(n, rows, status, x3d, written, nnew); n = -1 for a bad pair."""
    nkf = len(K["n"])
    bad = chain_bad(pairs, nkf)
    out = []
    hm = None
    for p, (i, j) in enumerate(pairs):
        if p == 0 or pairs[p - 1][0] != i:
            hm = K["has_mp"].copy()
        if bad[p]:
            out.append(dict(n=-1, rows=np.zeros((0, 2), np.int32), status=np.zeros(0, np.int32), x3d=np.zeros((0, 3), f32),
                            written=np.zeros(0, bool), nnew=0))
            continue
        n, rows = match(p, (i, j), hm)
        rows = np.asarray(rows, np.int32).reshape(-1, 2)
        status, x3d, written = triangulate_points(K["kps"][i], K["kps"][j], rows, pose[i], pose[j], cam, scale, sigma2, scale_factor,
                                                   trace)
        hm[i, rows[status == CREATED, 0]] = 1                   # mpCurrentKeyFrame->AddMapPoint(pMP, idx1), :624
        out.append(dict(n=int(n), rows=rows, status=status, x3d=x3d, written=written, nnew=int((status == CREATED).sum())))
    return out
