"""CPU restatement of Optimizer::PoseOptimization(Frame*, isCorner) (Optimizer.cc:666-1022) with the reference's g2o: SE3Quat
(se3quat.h), EdgeSE3ProjectXYZOnlyPose (types_six_dof_expmap.cpp), EdgeLineProjectXYZOnlyPose (lineEdge.h:155-240), the Huber kernel
and OptimizationAlgorithmLevenberg::solve (optimization_algorithm_levenberg.cpp:61-161), step by step in the reference's edge order.
It is the parity reference of sslpl_pose_optimization_batch_device (DESIGN.md, "Pose optimisation").  Inputs are read as given: f32
arrays as the device reads them, or f64 arrays for scenes that must be exact in double.  Also: synthetic scenes for the tests and the
timing tool."""
import math

import numpy as np

DELTA_MONO = float(np.float32(math.sqrt(5.991)))   # const float deltaMono = sqrt(5.991), widened by setDelta
DELTA_LINE = float(np.float32(math.sqrt(7.815)))   # deltaStereo, used for the line edges
CHI2_MONO = np.float32(5.991)
CHI2_LINE = np.float32(2) * CHI2_MONO              # 2 * chi2Mono[it], in float
ROUNDS, ITERS, TRIALS = 4, 10, 10


# ---------------------------------------------------------------- SE3Quat: q = (w, x, y, z), t
def quat_normalize_pos(q):
    q = np.array(q, np.float64)
    if q[0] < 0:
        q = -q
    return q * (1.0 / math.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]))


def quat_from_matrix(R):
    """Eigen's Quaternion(const Matrix3&), then SE3Quat::normalizeRotation."""
    R = np.asarray(R, np.float64)
    t = R[0, 0] + R[1, 1] + R[2, 2]
    q = np.zeros(4)
    if t > 0:
        t = math.sqrt(t + 1.0)
        q[0] = 0.5 * t
        t = 0.5 / t
        q[1] = (R[2, 1] - R[1, 2]) * t
        q[2] = (R[0, 2] - R[2, 0]) * t
        q[3] = (R[1, 0] - R[0, 1]) * t
    else:
        i = 0
        if R[1, 1] > R[0, 0]:
            i = 1
        if R[2, 2] > R[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = math.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0)
        v = np.zeros(3)
        v[i] = 0.5 * t
        t = 0.5 / t
        q[0] = (R[k, j] - R[j, k]) * t
        v[j] = (R[j, i] + R[i, j]) * t
        v[k] = (R[k, i] + R[i, k]) * t
        q[1:] = v
    return quat_normalize_pos(q)


def quat_to_matrix(q):
    w, x, y, z = q
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz, txx, txy, txz, tyy, tyz, tzz = tx * w, ty * w, tz * w, tx * x, ty * x, tz * x, ty * y, tz * y, tz * z
    return np.array([[1 - (tyy + tzz), txy - twz, txz + twy],
                     [txy + twz, 1 - (txx + tzz), tyz - twx],
                     [txz - twy, tyz + twx, 1 - (txx + tyy)]])


def quat_mul(a, b):
    return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
                     a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                     a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3],
                     a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]])


def se3_map(P, X):
    """SE3Quat::map of points X [k, 3]: Eigen's quaternion-vector product, then + t."""
    q, t = P
    u, w = q[1:], q[0]
    X = np.asarray(X, np.float64)
    uv = 2 * np.cross(u, X)
    return X + w * uv + np.cross(u, uv) + t


def se3_from_f32(T):
    """Converter::toSE3Quat of a 3x4 row-major pose (12 values)."""
    T = np.asarray(T).reshape(3, 4).astype(np.float64)
    return quat_from_matrix(T[:, :3]), T[:, 3].copy()


def se3_to_f32(P):
    """Converter::toCvMat(SE3Quat), narrowed to float: 12 values, 3x4 row-major."""
    return np.hstack([quat_to_matrix(P[0]), P[1][:, None]]).astype(np.float32).reshape(12)


def skew(w):
    return np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]], np.float64)


def se3_exp(d):
    """SE3Quat::exp of d = (omega, upsilon) -> (R, V, (q, t))."""
    d = np.asarray(d, np.float64)
    w = d[:3]
    theta = math.sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2])
    O = skew(w)
    O2 = O @ O
    if theta < 0.00001:
        R = np.eye(3) + O + O2
        V = R
    else:
        s, c = math.sin(theta), math.cos(theta)
        R = np.eye(3) + s / theta * O + (1 - c) / (theta * theta) * O2
        V = np.eye(3) + (1 - c) / (theta * theta) * O + (theta - s) / theta ** 3 * O2
    return R, V, (quat_from_matrix(R), V @ d[3:])


def se3_exp_mul(d, P):
    """VertexSE3Expmap::oplusImpl: SE3Quat::exp(d) * P."""
    E = se3_exp(d)[2]
    t = se3_map(E, P[1][None])[0]
    return quat_normalize_pos(quat_mul(E[0], P[0])), t


def rot_angle(Ra, Rb):
    """Angle in radians between two rotation matrices, accurate near 0 (also for matrices narrowed to float)."""
    M = np.asarray(Ra, np.float64).T @ np.asarray(Rb, np.float64)
    s = 0.5 * math.sqrt((M[2, 1] - M[1, 2]) ** 2 + (M[0, 2] - M[2, 0]) ** 2 + (M[1, 0] - M[0, 1]) ** 2)
    return math.atan2(s, (np.trace(M) - 1) / 2)


# ---------------------------------------------------------------- edges
def mono_edge(P, X, obs, cam, jac=False):
    """EdgeSE3ProjectXYZOnlyPose: e [k, 2] = obs - pi(P X) and, with jac, J [k, 2, 6] (types_six_dof_expmap.cpp:266-288)."""
    fx, fy, cx, cy = (float(c) for c in cam)
    Y = se3_map(P, X)
    obs = np.asarray(obs, np.float64)
    e = np.stack([obs[:, 0] - (Y[:, 0] / Y[:, 2] * fx + cx), obs[:, 1] - (Y[:, 1] / Y[:, 2] * fy + cy)], 1)
    if not jac:
        return e
    x, y, invz = Y[:, 0], Y[:, 1], 1.0 / Y[:, 2]
    invz2 = invz * invz
    z0 = np.zeros_like(x)
    J = np.stack([np.stack([x * y * invz2 * fx, -(1 + x * x * invz2) * fx, y * invz * fx, -invz * fx, z0, x * invz2 * fx], 1),
                  np.stack([(1 + y * y * invz2) * fy, -x * y * invz2 * fy, -x * invz * fy, z0, -invz * fy, y * invz2 * fy], 1)], 1)
    return e, J


def line_edge(P, X, l, cam, jac=False):
    """EdgeLineProjectXYZOnlyPose: e [k] = l0 u + l1 v + l2 and, with jac, its Jacobian row J [k, 6] (lineEdge.h:161-205)."""
    fx, fy, cx, cy = (float(c) for c in cam)
    Y = se3_map(P, X)
    l = np.asarray(l, np.float64)
    u, v = Y[:, 0] / Y[:, 2] * fx + cx, Y[:, 1] / Y[:, 2] * fy + cy
    e = l[:, 0] * u + l[:, 1] * v + l[:, 2]
    if not jac:
        return e
    x, y, invz = Y[:, 0], Y[:, 1], 1.0 / Y[:, 2]
    invz2 = invz * invz
    lx, ly = l[:, 0], l[:, 1]
    J = np.stack([-fy * ly - fx * lx * x * y * invz2 - fy * ly * y * y * invz2,
                  fx * lx + fx * lx * x * x * invz2 + fy * ly * x * y * invz2,
                  -fx * lx * y * invz + fy * ly * x * invz,
                  fx * lx * invz, fy * ly * invz, -(fx * lx * x + fy * ly * y) * invz2], 1)
    return e, J


def huber(e, delta):
    """RobustKernelHuber::robustify -> (rho, rho') of chi2 values e."""
    dsqr = delta * delta
    s = np.sqrt(np.maximum(e, 0))
    inl = e <= dsqr
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(inl, e, 2 * s * delta - dsqr), np.where(inl, 1.0, delta / s)


def ldlt6(A, b):
    """Dense LDLT of a 6 x 6 system without pivoting -> x, or None when a pivot is not positive."""
    L, D = np.eye(6), np.zeros(6)
    for j in range(6):
        d = A[j, j] - sum(L[j, p] * L[j, p] * D[p] for p in range(j))
        if not (d > 0) or not math.isfinite(d):
            return None
        D[j] = d
        for i in range(j + 1, 6):
            L[i, j] = (A[i, j] - sum(L[i, p] * L[j, p] * D[p] for p in range(j))) / d
    y = np.zeros(6)
    for i in range(6):
        y[i] = b[i] - sum(L[i, p] * y[p] for p in range(i))
    x = np.zeros(6)
    for i in range(5, -1, -1):
        x[i] = y[i] / D[i] - sum(L[p, i] * x[p] for p in range(i + 1, 6))
    return x


# ---------------------------------------------------------------- PoseOptimization
class _Edges:
    def __init__(self, obs, inv, Xp, lq, Xs, Xe, cam):
        self.obs, self.inv, self.Xp, self.lq, self.Xs, self.Xe, self.cam = obs, inv, Xp, lq, Xs, Xe, cam

    def system(self, P, out_p, out_l, robust, want):
        """Robust chi2 of the level-0 edges at P, and with `want` H (6 x 6) and b (OptimizableGraph's b: -sum rho' J^T Omega e)."""
        ap, al = ~out_p, ~out_l
        H, b, chi = np.zeros((6, 6)), np.zeros(6), 0.0
        if ap.any():
            r = mono_edge(P, self.Xp[ap], self.obs[ap], self.cam, want)
            e, J = r if want else (r, None)
            inv = self.inv[ap]
            c2 = e[:, 0] * (inv * e[:, 0]) + e[:, 1] * (inv * e[:, 1])
            r0, r1 = huber(c2, DELTA_MONO) if robust else (c2, np.ones_like(c2))
            chi += float(np.sum(r0))
            if want:
                w = r1 * inv
                H += np.einsum("k,kri,krj->ij", w, J, J)
                b -= np.einsum("k,kri,kr->i", w, J, e)
        if al.any():
            for X in (self.Xs[al], self.Xe[al]):
                r = line_edge(P, X, self.lq[al], self.cam, want)
                e, J = r if want else (r, None)
                c2 = e * e
                r0, r1 = huber(c2, DELTA_LINE) if robust else (c2, np.ones_like(c2))
                chi += float(np.sum(r0))
                if want:
                    H += np.einsum("k,ki,kj->ij", r1, J, J)
                    b -= np.einsum("k,ki,k->i", r1, J, e)
        return chi, H, b


def levenberg(edges, P, out_p, out_l, robust, trace=None):
    """One optimizer.optimize(10) from P -> (final estimate, pose of the last computeActiveErrors, iterations run)."""
    lam = ni = 0.0
    nbad_lm = 0
    x = np.zeros(6)
    last = P
    for it in range(ITERS):
        cur, H, b = edges.system(P, out_p, out_l, robust, True)
        ini = cur
        if it == 0:
            lam, ni, nbad_lm = 1e-5 * float(np.max(np.abs(np.diag(H)))), 2.0, 0
        q = 0
        while True:
            xs = ldlt6(H + lam * np.eye(6), b)
            ok = xs is not None
            if ok:
                x = xs
            trial = se3_exp_mul(x, P)
            last = trial
            tmp = edges.system(trial, out_p, out_l, robust, False)[0]
            if not ok:
                tmp = np.finfo(np.float64).max
            scale = float(sum(x[k] * (lam * x[k] + b[k]) for k in range(6))) + 1e-3
            with np.errstate(over="ignore", invalid="ignore"):
                rho = (cur - tmp) / scale
            if rho > 0 and math.isfinite(tmp):
                alpha = min(1.0 - (2 * rho - 1) ** 3, 2.0 / 3.0)
                lam *= max(1.0 / 3.0, alpha)
                ni = 2.0
                cur = tmp
                P = trial
            else:
                lam *= ni
                ni *= 2
            q += 1
            if not (rho < 0 and q < TRIALS):
                break
        if trace is not None:
            trace.append((cur, lam))
        if q == TRIALS or rho == 0:
            return P, last, it + 1
        nbad_lm = nbad_lm + 1 if (ini - cur) * 1e3 < ini else 0
        if nbad_lm >= 3:
            return P, last, it + 1
    return P, last, ITERS


def pose_optimization(obs, octave, fmp, mp, Tcw, cam, inv_level_sigma2, lineeq=None, fml=None, mlpos=None,
                      outlier=None, line_outlier=None):
    """One frame.  obs [n, 2] (mvKeysUn x, y), octave [n], fmp [n] element indices into mp [nmp, >= 3] (Xw; -1 or outside = NULL);
    lineeq [nl, 3], fml [nl] indices into mlpos [nml, 6] (fml None = no line edges); Tcw 12 values; cam fx fy cx cy.  Returns a dict:
    T (12 f32, what SetPose writes or the input), outlier / line_outlier (the given rows with the edges' flags written), ninlier (the
    return value, -1 for an octave outside the pyramid), pose (q, t) in double, rounds (one dict per round that ran)."""
    obs = np.asarray(obs)
    n = len(obs)
    fmp = np.asarray(fmp, np.int64).reshape(-1)[:n]
    mp = np.asarray(mp).reshape(len(mp), -1) if mp is not None and len(mp) else np.zeros((0, 3))
    octave = np.asarray(octave, np.int64).reshape(-1)[:n]
    inv_tab = np.asarray(inv_level_sigma2)
    out = np.zeros(n, np.uint8) if outlier is None else np.array(outlier, np.uint8)
    ip = np.nonzero((fmp >= 0) & (fmp < len(mp)))[0]
    if fml is not None:
        lineeq = np.asarray(lineeq).reshape(-1, 3)
        nl = len(lineeq)
        fml = np.asarray(fml, np.int64).reshape(-1)[:nl]
        mlpos = np.asarray(mlpos).reshape(-1, 6) if mlpos is not None and len(mlpos) else np.zeros((0, 6))
        il = np.nonzero((fml >= 0) & (fml < len(mlpos)))[0]
    else:
        nl, il = 0, np.zeros(0, np.int64)
    lout = np.zeros(nl, np.uint8) if line_outlier is None else np.array(line_outlier, np.uint8)
    T_in = np.asarray(Tcw, np.float32).reshape(12).copy()
    res = dict(T=T_in, outlier=out, line_outlier=lout, ninlier=0, pose=None, rounds=[])
    if len(ip) and ((octave[ip] < 0) | (octave[ip] >= len(inv_tab))).any():
        res["ninlier"] = -1
        return res
    out[ip] = 0
    lout[il] = 0
    Np, Nl = len(ip), len(il)
    nInit, E = Np + Nl, Np + 2 * Nl
    if nInit < 3:
        return res
    edges = _Edges(obs[ip].astype(np.float64), inv_tab[octave[ip]].astype(np.float64), mp[fmp[ip], :3].astype(np.float64),
                   lineeq[il].astype(np.float64) if Nl else np.zeros((0, 3)),
                   mlpos[fml[il], :3].astype(np.float64) if Nl else np.zeros((0, 3)),
                   mlpos[fml[il], 3:].astype(np.float64) if Nl else np.zeros((0, 3)), cam)
    P0 = se3_from_f32(Tcw)
    out_p, out_l = np.zeros(Np, bool), np.zeros(Nl, bool)
    nBad = 0
    P = P0
    for it in range(ROUNDS):
        robust = it < 3
        start_p, start_l = out_p.copy(), out_l.copy()
        active = int((~out_p).sum() + 2 * (~out_l).sum())
        P, last, iters = levenberg(edges, P0, out_p, out_l, robust) if active else (P0, P0, 0)
        # classification: active points keep the error of the last computeActiveErrors, the rest is recomputed at P
        cp = np.zeros(Np, np.float32)
        if Np:
            e_last = mono_edge(last, edges.Xp, edges.obs, cam)
            e_est = mono_edge(P, edges.Xp, edges.obs, cam)
            e = np.where(out_p[:, None], e_est, e_last)
            cp = (e[:, 0] * (edges.inv * e[:, 0]) + e[:, 1] * (edges.inv * e[:, 1])).astype(np.float32)
        cs = ce = np.zeros(Nl, np.float32)
        if Nl:
            es, ee = line_edge(P, edges.Xs, edges.lq, cam), line_edge(P, edges.Xe, edges.lq, cam)
            cs, ce = (es * es).astype(np.float32), (ee * ee).astype(np.float32)
        out_p = cp > CHI2_MONO
        out_l = (cs > CHI2_LINE) | (ce > CHI2_LINE)
        nBad = int(out_p.sum() + out_l.sum())
        res["rounds"].append(dict(start=P0, robust=robust, active_p=~start_p, active_l=~start_l, ran=bool(active), iters=iters,
                                  est=P, last=last, chi2_p=cp, chi2_s=cs, chi2_e=ce, nbad=nBad))
        if E < 10:
            break
    out[ip] = out_p
    lout[il] = out_l
    res.update(T=se3_to_f32(P), ninlier=nInit - nBad, pose=P)
    return res


def in_band(res, rel=1e-5):
    """Per point / per line of the frame's edges (in feature order): whether any round's chi2 lay within a relative `rel` of its
    threshold (the parity contract excuses those)."""
    bp = bl = None
    for r in res["rounds"]:
        p = np.abs(r["chi2_p"].astype(np.float64) - float(CHI2_MONO)) <= rel * float(CHI2_MONO)
        t = float(CHI2_LINE)
        l = (np.abs(r["chi2_s"].astype(np.float64) - t) <= rel * t) | (np.abs(r["chi2_e"].astype(np.float64) - t) <= rel * t)
        bp = p if bp is None else bp | p
        bl = l if bl is None else bl | l
    return bp, bl


# ---------------------------------------------------------------- synthetic scenes
def camera(width, height):
    """A pinhole camera for a width x height frame (fx = fy = 0.8 width)."""
    return np.array([0.8 * width, 0.8 * width, width / 2.0, height / 2.0], np.float32)


def pyramid(nlevels=8, scale=1.2):
    """mvLevelSigma2 and mvInvLevelSigma2 of an ORB pyramid, float."""
    s2 = np.array([scale ** (2 * l) for l in range(nlevels)], np.float32)
    return s2, (np.float32(1) / s2).astype(np.float32)


def random_pose(rng, max_deg=20.0, max_t=0.5):
    R = se3_exp(np.concatenate([rng.normal(size=3) * math.radians(max_deg) / 2, np.zeros(3)]))[0]
    return R, rng.uniform(-max_t, max_t, 3)


def perturb(R, t, rng, deg, dt):
    """(R, t) rotated by `deg` degrees about a random axis and moved by `dt` in a random direction."""
    a = rng.normal(size=3)
    a *= math.radians(deg) / np.linalg.norm(a)
    d = rng.normal(size=3)
    d *= dt / np.linalg.norm(d)
    return se3_exp(np.concatenate([a, np.zeros(3)]))[0] @ R, t + d


def pose12(R, t, dtype=np.float32):
    return np.hstack([R, np.asarray(t).reshape(3, 1)]).astype(dtype).reshape(12)


def make_scene(rng, width, height, npts, nlines, outlier_frac=0.0, noise=1.0, deg=2.0, dt=0.05, nlevels=8, dtype=np.float32):
    """A frame with npts points and nlines lines seen from a random ground-truth pose, an initial pose `deg` / `dt` away, Gaussian
    pixel noise of `noise` x the level's scale, and a fraction `outlier_frac` of gross outliers (a point, or both ends of a line,
    moved 20 to 200 px).  dtype float32 gives the device's input types; float64 keeps a noise-free scene exact."""
    cam = camera(width, height).astype(np.float64)
    fx, fy, cx, cy = cam
    R, t = random_pose(rng)
    s2, inv = pyramid(nlevels)

    def back(u, v, z):
        Xc = np.stack([(u - cx) / fx * z, (v - cy) / fy * z, z], 1)
        return (Xc - t) @ R                                            # R^T (Xc - t)

    def proj(X):
        Y = X @ R.T + t
        return np.stack([Y[:, 0] / Y[:, 2] * fx + cx, Y[:, 1] / Y[:, 2] * fy + cy], 1)

    def gross(k):                                                      # 20 to 200 px in a random direction
        a, r = rng.uniform(0, 2 * np.pi, k), rng.uniform(20, 200, k)
        return np.stack([r * np.cos(a), r * np.sin(a)], 1)

    oct_ = rng.integers(0, nlevels, npts)
    Xw = back(rng.uniform(0, width, npts), rng.uniform(0, height, npts), rng.uniform(1.0, 8.0, npts)).astype(dtype)
    obs = proj(Xw.astype(np.float64)) + noise * np.sqrt(s2[oct_])[:, None] * rng.normal(size=(npts, 2))
    bad_p = rng.random(npts) < outlier_frac
    obs[bad_p] += gross(bad_p.sum())
    zs, ze = rng.uniform(1.0, 8.0, nlines), rng.uniform(1.0, 8.0, nlines)
    S = back(rng.uniform(0, width, nlines), rng.uniform(0, height, nlines), zs)
    Ee = back(rng.uniform(0, width, nlines), rng.uniform(0, height, nlines), ze)
    mlpos = np.hstack([S, Ee])
    ps = proj(S) + noise * rng.normal(size=(nlines, 2))
    pe = proj(Ee) + noise * rng.normal(size=(nlines, 2))
    bad_l = rng.random(nlines) < outlier_frac
    ps[bad_l] += gross(bad_l.sum())
    pe[bad_l] += gross(bad_l.sum())
    hs = np.hstack([ps, np.ones((nlines, 1))])
    he = np.hstack([pe, np.ones((nlines, 1))])
    l = np.cross(hs, he)
    lineeq = l / np.sqrt(l[:, :1] ** 2 + l[:, 1:2] ** 2)               # the keyline function, normalised as the extractor does
    R0, t0 = perturb(R, t, rng, deg, dt)
    return dict(obs=obs.astype(dtype), octave=oct_.astype(np.int32), fmp=np.arange(npts, dtype=np.int32), mp=Xw,
                lineeq=lineeq, fml=np.arange(nlines, dtype=np.int32), mlpos=mlpos, T0=pose12(R0, t0, dtype), R=R, t=t,
                bad_p=bad_p, bad_l=bad_l, cam=cam.astype(dtype), inv=inv.astype(dtype) if dtype == np.float64 else inv,
                width=width, height=height)


def run_scene(sc, lines=True, points=True, **kw):
    """pose_optimization on a scene from make_scene; points / lines False drop that kind of edge."""
    fmp = sc["fmp"] if points else np.full_like(sc["fmp"], -1)
    return pose_optimization(sc["obs"], sc["octave"], fmp, sc["mp"], sc["T0"], sc["cam"], sc["inv"],
                             lineeq=sc["lineeq"], fml=sc["fml"] if lines else None, mlpos=sc["mlpos"], **kw)
