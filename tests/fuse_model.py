"""Inputs and host-side models for the batched Fuse tests (tests/test_kf_fuse_gpu.py, tests/test_kf_fuse_cpu.py):
LocalMapping::SearchInNeighbors (LocalMapping.cc:1178-1279) with ORBmatcher::Fuse (ORBmatcher.cc:828-973) and LSDmatcher::Fuse
(LSDmatcher.cpp:417-548) over a keyframe set of synthetic frames.

Keyframe k of the set is synthetic frame k of one group (tools/synth.py): the base image moved by a rotation about the image centre and a
translation.  With fx = fy = F, (cx, cy) = the image centre and the world = keyframe 0's camera, the pose Tcw = [R | t] with R the
in-plane rotation and t = shift * Z0 / F reproduces that motion exactly for points at depth Z0 and within a fraction of a pixel for the
depths used here, so that projections land next to the features they came from and fusions happen.

Elements (MapPoints, MapLines) are keyframe features back-projected at about Z0, with normals, distance ranges and predicted levels that
mostly pass the gates, as in scenarios.fuse_points_scenario / fuse_lines_scenario.  A few get one perturbation each, which one gate of
the projection or search stage then decides (POINT_GATES / LINE_GATES); the CPU test checks that undoing each one changes results."""
import numpy as np

from test_kf_triangulation_gpu import warp

F = 500.0
NLEV = 8
SF = (np.float32(1.2) ** np.arange(NLEV)).astype(np.float32)
INV_SIGMA2 = (np.float32(1.0) / (SF * SF)).astype(np.float32)
LOGS = np.float32(np.log(np.float32(1.2)))            # KeyFrame::mfLogScaleFactor = log(mfScaleFactor)
TH = 3.0                                               # Fuse's default th
TH_LOW = 50
Z0 = 3.0
INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
POINT_GATES = ("depth", "bounds", "range", "angle", "level", "chi2", "desc")
LINE_GATES = ("depth", "bounds", "range", "angle", "level", "pyramid", "desc")


def camera(W, H):
    return np.array([F, F, W / 2.0, H / 2.0], np.float32), np.array([0.0, W, 0.0, H], np.float32)


def poses(nkf, group, W, H):
    """pose[k][15] = Tcw (3x4 row-major), Ow of keyframe k (see the module docstring)."""
    P = np.zeros((nkf, 15), np.float32)
    for k in range(nkf):
        M = warp(k, group, W, H)
        s = np.array([4.0, -3.0]) * ((k % group) / (group - 1))
        T = np.zeros((3, 4)); T[:2, :2] = M[:2, :2]; T[2, 2] = 1.0; T[:2, 3] = s * Z0 / F
        T = T.astype(np.float32)
        P[k, :12] = T.reshape(-1)
        P[k, 12:] = -(T[:, :3].astype(np.float64).T @ T[:, 3].astype(np.float64))
    return P


def _backproject(k, x, y, z, group, W, H):
    p = np.linalg.inv(warp(k, group, W, H)) @ np.stack([x, y, np.ones_like(x)]).astype(np.float64)
    return np.stack([(p[0] - W / 2.0) / F * z, (p[1] - H / 2.0) / F * z, z], 1)


def _flip_bits(rng, d, p):
    d = d.copy(); m = rng.random(d.shape + (8,)) < p
    return d ^ np.packbits(m, axis=-1, bitorder="little").reshape(d.shape)


def _assign_gates(rng, m, gates, p):
    """One perturbation class per element: -1 none, else an index into `gates` (each class gets about p of the elements)."""
    u = rng.random(m)
    cls = np.full(m, -1, np.int32)
    for g in range(len(gates)):
        cls[(u >= g * p) & (u < (g + 1) * p)] = g
    return cls


def point_table(rng, src, kps, desc, P, group, W, H, p_gate=0.03):
    """MapPoints from keyframe features src = [(kf, idx)]: dict(mp [m, 9] f32 = Xw, normal, minInv, maxInv, maxRaw; desc [m, 32];
    gate [m] = the perturbation class; base = the unperturbed mp / desc)."""
    src = np.asarray(src, np.int64).reshape(-1, 2); m = len(src)
    kp = kps[src[:, 0], src[:, 1]]
    z = Z0 * (1 + rng.uniform(-0.08, 0.08, m))
    X = np.concatenate([_backproject(int(k), kp["x"][i:i + 1].astype(np.float64), kp["y"][i:i + 1].astype(np.float64), z[i:i + 1], group, W, H)
                        for i, k in enumerate(src[:, 0])]) if m else np.zeros((0, 3))
    Ow = P[src[:, 0], 12:].astype(np.float64)
    PO = X - Ow; dist = np.linalg.norm(PO, axis=1)
    nrm = PO / dist[:, None] + rng.normal(0, 0.2, (m, 3)); nrm /= np.linalg.norm(nrm, axis=1)[:, None]
    oct_ = kp["octave"].astype(np.float64)
    max_raw = dist * 1.2 ** (oct_ + rng.uniform(-0.9, -0.05, m))
    d = _flip_bits(rng, desc[src[:, 0], src[:, 1]], 0.02)
    base = _pack_points(X, nrm, max_raw)
    gate = _assign_gates(rng, m, POINT_GATES, p_gate)
    X2, n2, r2, d2 = X.copy(), nrm.copy(), max_raw.copy(), d.copy()
    g = dict(zip(POINT_GATES, range(len(POINT_GATES))))
    s = gate == g["depth"]; X2[s] = 2 * Ow[s] - X[s]                                  # mirrored through the camera: behind it
    s = gate == g["bounds"]; X2[s, 0] += X[s, 2] * W / F                               # one image width to the right
    s = gate == g["range"]; r2[s] = dist[s] * 0.5                                      # dist > maxInv
    s = gate == g["angle"]; n2[s] *= -1                                                # seen from behind
    s = gate == g["level"]; r2[s] = dist[s] * 1.2 ** (oct_[s] + 2.5)                   # predicted level 3 above the octave
    s = gate == g["chi2"]; X2[s, :2] += (1.9 * 1.2 ** oct_[s] * X[s, 2] / F)[:, None]   # inside the window, outside the chi-square
    s = gate == g["desc"]; d2[s] = _flip_bits(rng, d[s], 0.35)                         # nearest descriptor above TH_LOW
    return dict(mp=_pack_points(X2, n2, r2), desc=d2, gate=gate, base=base, base_desc=d, src=src)


def _pack_points(X, nrm, max_raw):
    max_raw = max_raw.astype(np.float32)
    min_raw = (max_raw / np.float32(1.2 ** (NLEV - 1))).astype(np.float32)
    return np.concatenate([X, nrm, (min_raw * np.float32(0.8))[:, None], (max_raw * np.float32(1.2))[:, None], max_raw[:, None]],
                          1).astype(np.float32)


def line_table(rng, src, kl, ldesc, P, group, W, H, p_gate=0.03):
    """MapLines from keyframe lines src = [(kf, idx)]: dict(ml [m, 12] f32 = SP, EP, normal, minInv, maxInv, maxRaw; desc; gate; base)."""
    src = np.asarray(src, np.int64).reshape(-1, 2); m = len(src)
    k = kl[src[:, 0], src[:, 1]]
    zs, ze = Z0 * (1 + rng.uniform(-0.05, 0.05, m)), Z0 * (1 + rng.uniform(-0.05, 0.05, m))
    SP = np.zeros((m, 3)); EP = np.zeros((m, 3))
    for i, f in enumerate(src[:, 0]):
        SP[i] = _backproject(int(f), k["startPointX"][i:i + 1].astype(np.float64), k["startPointY"][i:i + 1].astype(np.float64), zs[i:i + 1], group, W, H)
        EP[i] = _backproject(int(f), k["endPointX"][i:i + 1].astype(np.float64), k["endPointY"][i:i + 1].astype(np.float64), ze[i:i + 1], group, W, H)
    SP = SP.astype(np.float32).astype(np.float64); EP = EP.astype(np.float32).astype(np.float64)
    Ow = P[src[:, 0], 12:].astype(np.float64)
    OM = 0.5 * (SP + EP) - Ow; dist = np.linalg.norm(OM, axis=1)
    nrm = OM / dist[:, None] + rng.normal(0, 0.2, (m, 3)); nrm /= np.linalg.norm(nrm, axis=1)[:, None]
    max_raw = dist * 1.2 ** rng.uniform(-0.9, -0.05, m)
    d = _flip_bits(rng, ldesc[src[:, 0], src[:, 1]], 0.02)
    base = _pack_lines(SP, EP, nrm, max_raw)
    gate = _assign_gates(rng, m, LINE_GATES, p_gate)
    SP2, EP2, n2, r2, d2 = SP.copy(), EP.copy(), nrm.copy(), max_raw.copy(), d.copy()
    g = dict(zip(LINE_GATES, range(len(LINE_GATES))))
    s = gate == g["depth"]; SP2[s] = 2 * Ow[s] - SP[s]; EP2[s] = 2 * Ow[s] - EP[s]
    s = gate == g["bounds"]; SP2[s, 0] += SP[s, 2] * W / F; EP2[s, 0] += EP[s, 2] * W / F
    s = gate == g["range"]; r2[s] = dist[s] * 0.5
    s = gate == g["angle"]; n2[s] *= -1
    s = gate == g["level"]; r2[s] = dist[s] * 1.2 ** 2.5                               # level 3: the keylines are all octave 0
    s = gate == g["pyramid"]; r2[s] = dist[s] * 1.2 ** 7.5                             # level 8 = nlevels: outside the pyramid
    s = gate == g["desc"]; d2[s] = _flip_bits(rng, d[s], 0.35)
    return dict(ml=_pack_lines(SP2, EP2, n2, r2), desc=d2, gate=gate, base=base, base_desc=d, src=src)


def _pack_lines(SP, EP, nrm, max_raw):
    max_raw = max_raw.astype(np.float32)
    min_raw = (max_raw / np.float32(1.2 ** (NLEV - 1))).astype(np.float32)
    return np.concatenate([SP, EP, nrm, (min_raw * np.float32(0.8))[:, None], (max_raw * np.float32(1.2))[:, None], max_raw[:, None]],
                          1).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------- oracle per entry
def oracle_points(oracle, K, pose, mp, mpdesc, entries, skip, th=TH):
    """(best_idx, best_dist) per entry: orc_fuse_project_points then orc_fuse_points_search on the entry's keyframe; (-1, -1) for an
    index out of range.  K = dict(kps, desc, n, cam, bounds).  Also returns the projections per keyframe (for the single call)."""
    E = np.asarray(entries, np.int64).reshape(-1, 2); nkf = len(K["n"]); nmp = len(mp)
    bi = np.full(len(E), -1, np.int32); bd = np.full(len(E), -1, np.int32)
    ok = (E[:, 0] >= 0) & (E[:, 0] < nkf) & (E[:, 1] >= -1) & (E[:, 1] < nmp)
    per_kf = {}
    for k in np.unique(E[ok, 0]):
        sel = np.nonzero(ok & (E[:, 0] == k))[0]; e = E[sel, 1]
        rows = mp[np.maximum(e, 0)]; sk = (np.asarray(skip)[sel] != 0) | (e < 0)
        T = pose[k]; n = int(K["n"][k]); kp = K["kps"][k, :n]
        q = oracle.fuse_project_points(sk.astype(np.uint8), rows[:, :3], rows[:, 3:6], rows[:, 6], rows[:, 7], rows[:, 8], T[:12].reshape(3, 4), T[12:],
                                       np.append(K["cam"], 0.0), K["bounds"], NLEV, LOGS)
        d = mpdesc[np.maximum(e, 0)]
        args = (q, d, K["desc"][k, :n], kp["x"], kp["y"], kp["octave"].astype(np.int32), None, K["bounds"], SF, INV_SIGMA2, th)
        bi[sel], bd[sel] = oracle.fuse_points_search(*args)
        per_kf[int(k)] = (sel, args)
    return bi, bd, per_kf


def keyline_rows(kl):
    return np.stack([kl["pt_x"], kl["pt_y"], kl["angle"]], 1).astype(np.float32)


def oracle_lines(oracle, K, pose, ml, mldesc, entries, skip, th=TH):
    """As oracle_points for MapLines: orc_fuse_project_lines then orc_fuse_lines_search.  K = dict(kl, ldesc, nl, cam, bounds)."""
    E = np.asarray(entries, np.int64).reshape(-1, 2); nkf = len(K["nl"]); nml = len(ml)
    bi = np.full(len(E), -1, np.int32); bd = np.full(len(E), -1, np.int32)
    ok = (E[:, 0] >= 0) & (E[:, 0] < nkf) & (E[:, 1] >= -1) & (E[:, 1] < nml)
    per_kf = {}
    for k in np.unique(E[ok, 0]):
        sel = np.nonzero(ok & (E[:, 0] == k))[0]; e = E[sel, 1]
        rows = ml[np.maximum(e, 0)]; sk = (np.asarray(skip)[sel] != 0) | (e < 0)
        T = pose[k]; n = int(K["nl"][k]); kl = K["kl"][k, :n]
        q = oracle.fuse_project_lines(sk.astype(np.uint8), rows[:, :6], rows[:, 6:9], rows[:, 9], rows[:, 10], rows[:, 11], T[:12].reshape(3, 4), T[12:],
                                      np.append(K["cam"], 0.0), K["bounds"], NLEV, LOGS)
        args = (q, mldesc[np.maximum(e, 0)], K["ldesc"][k, :n], keyline_rows(kl), kl["octave"].astype(np.int32), SF, th)
        bi[sel], bd[sel] = oracle.fuse_lines_search(*args)
        per_kf[int(k)] = (sel, args)
    return bi, bd, per_kf


def oracle_levels(oracle, ratio, log_scale_factor, nlevels, chunk=1 << 20):
    """The oracle's own (int)ceil(logf(ratio) / logScaleFactor) of MapLine::PredictScale (not clamped), read from orc_fuse_project_lines'
    level output for a line whose mid-point is at distance exactly 1 from the camera (SP = EP = (0, 0, 1), Ow = 0, Tcw = I): its
    ratio is maxRaw / 1 = maxRaw, bit for bit, for every float, NaN and infinities included."""
    C = __import__("ctypes")
    ratio = np.ascontiguousarray(ratio, np.float32).reshape(-1)
    n = min(len(ratio), chunk)
    Pw = np.zeros((n, 6), np.float32); Pw[:, 2] = 1; Pw[:, 5] = 1
    nrm = np.zeros((n, 3), np.float32); nrm[:, 2] = 1
    mn = np.zeros(n, np.float32); mx = np.full(n, 2, np.float32); skip = np.zeros(n, np.uint8)
    T = np.eye(3, 4, dtype=np.float32); Ow = np.zeros(3, np.float32); cam = np.array([500, 500, 320, 240, 0], np.float32)
    bnd = np.array([0, 640, 0, 480], np.float32)
    act = np.empty(n, np.uint8); proj = np.empty((n, 4), np.float32)
    out = np.empty(len(ratio), np.int32)
    p = oracle._p
    for a in range(0, len(ratio), n):
        b = min(a + n, len(ratio))
        oracle.lib().orc_fuse_project_lines(b - a, p(skip), p(Pw), p(nrm), p(mn), p(mx), p(ratio[a:b]), p(T), p(Ow), p(cam), p(bnd), int(nlevels),
                                            C.c_float(log_scale_factor), p(act), p(proj), p(out[a:b]))
    return out


def window_levels(L, nlevels, clamp):
    """The oracle's raw level L in the form sslpl_matcher_debug_predict_scale returns it."""
    L = np.asarray(L, np.int64)
    if clamp:
        return np.clip(np.where(L == INT_MIN, 0, L), 0, nlevels - 1).astype(np.int32)
    return np.where(L == INT_MIN, INT_MIN, np.clip(L, -1, nlevels)).astype(np.int32)


def table_levels(thr, ratio, clamp):
    """The device rule over a threshold table, restated in numpy: count thr[k] <= ratio; non-finite or non-positive ratios as INT_MIN."""
    nlevels = len(thr) - 1
    c = np.zeros(len(ratio), np.int32)
    for t in thr:
        c += ratio >= t
    bad = ~((ratio > 0) & (ratio < np.inf))
    if clamp:
        return np.where(bad, 0, np.clip(c - 1, 0, nlevels - 1)).astype(np.int32)
    return np.where(bad, INT_MIN, c - 1).astype(np.int32)


# ---------------------------------------------------------------------------------------------------------------- replay model
class MapModel:
    """The bookkeeping of SearchInNeighbors' Fuse calls: keyframe slots, observations (KeyFrame -> index; iterated in keyframe-index
    order), Observations() counts, bad flags and descriptors.  MapPoint::Replace (MapPoint.cc:182-220) = MapLine::Replace
    (MapLine.cpp:183-219); AddObservation ignores a keyframe already observed (MapPoint.cc:103-114, monocular: +1);
    ComputeDistinctiveDescriptors (MapPoint.cc:247-312) = the medoid of the observed descriptors, first least median wins."""

    def __init__(self, kf_desc, n):
        self.kf_desc = kf_desc
        self.slot = [np.full(int(c), -1, np.int64) for c in n]
        self.obs, self.nobs, self.bad, self.desc, self.ver = [], [], [], [], []
        self.replaced = {"into_existing": 0, "into_incoming": 0}

    def add(self, observations):
        e = len(self.obs)
        self.obs.append({}); self.nobs.append(0); self.bad.append(False); self.desc.append(np.zeros(32, np.uint8)); self.ver.append(0)
        for k, i in observations:
            self.add_observation(e, k, i); self.slot[k][i] = e
        self.compute_desc(e)
        return e

    def add_observation(self, e, k, i):
        if k in self.obs[e]:
            return
        self.obs[e][k] = int(i); self.nobs[e] += 1

    def compute_desc(self, e):
        ds = np.array([self.kf_desc[k][i] for k, i in sorted(self.obs[e].items())], np.uint8)
        if len(ds) == 0:
            return
        D = np.unpackbits(ds[:, None, :] ^ ds[None, :, :], axis=-1).sum(-1)
        med = np.sort(D, axis=1)[:, int(0.5 * (len(ds) - 1))]
        self.desc[e] = ds[int(np.argmin(med))].copy(); self.ver[e] += 1

    def replace(self, this, other):
        if this == other:
            return
        o = self.obs[this]; self.obs[this] = {}; self.bad[this] = True
        for k, i in sorted(o.items()):
            if k not in self.obs[other]:
                self.slot[k][i] = other; self.add_observation(other, k, i)
            else:
                self.slot[k][i] = -1
        self.compute_desc(other)

    def apply(self, k, e, bi, bd):
        """The end of ORBmatcher::Fuse / LSDmatcher::Fuse for one element (ORBmatcher.cc:952-970): True when it counts as fused."""
        if not (bd <= TH_LOW and bi >= 0):
            return False
        inkf = int(self.slot[k][bi])
        if inkf >= 0:
            if not self.bad[inkf]:
                if self.nobs[inkf] > self.nobs[e]:
                    self.replace(e, inkf); self.replaced["into_existing"] += 1
                else:
                    self.replace(inkf, e); self.replaced["into_incoming"] += 1
        else:
            self.add_observation(e, k, bi); self.slot[k][bi] = e
        return True

    def state(self):
        return ([s.tolist() for s in self.slot], list(self.bad), [sorted(o.items()) for o in self.obs], list(self.nobs),
                [d.tobytes() for d in self.desc])


def replay_map(rng, kf_desc, n, kfs, p_own=0.5, p_extra=0.3):
    """Elements made from p_own of the features of every keyframe in kfs, each observed by its own keyframe; p_extra of them also observed
    by one or two other keyframes of kfs at free slots (so that Observations() differs and IsInKeyFrame holds for some targets)."""
    M = MapModel(kf_desc, n)
    src = []
    for k in kfs:
        for i in np.nonzero(rng.random(int(n[k])) < p_own)[0]:
            src.append((k, int(i)))
    for k, i in src:
        obs = [(k, i)]
        if rng.random() < p_extra:
            for k2 in rng.choice(kfs, int(rng.integers(1, 3)), replace=False):
                free = np.nonzero(M.slot[k2] < 0)[0]
                if k2 != k and len(free):
                    obs.append((int(k2), int(rng.choice(free))))
        M.add(obs)
    return M, src


def search_in_neighbors(M, cur, targets, run, points=True):
    """SearchInNeighbors' two Fuse phases (LocalMapping.cc:1203-1224 / :1240-1264) on the model.  run(entries, M, points) applies the
    entries in order through M.apply and returns whether each one fused.  Returns the fused counts of the reference's Fuse calls: one
    per target, then the candidate call."""
    matches = [int(e) for e in M.slot[cur]]                         # GetMapPointMatches(): NULL entries included
    A = [(k, e) for k in targets for e in matches]
    fusedA = run(A, M, points)
    counts = [int(sum(fusedA[j * len(matches):(j + 1) * len(matches)])) for j in range(len(targets))]
    seen, C = set(), []
    for k in targets:
        for e in M.slot[k]:
            e = int(e)
            if e < 0 or M.bad[e] or e in seen:
                continue
            seen.add(e); C.append((cur, e))
    counts.append(int(sum(run(C, M, points))))
    for e in M.slot[cur]:
        if e >= 0 and not M.bad[e]:
            M.compute_desc(int(e))
    return counts


def skipped(M, k, e, points):
    return e < 0 or M.bad[e] or (points and k in M.obs[e])


def run_sequential(one):
    """The reference's order: every entry is projected and searched with the map as the earlier entries left it.
    one(k, e, M) -> (best_idx, best_dist) for element e's current state."""
    def run(entries, M, points=True):
        out = []
        for k, e in entries:
            if skipped(M, k, e, points):
                out.append(False); continue
            out.append(M.apply(k, e, *one(k, e, M)))
        return out
    return run


def run_batched(batch, stats):
    """One batched call per phase with the skip flags as they are at the call, then the caller's rule: apply in entry order, re-test
    isBad / IsInKeyFrame, re-submit an entry whose element's descriptor was recomputed since the call.
    batch(entries, skip, M) -> (best_idx, best_dist) arrays."""
    def run(entries, M, points=True):
        if not entries:
            return []
        skip = np.array([skipped(M, k, e, points) for k, e in entries], np.uint8)
        ver = list(M.ver)
        bi, bd = batch(entries, skip, M)
        stats["calls"] += 1
        out = []
        for j, (k, e) in enumerate(entries):
            if skipped(M, k, e, points):
                out.append(False); continue
            b, d = int(bi[j]), int(bd[j])
            if M.ver[e] != ver[e]:
                (b,), (d,) = batch([(k, e)], np.zeros(1, np.uint8), M)
                stats["resubmitted"] += 1
            out.append(M.apply(k, e, b, d))
        return out
    return run
