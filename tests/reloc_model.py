"""NumPy restatement of the relocalisation matchers of Tracking::Relocalization (Tracking.cc:1961-2121):
ORBmatcher::SearchByProjection(Frame &F, KeyFrame *pKF, sAlreadyFound, th, ORBdist) (ORBmatcher.cc:1475-1602) and the candidate table as a
pair list.  The float work follows the reference's operation order in float32 (no contraction); Frame::GetFeaturesInArea and the
(int)ceil(logf(ratio) / mfLogScaleFactor) of MapPoint::PredictScale come from the CPU oracle.  Also the ctypes entry to the reference's own
matcher (oracle/_ref/libref_reloc.so, built by oracle/ref_reloc_build.sh)."""
import ctypes as C
import os

import numpy as np

from fuse_model import oracle_levels, window_levels

f32, f64 = np.float32, np.float64
HISTO_LENGTH = 30
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libref_reloc.so")


def rot_bin(a1, a2):
    """ORBmatcher.cc:1568-1573: rot = a1 - a2 (+360 when negative), bin = round(rot / 30) with C's roundf, 30 -> 0."""
    rot = f32(f32(a1) - f32(a2))
    if rot < 0:
        rot = f32(rot + f32(360.0))
    x = f32(rot * f32(f32(1.0) / f32(HISTO_LENGTH)))
    t = np.floor(x)
    b = int(t) + (1 if x - t >= 0.5 else 0)
    return 0 if b == HISTO_LENGTH else b


def three_maxima(hist):
    """ComputeThreeMaxima (ORBmatcher.cc:1604-1645): the kept bins, -1 for a dropped one."""
    m1 = m2 = m3 = 0; i1 = i2 = i3 = -1
    for i, s in enumerate(hist):
        if s > m1: m3, m2, m1, i3, i2, i1 = m2, m1, s, i2, i1, i
        elif s > m2: m3, m2, i3, i2 = m2, s, i2, i
        elif s > m3: m3, i3 = s, i
    if f32(m2) < f32(0.1) * f32(m1): i2 = i3 = -1
    elif f32(m3) < f32(0.1) * f32(m1): i3 = -1
    return i1, i2, i3


def element_table(Xw, mindist, maxdist):
    """d_mp[m][9] = Xw, normal (unused here, 0), GetMinDistanceInvariance() = 0.8f * mfMinDistance, GetMaxDistanceInvariance() =
    1.2f * mfMaxDistance, mfMaxDistance."""
    el = np.zeros((len(Xw), 9), f32)
    el[:, :3] = Xw
    el[:, 6] = f32(0.8) * np.asarray(mindist, f32); el[:, 7] = f32(1.2) * np.asarray(maxdist, f32); el[:, 8] = maxdist
    return el


def search_by_projection_kf(oracle, kf_kps, kfmp, el, eldesc, bad, found, kps, desc, held, Tcw, cam, bounds, sf, log_sf, th, orb_dist,
                            check_ori=True):
    """SearchByProjection(F, pKF, sAlreadyFound, th, ORBdist).  Keyframe feature i holds element kfmp[i] (< 0 or >= len(el): NULL) of the
    table el[m][9] (element_table) / eldesc[m][32], bad[m] = isBad() (None = none), found[i] = sAlreadyFound.count(vpMPs[i]) (None = none).
    Frame: keypoints kps (mvKeysUn), descriptors, held[j] = mvpMapPoints[j] != NULL (None = none), pose Tcw 3x4.  Returns (nmatches,
    assign[j]): keyframe feature index, -1 untouched, -2 written then NULLed by the rotation check."""
    T = np.asarray(Tcw, f32).reshape(-1)[:12]
    fx, fy, cx, cy = (f32(c) for c in cam[:4])
    minX, maxX, minY, maxY = (f32(b) for b in bounds)
    n1, n2, nel = len(kfmp), len(kps), len(el)
    # Ow = -Rcw.t()*tcw: cv::gemm's general path (double accumulation, one rounding)
    Td = T.astype(f64)
    Ow = np.array([-((Td[r] * Td[3] + Td[4 + r] * Td[7]) + Td[8 + r] * Td[11]) for r in range(3)]).astype(f32)
    e = np.asarray(kfmp, np.int64)
    ok = (e >= 0) & (e < nel)
    ee = np.where(ok, e, 0)
    if bad is not None: ok &= np.asarray(bad, np.uint8)[ee] == 0
    if found is not None: ok &= np.asarray(found, np.uint8)[:n1] == 0
    X = el[ee, :3]
    row = lambda k: ((T[k] * X[:, 0] + T[k + 1] * X[:, 1]) + T[k + 2] * X[:, 2]) + T[k + 3]    # Rcw*x3Dw+tcw in float (plain gemm)
    with np.errstate(all="ignore"):
        xc, yc, zc = row(0), row(4), row(8)
        invz = (1.0 / zc.astype(f64)).astype(f32)
        u = (fx * xc) * invz + cx; v = (fy * yc) * invz + cy
        ok &= ~((u < minX) | (u > maxX) | (v < minY) | (v > maxY))
        PO = (X - Ow).astype(f64)
        dist = np.sqrt((PO[:, 0] * PO[:, 0] + PO[:, 1] * PO[:, 1]) + PO[:, 2] * PO[:, 2]).astype(f32)
        ok &= ~((dist < el[ee, 6]) | (dist > el[ee, 7]))
        ratio = (el[ee, 8] / dist).astype(f32)
    lvl = window_levels(oracle_levels(oracle, ratio, log_sf, len(sf)), len(sf), True) if n1 else np.zeros(0, np.int32)
    kx, ky = np.asarray(kps["x"], f32), np.asarray(kps["y"], f32)
    oct2 = np.asarray(kps["octave"], np.int32)
    claimed = np.zeros(n2, bool) if held is None else np.asarray(held[:n2]) != 0
    assign = np.full(n2, -1, np.int32)
    hist = [[] for _ in range(HISTO_LENGTH)]
    nm = 0
    for i in np.nonzero(ok)[0]:
        L = int(lvl[i])
        r = f32(f32(th) * f32(sf[L]))
        win = oracle.features_in_area(kx, ky, oct2, bounds, u[i], v[i], r, L - 1, L + 1)
        best, bj = 256, -1
        win = win[~claimed[win]]
        if len(win):
            dd = np.unpackbits(np.bitwise_xor(desc[win], eldesc[ee[i]]), axis=1).sum(1)
            k = int(np.argmin(dd))                                   # the first strict minimum in window order
            best, bj = int(dd[k]), int(win[k])
        if best <= orb_dist:
            assign[bj] = i; claimed[bj] = True; nm += 1
            if check_ori: hist[rot_bin(kf_kps["angle"][i], kps["angle"][bj])].append(bj)
    if check_ori:
        keep = three_maxima([len(h) for h in hist])
        for b in range(HISTO_LENGTH):
            if b in keep: continue
            for j in hist[b]:
                assign[j] = -2; nm -= 1
    return nm, assign


def reloc_pairs(query, cand, ncand, kmax):
    """The pair list of sslpl_reloc_pairs_batch_device: slot q * kmax + k = (cand[q][k], query[q]) for k < min(ncand[q], kmax, ndb)."""
    nq = len(query)
    out = np.full((nq * kmax, 2), -1, np.int32)
    for q in range(nq):
        for k in range(min(int(ncand[q]), kmax, cand.shape[1])):
            out[q * kmax + k] = (cand[q][k], query[q])
    return out


def ref_available():
    return os.path.exists(REF_LIB)


_ref = None


def ref_search_by_projection_kf(kf_kps, kfmp, Xw, mindist, maxdist, eldesc, bad, found_el, kps, desc, held, Tcw, cam, bounds, nlevels,
                                scale_factor, th, orb_dist, check_ori=True, seconds=None):
    """The reference's own SearchByProjection(F, pKF, sAlreadyFound, th, ORBdist) (tests/ref_reloc.cpp).  Elements: Xw, raw mfMinDistance /
    mfMaxDistance, descriptor, bad and found_el[m] = in sAlreadyFound.  Returns (nmatches, assign[j] = ELEMENT index of the MapPoint left in
    mvpMapPoints[j], -1 none, -3 the one held on entry).  seconds: a ctypes double that receives the matcher call's wall time."""
    global _ref
    if _ref is None:
        _ref = C.CDLL(REF_LIB)
        _ref.ref_search_by_projection_kf.restype = C.c_int
    p = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    c = lambda a, t: np.ascontiguousarray(a, t)
    kf_kps = np.ascontiguousarray(kf_kps); kps = np.ascontiguousarray(kps)
    assert kf_kps.dtype.itemsize == 28 and kps.dtype.itemsize == 28
    nel = len(Xw)
    cam8 = np.array([cam[0], cam[1], cam[2], cam[3], bounds[0], bounds[1], bounds[2], bounds[3]], f32)
    out = np.full(max(len(kps), 1), -1, np.int32)
    n = _ref.ref_search_by_projection_kf(len(kfmp), p(kf_kps), p(c(kfmp, np.int32)), nel, p(c(Xw, f32)), p(c(mindist, f32)), p(c(maxdist, f32)),
                                         p(c(eldesc, np.uint8)), p(c(bad, np.uint8)), p(c(found_el, np.uint8)), len(kps), p(kps),
                                         p(c(desc, np.uint8)), p(None if held is None else c(held, np.uint8)), p(c(np.asarray(Tcw, f32).reshape(-1)[:12], f32)),
                                         p(cam8), int(nlevels), C.c_float(scale_factor), C.c_float(th), int(orb_dist), int(check_ori), p(out),
                                         None if seconds is None else C.byref(seconds))
    return n, out[:len(kps)]


def _rot(ang):
    Rx = np.array([[1, 0, 0], [0, np.cos(ang[0]), -np.sin(ang[0])], [0, np.sin(ang[0]), np.cos(ang[0])]])
    Ry = np.array([[np.cos(ang[1]), 0, np.sin(ang[1])], [0, 1, 0], [-np.sin(ang[1]), 0, np.cos(ang[1])]])
    Rz = np.array([[np.cos(ang[2]), -np.sin(ang[2]), 0], [np.sin(ang[2]), np.cos(ang[2]), 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


CAM = (481.2, 480.0, 319.5, 239.5)                    # Examples/ICL.yaml (|fy|)
BOUNDS = (0.0, 640.0, 0.0, 480.0)
SF = (f32(1.2) ** np.arange(8)).astype(f32)
LOG_SF = f32(np.log(f32(1.2)))                        # Frame::mfLogScaleFactor = log(mfScaleFactor)


def reloc_scene(oracle, synth, seed, f0=0, p_null=0.1, p_bad=0.05, p_found=0.1, p_held=0.05, p_behind=0.03, p_edge=0.05, identity=False):
    """A keyframe made from synthetic frame f0 (camera = world) whose features see MapPoints at random depths, and frame f0 + 1 posed by a
    small rigid motion (a PnP pose).  Covers NULL, bad and already-found MapPoints, one MapPoint at two keyframe indices, held frame
    features, points behind the camera, distances just inside / outside the invariance range and predicted levels from 0 to the top.
    identity: Tcw = I and two MapPoints on the camera plane (z = 0: one at the centre, which projects to NaN, one off it, to inf).
    Returns a dict with the keyframe (kf_kps, kfmp), the elements (Xw, mindist, maxdist, eldesc, bad, found_el), the frame (kps, desc,
    held) and Tcw."""
    rng = np.random.default_rng(seed)
    orc = oracle.OrbOracle(1000, 1.2, 8, 20, 7)
    k1, d1 = orc.extract(synth.frame(640, 480, f0))
    k2, d2 = orc.extract(synth.frame(640, 480, f0 + 1))
    fx, fy, cx, cy = CAM
    n1 = len(k1)
    z = rng.uniform(1.0, 6.0, n1).astype(f32)
    Xw = np.stack([(k1["x"] - cx) / fx * z, (k1["y"] - cy) / fy * z, z], 1).astype(f32)
    beh = rng.random(n1) < p_behind
    Xw[beh] *= f32(-1)                                                            # behind the camera, mirrored into the image
    Tcw = np.eye(4, dtype=f32)
    if not identity:
        Tcw[:3, :3] = _rot(rng.normal(0, 0.01, 3)).astype(f32); Tcw[:3, 3] = rng.normal(0, 0.03, 3).astype(f32)
    else:
        Xw[0] = 0; Xw[1] = (0.5, -0.25, 0)
    eldesc = d1.copy(); flip = rng.random(eldesc.shape) < 0.02
    eldesc[flip] ^= (1 << rng.integers(0, 8, flip.sum())).astype(np.uint8)
    # invariance range around the distance the frame will measure: predicted levels spread over the pyramid and past both ends
    T = Tcw[:3].reshape(-1).astype(f64)
    Ow = np.array([-((T[r] * T[3] + T[4 + r] * T[7]) + T[8 + r] * T[11]) for r in range(3)]).astype(f32)
    PO = (Xw - Ow).astype(f64)
    dist = np.sqrt((PO[:, 0] * PO[:, 0] + PO[:, 1] * PO[:, 1]) + PO[:, 2] * PO[:, 2]).astype(f32)
    maxdist = (dist * f32(1.2) ** rng.uniform(-0.5, 8.5, n1).astype(f32)).astype(f32)
    mindist = (maxdist / f32(1.2) ** 7).astype(f32)
    edge = np.nonzero(rng.random(n1) < p_edge)[0]
    for k, i in enumerate(edge):                                                  # 1.2f * maxdist or 0.8f * mindist at dist, one ulp either way
        if k % 2:
            m = f32(dist[i] / f32(1.2))
            while f32(1.2) * m > dist[i]: m = np.nextafter(m, f32(0))
            while f32(1.2) * m < dist[i]: m = np.nextafter(m, f32(np.inf))
            maxdist[i] = m if k % 4 == 1 else np.nextafter(m, f32(0))
        else:
            m = f32(dist[i] / f32(0.8))
            while f32(0.8) * m < dist[i]: m = np.nextafter(m, f32(np.inf))
            while f32(0.8) * m > dist[i]: m = np.nextafter(m, f32(0))
            mindist[i] = m if k % 4 == 0 else np.nextafter(m, f32(np.inf))
    if identity:
        mindist[:2] = 0
    kfmp = np.arange(n1, dtype=np.int32)
    kfmp[rng.random(n1) < p_null] = -1
    a, b = rng.choice(n1, 2, replace=False)
    kfmp[b] = kfmp[a] = a                                                         # one MapPoint at two keyframe indices
    bad = (rng.random(n1) < p_bad).astype(np.uint8)
    found_el = (rng.random(n1) < p_found).astype(np.uint8)
    held = (rng.random(len(k2)) < p_held).astype(np.uint8)
    return dict(kf_kps=k1, kfmp=kfmp, Xw=Xw, mindist=mindist, maxdist=maxdist, eldesc=eldesc, bad=bad, found_el=found_el,
                kps=k2, desc=d2, held=held, Tcw=Tcw[:3].copy())


def scene_model(oracle, S, th, orb_dist, check_ori=True):
    """search_by_projection_kf on a reloc_scene."""
    el = element_table(S["Xw"], S["mindist"], S["maxdist"])
    found = np.where(S["kfmp"] >= 0, S["found_el"][np.maximum(S["kfmp"], 0)], 0).astype(np.uint8)
    return search_by_projection_kf(oracle, S["kf_kps"], S["kfmp"], el, S["eldesc"], S["bad"], found, S["kps"], S["desc"], S["held"],
                                   S["Tcw"], CAM, BOUNDS, SF, LOG_SF, th, orb_dist, check_ori)


def as_elements(S, assign):
    """Keyframe-feature indices of a reloc_scene result as the reference entry point reports them: the element of the MapPoint, -3 for
    a feature that keeps the MapPoint it held."""
    out = np.where(assign >= 0, S["kfmp"][np.maximum(assign, 0)], -1)
    return np.where((out == -1) & (S["held"] != 0), -3, out).astype(np.int32)


def scene_ref(S, th, orb_dist, check_ori=True):
    return ref_search_by_projection_kf(S["kf_kps"], S["kfmp"], S["Xw"], S["mindist"], S["maxdist"], S["eldesc"], S["bad"], S["found_el"],
                                       S["kps"], S["desc"], S["held"], S["Tcw"], CAM, BOUNDS, len(SF), 1.2, th, orb_dist, check_ori)


class DeviceRows:
    """The scenes as a row set (row 2 s = keyframe of scene s, row 2 s + 1 = its frame) with one element table."""

    def __init__(self, torch, scenes, cap):
        nrows = 2 * len(scenes)
        kps = np.zeros((nrows, cap), scenes[0]["kps"].dtype); desc = np.zeros((nrows, cap, 32), np.uint8)
        n = np.zeros(nrows, np.int32); kfmp = np.full((nrows, cap), -1, np.int32)
        els, descs, bads, self.off = [], [], [], []
        base = 0
        for s, S in enumerate(scenes):
            n1, n2 = len(S["kf_kps"]), len(S["kps"])
            kps[2 * s, :n1] = S["kf_kps"]; kps[2 * s + 1, :n2] = S["kps"]; desc[2 * s + 1, :n2] = S["desc"]
            n[2 * s], n[2 * s + 1] = n1, n2
            kfmp[2 * s, :n1] = np.where(S["kfmp"] >= 0, S["kfmp"] + base, -1)
            els.append(element_table(S["Xw"], S["mindist"], S["maxdist"])); descs.append(S["eldesc"]); bads.append(S["bad"])
            self.off.append(base); base += len(S["Xw"])
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        self.kps, self.desc, self.n, self.kfmp = dev(kps.view(np.uint8)), dev(desc), dev(n), dev(kfmp)
        self.el, self.eldesc, self.bad = dev(np.concatenate(els)), dev(np.concatenate(descs)), dev(np.concatenate(bads))
        self.nrows, self.cap, self.nel = nrows, cap, base
