"""TEST INFRASTRUCTURE: a NumPy restatement of the map-element refresh of include/sslpl_map.h, bit for bit:
MapPoint::ComputeDistinctiveDescriptors / UpdateNormalAndDepth (MapPoint.cc:247-312, 335-376) and MapLine::ComputeDistinctiveDescriptors /
UpdateAverageDir (MapLine.cpp:246-317, 325-372), with the entry rules of sslpl_update_map_*_batch_device (statuses, first entry wins).
Rounding rules (tools/probe_cv_matexpr.py, cv2 4.13):
  - normal + normali / cv::norm(normali) is scaleAdd(normali, 1.0 / norm, normal): one fused multiply-add with the scale narrowed to
    float.  NumPy has no fma, so scale_add rounds the exact double sum to odd and then to float, which is the correctly rounded fma;
  - normal / n is convertTo with the scale 1.0 / n narrowed to float (create_points_model.convert_scale);
  - 0.5 * (SP + EP) is addWeighted(SP, 0.5, EP, 0.5, 0) (create_points_model.add_weighted); the line normal is Eigen's double arithmetic.
`rounding` selects the cv::Mat expression rules: "cv2" (above; what the device is held to) or "minicv", the rules of the OpenCV stand-in
the reference is compiled against in oracle/_ref/libref.so (oracle/refshim/minicv.cpp: Mat * double and Mat / double in double, rounded
once to float; Mat + Mat and Mat - Mat in float), with which the model equals the reference's own member functions
(tests/test_map_update_ref_cpu.py).  The two differ only in the last bits of the point normal and of the line mid-point.
No libm: +, -, *, / and sqrt only, each correctly rounded in NumPy."""
import numpy as np

from create_points_model import add_weighted, convert_scale, norm3

f32, f64 = np.float32, np.float64

DESC, GEOM = 1, 2
OK, NO_OBS, NO_GOOD_KF, REF_OCTAVE, BAD = 0, 1, 2, 3, -1


def scale_add(a, alpha, b):
    """cv::scaleAdd(a, alpha, b) on CV_32F as cv2 4.13 evaluates it: fma(a, (float)alpha, b), elementwise."""
    a = np.asarray(a, f32).astype(f64); b = np.asarray(b, f32).astype(f64)
    p = a * f64(f32(alpha))                                  # exact: two 24-bit significands
    with np.errstate(all="ignore"):
        s = p + b
        t = s - p
        e = (p - (s - t)) + (b - t)                          # s + e = p + b exactly (TwoSum)
        odd = (e != 0) & ((np.asarray(s, f64).view(np.uint64) & 1) == 0)
        s = np.where(odd, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(f32)


def two_roundings(a, alpha, b):
    """The rule scale_add is told apart from: fl(fl(a * (float)alpha) + b)."""
    return (np.asarray(a, f32) * f32(alpha)) + np.asarray(b, f32)


def medoid(ds):
    """Index of the descriptor with the least median Hamming distance to the rows ds [N, 32] (median = sorted[int(0.5 (N - 1))], the
    self-distance included, first least median wins); -1 when N = 0."""
    ds = np.asarray(ds, np.uint8).reshape(-1, 32)
    if len(ds) == 0:
        return -1
    D = np.unpackbits(ds[:, None, :] ^ ds[None, :, :], axis=-1).sum(-1)
    return int(np.argmin(np.sort(D, axis=1)[:, int(0.5 * (len(ds) - 1))]))


def _entry_ok(e, nel, first, u, refkf, obs, n, nkf, geom):
    """SSLPL_MAPUPD_BAD tests of one entry before and after the empty-list test: (bad, empty)."""
    if not (0 <= e < nel) or first[e] != u or len(obs) > nkf or (geom and not (0 <= refkf < nkf)):
        return True, False
    if len(obs) == 0:
        return False, True
    ks = [k for k, _ in obs]
    if any(not (0 <= k < nkf) or not (0 <= i < n[k]) for k, i in obs) or len(set(ks)) != len(ks):
        return True, False
    if geom and (dict(obs).get(refkf, 0) >= n[refkf]):
        return True, False
    return False, False


def _first(elems, nel):
    first = {}
    for u, e in enumerate(elems):
        if 0 <= e < nel and e not in first:
            first[e] = u
    return first


def _scaled(x, s):
    """minicv's Mat * double on CV_32F: (float)((double)x * s)."""
    return (np.asarray(x, f32).astype(f64) * f64(s)).astype(f32)


def _update(lines, feat, desc, n, pose, kfbad, table, tdesc, entries, scale, what, pos=None, nrm64=None, rounding="cv2"):
    assert rounding in ("cv2", "minicv")
    nkf = len(n)
    n = [int(c) for c in n]
    nlev = len(scale)
    scale = np.asarray(scale, f32)
    kfbad = np.zeros(nkf, bool) if kfbad is None else np.asarray(kfbad) != 0
    table = np.array(table, f32); tdesc = np.array(tdesc, np.uint8)
    nrm64 = None if nrm64 is None else np.array(nrm64, f64)
    geom, dsc = bool(what & GEOM), bool(what & DESC)
    first = _first([e for e, _, _ in entries], len(table))
    status = np.zeros(len(entries), np.int32)
    for u, (e, rk, obs) in enumerate(entries):
        obs = [(int(k), int(i)) for k, i in obs]
        bad, empty = _entry_ok(e, len(table), first, u, rk, obs, n, nkf, geom)
        if bad or empty:
            status[u] = BAD if bad else NO_OBS
            continue
        st = OK
        if dsc:
            good = [(k, i) for k, i in obs if not kfbad[k]]
            if not good:
                st = NO_GOOD_KF
            else:
                ds = np.array([desc[k][i] for k, i in good], np.uint8)
                tdesc[e] = ds[medoid(ds)]
        if geom:
            Ow = [np.asarray(pose[k][12:15], f32) for k, _ in obs]
            if not lines:
                X = table[e, :3].copy()
                s = np.zeros(3, f32)
                for o in Ow:
                    q = X - o
                    with np.errstate(divide="ignore"):
                        alpha = f64(1.0) / f64(norm3(q))            # inf for a point at the camera centre, as on the device
                    s = scale_add(q, alpha, s) if rounding == "cv2" else s + _scaled(q, alpha)
                nf = convert_scale(s, 1.0 / len(obs)) if rounding == "cv2" else _scaled(s, 1.0 / len(obs))
            else:
                W = np.asarray(pos[e], f64)
                mid = 0.5 * (W[:3] + W[3:])
                s = np.zeros(3, f64)
                for o in Ow:
                    q = mid - o.astype(f64)
                    with np.errstate(divide="ignore", invalid="ignore"):
                        s = s + q / np.sqrt((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2])
                s = s / f64(len(obs))
                if nrm64 is not None:
                    nrm64[e] = s
                nf = s.astype(f32)
                SP, EP = W[:3].astype(f32), W[3:].astype(f32)
                X = add_weighted(SP, 0.5, EP, 0.5) if rounding == "cv2" else _scaled(SP + EP, 0.5)
            w = table.shape[1]
            table[e, w - 6:w - 3] = nf
            oct_ = int(feat[rk][dict(obs).get(rk, 0)]["octave"])
            if not (0 <= oct_ < nlev):
                st = REF_OCTAVE
            else:
                dist = f32(norm3(X - np.asarray(pose[rk][12:15], f32)))
                mx = dist * scale[oct_]
                mn = mx / scale[nlev - 1]
                table[e, w - 3:] = (f32(0.8) * mn, f32(1.2) * mx, mx)
        status[u] = st
    return table, tdesc, nrm64, status


def update_points(kps, desc, n, pose, kfbad, mp, mpdesc, entries, scale, what, rounding="cv2"):
    """sslpl_update_map_points_batch_device on host arrays: kps [nkf, cap] KEYPOINT_DTYPE (mvKeysUn), desc [nkf, cap, 32], n [nkf],
    pose [nkf, 15], kfbad [nkf] or None, mp [nmp, 9], mpdesc [nmp, 32], entries = [(element, refkf, [(kf, idx), ...])] ->
    (mp, mpdesc, status), new arrays."""
    mp, mpdesc, _, st = _update(False, kps, desc, n, pose, kfbad, mp, mpdesc, entries, scale, what, rounding=rounding)
    return mp, mpdesc, st


def update_lines(kl, ldesc, nl, pose, kfbad, mlpos, ml, mldesc, mlnormal, entries, scale, what, rounding="cv2"):
    """sslpl_update_map_lines_batch_device on host arrays: kl [nkf, capl] KEYLINE_DTYPE, mlpos [nml, 6] f64, ml [nml, 12],
    mlnormal [nml, 3] f64 or None -> (ml, mldesc, mlnormal, status)."""
    return _update(True, kl, ldesc, nl, pose, kfbad, ml, mldesc, entries, scale, what, pos=mlpos, nrm64=mlnormal, rounding=rounding)


def csr(entries):
    """(elem, refkf, obs_off, obs) int32 arrays of an entry list, as the batched calls take them."""
    elem = np.array([e for e, _, _ in entries], np.int32)
    refkf = np.array([r for _, r, _ in entries], np.int32)
    off = np.zeros(len(entries) + 1, np.int32)
    off[1:] = np.cumsum([len(o) for _, _, o in entries])
    obs = np.array([p for _, _, o in entries for p in o], np.int32).reshape(-1, 2)
    return elem, refkf, off, obs
