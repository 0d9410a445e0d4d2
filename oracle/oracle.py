"""ctypes bindings of the CPU oracle (oracle/liboracle.so).

TEST INFRASTRUCTURE ONLY: import from tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference legs.  The product package never imports this module.
"""
import ctypes as C
import os
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "liboracle.so")

KEYPOINT_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                           ("octave", "<i4"), ("class_id", "<i4")])
KEYLINE_DTYPE = np.dtype([("angle", "<f4"), ("class_id", "<i4"), ("octave", "<i4"), ("pt_x", "<f4"), ("pt_y", "<f4"),
                          ("response", "<f4"), ("size", "<f4"),
                          ("startPointX", "<f4"), ("startPointY", "<f4"), ("endPointX", "<f4"), ("endPointY", "<f4"),
                          ("sPointInOctaveX", "<f4"), ("sPointInOctaveY", "<f4"),
                          ("ePointInOctaveX", "<f4"), ("ePointInOctaveY", "<f4"),
                          ("lineLength", "<f4"), ("numOfPixels", "<i4")])
assert KEYPOINT_DTYPE.itemsize == 28 and KEYLINE_DTYPE.itemsize == 68


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith((".cpp", ".h", ".inc")) or f == "Makefile"]
    stale = (not os.path.exists(_LIB)) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in srcs)
    if force or stale:
        subprocess.run(["make", "-C", _HERE, "-s"], check=True)
    return _LIB


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.orc_fast_atan2.restype = C.c_float
        _lib.orc_fast_atan2.argtypes = [C.c_float, C.c_float]
        _lib.orc_orb_create.restype = C.c_void_p
        _lib.orc_orb_create.argtypes = [C.c_int, C.c_float, C.c_int, C.c_int, C.c_int]
        if hasattr(_lib, "orc_line_create"):
            _lib.orc_line_create.restype = C.c_void_p
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _u8(img):
    img = np.ascontiguousarray(img, dtype=np.uint8)
    assert img.ndim == 2
    return img


def resize_linear(img, dw, dh):
    img = _u8(img)
    out = np.empty((dh, dw), np.uint8)
    lib().orc_resize_linear_u8(_p(img), img.shape[1], img.shape[0], img.strides[0], _p(out), dw, dh, dw)
    return out


def border_reflect101(img, b):
    img = _u8(img)
    out = np.empty((img.shape[0] + 2 * b, img.shape[1] + 2 * b), np.uint8)
    lib().orc_border_reflect101_u8(_p(img), img.shape[1], img.shape[0], img.strides[0], _p(out), out.strides[0], b)
    return out


def sepfilter_fixed(img, taps):
    img = _u8(img)
    taps = np.ascontiguousarray(taps, np.int32)
    out = np.empty_like(img)
    lib().orc_sepfilter_fixed_u8(_p(img), img.shape[1], img.shape[0], img.strides[0], _p(out), out.strides[0],
                                 _p(taps), len(taps))
    return out


def gauss7_sigma2(img):
    return sepfilter_fixed(img, [18, 34, 48, 56, 48, 34, 18])


def fast9_16(img, threshold, cap=1 << 16):
    img = _u8(img)
    xs = np.empty(cap, np.int32); ys = np.empty(cap, np.int32); ss = np.empty(cap, np.int32)
    n = lib().orc_fast9_16(_p(img), img.shape[1], img.shape[0], img.strides[0], int(threshold), _p(xs), _p(ys), _p(ss), cap)
    assert n <= cap
    return xs[:n].copy(), ys[:n].copy(), ss[:n].copy()


def fast_atan2(y, x):
    return float(lib().orc_fast_atan2(float(y), float(x)))


def line_nfa(n, k, p, log_nt, threads=1):
    """nfa() of lsd.cpp on arrays -> (log_nfa float64, stop int32: loop index of the early stop, n + 1 when the tail loop ran out,
    -1 for the early returns).  threads > 1 splits the arrays over a thread pool (the C call releases the GIL)."""
    n = np.ascontiguousarray(n, np.int32).reshape(-1); k = np.ascontiguousarray(k, np.int32).reshape(-1)
    p = np.ascontiguousarray(np.broadcast_to(np.asarray(p, np.float64), n.shape))
    out = np.empty(len(n)); stop = np.empty(len(n), np.int32)
    f = lib().orc_line_nfa_array
    f.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p]

    def run(a, b):
        if b > a:
            f(b - a, _p(n[a:]), _p(k[a:]), _p(p[a:]), float(log_nt), _p(out[a:]), _p(stop[a:]))
    if threads <= 1:
        run(0, len(n))
    else:
        from concurrent.futures import ThreadPoolExecutor
        step = 4096                     # small chunks: the cost of one entry varies with n by orders of magnitude
        with ThreadPoolExecutor(threads) as ex:
            list(ex.map(lambda a: run(a, min(a + step, len(n))), range(0, len(n), step)))
    return out, stop


def ddtrig_sincos(x, full=False):
    """Host form of csrc/ddtrig.h -> (sin, cos, quick_ok): sincos_cr (full=False) or sincos_cr_full; quick_ok = 1 where the quick
    evaluation's round_safe accepted both results."""
    x = np.ascontiguousarray(x, np.float64).reshape(-1)
    s = np.empty_like(x); c = np.empty_like(x); q = np.empty(len(x), np.uint8)
    lib().orc_ddtrig_sincos(len(x), _p(x), int(bool(full)), _p(s), _p(c), _p(q))
    return s, c, q


def octree(xs, ys, resp, minX, maxX, minY, maxY, N):
    xs = np.ascontiguousarray(xs, np.int32); ys = np.ascontiguousarray(ys, np.int32); resp = np.ascontiguousarray(resp, np.int32)
    out = np.empty(len(xs) + 8, np.int32)
    n = lib().orc_octree(_p(xs), _p(ys), _p(resp), len(xs), minX, maxX, minY, maxY, N, _p(out), len(out))
    return out[:n].copy()


class OrbOracle:
    """ORBextractor restatement (ORBextractor.cc:410-470 ctor, :1043 operator())."""

    def __init__(self, nfeatures=1000, scale_factor=1.2, nlevels=8, ini_th=20, min_th=7):
        self.nlevels = nlevels
        self.nfeatures = nfeatures
        self.h = C.c_void_p(lib().orc_orb_create(nfeatures, scale_factor, nlevels, ini_th, min_th))

    def ic_angles(self, img, xs, ys):
        """IC_Angle (ORBextractor.cc:77-104) at integer positions of an un-blurred image."""
        img = _u8(img); xs = np.ascontiguousarray(xs, np.int32); ys = np.ascontiguousarray(ys, np.int32)
        out = np.empty(max(len(xs), 1), np.float32)
        lib().orc_ic_angles(self.h, _p(img), img.shape[1], img.shape[0], img.strides[0], _p(xs), _p(ys), len(xs), _p(out))
        return out[:len(xs)]

    @staticmethod
    def brief_descriptors(blurred, xs, ys, angles):
        """computeOrbDescriptor (ORBextractor.cc:107-147) at integer positions of an ALREADY blurred image."""
        blurred = _u8(blurred); xs = np.ascontiguousarray(xs, np.int32); ys = np.ascontiguousarray(ys, np.int32)
        angles = np.ascontiguousarray(angles, np.float32)
        out = np.empty((max(len(xs), 1), 32), np.uint8)
        lib().orc_brief_descriptors(_p(blurred), blurred.shape[1], blurred.shape[0], blurred.strides[0], _p(xs), _p(ys), _p(angles), len(xs), _p(out))
        return out[:len(xs)]

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_orb_destroy(self.h)
            self.h = None

    def tables(self):
        L = self.nlevels
        sc, isc, s2, is2 = (np.empty(L, np.float32) for _ in range(4))
        nf = np.empty(L, np.int32); um = np.empty(16, np.int32)
        lib().orc_orb_tables(self.h, _p(sc), _p(isc), _p(s2), _p(is2), _p(nf), _p(um))
        return dict(scale=sc, invscale=isc, sigma2=s2, invsigma2=is2, nfeat=nf, umax=um)

    def extract(self, img):
        """(keypoints, descriptors) of every level.  The C side returns the full count; a level may keep more keypoints than its
        share of nfeatures (up to 4 * nIni after the octree's first split), so a short buffer is sized again from that count."""
        img = _u8(img)
        cap = self.nfeatures + 4 * self.nlevels + 64
        while True:
            kps = np.zeros(cap, KEYPOINT_DTYPE); desc = np.zeros((cap, 32), np.uint8)
            n = lib().orc_orb_extract(self.h, _p(img), img.shape[1], img.shape[0], img.strides[0], _p(kps), _p(desc), cap)
            if n <= cap:
                return kps[:n].copy(), desc[:n].copy()
            cap = n

    def level_size(self, l):
        w = C.c_int(); h = C.c_int()
        lib().orc_orb_level_size(self.h, l, C.byref(w), C.byref(h))
        return w.value, h.value

    def level(self, l, bordered=False):
        w, h = self.level_size(l)
        b = 19 if bordered else 0
        out = np.empty((h + 2 * b, w + 2 * b), np.uint8)
        lib().orc_orb_level_copy(self.h, l, int(bordered), _p(out), out.strides[0])
        return out

    def blurred(self, l):
        w, h = self.level_size(l)
        out = np.zeros((h, w), np.uint8)
        lib().orc_orb_blur_copy(self.h, l, _p(out), out.strides[0])
        return out

    def candidates(self, l, cap=1 << 16):
        """FAST candidates of level l of the last call; the C side returns the full count, and a short buffer is sized again."""
        xs = np.empty(cap, np.int32); ys = np.empty(cap, np.int32); rs = np.empty(cap, np.int32)
        n = lib().orc_orb_candidates(self.h, l, _p(xs), _p(ys), _p(rs), cap)
        if n > cap:
            return self.candidates(l, n)
        return xs[:n].copy(), ys[:n].copy(), rs[:n].copy()

    def level_keypoints(self, l, cap=1 << 14):
        xs = np.empty(cap, np.int32); ys = np.empty(cap, np.int32); rs = np.empty(cap, np.int32); an = np.empty(cap, np.float32)
        n = lib().orc_orb_level_keypoints(self.h, l, _p(xs), _p(ys), _p(rs), _p(an), cap)
        if n > cap:
            return self.level_keypoints(l, n)
        return xs[:n].copy(), ys[:n].copy(), rs[:n].copy(), an[:n].copy()

    def stage_ms(self):
        ms = np.empty(6, np.float64)
        lib().orc_orb_stage_ms(self.h, _p(ms))
        return dict(zip(["pyramid", "fast", "octree", "orient", "blur", "brief"], ms.tolist()))


# ---------------- matching ----------------
def descriptor_distance(a, b):
    a = np.ascontiguousarray(a, np.uint8); b = np.ascontiguousarray(b, np.uint8)
    return int(lib().orc_descriptor_distance(_p(a), _p(b)))


def knn2(q, t):
    q = np.ascontiguousarray(q, np.uint8).reshape(-1, 32); t = np.ascontiguousarray(t, np.uint8).reshape(-1, 32)
    out = np.empty((max(len(q), 1), 4), np.int32)
    lib().orc_knn2(_p(q), len(q), _p(t), len(t), _p(out))
    return out[:len(q)]


def bow_assign(desc, centroids):
    desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32); centroids = np.ascontiguousarray(centroids, np.uint8).reshape(-1, 32)
    node = np.empty(max(len(desc), 1), np.int32)
    lib().orc_bow_assign(_p(desc), len(desc), _p(centroids), len(centroids), _p(node))
    return node[:len(desc)]


def vocab_transform(L, parent, ndesc, weight, is_leaf, feats, levelsup=4):
    """DBoW2 transform (TemplatedVocabulary.h:1127-1259) on a tree given as arrays -> (word, node, weight) per feature."""
    parent = np.ascontiguousarray(parent, np.int32); ndesc = np.ascontiguousarray(ndesc, np.uint8).reshape(-1, 32)
    weight = np.ascontiguousarray(weight, np.float64); is_leaf = np.ascontiguousarray(is_leaf, np.uint8)
    feats = np.ascontiguousarray(feats, np.uint8).reshape(-1, 32)
    n = len(feats)
    word = np.empty(max(n, 1), np.int32); node = np.empty(max(n, 1), np.int32); w = np.empty(max(n, 1), np.float64)
    lib().orc_vocab_transform.restype = C.c_int
    nw = lib().orc_vocab_transform(int(L), len(parent), _p(parent), _p(ndesc), _p(weight), _p(is_leaf), _p(feats), n, int(levelsup),
                                   _p(word), _p(node), _p(w))
    assert nw >= 0, "malformed vocabulary tree"
    return word[:n], node[:n], w[:n]


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def search_by_projection_frame(last, cur, Tcw, Tlw, cam, bounds, scale_factors, th, mono=True, check_ori=True):
    """ORBmatcher::SearchByProjection(Frame&, const Frame&, th, bMono) (ORBmatcher.cc:1331-1473).
    last = dict(valid, obs, Xw[n,3], dmp[n,32], oct, angle); cur = dict(desc[n,32], x, y, oct, angle, uright|None, claimed|None).
    Returns (nmatches, assign2)."""
    n1, n2 = len(last["valid"]), len(cur["x"])
    v1 = np.ascontiguousarray(last["valid"], np.uint8); o1 = np.ascontiguousarray(last["obs"], np.uint8)
    Xw = _f32(last["Xw"]).reshape(-1, 3); dmp = np.ascontiguousarray(last["dmp"], np.uint8).reshape(-1, 32)
    oc1 = np.ascontiguousarray(last["oct"], np.int32); a1 = _f32(last["angle"])
    d2 = np.ascontiguousarray(cur["desc"], np.uint8).reshape(-1, 32); x2 = _f32(cur["x"]); y2 = _f32(cur["y"])
    oc2 = np.ascontiguousarray(cur["oct"], np.int32); a2 = _f32(cur["angle"])
    ur = _f32(cur["uright"]) if cur.get("uright") is not None else None
    cl = np.ascontiguousarray(cur["claimed"], np.uint8) if cur.get("claimed") is not None else None
    Tc = _f32(Tcw).reshape(-1)[:12].copy(); Tl = _f32(Tlw).reshape(-1)[:12].copy() if Tlw is not None else None
    camv = _f32(cam); bnd = _f32(bounds); sf = _f32(scale_factors)
    out = np.full(max(n2, 1), -1, np.int32)
    lib().orc_search_by_projection_frame.restype = C.c_int
    n = lib().orc_search_by_projection_frame(n1, _p(v1), _p(o1), _p(Xw), _p(dmp), _p(oc1), _p(a1),
                                             n2, _p(d2), _p(x2), _p(y2), _p(oc2), _p(a2), _p(ur) if ur is not None else None,
                                             _p(cl) if cl is not None else None, _p(Tc), _p(Tl) if Tl is not None else None,
                                             _p(camv), _p(bnd), _p(sf), C.c_float(th), int(mono), int(check_ori), _p(out))
    return n, out[:n2]


def search_by_projection_mps(mp, cur, bounds, scale_factors, nnratio=0.8, th=1.0):
    """ORBmatcher::SearchByProjection(Frame&, const vector<MapPoint*>&, th) (ORBmatcher.cc:45-129).
    mp = dict(inview, bad, obs, projx, projy, level, viewcos, desc[, projxr]); cur = dict(desc, x, y, oct[, uright, held])."""
    nmp = len(mp["inview"]); n2 = len(cur["x"])
    u8 = lambda a: np.ascontiguousarray(a, np.uint8)
    iv, bad, obs = u8(mp["inview"]), u8(mp["bad"]), u8(mp["obs"])
    px, py = _f32(mp["projx"]), _f32(mp["projy"]); pxr = _f32(mp["projxr"]) if mp.get("projxr") is not None else None
    lv = np.ascontiguousarray(mp["level"], np.int32); vc = _f32(mp["viewcos"]); dmp = u8(mp["desc"]).reshape(-1, 32)
    d2 = u8(cur["desc"]).reshape(-1, 32); x2, y2 = _f32(cur["x"]), _f32(cur["y"]); oc2 = np.ascontiguousarray(cur["oct"], np.int32)
    ur = _f32(cur["uright"]) if cur.get("uright") is not None else None
    held = u8(cur["held"]) if cur.get("held") is not None else None
    out = np.full(max(n2, 1), -1, np.int32)
    lib().orc_search_by_projection_mps.restype = C.c_int
    n = lib().orc_search_by_projection_mps(nmp, _p(iv), _p(bad), _p(obs), _p(px), _p(py), _p(pxr) if pxr is not None else None, _p(lv), _p(vc), _p(dmp),
                                           n2, _p(d2), _p(x2), _p(y2), _p(oc2), _p(ur) if ur is not None else None, _p(held) if held is not None else None,
                                           _p(_f32(bounds)), _p(_f32(scale_factors)), C.c_float(nnratio), C.c_float(th), _p(out))
    return n, out[:n2]


def search_for_initialization(d1, k1, d2, k2, prev, bounds, nnratio=0.9, check_ori=True, window=100):
    """ORBmatcher::SearchForInitialization (ORBmatcher.cc:408-523) -> (nmatches, matches12, prev_out)."""
    d1 = np.ascontiguousarray(d1, np.uint8).reshape(-1, 32); d2 = np.ascontiguousarray(d2, np.uint8).reshape(-1, 32)
    prev = _f32(prev).reshape(-1, 2).copy()
    m12 = np.full(max(len(k1), 1), -1, np.int32)
    lib().orc_search_for_initialization.restype = C.c_int
    n = lib().orc_search_for_initialization(len(k1), _p(d1), _p(np.ascontiguousarray(k1["octave"], np.int32)), _p(_f32(k1["angle"])),
                                            len(k2), _p(d2), _p(_f32(k2["x"])), _p(_f32(k2["y"])), _p(np.ascontiguousarray(k2["octave"], np.int32)),
                                            _p(_f32(k2["angle"])), _p(prev), _p(_f32(bounds)), C.c_float(nnratio), int(check_ori), int(window), _p(m12))
    return n, m12[:len(k1)], prev


def _u8(a):
    return np.ascontiguousarray(a, np.uint8)


def _i32(a):
    return np.ascontiguousarray(a, np.int32)


def line_project_frame(valid1, Pw, oct1, Tcw, Tlw, cam5, bounds, scale_factors, th, mono=True):
    """Projection stage of LSDmatcher::SearchByProjection(Frame&, const Frame&, th, bMono) (LSDmatcher.cpp:22-96)
    -> dict(active, proj[n,4], radius, min_level, max_level)."""
    n = len(valid1)
    out = dict(active=np.zeros(n, np.uint8), proj=np.zeros((n, 4), np.float32), radius=np.zeros(n, np.float32),
               min_level=np.zeros(n, np.int32), max_level=np.zeros(n, np.int32))
    lib().orc_line_project_frame(n, _p(_u8(valid1)), _p(_f32(Pw)), _p(_i32(oct1)), _p(_f32(Tcw)), _p(_f32(Tlw)), _p(_f32(cam5)), _p(_f32(bounds)),
                                 _p(_f32(scale_factors)), C.c_float(th), int(mono), _p(out["active"]), _p(out["proj"]), _p(out["radius"]),
                                 _p(out["min_level"]), _p(out["max_level"]))
    return out


def line_project_mls(inview, bad, level, viewcos, scale_factors, th=1.0):
    """Projection stage of LSDmatcher::SearchByProjection(Frame&, const vector<MapLine*>&, th) (LSDmatcher.cpp:185-208)."""
    n = len(inview)
    out = dict(active=np.zeros(n, np.uint8), radius=np.zeros(n, np.float32), min_level=np.zeros(n, np.int32), max_level=np.zeros(n, np.int32))
    lib().orc_line_project_mls(n, _p(_u8(inview)), _p(_u8(bad)), _p(_i32(level)), _p(_f32(viewcos)), _p(_f32(scale_factors)), C.c_float(th),
                               _p(out["active"]), _p(out["radius"]), _p(out["min_level"]), _p(out["max_level"]))
    return out


def line_window_search(q, obs, dml, ld2, kl2, oct2, held2=None, nnratio=0.8):
    """Search stage of both line SearchByProjection overloads (LSDmatcher.cpp:98-137, :210-251).  q = dict(active, proj, radius,
    min_level, max_level); kl2[n,3] = pt.x, pt.y, angle -> (nmatches, assign2)."""
    nml = len(q["active"]); nl2 = len(oct2)
    out = np.full(max(nl2, 1), -1, np.int32)
    lib().orc_line_window_search.restype = C.c_int
    n = lib().orc_line_window_search(nml, _p(_u8(q["active"])), _p(_u8(obs)), _p(_f32(q["proj"])), _p(_f32(q["radius"])), _p(_i32(q["min_level"])),
                                     _p(_i32(q["max_level"])), _p(_u8(dml)), nl2, _p(_u8(ld2)), _p(_f32(kl2)), _p(_i32(oct2)),
                                     _p(_u8(held2)) if held2 is not None else None, C.c_float(nnratio), _p(out))
    return n, out[:nl2]


def fuse_project_points(skip, Xw, normal, min_inv, max_inv, max_raw, Tcw, Ow, cam5, bounds, nlevels, log_scale_factor):
    """Projection stage of ORBmatcher::Fuse (ORBmatcher.cc:828-894) -> dict(active, u, v, ur, level)."""
    n = len(skip)
    out = dict(active=np.zeros(n, np.uint8), u=np.zeros(n, np.float32), v=np.zeros(n, np.float32), ur=np.zeros(n, np.float32), level=np.zeros(n, np.int32))
    lib().orc_fuse_project_points(n, _p(_u8(skip)), _p(_f32(Xw)), _p(_f32(normal)), _p(_f32(min_inv)), _p(_f32(max_inv)), _p(_f32(max_raw)),
                                  _p(_f32(Tcw)), _p(_f32(Ow)), _p(_f32(cam5)), _p(_f32(bounds)), int(nlevels), C.c_float(log_scale_factor),
                                  _p(out["active"]), _p(out["u"]), _p(out["v"]), _p(out["ur"]), _p(out["level"]))
    return out


def fuse_points_search(q, dmp, d2, x2, y2, oct2, uright2, bounds, scale_factors, inv_level_sigma2, th=3.0):
    """Search stage of ORBmatcher::Fuse (ORBmatcher.cc:896-950) -> (best_idx, best_dist)."""
    n = len(q["active"])
    bi = np.full(max(n, 1), -1, np.int32); bd = np.full(max(n, 1), 256, np.int32)
    lib().orc_fuse_points_search(n, _p(_u8(q["active"])), _p(_f32(q["u"])), _p(_f32(q["v"])), _p(_f32(q["ur"])), _p(_i32(q["level"])), _p(_u8(dmp)),
                                 len(x2), _p(_u8(d2)), _p(_f32(x2)), _p(_f32(y2)), _p(_i32(oct2)), _p(_f32(uright2)) if uright2 is not None else None,
                                 _p(_f32(bounds)), _p(_f32(scale_factors)), _p(_f32(inv_level_sigma2)), C.c_float(th), _p(bi), _p(bd))
    return bi[:n], bd[:n]


def fuse_project_lines(skip, Pw, normal, min_inv, max_inv, max_raw, Tcw, Ow, cam5, bounds, nlevels, log_scale_factor):
    """Projection stage of LSDmatcher::Fuse (LSDmatcher.cpp:417-497) -> dict(active, proj[n,4], level)."""
    n = len(skip)
    out = dict(active=np.zeros(n, np.uint8), proj=np.zeros((n, 4), np.float32), level=np.zeros(n, np.int32))
    lib().orc_fuse_project_lines(n, _p(_u8(skip)), _p(_f32(Pw)), _p(_f32(normal)), _p(_f32(min_inv)), _p(_f32(max_inv)), _p(_f32(max_raw)),
                                 _p(_f32(Tcw)), _p(_f32(Ow)), _p(_f32(cam5)), _p(_f32(bounds)), int(nlevels), C.c_float(log_scale_factor),
                                 _p(out["active"]), _p(out["proj"]), _p(out["level"]))
    return out


def fuse_lines_search(q, dml, ld2, kl2, oct2, scale_factors, th=3.0):
    """Search stage of LSDmatcher::Fuse (LSDmatcher.cpp:499-523) -> (best_idx, best_dist)."""
    n = len(q["active"])
    bi = np.full(max(n, 1), -1, np.int32); bd = np.full(max(n, 1), 0x7fffffff, np.int32)
    lib().orc_fuse_lines_search(n, _p(_u8(q["active"])), _p(_f32(q["proj"])), _p(_i32(q["level"])), _p(_u8(dml)), len(oct2), _p(_u8(ld2)), _p(_f32(kl2)),
                                _p(_i32(oct2)), _p(_f32(scale_factors)), C.c_float(th), _p(bi), _p(bd))
    return bi[:n], bd[:n]


def features_in_area(kx, ky, oct, bounds, x, y, r, min_level=-1, max_level=-1):
    """Frame::GetFeaturesInArea (Frame.cc:368-421) over a freshly built grid (AssignFeaturesToGrid, :133-148)."""
    kx = _f32(kx); ky = _f32(ky); oct = np.ascontiguousarray(oct, np.int32)
    invw = np.float32(64) / (np.float32(bounds[1]) - np.float32(bounds[0])); invh = np.float32(48) / (np.float32(bounds[3]) - np.float32(bounds[2]))
    out = np.empty(max(len(kx), 1), np.int32)
    lib().orc_features_in_area.restype = C.c_int
    n = lib().orc_features_in_area(len(kx), _p(kx), _p(ky), _p(oct), C.c_float(bounds[0]), C.c_float(bounds[2]), C.c_float(invw), C.c_float(invh),
                                   C.c_float(x), C.c_float(y), C.c_float(r), int(min_level), int(max_level), _p(out), len(out))
    return out[:n]


def descriptor_medoid(desc, off):
    """ComputeDistinctiveDescriptors (MapPoint.cc:247-312) for CSR groups: (best index inside each group, its median distance)."""
    desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32); off = np.ascontiguousarray(off, np.int32)
    ng = len(off) - 1
    bi = np.empty(max(ng, 1), np.int32); bm = np.empty(max(ng, 1), np.int32)
    lib().orc_descriptor_medoid(_p(desc), _p(off), ng, _p(bi), _p(bm))
    return bi[:ng], bm[:ng]


def feature_vector_csr(node):
    """DBoW2::FeatureVector (std::map<NodeId, vector<unsigned>>, FeatureVector.cpp:31-45) flattened to CSR:
    node ids ascending, feature indices ascending inside a node."""
    node = np.asarray(node, np.int32)
    order = np.argsort(node, kind="stable").astype(np.int32)
    ids, counts = np.unique(node, return_counts=True)
    off = np.zeros(len(ids) + 1, np.int32)
    off[1:] = np.cumsum(counts)
    return ids.astype(np.int32), off, order


def _csr(args):
    return [np.ascontiguousarray(a, np.int32) for a in args]


def search_by_bow(d1, d2, fv1, fv2, valid1, angle1, angle2, nnratio=0.7, check_ori=True):
    d1 = np.ascontiguousarray(d1, np.uint8); d2 = np.ascontiguousarray(d2, np.uint8)
    n1s, o1, i1 = _csr(fv1); n2s, o2, i2 = _csr(fv2)
    valid1 = np.ascontiguousarray(valid1, np.uint8)
    angle1 = np.ascontiguousarray(angle1, np.float32); angle2 = np.ascontiguousarray(angle2, np.float32)
    m = np.empty(max(len(d2), 1), np.int32)
    n = lib().orc_search_by_bow(_p(d1), len(d1), _p(d2), len(d2), _p(n1s), _p(o1), _p(i1), len(n1s),
                                _p(n2s), _p(o2), _p(i2), len(n2s), _p(valid1), _p(angle1), _p(angle2),
                                C.c_float(nnratio), int(check_ori), _p(m))
    return n, m[:len(d2)]


def search_by_bow_kf(d1, d2, fv1, fv2, valid1, valid2, angle1, angle2, nnratio=0.7, check_ori=True):
    d1 = np.ascontiguousarray(d1, np.uint8); d2 = np.ascontiguousarray(d2, np.uint8)
    n1s, o1, i1 = _csr(fv1); n2s, o2, i2 = _csr(fv2)
    valid1 = np.ascontiguousarray(valid1, np.uint8); valid2 = np.ascontiguousarray(valid2, np.uint8)
    angle1 = np.ascontiguousarray(angle1, np.float32); angle2 = np.ascontiguousarray(angle2, np.float32)
    m = np.empty(max(len(d1), 1), np.int32)
    n = lib().orc_search_by_bow_kf(_p(d1), len(d1), _p(d2), len(d2), _p(n1s), _p(o1), _p(i1), len(n1s),
                                   _p(n2s), _p(o2), _p(i2), len(n2s), _p(valid1), _p(valid2), _p(angle1), _p(angle2),
                                   C.c_float(nnratio), int(check_ori), _p(m))
    return n, m[:len(d1)]


def search_for_triangulation(d1, d2, fv1, fv2, has_mp1, has_mp2, kp1, kp2, F12, ex, ey, scale, sigma2, check_ori=True):
    """kp1/kp2: structured KEYPOINT arrays (x, y, angle, octave used)."""
    d1 = np.ascontiguousarray(d1, np.uint8); d2 = np.ascontiguousarray(d2, np.uint8)
    n1s, o1, i1 = _csr(fv1); n2s, o2, i2 = _csr(fv2)
    has_mp1 = np.ascontiguousarray(has_mp1, np.uint8); has_mp2 = np.ascontiguousarray(has_mp2, np.uint8)
    f = lambda a: np.ascontiguousarray(a, np.float32)
    x1, y1, a1 = f(kp1["x"]), f(kp1["y"]), f(kp1["angle"])
    x2, y2, a2 = f(kp2["x"]), f(kp2["y"]), f(kp2["angle"])
    oc2 = np.ascontiguousarray(kp2["octave"], np.int32)
    F12 = f(F12).reshape(9); scale = f(scale); sigma2 = f(sigma2)
    pairs = np.empty((max(len(d1), 1), 2), np.int32)
    n = lib().orc_search_for_triangulation(_p(d1), len(d1), _p(d2), len(d2), _p(n1s), _p(o1), _p(i1), len(n1s),
                                           _p(n2s), _p(o2), _p(i2), len(n2s), _p(has_mp1), _p(has_mp2),
                                           _p(x1), _p(y1), _p(a1), _p(x2), _p(y2), _p(a2), _p(oc2),
                                           _p(F12), C.c_float(ex), C.c_float(ey), _p(scale), _p(sigma2),
                                           int(check_ori), _p(pairs))
    return n, pairs[:n].copy()


def line_mad(knn):
    knn = np.ascontiguousarray(knn, np.int32)
    a = C.c_double(); b = C.c_double()
    lib().orc_line_mad(_p(knn), len(knn), C.byref(a), C.byref(b))
    return a.value, b.value


def line_match(mode, d1, d2, has_ml1=None, has_ml2=None):
    d1 = np.ascontiguousarray(d1, np.uint8).reshape(-1, 32); d2 = np.ascontiguousarray(d2, np.uint8).reshape(-1, 32)
    has_ml1 = np.ascontiguousarray(has_ml1 if has_ml1 is not None else np.zeros(len(d1)), np.uint8)
    has_ml2 = np.ascontiguousarray(has_ml2 if has_ml2 is not None else np.zeros(len(d2)), np.uint8)
    out = np.full(2 * max(len(d1), len(d2), 1), -1, np.int32)
    k = C.c_int()
    n = lib().orc_line_match(mode, _p(d1), len(d1), _p(d2), len(d2), _p(has_ml1), _p(has_ml2), _p(out), C.byref(k))
    if mode == 0:
        return n, out[:len(d2)].copy()
    if mode == 2:
        return n, out[:len(d1)].copy()
    return n, out[:2 * k.value].reshape(-1, 2).copy()


# ---------------- lines ----------------
def lsd_detect_scaled(img, cap=1 << 14):
    """cv::createLineSegmentDetector(LSD_REFINE_ADV, scale=1.0).detect(img): float32 [n,4]."""
    img = _u8(img)
    seg = np.empty((cap, 4), np.float32)
    n = lib().orc_lsd_detect_scaled(_p(img), img.shape[1], img.shape[0], img.strides[0], _p(seg), cap)
    assert n <= cap
    return seg[:n].copy()


def lbd_prep(img):
    img = _u8(img)
    dx = np.empty(img.shape, np.int16); dy = np.empty(img.shape, np.int16)
    lib().orc_lbd_prep(_p(img), img.shape[1], img.shape[0], img.strides[0], _p(dx), _p(dy))
    return dx, dy


class LineOracle:
    """LineSegment::ExtractLineSegment restatement (ExtractLineSegment.cpp:18-69)."""

    def __init__(self, lsd_nfeatures=40, cr_trig=False):
        """cr_trig=True: region2rect takes cos / sin(theta) from the host form of the device's correctly-rounded ddtrig::sincos_cr_full
        instead of glibc, so that rectangles can be compared with the device's bit for bit."""
        self.nfeat = lsd_nfeatures
        self.h = C.c_void_p(lib().orc_line_create(lsd_nfeatures))
        if cr_trig:
            lib().orc_line_set_cr_trig(self.h, 1)

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_line_destroy(self.h)
            self.h = None

    def extract(self, img):
        img = _u8(img)
        cap = self.nfeat
        kl = np.zeros(cap, KEYLINE_DTYPE); ld = np.zeros((cap, 32), np.uint8); eq = np.zeros((cap, 3), np.float64)
        n = lib().orc_line_extract(self.h, _p(img), img.shape[1], img.shape[0], img.strides[0], _p(kl), _p(ld), _p(eq), cap)
        return kl[:n].copy(), ld[:n].copy(), eq[:n].copy()

    def raw_segments(self, cap=1 << 14):
        seg = np.empty((cap, 4), np.float32)
        n = lib().orc_line_raw_segments(self.h, _p(seg), cap)
        return seg[:n].copy()

    def scaled(self):
        w = C.c_int(); h = C.c_int()
        lib().orc_line_scaled_copy(self.h, None, 0, C.byref(w), C.byref(h))
        out = np.empty((h.value, w.value), np.uint8)
        lib().orc_line_scaled_copy(self.h, _p(out), out.strides[0], C.byref(w), C.byref(h))
        return out

    def trace(self, cap=1 << 16):
        out = np.empty((cap, 10), np.float64)
        n = lib().orc_line_trace(self.h, _p(out), cap)
        return out[:min(n, cap)].copy()

    def stage_ms(self):
        ms = np.empty(4, np.float64)
        lib().orc_line_stage_ms(self.h, _p(ms))
        return dict(zip(["prep", "lsd", "keylines", "lbd"], ms.tolist()))
