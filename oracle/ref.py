"""ctypes bindings of oracle/_ref/libref.so — the REFERENCE ITSELF (its hot-path sources compiled unmodified by
oracle/ref_build.sh against the stand-ins in oracle/refshim/), behind the C entry points of oracle/ref_harness.cpp.

TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/make_ref_golden.py to pin the oracle's restatement; the product
never loads it.  /root/reference is needed to BUILD the library (this container); the GPU box uses the prebuilt file.
"""
import ctypes as C
import os
import subprocess
import numpy as np

from .oracle import KEYPOINT_DTYPE, KEYLINE_DTYPE, _p, _u8, _csr, _f32

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "_ref", "libref.so")
_lib = None


def available():
    return os.path.exists(_LIB) or os.path.isdir("/root/reference/src")


def lib():
    global _lib
    if _lib is None:
        if os.path.isdir("/root/reference/src"):
            subprocess.run(["bash", os.path.join(_HERE, "ref_build.sh")], check=True, stdout=subprocess.DEVNULL)
        _lib = C.CDLL(_LIB)
        _lib.ref_vocab_load_text.restype = C.c_void_p
        _lib.ref_vocab_load_text.argtypes = [C.c_char_p]
    return _lib


CAM640 = np.array([500, 500, 320, 240, 0, 640, 0, 480], np.float32)


def cam(fx, fy, cx, cy, minx, maxx, miny, maxy):
    return np.array([fx, fy, cx, cy, minx, maxx, miny, maxy], np.float32)


def _kp(k):
    k = np.ascontiguousarray(k, KEYPOINT_DTYPE)
    return k


def orb_extract(img, nfeatures=1000, scale=1.2, nlevels=8, ini=20, mn=7, cap=None):
    """ORBextractor::operator() of the reference (bump allocator): (keypoints, descriptors, per-level counts)."""
    img = _u8(img)
    cap = cap or (nfeatures * 2 + 64 * nlevels)
    kps = np.zeros(cap, KEYPOINT_DTYPE); desc = np.zeros((cap, 32), np.uint8); lc = np.zeros(nlevels, np.int32)
    n = lib().ref_orb_extract(nfeatures, C.c_float(scale), nlevels, ini, mn, _p(img), img.shape[1], img.shape[0], img.strides[0],
                              _p(kps), _p(desc), cap, _p(lc))
    if n > cap:             # wide frames and small budgets keep more than 2 * nfeatures: run again with room for the full count
        return orb_extract(img, nfeatures, scale, nlevels, ini, mn, n)
    return kps[:n].copy(), desc[:n].copy(), lc


def orb_tables(nfeatures=1000, scale=1.2, nlevels=8):
    s = [np.zeros(nlevels, np.float32) for _ in range(4)]
    nf = np.zeros(nlevels, np.int32); um = np.zeros(16, np.int32)
    lib().ref_orb_tables(nfeatures, C.c_float(scale), nlevels, _p(s[0]), _p(s[1]), _p(s[2]), _p(s[3]), _p(nf), _p(um))
    return dict(scale=s[0], invscale=s[1], sigma2=s[2], invsigma2=s[3], nfeat=nf, umax=um)


def orb_pyramid_level(img, level, bordered=False, scale=1.2, nlevels=8):
    img = _u8(img)
    buf = np.zeros((img.shape[0] + 38) * (img.shape[1] + 38), np.uint8)
    w = C.c_int(); h = C.c_int()
    rc = lib().ref_orb_pyramid_level(_p(img), img.shape[1], img.shape[0], img.strides[0], C.c_float(scale), nlevels, level, int(bordered),
                                     _p(buf), buf.size, C.byref(w), C.byref(h))
    assert rc == 0
    return buf[:w.value * h.value].reshape(h.value, w.value).copy()


def octree(xs, ys, resp, minX, maxX, minY, maxY, N):
    xs = np.ascontiguousarray(xs, np.int32); ys = np.ascontiguousarray(ys, np.int32); resp = np.ascontiguousarray(resp, np.int32)
    out = np.zeros(N + 64, np.int32)
    n = lib().ref_octree(_p(xs), _p(ys), _p(resp), len(xs), minX, maxX, minY, maxY, N, _p(out), len(out))
    return out[:n].copy()


def descriptor_distance(a, b, line=False):
    a = np.ascontiguousarray(a, np.uint8); b = np.ascontiguousarray(b, np.uint8)
    f = lib().ref_line_descriptor_distance if line else lib().ref_descriptor_distance
    return f(_p(a), _p(b))


def search_by_bow(d1, k1, d2, k2, fv1, fv2, state1, nnratio=0.7, check_ori=True):
    d1 = np.ascontiguousarray(d1, np.uint8); d2 = np.ascontiguousarray(d2, np.uint8); k1 = _kp(k1); k2 = _kp(k2)
    n1s, o1, i1 = _csr(fv1); n2s, o2, i2 = _csr(fv2)
    state1 = np.ascontiguousarray(state1, np.uint8)
    m = np.empty(max(len(d2), 1), np.int32)
    n = lib().ref_search_by_bow(_p(d1), len(d1), _p(k1), _p(d2), len(d2), _p(k2), _p(n1s), _p(o1), _p(i1), len(n1s),
                                _p(n2s), _p(o2), _p(i2), len(n2s), _p(state1), C.c_float(nnratio), int(check_ori), _p(m))
    return n, m[:len(d2)]


def search_by_bow_kf(d1, k1, d2, k2, fv1, fv2, state1, state2, nnratio=0.7, check_ori=True):
    d1 = np.ascontiguousarray(d1, np.uint8); d2 = np.ascontiguousarray(d2, np.uint8); k1 = _kp(k1); k2 = _kp(k2)
    n1s, o1, i1 = _csr(fv1); n2s, o2, i2 = _csr(fv2)
    state1 = np.ascontiguousarray(state1, np.uint8); state2 = np.ascontiguousarray(state2, np.uint8)
    m = np.empty(max(len(d1), 1), np.int32)
    n = lib().ref_search_by_bow_kf(_p(d1), len(d1), _p(k1), _p(d2), len(d2), _p(k2), _p(n1s), _p(o1), _p(i1), len(n1s),
                                   _p(n2s), _p(o2), _p(i2), len(n2s), _p(state1), _p(state2), C.c_float(nnratio), int(check_ori), _p(m))
    return n, m[:len(d1)]


def search_for_triangulation(d1, k1, d2, k2, fv1, fv2, has_mp1, has_mp2, camv, Tcw1, Tcw2, F12, check_ori=True):
    """Returns (n, pairs[n,2], (ex, ey)) — the epipole as the reference computes it from the two poses."""
    d1 = np.ascontiguousarray(d1, np.uint8); d2 = np.ascontiguousarray(d2, np.uint8); k1 = _kp(k1); k2 = _kp(k2)
    n1s, o1, i1 = _csr(fv1); n2s, o2, i2 = _csr(fv2)
    has_mp1 = np.ascontiguousarray(has_mp1, np.uint8); has_mp2 = np.ascontiguousarray(has_mp2, np.uint8)
    camv = _f32(camv); T1 = _f32(Tcw1).reshape(-1)[:12].copy(); T2 = _f32(Tcw2).reshape(-1)[:12].copy(); F = _f32(F12).reshape(9)
    pairs = np.empty((max(len(d1), 1), 2), np.int32); epi = np.zeros(2, np.float32)
    n = lib().ref_search_for_triangulation(_p(d1), len(d1), _p(k1), _p(d2), len(d2), _p(k2), _p(n1s), _p(o1), _p(i1), len(n1s),
                                           _p(n2s), _p(o2), _p(i2), len(n2s), _p(has_mp1), _p(has_mp2), _p(camv), _p(T1), _p(T2),
                                           _p(F), int(check_ori), _p(pairs), _p(epi))
    return n, pairs[:n].copy(), (float(epi[0]), float(epi[1]))


def search_by_projection_frame(last, cur, Tcw, Tlw, camv, nlevels, scale, th, mono=True, check_ori=True, mbf=0.0):
    """last = dict(valid, obs|None, Xw[n,3], dmp[n,32], kps); cur = dict(desc, kps, claimed|None, uright|None)."""
    v1 = np.ascontiguousarray(last["valid"], np.uint8); n1 = len(v1)
    o1 = np.ascontiguousarray(last["obs"], np.uint8) if last.get("obs") is not None else None
    Xw = _f32(last["Xw"]).reshape(-1, 3); dmp = np.ascontiguousarray(last["dmp"], np.uint8).reshape(-1, 32); k1 = _kp(last["kps"])
    d2 = np.ascontiguousarray(cur["desc"], np.uint8).reshape(-1, 32); k2 = _kp(cur["kps"]); n2 = len(k2)
    cl = np.ascontiguousarray(cur["claimed"], np.uint8) if cur.get("claimed") is not None else None
    Tc = _f32(Tcw).reshape(-1)[:12].copy(); Tl = _f32(Tlw).reshape(-1)[:12].copy()
    out = np.full(max(n2, 1), -1, np.int32)
    ur = _f32(cur["uright"]) if cur.get("uright") is not None else None
    n = lib().ref_search_by_projection_frame(n1, _p(v1), _p(o1) if o1 is not None else None, _p(Xw), _p(dmp), _p(k1), n2, _p(d2), _p(k2),
                                             _p(cl) if cl is not None else None, _p(ur) if ur is not None else None, C.c_float(mbf), _p(Tc), _p(Tl), _p(_f32(camv)), nlevels, C.c_float(scale),
                                             C.c_float(th), int(mono), int(check_ori), _p(out))
    return n, out[:n2]


def search_by_projection_mps(mp, cur, camv, nlevels=8, scale=1.2, nnratio=0.8, th=1.0):
    """mp = dict(inview, bad, obs, projx, projy, level, viewcos, desc); cur = dict(desc, kps, claimed|None) (claimed: 0 / 1 / 2)."""
    nmp = len(mp["inview"])
    iv = np.ascontiguousarray(mp["inview"], np.uint8); bad = np.ascontiguousarray(mp["bad"], np.uint8); obs = np.ascontiguousarray(mp["obs"], np.uint8)
    px = _f32(mp["projx"]); py = _f32(mp["projy"]); lv = np.ascontiguousarray(mp["level"], np.int32); vc = _f32(mp["viewcos"])
    dmp = np.ascontiguousarray(mp["desc"], np.uint8).reshape(-1, 32)
    d2 = np.ascontiguousarray(cur["desc"], np.uint8).reshape(-1, 32); k2 = _kp(cur["kps"]); n2 = len(k2)
    cl = np.ascontiguousarray(cur["claimed"], np.uint8) if cur.get("claimed") is not None else None
    out = np.full(max(n2, 1), -1, np.int32)
    n = lib().ref_search_by_projection_mps(nmp, _p(iv), _p(bad), _p(obs), _p(px), _p(py), _p(lv), _p(vc), _p(dmp), n2, _p(d2), _p(k2),
                                           _p(cl) if cl is not None else None, _p(_f32(camv)), nlevels, C.c_float(scale),
                                           C.c_float(nnratio), C.c_float(th), _p(out))
    return n, out[:n2]


def search_for_initialization(d1, k1, d2, k2, prev, camv, nlevels=8, scale=1.2, nnratio=0.9, check_ori=True, window=100):
    d1 = np.ascontiguousarray(d1, np.uint8); d2 = np.ascontiguousarray(d2, np.uint8); k1 = _kp(k1); k2 = _kp(k2)
    prev = _f32(prev).reshape(-1, 2).copy()
    m12 = np.full(max(len(k1), 1), -1, np.int32)
    n = lib().ref_search_for_initialization(len(k1), _p(d1), _p(k1), len(k2), _p(d2), _p(k2), _p(prev), _p(_f32(camv)), nlevels,
                                            C.c_float(scale), C.c_float(nnratio), int(check_ori), int(window), _p(m12))
    return n, m12[:len(k1)], prev


def _u8(a):
    return np.ascontiguousarray(a, np.uint8)


def _i32(a):
    return np.ascontiguousarray(a, np.int32)


def _f64(a):
    return np.ascontiguousarray(a, np.float64)


def line_projection_frame(last, cur, Tcw, Tlw, camv, mb, nlevels=8, scale=1.2, nnratio=0.8, th=3.0, mono=True):
    """LSDmatcher::SearchByProjection(Frame&, const Frame&, th, bMono) :22-141.  last = dict(state, obs, Pw[n,6] f64, dml, oct);
    cur = dict(ld, kl[n,3], oct, held) -> (nmatches, assign2)."""
    nl1, nl2 = len(last["state"]), len(cur["oct"])
    out = np.full(max(nl2, 1), -1, np.int32)
    lib().ref_line_projection_frame.restype = C.c_int
    n = lib().ref_line_projection_frame(nl1, _p(_u8(last["state"])), _p(_u8(last["obs"])), _p(_f64(last["Pw"])), _p(_u8(last["dml"])), _p(_i32(last["oct"])),
                                        nl2, _p(_u8(cur["ld"])), _p(_f32(cur["kl"])), _p(_i32(cur["oct"])),
                                        _p(_u8(cur["held"])) if cur.get("held") is not None else None,
                                        _p(_f32(np.asarray(Tcw)[:3, :4])), _p(_f32(np.asarray(Tlw)[:3, :4])), _p(_f32(camv)), C.c_float(mb), nlevels,
                                        C.c_float(scale), C.c_float(nnratio), C.c_float(th), int(mono), _p(out))
    return n, out[:nl2]


def line_projection_mls(ml, cur, camv, nlevels=8, scale=1.2, nnratio=0.8, th=1.0):
    """LSDmatcher::SearchByProjection(Frame&, const vector<MapLine*>&, th) :185-255."""
    nml, nl2 = len(ml["inview"]), len(cur["oct"])
    out = np.full(max(nl2, 1), -1, np.int32)
    lib().ref_line_projection_mls.restype = C.c_int
    n = lib().ref_line_projection_mls(nml, _p(_u8(ml["inview"])), _p(_u8(ml["bad"])), _p(_u8(ml["obs"])), _p(_f32(ml["proj"])), _p(_i32(ml["level"])),
                                      _p(_f32(ml["viewcos"])), _p(_u8(ml["desc"])), nl2, _p(_u8(cur["ld"])), _p(_f32(cur["kl"])), _p(_i32(cur["oct"])),
                                      _p(_u8(cur["held"])) if cur.get("held") is not None else None, _p(_f32(camv)), nlevels, C.c_float(scale),
                                      C.c_float(nnratio), C.c_float(th), _p(out))
    return n, out[:nl2]


def fuse_points(mp, kf, Tcw, camv, mbf, nlevels=8, scale=1.2, th=3.0):
    """ORBmatcher::Fuse(KeyFrame*, const vector<MapPoint*>&, th) :828-973 -> (nFused, fused_idx, dict(Ow, min_inv, max_inv, log_scale))."""
    nmp = len(mp["state"]); k2 = _kp(kf["kps"]); n2 = len(k2)
    fi = np.full(max(nmp, 1), -1, np.int32); Ow = np.zeros(3, np.float32); mi = np.zeros(max(nmp, 1), np.float32); ma = np.zeros(max(nmp, 1), np.float32)
    ls = C.c_float()
    ur = _f32(kf["uright"]) if kf.get("uright") is not None else None
    lib().ref_fuse_points.restype = C.c_int
    n = lib().ref_fuse_points(nmp, _p(_u8(mp["state"])), _p(_i32(mp["nobs"])), _p(_f32(mp["Xw"])), _p(_f32(mp["normal"])), _p(_f32(mp["min_raw"])),
                              _p(_f32(mp["max_raw"])), _p(_u8(mp["desc"])), n2, _p(_u8(kf["desc"])), _p(k2), _p(ur) if ur is not None else None,
                              _p(_i32(kf["kfobs"])), _p(_f32(np.asarray(Tcw)[:3, :4])), _p(_f32(camv)), C.c_float(mbf), nlevels, C.c_float(scale), C.c_float(th),
                              _p(fi), _p(Ow), _p(mi), _p(ma), C.byref(ls))
    return n, fi[:nmp], dict(Ow=Ow, min_inv=mi[:nmp], max_inv=ma[:nmp], log_scale=ls.value)


def fuse_lines(ml, kf, Tcw, camv, nlevels=8, scale=1.2, th=3.0):
    """LSDmatcher::Fuse(KeyFrame*, const vector<MapLine*>&, th) :417-548 -> (nFused, fused_idx, dict(Ow, min_inv, max_inv, log_scale))."""
    nml = len(ml["state"]); nl2 = len(kf["oct"])
    fi = np.full(max(nml, 1), -1, np.int32); Ow = np.zeros(3, np.float32); mi = np.zeros(max(nml, 1), np.float32); ma = np.zeros(max(nml, 1), np.float32)
    ls = C.c_float()
    lib().ref_fuse_lines.restype = C.c_int
    n = lib().ref_fuse_lines(nml, _p(_u8(ml["state"])), _p(_i32(ml["nobs"])), _p(_f64(ml["Pw"])), _p(_f64(ml["normal"])), _p(_f32(ml["min_raw"])),
                             _p(_f32(ml["max_raw"])), _p(_u8(ml["desc"])), nl2, _p(_u8(kf["ld"])), _p(_f32(kf["kl"])), _p(_i32(kf["oct"])), _p(_i32(kf["kfobs"])),
                             _p(_f32(np.asarray(Tcw)[:3, :4])), _p(_f32(camv)), nlevels, C.c_float(scale), C.c_float(th),
                             _p(fi), _p(Ow), _p(mi), _p(ma), C.byref(ls))
    return n, fi[:nml], dict(Ow=Ow, min_inv=mi[:nml], max_inv=ma[:nml], log_scale=ls.value)


def features_in_area(kps, camv, x, y, r, min_level=-1, max_level=-1):
    k = _kp(kps); out = np.empty(max(len(k), 1), np.int32)
    n = lib().ref_features_in_area(len(k), _p(k), _p(_f32(camv)), C.c_float(x), C.c_float(y), C.c_float(r), int(min_level), int(max_level),
                                   _p(out), len(out))
    return out[:n].copy()


def descriptor_medoid(desc, off):
    desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32); off = np.ascontiguousarray(off, np.int32)
    bi = np.empty(max(len(off) - 1, 1), np.int32)
    lib().ref_descriptor_medoid(_p(desc), _p(off), len(off) - 1, _p(bi))
    return bi[:len(off) - 1]


def line_match(mode, d1, d2, has_ml1=None, has_ml2=None):
    """Same modes and outputs as oracle.line_match (+ mode 4 = SearchByDescriptor(KF,F)); also returns (nn_mad, nn12_mad)."""
    d1 = np.ascontiguousarray(d1, np.uint8).reshape(-1, 32); d2 = np.ascontiguousarray(d2, np.uint8).reshape(-1, 32)
    has_ml1 = np.ascontiguousarray(has_ml1 if has_ml1 is not None else np.zeros(len(d1)), np.uint8)
    has_ml2 = np.ascontiguousarray(has_ml2 if has_ml2 is not None else np.zeros(len(d2)), np.uint8)
    out = np.full(2 * max(len(d1), len(d2), 1), -1, np.int32)
    k = C.c_int(); mad = np.zeros(2, np.float64)
    n = lib().ref_line_match(mode, _p(d1), len(d1), _p(d2), len(d2), _p(has_ml1), _p(has_ml2), _p(out), C.byref(k), _p(mad))
    if mode in (0, 4):
        return n, out[:len(d2)].copy(), tuple(mad)
    if mode == 2:
        return n, out[:len(d1)].copy(), tuple(mad)
    return n, out[:2 * k.value].reshape(-1, 2).copy(), tuple(mad)


class Vocabulary:
    """The reference's ORBVocabulary (DBoW2::TemplatedVocabulary<FORB>) loaded with its own loadFromTextFile."""

    def __init__(self, path):
        self.h = lib().ref_vocab_load_text(path.encode())
        assert self.h, path

    def __del__(self):
        if getattr(self, "h", None):
            lib().ref_vocab_destroy(C.c_void_p(self.h)); self.h = None

    def __len__(self):
        return lib().ref_vocab_size(C.c_void_p(self.h))

    def transform(self, desc, levelsup=4):
        """(node per feature, bow word ids, bow weights) — Frame::ComputeBoW's call (Frame.cc:479)."""
        desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32); n = len(desc)
        node = np.empty(max(n, 1), np.int32); ids = np.empty(max(n, 1), np.int32); w = np.empty(max(n, 1), np.float64)
        k = lib().ref_vocab_transform(C.c_void_p(self.h), _p(desc), n, levelsup, _p(node), _p(ids), _p(w), len(ids))
        return node[:n].copy(), ids[:k].copy(), w[:k].copy()

    def words(self, desc):
        desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32); n = len(desc)
        word = np.empty(max(n, 1), np.int32); w = np.empty(max(n, 1), np.float64)
        lib().ref_vocab_words(C.c_void_p(self.h), _p(desc), n, _p(word), _p(w))
        return word[:n].copy(), w[:n].copy()


def line_extract(img, cap=64):
    """LineSegment::ExtractLineSegment (ExtractLineSegment.cpp:18-69; lsdNFeatures = 40 is hard-coded there)."""
    img = _u8(img)
    kl = np.zeros(cap, KEYLINE_DTYPE); ld = np.zeros((cap, 32), np.uint8); eq = np.zeros((cap, 3), np.float64)
    n = lib().ref_line_extract(_p(img), img.shape[1], img.shape[0], img.strides[0], _p(kl), _p(ld), _p(eq), cap)
    return kl[:n].copy(), ld[:n].copy(), eq[:n].copy()


def frame_from_image(img, nfeatures=1000, scale=1.2, nlevels=8, ini=20, mn=7, K=(500, 500, 320, 240), dist=(0, 0, 0, 0)):
    """Frame::Frame(imGray, ...) (Frame.cc:69-131): dict(keys, keysUn, desc, keylines, ldesc, lineeq, grid_off, grid_idx, bounds).
    dist: k1 k2 p1 p2 [k3], 4 or 5 coefficients as Tracking.cc:61-72 builds mDistCoef."""
    img = _u8(img)
    dist = _f32(dist)
    assert len(dist) in (4, 5)
    cap = nfeatures * 2 + 64 * nlevels; lcap = 64
    keys = np.zeros(cap, KEYPOINT_DTYPE); keysun = np.zeros(cap, KEYPOINT_DTYPE); desc = np.zeros((cap, 32), np.uint8)
    kl = np.zeros(lcap, KEYLINE_DTYPE); ld = np.zeros((lcap, 32), np.uint8); eq = np.zeros((lcap, 3), np.float64)
    NL = C.c_int(); goff = np.zeros(64 * 48 + 1, np.int32); gidx = np.zeros(cap, np.int32); b = np.zeros(4, np.float32)
    n = lib().ref_frame_from_image(_p(img), img.shape[1], img.shape[0], img.strides[0], nfeatures, C.c_float(scale), nlevels, ini, mn,
                                   _p(_f32(K)), _p(dist), len(dist), _p(keys), _p(keysun), _p(desc), cap, _p(kl), _p(ld), _p(eq), lcap,
                                   C.byref(NL), _p(goff), _p(gidx), _p(b))
    nl = NL.value
    return dict(keys=keys[:n].copy(), keysUn=keysun[:n].copy(), desc=desc[:n].copy(), keylines=kl[:nl].copy(), ldesc=ld[:nl].copy(),
                lineeq=eq[:nl].copy(), grid_off=goff, grid_idx=gidx[:goff[-1]].copy(), bounds=b)


def cvt_gray(img, rgb):
    img = np.ascontiguousarray(img, np.uint8); h, w, cn = img.shape
    out = np.empty((h, w), np.uint8)
    lib().ref_cvt_gray(_p(img), w, h, cn, int(rgb), _p(out))
    return out
