"""structure-slam-pointline_b200 — host-side Python mirror of the reference interface over libsslpl_b200.so.

The product is the C-ABI shared library (include/sslpl.h) built from csrc/*.cu for sm_90a; the C++
adapters with the reference's own class signatures live in host/.  This module is the thin ctypes layer
the tests and bench.py use; its classes carry the reference's names and argument meaning:

    ORBextractor(nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST)   include/ORBextractor.h:45-111
        __call__(image) -> (keypoints, descriptors)                       src/ORBextractor.cc:1043
    LineSegment().ExtractLineSegment(img) -> (keylines, ldesc, keylineFunctions)   src/ExtractLineSegment.cpp:18
    ORBmatcher(nnratio, checkOri).SearchByBoW / SearchForTriangulation    src/ORBmatcher.cc:159,525,660
    LSDmatcher().SearchByProjection / SerachForInitialize / ...           src/LSDmatcher.cpp:143,257,286,329,382

There is no CPU fallback and nothing here imports oracle/: if the CUDA library is missing or no GPU is
present, construction raises.  (The package directory name contains '-', so import it through
`__graft_entry__.load_package()`, which registers it as module `sslpl_b200`.)
"""
import ctypes as C
import os
import re
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsslpl_b200.so")

KEYPOINT_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                           ("octave", "<i4"), ("class_id", "<i4")])
KEYLINE_DTYPE = np.dtype([("angle", "<f4"), ("class_id", "<i4"), ("octave", "<i4"), ("pt_x", "<f4"), ("pt_y", "<f4"),
                          ("response", "<f4"), ("size", "<f4"),
                          ("startPointX", "<f4"), ("startPointY", "<f4"), ("endPointX", "<f4"), ("endPointY", "<f4"),
                          ("sPointInOctaveX", "<f4"), ("sPointInOctaveY", "<f4"),
                          ("ePointInOctaveX", "<f4"), ("ePointInOctaveY", "<f4"),
                          ("lineLength", "<f4"), ("numOfPixels", "<i4")])
assert KEYPOINT_DTYPE.itemsize == 28 and KEYLINE_DTYPE.itemsize == 68


class SslplError(RuntimeError):
    pass


class OrbParams(C.Structure):
    _fields_ = [("nfeatures", C.c_int), ("scaleFactor", C.c_float), ("nlevels", C.c_int), ("iniThFAST", C.c_int),
                ("minThFAST", C.c_int), ("max_width", C.c_int), ("max_height", C.c_int), ("max_batch", C.c_int),
                ("device", C.c_int)]


class MatcherParams(C.Structure):
    _fields_ = [("max_features", C.c_int), ("max_lines", C.c_int), ("max_nodes", C.c_int), ("max_batch", C.c_int),
                ("device", C.c_int)]


class LineParams(C.Structure):
    _fields_ = [("lsdNFeatures", C.c_int), ("max_width", C.c_int), ("max_height", C.c_int), ("max_batch", C.c_int),
                ("device", C.c_int)]


class FeatVec(C.Structure):
    _fields_ = [("nodes", C.c_void_p), ("off", C.c_void_p), ("idx", C.c_void_p), ("nn", C.c_int)]


_SCALARS = {"int": C.c_int, "float": C.c_float, "double": C.c_double, "size_t": C.c_size_t, "long long": C.c_longlong}


def _prototypes(text):
    """{name: (restype, argtypes)} of every sslpl_* function declared in `text`, the source of include/sslpl.h.  Every pointer is a
    c_void_p, except that a const char* return comes back as bytes.  A scalar type outside _SCALARS raises, so no argument of a new
    type reaches C without a conversion."""
    def ctype(decl, name, named):
        if "*" in decl:
            return C.c_void_p
        words = [w for w in decl.split() if w != "const"]
        t = " ".join(words[:-1] if named else words)
        if t not in _SCALARS:
            raise SslplError(f"include/sslpl.h: {name} uses {t!r}, which has no ctypes type here")
        return _SCALARS[t]

    protos = {}
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    for ret, name, params in re.findall(r"^\s*([A-Za-z_][\w ]*\**)\s*(sslpl_\w+)\s*\(([^)]*)\)\s*;", text, flags=re.M):
        ret = " ".join(ret.split())
        restype = None if ret == "void" else C.c_char_p if ret == "const char*" else ctype(ret, name, False)
        argtypes = [] if params.strip() == "void" else [ctype(p, name, True) for p in params.split(",")]
        protos[name] = (restype, argtypes)
    return protos


_lib = None


def lib():
    """Load libsslpl_b200.so with the prototypes of include/sslpl.h and include/sslpl_map.h on every function (fails loudly when it has
    not been built: run __graft_entry__.build())."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SslplError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'`"
                             " (there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        for header in ("sslpl.h", "sslpl_map.h"):
            with open(os.path.join(_HERE, "..", "include", header)) as f:
                for name, (restype, argtypes) in _prototypes(f.read()).items():
                    fn = getattr(L, name)
                    fn.restype, fn.argtypes = restype, argtypes
        _lib = L
    return _lib


def _check(rc):
    if rc != 0:
        raise SslplError(f"sslpl error {rc}: {lib().sslpl_last_error().decode(errors='replace')}")


def _p(a):
    """An ndarray as a pointer argument (a c_void_p argtype rejects the array itself); the result keeps the array alive through the
    call.  None stays NULL."""
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _u8(a):
    return None if a is None else np.ascontiguousarray(a, np.uint8)


def _i32(a):
    return None if a is None else np.ascontiguousarray(a, np.int32)


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, np.float32)


def _f64(a):
    return None if a is None else np.ascontiguousarray(a, np.float64)


class _Handle:
    """A handle of include/sslpl.h.  A subclass names its kind, the <kind> of the sslpl_<kind>_* functions, and takes the lifecycle
    methods the header declares for that kind: class Matcher(_Handle, kind="matcher", lifecycle=("sync", ...)).  A borrowed handle
    belongs to another one (Frame's extractors): same methods, never destroyed from here."""
    _h = None
    _borrowed = False

    def __init_subclass__(cls, kind, lifecycle=()):
        cls._kind = kind
        for name in lifecycle:
            setattr(cls, name, getattr(_Handle, "_" + name))

    def _fn(self, name):
        return getattr(lib(), f"sslpl_{self._kind}_{name}")

    def _create(self, params):
        self._h = C.c_void_p()
        _check(self._fn("create")(C.byref(params), C.byref(self._h)))

    @classmethod
    def _borrow(cls, ptr, **attrs):
        self = cls.__new__(cls)
        self.__dict__.update(attrs, _h=C.c_void_p(ptr), _borrowed=True)
        return self

    def close(self):
        if self._h is not None and self._h.value and not self._borrowed:
            self._fn("destroy")(self._h)
            self._h = C.c_void_p()

    __del__ = close

    # the lifecycle methods, public under their names without the underscore in the classes that take them
    def _sync(self):
        _check(self._fn("sync")(self._h))

    def _set_stream(self, cuda_stream):
        _check(self._fn("set_stream")(self._h, cuda_stream))

    _stream = property(lambda self: self._fn("stream")(self._h))
    _launch_count = property(lambda self: self._fn("launch_count")(self._h))

    def _set_profiling(self, on=True):
        _check(self._fn("set_profiling")(self._h, int(on)))

    def _stage_ms(self):
        ms = (C.c_float * 16)(); names = (C.c_char_p * 16)(); n = C.c_int()
        _check(self._fn("stage_ms")(self._h, ms, 16, names, C.byref(n)))
        return {names[i].decode(): float(ms[i]) for i in range(n.value)}


def device_count():
    return lib().sslpl_device_count()


def host_alloc(shape, dtype=np.uint8):
    """Pinned host ndarray (sslpl_host_alloc); keeps the allocation alive through .base."""
    dtype = np.dtype(dtype)
    nbytes = int(np.prod(shape)) * dtype.itemsize
    ptr = C.c_void_p()
    _check(lib().sslpl_host_alloc(C.byref(ptr), max(nbytes, 1)))
    buf = (C.c_uint8 * max(nbytes, 1)).from_address(ptr.value)
    arr = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)
    return arr


class ORBextractor(_Handle, kind="orb", lifecycle=("sync", "set_stream", "stream", "launch_count", "set_profiling", "stage_ms")):
    """Mirror of StructureSLAM::ORBextractor (include/ORBextractor.h:45-111)."""

    def __init__(self, nfeatures=1000, scaleFactor=1.2, nlevels=8, iniThFAST=20, minThFAST=7,
                 max_width=1280, max_height=960, max_batch=1, device=0):
        self.nfeatures, self.scaleFactor, self.nlevels = nfeatures, scaleFactor, nlevels
        self._create(OrbParams(nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST, max_width, max_height, max_batch, device))
        self.max_batch = max_batch
        self.cap = lib().sslpl_orb_max_keypoints(self._h)

    # ORBextractor.h:60-77
    def GetLevels(self):
        return self.nlevels

    def GetScaleFactor(self):
        return self.scaleFactor

    def _tables(self):
        L = self.nlevels
        sc, isc, s2, is2 = (np.empty(L, np.float32) for _ in range(4))
        nf = np.empty(L, np.int32); um = np.empty(16, np.int32)
        _check(lib().sslpl_orb_tables(self._h, _p(sc), _p(isc), _p(s2), _p(is2), _p(nf), _p(um)))
        return dict(scale=sc, invscale=isc, sigma2=s2, invsigma2=is2, nfeat=nf, umax=um)

    def GetScaleFactors(self):
        return self._tables()["scale"]

    def GetInverseScaleFactors(self):
        return self._tables()["invscale"]

    def GetScaleSigmaSquares(self):
        return self._tables()["sigma2"]

    def GetInverseScaleSigmaSquares(self):
        return self._tables()["invsigma2"]

    def __call__(self, image, mask=None):
        """operator()(image, mask /*ignored*/, keypoints, descriptors) — ORBextractor.cc:1043."""
        if image is None or image.size == 0:
            return np.zeros(0, KEYPOINT_DTYPE), np.zeros((0, 32), np.uint8)      # silent return, ORBextractor.cc:1046
        assert image.dtype == np.uint8 and image.ndim == 2, "CV_8UC1 expected (ORBextractor.cc:1050)"
        if image.strides[1] != 1:
            image = np.ascontiguousarray(image)
        kps = np.zeros(self.cap, KEYPOINT_DTYPE); desc = np.zeros((self.cap, 32), np.uint8)
        n = C.c_int()
        _check(lib().sslpl_orb_extract(self._h, _p(image), image.shape[1], image.shape[0], image.strides[0],
                                       _p(kps), _p(desc), self.cap, C.byref(n)))
        return kps[:n.value].copy(), desc[:n.value].copy()

    def extract_batch(self, frames, out=None):
        """frames: (B,H,W) uint8 host array (pinned for full H2D speed). Returns (kps[B,cap], desc[B,cap,32], n[B])."""
        assert frames.dtype == np.uint8 and frames.ndim == 3 and frames.strides[2] == 1
        B, H, W = frames.shape
        if out is None:
            out = (np.zeros((B, self.cap), KEYPOINT_DTYPE), np.zeros((B, self.cap, 32), np.uint8), np.zeros(B, np.int32))
        kps, desc, n = out
        _check(lib().sslpl_orb_extract_batch(self._h, _p(frames), B, W, H, frames.strides[1], frames.strides[0],
                                             _p(kps), _p(desc), self.cap, _p(n)))
        return kps, desc, n

    def extract_batch_begin(self, frames, out):
        """Asynchronous host-buffer form: returns immediately; `out` (pinned) is valid after sync()."""
        B, H, W = frames.shape
        kps, desc, n = out
        _check(lib().sslpl_orb_extract_batch_begin(self._h, _p(frames), B, W, H, frames.strides[1], frames.strides[0],
                                                   _p(kps), _p(desc), self.cap, _p(n)))

    def extract_batch_device(self, d_ptr, nframes, width, height, pitch, frame_stride):
        """Frames already in HBM (raw device pointer, e.g. torch_tensor.data_ptr()); asynchronous."""
        _check(lib().sslpl_orb_extract_batch_device(self._h, d_ptr, nframes, width, height, pitch, frame_stride))

    def device_results(self):
        kps = C.c_void_p(); desc = C.c_void_p(); n = C.c_void_p(); cap = C.c_int()
        _check(lib().sslpl_orb_device_results(self._h, C.byref(kps), C.byref(desc), C.byref(n), C.byref(cap)))
        return kps.value, desc.value, n.value, cap.value

    # ---- stage intermediates (parity tests) ----
    def level_size(self, l):
        w = C.c_int(); h = C.c_int()
        _check(lib().sslpl_orb_level_size(self._h, l, C.byref(w), C.byref(h)))
        return w.value, h.value

    def level(self, l, frame=0, bordered=False):
        """mvImagePyramid[l] (ORBextractor.h:79)."""
        w, h = self.level_size(l)
        b = 19 if bordered else 0
        out = np.empty((h + 2 * b, w + 2 * b), np.uint8)
        _check(lib().sslpl_orb_download_level(self._h, frame, l, int(bordered), _p(out), out.strides[0]))
        return out

    def blurred(self, l, frame=0):
        w, h = self.level_size(l)
        out = np.empty((h, w), np.uint8)
        _check(lib().sslpl_orb_download_blurred(self._h, frame, l, _p(out), out.strides[0]))
        return out

    def candidates(self, l, frame=0, cap=1 << 17):
        xs = np.empty(cap, np.int32); ys = np.empty(cap, np.int32); rs = np.empty(cap, np.int32); n = C.c_int()
        _check(lib().sslpl_orb_download_candidates(self._h, frame, l, _p(xs), _p(ys), _p(rs), cap, C.byref(n)))
        if n.value > cap:                  # *n is the full count: a wide level of noise can hold more
            return self.candidates(l, frame, n.value)
        return xs[:n.value].copy(), ys[:n.value].copy(), rs[:n.value].copy()

    def level_keypoints(self, l, frame=0, cap=1 << 15):
        xs = np.empty(cap, np.int32); ys = np.empty(cap, np.int32); rs = np.empty(cap, np.int32); n = C.c_int()
        _check(lib().sslpl_orb_download_level_keypoints(self._h, frame, l, _p(xs), _p(ys), _p(rs), cap, C.byref(n)))
        if n.value > cap:
            return self.level_keypoints(l, frame, n.value)
        return xs[:n.value].copy(), ys[:n.value].copy(), rs[:n.value].copy()


# =====================================================================================================
# Matching
# =====================================================================================================
def _featvec(fv):
    """(nodes, off, idx) int32 arrays -> FeatVec struct (keeps references alive)."""
    nodes, off, idx = (_i32(a) for a in fv)
    s = FeatVec(_p(nodes) if len(nodes) else None, _p(off), _p(idx) if len(idx) else None, len(nodes))
    s._keep = (nodes, off, idx)
    return s


def feature_vector_csr(node):
    """DBoW2::FeatureVector (std::map<NodeId, vector<unsigned>>; FeatureVector.cpp:31-45) flattened to CSR."""
    node = np.asarray(node, np.int32)
    order = np.argsort(node, kind="stable").astype(np.int32)
    ids, counts = np.unique(node, return_counts=True)
    off = np.zeros(len(ids) + 1, np.int32)
    off[1:] = np.cumsum(counts)
    return ids.astype(np.int32), off, order


class Matcher(_Handle, kind="matcher", lifecycle=("sync", "set_stream", "stream", "launch_count")):
    """Device context shared by ORBmatcher / LSDmatcher below (one stream + workspace; create one per thread)."""

    def __init__(self, max_features=4096, max_lines=512, max_nodes=1024, max_batch=1, device=0):
        self._create(MatcherParams(max_features, max_lines, max_nodes, max_batch, device))
        self.max_features, self.max_lines = max_features, max_lines

    def descriptor_distance(self, a, b):
        a = _u8(a).reshape(-1, 32); b = _u8(b).reshape(-1, 32)
        out = np.empty(len(a), np.int32)
        _check(lib().sslpl_descriptor_distance(self._h, _p(a), _p(b), len(a), _p(out)))
        return out

    def knn2(self, q, t):
        """cv::BFMatcher(NORM_HAMMING).knnMatch(q, t, k=2) -> int32 [nq,4] = idx0, d0, idx1, d1."""
        q = _u8(q).reshape(-1, 32); t = _u8(t).reshape(-1, 32)
        out = np.empty((len(q), 4), np.int32)
        _check(lib().sslpl_hamming_knn2(self._h, _p(q), len(q), _p(t), len(t), _p(out)))
        return out

    def bow_assign(self, desc, centroids):
        desc = _u8(desc).reshape(-1, 32); centroids = _u8(centroids).reshape(-1, 32)
        node = np.empty(len(desc), np.int32)
        _check(lib().sslpl_bow_assign(self._h, _p(desc), len(desc), _p(centroids), len(centroids), _p(node)))
        return node

    def match_bow_batch_device(self, d_desc, d_kps, d_n, nframes, cap, d_centroids, nc, nnratio, check_ori, d_match, d_nmatch):
        _check(lib().sslpl_match_bow_batch_device(self._h, d_desc, d_kps, d_n, nframes, cap, d_centroids, nc, nnratio, int(check_ori),
                                                  d_match, d_nmatch))

    def match_bow_batch_device_vocab(self, d_desc, d_kps, d_n, nframes, cap, vocab, levelsup, nnratio, check_ori, d_match, d_nmatch,
                                     d_word=0, d_node=0, d_weight=0):
        """Batched SearchByBoW with the DBoW2 tree transform (optional per-feature word / node / weight outputs in HBM)."""
        _check(lib().sslpl_match_bow_batch_device_vocab(self._h, d_desc, d_kps, d_n, nframes, cap, vocab._h, levelsup, nnratio,
                                                        int(check_ori), d_match, d_nmatch, d_word or None, d_node or None, d_weight or None))

    def bow_transform(self, vocab, desc, levelsup=4):
        """TemplatedVocabulary::transform per feature (TemplatedVocabulary.h:1218-1259): (word, node, weight) arrays."""
        desc = _u8(desc).reshape(-1, 32)
        n = len(desc)
        word = np.empty(max(n, 1), np.int32); node = np.empty(max(n, 1), np.int32); w = np.empty(max(n, 1), np.float64)
        _check(lib().sslpl_bow_transform(self._h, vocab._h, _p(desc), n, levelsup, _p(word), _p(node), _p(w)))
        return word[:n], node[:n], w[:n]

    def search_by_projection_mps(self, mp, cur, bounds, scale_factors, nnratio=0.8, th=1.0):
        """ORBmatcher::SearchByProjection(Frame&, const vector<MapPoint*>&, th) (ORBmatcher.cc:45-129).
        mp = dict(inview, bad, obs, projx, projy, level, viewcos, desc[, projxr]); cur = dict(desc, x, y, oct[, uright, held])."""
        nmp = len(mp["inview"]); n2 = len(cur["x"])
        iv, bad, obs = _u8(mp["inview"]), _u8(mp["bad"]), _u8(mp["obs"])
        px, py, pxr = _f32(mp["projx"]), _f32(mp["projy"]), _f32(mp.get("projxr"))
        lv = _i32(mp["level"]); vc = _f32(mp["viewcos"]); dmp = _u8(mp["desc"]).reshape(-1, 32)
        d2 = _u8(cur["desc"]).reshape(-1, 32); x2, y2 = _f32(cur["x"]), _f32(cur["y"]); oc2 = _i32(cur["oct"])
        ur, held = _f32(cur.get("uright")), _u8(cur.get("held"))
        sf = _f32(scale_factors); out = np.full(max(n2, 1), -1, np.int32); nm = C.c_int()
        _check(lib().sslpl_search_by_projection_mps(self._h, nmp, _p(iv), _p(bad), _p(obs), _p(px), _p(py), _p(pxr), _p(lv), _p(vc), _p(dmp),
                                                    n2, _p(d2), _p(x2), _p(y2), _p(oc2), _p(ur), _p(held), _p(_f32(bounds)), _p(sf), len(sf),
                                                    nnratio, th, _p(out), C.byref(nm)))
        return nm.value, out[:n2]

    def line_search_by_projection(self, q, obs, dml, ld2, kl2, oct2, held2=None, nnratio=0.8):
        """Search stage of LSDmatcher::SearchByProjection(Frame&, const Frame&, th, bMono) (LSDmatcher.cpp:98-137) and of
        LSDmatcher::SearchByProjection(Frame&, const vector<MapLine*>&, th) (:210-251).  q = dict(active, proj[n,4], radius, min_level,
        max_level) per MapLine (the projection stage's outputs), obs = Observations() > 0, dml their descriptors; ld2 / kl2[n,3] (pt.x,
        pt.y, angle) / oct2 / held2 the frame's lines -> (nmatches, assign2)."""
        nml = len(q["active"]); nl2 = len(oct2)
        out = np.full(max(nl2, 1), -1, np.int32); nm = C.c_int()
        _check(lib().sslpl_line_search_by_projection(self._h, nml, _p(_u8(q["active"])), _p(_u8(obs)), _p(_f32(q["proj"])), _p(_f32(q["radius"])),
                                                     _p(_i32(q["min_level"])), _p(_i32(q["max_level"])), _p(_u8(dml)), nl2, _p(_u8(ld2)), _p(_f32(kl2)), _p(_i32(oct2)),
                                                     _p(_u8(held2)), nnratio, _p(out), C.byref(nm)))
        return nm.value, out[:nl2]

    def fuse_lines_search(self, q, dml, ld2, kl2, oct2, scale_factors, th=3.0):
        """Search stage of LSDmatcher::Fuse (LSDmatcher.cpp:495-523).  q = dict(active, proj[n,4], level) -> (best_idx, best_dist)."""
        n = len(q["active"]); sf = _f32(scale_factors)
        bi = np.full(max(n, 1), -1, np.int32); bd = np.full(max(n, 1), 0x7fffffff, np.int32)
        _check(lib().sslpl_fuse_lines_search(self._h, n, _p(_u8(q["active"])), _p(_f32(q["proj"])), _p(_i32(q["level"])), _p(_u8(dml)), len(oct2), _p(_u8(ld2)),
                                             _p(_f32(kl2)), _p(_i32(oct2)), _p(sf), len(sf), th, _p(bi), _p(bd)))
        return bi[:n], bd[:n]

    def fuse_points_search(self, q, dmp, d2, x2, y2, oct2, uright2, bounds, scale_factors, inv_level_sigma2, th=3.0):
        """Search stage of ORBmatcher::Fuse (ORBmatcher.cc:889-950).  q = dict(active, u, v, ur, level) -> (best_idx, best_dist)."""
        n = len(q["active"]); sf = _f32(scale_factors)
        bi = np.full(max(n, 1), -1, np.int32); bd = np.full(max(n, 1), 256, np.int32)
        _check(lib().sslpl_fuse_points_search(self._h, n, _p(_u8(q["active"])), _p(_f32(q["u"])), _p(_f32(q["v"])), _p(_f32(q["ur"])), _p(_i32(q["level"])), _p(_u8(dmp)),
                                              len(x2), _p(_u8(d2)), _p(_f32(x2)), _p(_f32(y2)), _p(_i32(oct2)), _p(_f32(uright2)),
                                              _p(_f32(bounds)), _p(sf), _p(_f32(inv_level_sigma2)), len(sf), th, _p(bi), _p(bd)))
        return bi[:n], bd[:n]

    def search_for_initialization(self, d1, k1, d2, k2, prev, bounds, nnratio=0.9, check_ori=True, window=100):
        """ORBmatcher::SearchForInitialization (ORBmatcher.cc:408-523) -> (nmatches, matches12, prev_out)."""
        d1 = _u8(d1).reshape(-1, 32); d2 = _u8(d2).reshape(-1, 32)
        prev = _f32(prev).reshape(-1, 2).copy()
        m12 = np.full(max(len(k1), 1), -1, np.int32); nm = C.c_int()
        _check(lib().sslpl_search_for_initialization(self._h, len(k1), _p(d1), _p(_i32(k1["octave"])), _p(_f32(k1["angle"])), _p(prev),
                                                     len(k2), _p(d2), _p(_f32(k2["x"])), _p(_f32(k2["y"])), _p(_i32(k2["octave"])),
                                                     _p(_f32(k2["angle"])), _p(_f32(bounds)), nnratio, int(check_ori), window, _p(m12), C.byref(nm)))
        return nm.value, m12[:len(k1)], prev

    def search_for_initialization_batch_device(self, d_kps, d_desc, d_n, nrows, cap, npairs, d_pair, d_prev0, bounds, nnratio, check_ori,
                                               window, d_match12, d_prev, d_nmatch):
        """ORBmatcher::SearchForInitialization (ORBmatcher.cc:408-523) over the chains of a pair list of a row set in HBM (see
        sslpl_search_for_initialization_batch_device): d_kps / d_desc / d_n as the extractors give them (2 x nFeatures), d_pair [npairs, 2]
        i32 (init row, current row), d_prev0 [npairs, cap, 2] f32 or 0 (the init rows' keypoints), host bounds -> d_match12 [npairs, cap]
        i32, d_prev [npairs, cap, 2] f32 (vbPrevMatched after each pair), d_nmatch [npairs] i32 (-1: bad pair).  Asynchronous on the
        matcher's stream."""
        _check(lib().sslpl_search_for_initialization_batch_device(self._h, d_kps, d_desc, d_n, nrows, cap, npairs, d_pair, d_prev0 or None,
                                                                  _p(_f32(bounds)), nnratio, int(check_ori), window, d_match12, d_prev,
                                                                  d_nmatch))

    def search_by_projection_frame(self, last, cur, Tcw, Tlw, cam, bounds, scale_factors, th, mono=True, check_ori=True, raw=False):
        """ORBmatcher::SearchByProjection(Frame &CurrentFrame, const Frame &LastFrame, th, bMono) (ORBmatcher.cc:1331-1473).
        last = dict(valid, obs, Xw[n,3], dmp[n,32], oct, angle); cur = dict(desc[n,32], x, y, oct, angle, uright|None, claimed|None);
        Tcw / Tlw 3x4 (or 4x4) row-major; cam = (fx, fy, cx, cy, mbf, mb); bounds = (minX, maxX, minY, maxY).
        Returns (nmatches, assign2) with assign2[j] = index of the last-frame MapPoint given to current feature j or -1."""
        n1, n2 = len(last["valid"]), len(cur["x"])
        v1 = _u8(last["valid"]); o1 = _u8(last["obs"])
        Xw = _f32(last["Xw"]).reshape(-1, 3); dmp = _u8(last["dmp"]).reshape(-1, 32)
        oc1 = _i32(last["oct"]); a1 = _f32(last["angle"])
        d2 = _u8(cur["desc"]).reshape(-1, 32); x2 = _f32(cur["x"]); y2 = _f32(cur["y"])
        oc2 = _i32(cur["oct"]); a2 = _f32(cur["angle"])
        ur, cl = _f32(cur.get("uright")), _u8(cur.get("claimed"))
        Tc = _f32(Tcw).reshape(-1)[:12].copy(); Tl = _f32(Tlw).reshape(-1)[:12].copy() if Tlw is not None else None
        camv = _f32(cam); bnd = _f32(bounds); sf = _f32(scale_factors)
        out = np.full(max(n2, 1), -1, np.int32); nm = C.c_int()
        _check(lib().sslpl_search_by_projection_frame(self._h, n1, _p(v1), _p(o1), _p(Xw), _p(dmp), _p(oc1), _p(a1),
                                                      n2, _p(d2), _p(x2), _p(y2), _p(oc2), _p(a2), _p(ur), _p(cl), _p(Tc), _p(Tl),
                                                      _p(camv), _p(bnd), _p(sf), len(sf), th, int(mono), int(check_ori),
                                                      _p(out), C.byref(nm)))
        # -2 = assigned, then removed by the rotation check (the reference writes NULL there, ORBmatcher.cc:1461); -1 = never assigned
        return nm.value, (out[:n2] if raw else np.where(out[:n2] == -2, -1, out[:n2]).astype(np.int32))

    def search_by_projection_frame_batch_device(self, d_kps, d_desc, d_n, nframes, cap, d_Xw, d_mpflag, d_dmp, d_Tcw, cam, bounds,
                                                scale_factors, th, check_ori=True, retry_below=20, d_assign=0, d_nmatch=0):
        """SearchByProjection(CurrentFrame, LastFrame, th, bMono=true) (ORBmatcher.cc:1331-1473) over consecutive frames in HBM, with
        TrackWithMotionModel's 2 * th retry below `retry_below` matches (Tracking.cc:1240-1244; 0 = no retry).  Raw device pointers:
        d_kps / d_desc / d_n as sslpl_orb_device_results gives them, d_Xw [nframes, cap, 3] f32, d_mpflag [nframes, cap] u8 (bit0 has
        MapPoint and not outlier, bit1 Observations() > 0), d_dmp [nframes, cap, 32] or 0 (= d_desc), d_Tcw [nframes, 12] f32 ->
        d_assign [nframes - 1, cap] i32 (-1 never assigned, -2 removed by the rotation check), d_nmatch [nframes - 1] i32.
        Asynchronous on the matcher's stream."""
        sf = _f32(scale_factors)
        _check(lib().sslpl_search_by_projection_frame_batch_device(
            self._h, d_kps, d_desc, d_n, nframes, cap, d_Xw, d_mpflag, d_dmp or None, d_Tcw, _p(_f32(cam)[:4].copy()), _p(_f32(bounds)),
            _p(sf), len(sf), th, int(check_ori), retry_below, d_assign, d_nmatch))

    def descriptor_medoid(self, desc, off):
        """ComputeDistinctiveDescriptors (MapPoint.cc:247-312 / MapLine.cpp:246-317) for CSR groups of descriptors."""
        desc = _u8(desc).reshape(-1, 32); off = _i32(off)
        ng = len(off) - 1
        bi = np.empty(max(ng, 1), np.int32); bm = np.empty(max(ng, 1), np.int32)
        _check(lib().sslpl_descriptor_medoid_batch(self._h, _p(desc), _p(off), ng, _p(bi), _p(bm)))
        return bi[:ng], bm[:ng]

    def match_lines_batch_device(self, d_ldesc, d_nl, nframes, capl, d_lmatch, d_nlmatch):
        _check(lib().sslpl_match_lines_batch_device(self._h, d_ldesc, d_nl, nframes, capl, d_lmatch, d_nlmatch))

    def search_for_triangulation_batch_device(self, d_kps, d_desc, d_n, nkf, cap, d_has_mp, vocab, levelsup, npairs, d_pair, d_geom,
                                              scale, sigma2, check_ori, d_pairs, d_nmatch):
        """ORBmatcher::SearchForTriangulation(pKF1, pKF2, F12, pairs, false) (ORBmatcher.cc:660-826) for npairs keyframe pairs in HBM.
        Raw device pointers: d_kps / d_desc / d_n the keyframe set (mvKeysUn, cap rows each), d_has_mp [nkf, cap] u8, d_pair [npairs, 2]
        i32 (kf1, kf2), d_geom [npairs, 11] f32 (F12 row-major, ex, ey); scale / sigma2 host arrays (nlevels = len(scale)) ->
        d_pairs [npairs, cap, 2] i32 ((idx1, idx2) ascending idx1, -1 after the count), d_nmatch [npairs] i32 (-1: pair index out of
        range).  Asynchronous on the matcher's stream."""
        sc = _f32(scale); s2 = _f32(sigma2)
        assert len(s2) >= len(sc)
        _check(lib().sslpl_search_for_triangulation_batch_device(
            self._h, d_kps, d_desc, d_n, nkf, cap, d_has_mp, vocab._h, levelsup, npairs, d_pair, d_geom, _p(sc), _p(s2), len(sc),
            int(check_ori), d_pairs, d_nmatch))

    def line_search_for_triangulation_batch_device(self, d_ldesc, d_nl, nkf, capl, d_has_ml, npairs, d_pair, d_lpairs, d_nlmatch):
        """LSDmatcher::SearchForTriangulation(pKF1, pKF2, pairs) (LSDmatcher.cpp:382-415) for npairs keyframe pairs in HBM, with
        KeyFrame::lineDescriptorMAD on the device.  d_ldesc [nkf, capl, 32], d_nl [nkf], d_has_ml [nkf, capl] u8, d_pair [npairs, 2] ->
        d_lpairs [npairs, capl, 2] ((qdx, tdx) ascending qdx, -1 after the count), d_nlmatch [npairs] (-1: pair index out of range, or
        KF1 has lines and KF2 fewer than 2).  Asynchronous on the matcher's stream."""
        _check(lib().sslpl_line_search_for_triangulation_batch_device(self._h, d_ldesc, d_nl, nkf, capl, d_has_ml, npairs, d_pair,
                                                                      d_lpairs, d_nlmatch))

    def line_search_for_initialize_batch_device(self, d_ldesc, d_nl, nrows, capl, npairs, d_pair, d_lpairs, d_nlmatch):
        """LSDmatcher::SerachForInitialize (LSDmatcher.cpp:257-284) for npairs (init row, current row) pairs of a line row set in HBM,
        with Frame::lineDescriptorMAD on the device.  d_ldesc [nrows, capl, 32], d_nl [nrows], d_pair [npairs, 2] -> d_lpairs [npairs,
        capl, 2] ((qdx, tdx) ascending qdx, -1 after the count), d_nlmatch [npairs] (-1: a row out of range, or an init row with lines
        against a row with fewer than 2).  Asynchronous on the matcher's stream."""
        _check(lib().sslpl_line_search_for_initialize_batch_device(self._h, d_ldesc, d_nl, nrows, capl, npairs, d_pair, d_lpairs, d_nlmatch))

    def create_new_map_points_batch_device(self, d_kps, d_desc, d_n, nkf, cap, d_has_mp, vocab, levelsup, npairs, d_pair, d_geom, d_kfpose,
                                           cam, scale_factors, level_sigma2, scale_factor, d_pairs, d_nmatch, d_status, d_x3d, d_nnew):
        """LocalMapping::CreateNewMapPoints (LocalMapping.cc:371-637, monocular) for the chains of a pair list in HBM: per pair the
        SearchForTriangulation rows under the mask the reference sees at that neighbour, a status per row and the triangulated point
        (see sslpl_create_new_map_points_batch_device).  Inputs as search_for_triangulation_batch_device, plus d_kfpose [nkf, 15] f32 (Tcw
        3x4, Ow) and host cam = fx fy cx cy invfx invfy, scale_factors / level_sigma2 (nlevels = len) and scale_factor -> d_pairs [npairs,
        cap, 2], d_nmatch [npairs], d_status [npairs, cap] i32, d_x3d [npairs, cap, 3] f32, d_nnew [npairs].  Asynchronous."""
        sc = _f32(scale_factors); s2 = _f32(level_sigma2); cm = _f32(cam)
        assert len(s2) >= len(sc) and len(cm) == 6
        _check(lib().sslpl_create_new_map_points_batch_device(
            self._h, d_kps, d_desc, d_n, nkf, cap, d_has_mp, vocab._h, levelsup, npairs, d_pair, d_geom, d_kfpose, _p(cm), _p(sc), _p(s2),
            len(sc), scale_factor, d_pairs, d_nmatch, d_status, d_x3d, d_nnew))

    def create_new_map_lines_batch_device(self, d_kl, d_ldesc, d_lineeq, d_nl, nkf, capl, d_has_ml, npairs, d_pair, d_kfpose, d_kfdepth,
                                          cam, d_lpairs, d_nlmatch, d_status, d_line3d, d_nnew):
        """LocalMapping::CreateNewMapLines2 (LocalMapping.cc:911-1173, monocular) for the chains of a pair list in HBM: per pair the
        LSDmatcher::SearchForTriangulation rows under the mask the reference sees at that neighbour, a status per row and both
        triangulated end points (see sslpl_create_new_map_lines_batch_device).  d_kl [nkf, capl] sslpl_keyline, d_ldesc [nkf, capl, 32],
        d_lineeq [nkf, capl, 3] f64, d_nl [nkf] as sslpl_line_device_results gives them, d_has_ml [nkf, capl] u8, d_pair [npairs, 2]
        (the caller's pair list: baseline gate 0.1, nn = 10), d_kfpose [nkf, 15] f32 (Tcw 3x4, Ow), d_kfdepth [nkf] f32
        (ComputeSceneMedianDepth(2)) and host cam = fx fy cx cy invfx invfy -> d_lpairs [npairs, capl, 2], d_nlmatch [npairs],
        d_status [npairs, capl] i32, d_line3d [npairs, capl, 6] f32 (s3D, e3D), d_nnew [npairs].  Asynchronous."""
        cm = _f32(cam)
        assert len(cm) == 6
        _check(lib().sslpl_create_new_map_lines_batch_device(
            self._h, d_kl, d_ldesc, d_lineeq, d_nl, nkf, capl, d_has_ml, npairs, d_pair, d_kfpose, d_kfdepth, _p(cm), d_lpairs, d_nlmatch,
            d_status, d_line3d, d_nnew))

    def debug_svd4(self, A, hx=None, hy=None):
        """The device's 4x4 SVD (cv::SVD::compute on CV_32F) of host matrices A [n, 4, 4] -> (W [n, 4], Vt [n, 4, 4]), and its glibc
        hypot of hx, hy (float64) -> h.  Synchronous."""
        A = _f32(A).reshape(-1, 16)
        hx = _f64(hx if hx is not None else []).reshape(-1)
        hy = _f64(hy if hy is not None else []).reshape(-1)
        assert hx.shape == hy.shape
        n, nh = len(A), len(hx)
        W = np.empty((max(n, 1), 4), np.float32); Vt = np.empty((max(n, 1), 4, 4), np.float32); h = np.empty(max(nh, 1), np.float64)
        _check(lib().sslpl_matcher_debug_svd4(self._h, n, _p(A), _p(W), _p(Vt), nh, _p(hx), _p(hy), _p(h)))
        return W[:n], Vt[:n], h[:nh]

    def fuse_points_batch_device(self, d_kps, d_desc, d_n, nkf, cap, d_kfpose, nmp, d_mp, d_mpdesc, nentries, d_entry, d_skip,
                                 cam, bounds, scale_factors, inv_level_sigma2, log_scale_factor, th, d_best_idx, d_best_dist):
        """ORBmatcher::Fuse(pKF, vpMapPoints, th) (ORBmatcher.cc:828-973, monocular) for a flat list of (keyframe, MapPoint) entries in
        HBM, projection stage (with PredictScale) included.  Raw device pointers: d_kps / d_desc / d_n the keyframe set (mvKeysUn, cap rows
        each), d_kfpose [nkf, 15] f32 (Tcw 3x4, Ow), d_mp [nmp, 9] f32 (Xw, normal, minInv, maxInv, maxRaw), d_mpdesc [nmp, 32] u8,
        d_entry [nentries, 2] i32 (kf, mp; mp = -1 NULL), d_skip [nentries] u8 or 0; cam = fx fy cx cy, bounds, scale_factors (nlevels =
        len), inv_level_sigma2 host arrays -> d_best_idx / d_best_dist [nentries] i32 ((-1, 256) no candidate, (-1, -1) index out of
        range).  Asynchronous on the matcher's stream."""
        sf = _f32(scale_factors); isg = _f32(inv_level_sigma2)
        assert len(isg) >= len(sf)
        _check(lib().sslpl_fuse_points_batch_device(
            self._h, d_kps, d_desc, d_n, nkf, cap, d_kfpose, nmp, d_mp, d_mpdesc, nentries, d_entry, d_skip or None, _p(_f32(cam)[:4].copy()),
            _p(_f32(bounds)), _p(sf), _p(isg), len(sf), log_scale_factor, th, d_best_idx, d_best_dist))

    def fuse_lines_batch_device(self, d_kl, d_ldesc, d_nl, nkf, capl, d_kfpose, nml, d_ml, d_mldesc, nentries, d_entry, d_skip,
                                cam, bounds, scale_factors, log_scale_factor, th, d_best_idx, d_best_dist):
        """LSDmatcher::Fuse(pKF, vpMapLines, th) (LSDmatcher.cpp:417-548) for a flat list of (keyframe, MapLine) entries in HBM.  d_kl /
        d_ldesc / d_nl as sslpl_line_device_results gives them, d_ml [nml, 12] f32 (SP, EP, normal, minInv, maxInv, maxRaw), d_mldesc
        [nml, 32]; the rest as fuse_points_batch_device -> (-1, INT_MAX) no candidate (a level outside the pyramid included), (-1, -1)
        index out of range.  Asynchronous on the matcher's stream."""
        sf = _f32(scale_factors)
        _check(lib().sslpl_fuse_lines_batch_device(
            self._h, d_kl, d_ldesc, d_nl, nkf, capl, d_kfpose, nml, d_ml, d_mldesc, nentries, d_entry, d_skip or None, _p(_f32(cam)[:4].copy()),
            _p(_f32(bounds)), _p(sf), len(sf), log_scale_factor, th, d_best_idx, d_best_dist))

    def bow_vectors_batch_device(self, vocab, d_desc, d_n, nrows, cap, d_bow_word, d_bow_val, d_bow_n):
        """Frame::ComputeBoW's mBowVec of nrows rows in HBM (see sslpl_bow_vectors_batch_device): d_desc [nrows, cap, 32] u8, d_n
        [nrows] i32 -> d_bow_word [nrows, cap] i32, d_bow_val [nrows, cap] f64, d_bow_n [nrows] i32.  TF_IDF / L1_NORM vocabularies
        only.  Asynchronous on the matcher's stream."""
        if (vocab.scoring, vocab.weighting) != (0, 0):
            raise SslplError("BowVectors are built for TF_IDF weighting and L1 scoring only")
        _check(lib().sslpl_bow_vectors_batch_device(self._h, vocab._h, d_desc, d_n, nrows, cap, d_bow_word, d_bow_val, d_bow_n))

    def bow_score_batch_device(self, d_bow_word, d_bow_val, d_bow_n, nrows, cap, npairs, d_pair, d_score):
        """TemplatedVocabulary::score (L1) of row pairs d_pair [npairs, 2] i32 -> d_score [npairs] f64 (NaN: a row out of range)."""
        _check(lib().sslpl_bow_score_batch_device(self._h, d_bow_word, d_bow_val, d_bow_n, nrows, cap, npairs, d_pair, d_score))

    def detect_loop_candidates_batch_device(self, d_bow_word, d_bow_val, d_bow_n, nrows, cap, d_db, ndb, d_query, nq, d_covis,
                                            d_conn_off, d_conn, nconn, d_minscore, d_cand, d_ncand, d_words, d_score):
        """KeyFrameDatabase::DetectLoopCandidates for nq query rows against the database rows d_db (add order, erased ones left out):
        d_covis [nrows, 10] i32, d_conn_off [nq + 1] / d_conn [nconn] i32, d_minscore [nq] f32 -> d_cand [nq, ndb] / d_ncand [nq] /
        d_words [nq, ndb] i32, d_score [nq, ndb] f32.  Asynchronous on the matcher's stream."""
        _check(lib().sslpl_detect_loop_candidates_batch_device(self._h, d_bow_word, d_bow_val, d_bow_n, nrows, cap, d_db, ndb, d_query, nq,
                                                               d_covis, d_conn_off, d_conn, nconn, d_minscore, d_cand, d_ncand, d_words,
                                                               d_score))

    def detect_relocalization_candidates_batch_device(self, d_bow_word, d_bow_val, d_bow_n, nrows, cap, d_db, ndb, d_query, nq, d_covis,
                                                      d_relocscore, d_cand, d_ncand, d_words, d_score):
        """KeyFrameDatabase::DetectRelocalizationCandidates for nq query rows in sequence; d_relocscore [nrows] f32 is the keyframes'
        mRelocScore, read and updated (see sslpl_detect_relocalization_candidates_batch_device).  Outputs as the loop call."""
        _check(lib().sslpl_detect_relocalization_candidates_batch_device(self._h, d_bow_word, d_bow_val, d_bow_n, nrows, cap, d_db, ndb,
                                                                         d_query, nq, d_covis, d_relocscore, d_cand, d_ncand, d_words,
                                                                         d_score))

    def reloc_pairs_batch_device(self, d_query, d_cand, d_ncand, nq, ndb, kmax, d_pair):
        """The candidate table of detect_relocalization_candidates_batch_device as pairs: d_pair [nq * kmax, 2] i32 = (candidate row,
        query row) in rank order, (-1, -1) past min(ncand, kmax).  Asynchronous on the matcher's stream."""
        _check(lib().sslpl_reloc_pairs_batch_device(self._h, d_query, d_cand, d_ncand, nq, ndb, kmax, d_pair))

    def search_by_projection_kf(self, kf, cur, Tcw, cam, bounds, scale_factors, log_scale_factor, th, orb_dist, check_ori=True):
        """ORBmatcher::SearchByProjection(Frame &F, KeyFrame *pKF, sAlreadyFound, th, ORBdist) (ORBmatcher.cc:1475-1602).
        kf = dict(flag (MapPoint, not bad, not already found), Xw[n,3], dmp[n,32], dist3[n,3] (minInv, maxInv, mfMaxDistance), angle);
        cur = dict(desc[n,32], x, y, oct, angle, held|None); Tcw 3x4 (or 4x4); cam = (fx, fy, cx, cy); bounds = (minX, maxX, minY, maxY).
        Returns (nmatches, assign2): assign2[j] = keyframe feature written to mvpMapPoints[j], -1 untouched, -2 removed by the rotation
        check."""
        n1, n2 = len(kf["flag"]), len(cur["x"])
        fl = _u8(kf["flag"]); Xw = _f32(kf["Xw"]).reshape(-1, 3); dmp = _u8(kf["dmp"]).reshape(-1, 32)
        d3 = _f32(kf["dist3"]).reshape(-1, 3); a1 = _f32(kf["angle"])
        d2 = _u8(cur["desc"]).reshape(-1, 32)
        sf = _f32(scale_factors)
        out = np.full(max(n2, 1), -1, np.int32); nm = C.c_int()
        _check(lib().sslpl_search_by_projection_kf(self._h, n1, _p(fl), _p(Xw), _p(dmp), _p(d3), _p(a1), n2, _p(d2), _p(_f32(cur["x"])),
                                                   _p(_f32(cur["y"])), _p(_i32(cur["oct"])), _p(_f32(cur["angle"])), _p(_u8(cur.get("held"))),
                                                   _p(_f32(Tcw).reshape(-1)[:12].copy()), _p(_f32(cam)[:4].copy()), _p(_f32(bounds)), _p(sf),
                                                   len(sf), log_scale_factor, th, orb_dist, int(check_ori), _p(out), C.byref(nm)))
        return nm.value, out[:n2]

    def search_by_projection_kf_batch_device(self, d_kps, d_desc, d_n, nrows, cap, d_kfmp, d_mpbad, nmp, d_mp, d_mpdesc, npairs, d_pair,
                                             d_Tcw, d_found, d_held, cam, bounds, scale_factors, log_scale_factor, th, orb_dist,
                                             check_ori, d_assign, d_nmatch):
        """SearchByProjection(Frame, KeyFrame, sAlreadyFound, th, ORBdist) over (keyframe row, frame row) pairs of a row set in HBM:
        d_kfmp [nrows, cap] i32 element indices (-1 NULL), d_mpbad [nmp] u8 or 0, d_mp [nmp, 9] f32 / d_mpdesc [nmp, 32] (the Fuse
        table), d_pair [npairs, 2] i32, d_Tcw [npairs, 12] f32, d_found [npairs, cap] u8 or 0, d_held [npairs, cap] u8 or 0 ->
        d_assign [npairs, cap] i32, d_nmatch [npairs] i32 (-1 for a pair outside the rows).  Asynchronous on the matcher's stream."""
        sf = _f32(scale_factors)
        _check(lib().sslpl_search_by_projection_kf_batch_device(
            self._h, d_kps, d_desc, d_n, nrows, cap, d_kfmp, d_mpbad or None, nmp, d_mp, d_mpdesc, npairs, d_pair, d_Tcw, d_found or None,
            d_held or None, _p(_f32(cam)[:4].copy()), _p(_f32(bounds)), _p(sf), len(sf), log_scale_factor, th, orb_dist, int(check_ori),
            d_assign, d_nmatch))

    def search_by_bow_batch_device(self, d_kps, d_desc, d_n, nrows, cap, d_kfmp, d_mpbad, nmp, vocab, levelsup, npairs, d_pair, nnratio,
                                   check_ori, d_match, d_nmatch):
        """ORBmatcher::SearchByBoW(KeyFrame*, Frame&) (ORBmatcher.cc:159-291) over (keyframe row, frame row) pairs of a row set in HBM
        (see sslpl_search_by_bow_batch_device): the rows and d_kfmp [nrows, cap] i32 / d_mpbad [nmp] u8 or 0 as
        search_by_projection_kf_batch_device, d_pair [npairs, 2] i32 -> d_match [npairs, cap] i32 (keyframe feature of frame feature j,
        -1 none), d_nmatch [npairs] i32 (-1 for a pair outside the rows).  Asynchronous on the matcher's stream."""
        _check(lib().sslpl_search_by_bow_batch_device(self._h, d_kps, d_desc, d_n, nrows, cap, d_kfmp, d_mpbad or None, nmp, vocab._h,
                                                      levelsup, npairs, d_pair, nnratio, int(check_ori), d_match, d_nmatch))

    def match_lines_kf_batch_device(self, d_ldesc, d_nl, nrows, capl, d_kfml, nml, npairs, d_pair, d_lmatch, d_nlmatch):
        """LSDmatcher::SearchByProjection(KeyFrame*, Frame&) (LSDmatcher.cpp:143-183) over (keyframe row, frame row) pairs of a line row
        set in HBM (see sslpl_match_lines_kf_batch_device): d_ldesc [nrows, capl, 32], d_nl [nrows], d_kfml [nrows, capl] i32 element
        indices (-1 NULL), d_pair [npairs, 2] -> d_lmatch [npairs, capl] i32 (the last accepted qdx per tdx, -1 none), d_nlmatch
        [npairs] i32 (-1: a row outside the set, or a keyframe with lines against a frame with fewer than 2).  Asynchronous on the
        matcher's stream."""
        _check(lib().sslpl_match_lines_kf_batch_device(self._h, d_ldesc, d_nl, nrows, capl, d_kfml, nml, npairs, d_pair, d_lmatch,
                                                       d_nlmatch))

    def pose_optimization_batch_device(self, d_kps, d_n, nframes, cap, d_fmp, nmp, d_mp, d_lineeq, d_nl, capl, d_fml, nml, d_mlpos,
                                       d_Tcw, cam, inv_level_sigma2, d_Tcw_out, d_outlier, d_line_outlier, d_ninlier):
        """Optimizer::PoseOptimization (Optimizer.cc:666-1022, monocular) for nframes frames in HBM (see
        sslpl_pose_optimization_batch_device).  Raw device pointers: d_kps [nframes, cap] sslpl_keypoint (mvKeysUn), d_n [nframes] i32,
        d_fmp [nframes, cap] i32 element indices into d_mp [nmp, 9] f32 (-1 NULL); d_lineeq [nframes, capl, 3] f64, d_nl [nframes],
        d_fml [nframes, capl] i32 element indices into d_mlpos [nml, 6] f64, or d_fml = 0 for no line edges; d_Tcw [nframes, 12] f32;
        host cam = fx fy cx cy and inv_level_sigma2 (nlevels = len) -> d_Tcw_out [nframes, 12] f32 (may be d_Tcw), d_outlier
        [nframes, cap] / d_line_outlier [nframes, capl] u8 (written where a feature has an edge), d_ninlier [nframes] i32 (-1: an octave
        outside the pyramid).  Asynchronous on the matcher's stream."""
        isg = _f32(inv_level_sigma2)
        _check(lib().sslpl_pose_optimization_batch_device(
            self._h, d_kps, d_n, nframes, cap, d_fmp, nmp, d_mp or None, d_lineeq or None, d_nl or None, capl, d_fml or None, nml,
            d_mlpos or None, d_Tcw, _p(_f32(cam)[:4].copy()), _p(isg), len(isg), d_Tcw_out, d_outlier, d_line_outlier or None, d_ninlier))

    def debug_predict_scale(self, ratio, log_scale_factor, nlevels, clamp=True):
        """MapPoint / MapLine::PredictScale on the device for host ratios (see sslpl_matcher_debug_predict_scale) -> int32 levels."""
        r = _f32(ratio).reshape(-1)
        out = np.empty(max(len(r), 1), np.int32)
        _check(lib().sslpl_matcher_debug_predict_scale(self._h, len(r), _p(r), log_scale_factor, nlevels, int(clamp), _p(out)))
        return out[:len(r)]


def predict_scale_table(log_scale_factor, nlevels):
    """The nlevels + 1 PredictScale thresholds of sslpl_predict_scale_table (host only, no device): thr[k] = the smallest positive float
    ratio whose level (int)ceil(logf(ratio) / log_scale_factor) is >= k."""
    thr = np.empty(int(nlevels) + 1, np.float32)
    _check(lib().sslpl_predict_scale_table(log_scale_factor, nlevels, _p(thr)))
    return thr


class Vocabulary(_Handle, kind="vocab"):
    """DBoW2 ORB vocabulary tree on the device (the reference's ORBVocabulary = TemplatedVocabulary<FORB::TDescriptor, FORB>,
    include/ORBVocabulary.h; used by Frame::ComputeBoW Frame.cc:474-481 with levelsup = 4).

    Vocabulary(k, L, parent, desc, weight, is_leaf)   from arrays (node 0 = root)
    Vocabulary.load_text(path)                          ORBvoc.txt (TemplatedVocabulary.h:1338-1420)
    Vocabulary.random(k, L, seed)                       synthetic tree for tests / benchmarks"""
    # scoring / weighting enums of DBoW2 (BowVector.h): the defaults of ORBvoc.txt are L1_NORM (0) and TF_IDF (0)
    TF_IDF, TF, IDF, BINARY = 0, 1, 2, 3

    def __init__(self, k, L, parent, desc, weight, is_leaf, device=0, scoring=0, weighting=0):
        self.parent = _i32(parent); self.desc = _u8(desc).reshape(-1, 32)
        self.weight = _f64(weight); self.is_leaf = _u8(is_leaf)
        self.k, self.L, self.scoring, self.weighting = int(k), int(L), int(scoring), int(weighting)
        self._h = C.c_void_p()
        _check(lib().sslpl_vocab_create(device, self.k, self.L, len(self.parent), _p(self.parent), _p(self.desc), _p(self.weight),
                                        _p(self.is_leaf), C.byref(self._h)))

    @classmethod
    def load_text(cls, path, device=0):
        self = cls.__new__(cls)
        self._h = C.c_void_p(); sc = C.c_int(); we = C.c_int()
        _check(lib().sslpl_vocab_load_text(device, str(path).encode(), C.byref(self._h), C.byref(sc), C.byref(we)))
        k = C.c_int(); L = C.c_int()
        _check(lib().sslpl_vocab_info(self._h, C.byref(k), C.byref(L), None, None))
        self.k, self.L, self.scoring, self.weighting = k.value, L.value, sc.value, we.value
        self.parent = self.desc = self.weight = self.is_leaf = None
        return self

    @staticmethod
    def random_arrays(k, L, seed=0, stop_fraction=0.0, early_leaf_fraction=0.0):
        """A random k-ary tree of depth L as arrays, in the node order loadFromTextFile produces for a file written level by
        level is NOT required: any order with parent[i] < i works.  Some leaves can be 'stopped' (weight 0) or sit above L."""
        rng = np.random.default_rng(seed)
        parent = [-1]; depth = [0]; frontier = [0]
        for d in range(1, L + 1):
            nxt = []
            for p in frontier:
                if d > 1 and rng.random() < early_leaf_fraction:
                    continue                                        # p stays a leaf above the last level
                for _ in range(k):
                    parent.append(p); depth.append(d); nxt.append(len(parent) - 1)
            frontier = nxt
        n = len(parent)
        parent = np.array(parent, np.int32)
        has_child = np.zeros(n, bool); has_child[parent[1:]] = True
        is_leaf = (~has_child).astype(np.uint8); is_leaf[0] = 0
        desc = rng.integers(0, 256, (n, 32), dtype=np.uint8)
        weight = np.where(is_leaf == 1, rng.random(n) * 5 + 0.1, 0.0)
        weight[(is_leaf == 1) & (rng.random(n) < stop_fraction)] = 0.0
        return parent, desc, weight.astype(np.float64), is_leaf

    @classmethod
    def random(cls, k=10, L=3, seed=0, device=0, **kw):
        parent, desc, weight, is_leaf = cls.random_arrays(k, L, seed, **kw)
        return cls(k, L, parent, desc, weight, is_leaf, device=device)

    def info(self):
        k = C.c_int(); L = C.c_int(); nn = C.c_int(); nw = C.c_int()
        _check(lib().sslpl_vocab_info(self._h, C.byref(k), C.byref(L), C.byref(nn), C.byref(nw)))
        return {"k": k.value, "L": L.value, "nodes": nn.value, "words": nw.value}

    def level_nodes(self, levelsup=4):
        c = C.c_int()
        _check(lib().sslpl_vocab_level_nodes(self._h, levelsup, C.byref(c)))
        return c.value

    def bow_vector(self, word, weight):
        """BowVector assembly of TemplatedVocabulary::transform (:1145-1195) from the per-feature arrays: a word -> value map
        (ascending word id), TF_IDF / TF: weights added in feature order then divided by the number of words unless the scoring
        normalises (L1 / L2 scoring types 0, 1 do); IDF / BINARY: first weight kept."""
        bv = {}
        for wid, w in zip(np.asarray(word).tolist(), np.asarray(weight).tolist()):
            if not w > 0:
                continue
            if self.weighting in (self.TF_IDF, self.TF):
                bv[wid] = bv.get(wid, 0.0) + w
            else:
                bv.setdefault(wid, w)
        must, l2 = self.scoring in (0, 1), self.scoring == 1      # L1_NORM, L2_NORM normalise (ScoringObject.cpp)
        keys = sorted(bv)
        if self.weighting in (self.TF_IDF, self.TF) and bv and not must:
            nd = float(len(bv))
            for kk in keys:
                bv[kk] /= nd
        if must and bv:
            norm = 0.0
            for kk in keys:
                norm += bv[kk] * bv[kk] if l2 else abs(bv[kk])
            if l2:
                norm = float(np.sqrt(norm))
            if norm > 0.0:
                for kk in keys:
                    bv[kk] /= norm
        return np.array(keys, np.int32), np.array([bv[kk] for kk in keys], np.float64)

    @staticmethod
    def feature_vector(node, weight):
        """FeatureVector (node id -> ascending feature indices) as CSR, without the stopped words (:1162-1166)."""
        node = np.asarray(node, np.int32); keep = np.nonzero(np.asarray(weight) > 0)[0].astype(np.int32)
        order = keep[np.argsort(node[keep], kind="stable")]
        ids, counts = np.unique(node[keep], return_counts=True)
        off = np.zeros(len(ids) + 1, np.int32); off[1:] = np.cumsum(counts)
        return ids.astype(np.int32), off, order.astype(np.int32)


class ORBmatcher:
    """Mirror of StructureSLAM::ORBmatcher (include/ORBmatcher.h:36-101) on indices + masks instead of
    KeyFrame*/MapPoint* (the C++ adapter in host/ maps indices back to pointers)."""
    TH_HIGH, TH_LOW, HISTO_LENGTH = 100, 50, 30

    def __init__(self, nnratio=0.6, checkOri=True, ctx=None):
        self.mfNNratio, self.mbCheckOrientation = float(nnratio), bool(checkOri)
        self.ctx = ctx or Matcher()

    def DescriptorDistance(self, a, b):
        return int(self.ctx.descriptor_distance(a, b)[0])

    def SearchByBoW(self, d1, fv1, valid1, angle1, d2, fv2, angle2, valid2=None):
        """KeyFrame-vs-Frame (valid2 is None; ORBmatcher.cc:159) -> (nmatches, match2[n2] = KF index or -1);
        KeyFrame-vs-KeyFrame (valid2 given; ORBmatcher.cc:525) -> (nmatches, match12[n1] = KF2 index or -1)."""
        d1 = _u8(d1).reshape(-1, 32); d2 = _u8(d2).reshape(-1, 32)
        f1, f2 = _featvec(fv1), _featvec(fv2)
        valid1 = _u8(valid1)
        angle1 = _f32(angle1); angle2 = _f32(angle2)
        nm = C.c_int()
        if valid2 is None:
            out = np.empty(len(d2), np.int32)
            _check(lib().sslpl_search_by_bow(self.ctx._h, _p(d1), len(d1), _p(d2), len(d2), C.byref(f1), C.byref(f2),
                                             _p(valid1), _p(angle1), _p(angle2), self.mfNNratio, self.mbCheckOrientation, _p(out), C.byref(nm)))
        else:
            valid2 = _u8(valid2)
            out = np.empty(len(d1), np.int32)
            _check(lib().sslpl_search_by_bow_kf(self.ctx._h, _p(d1), len(d1), _p(d2), len(d2), C.byref(f1), C.byref(f2),
                                                _p(valid1), _p(valid2), _p(angle1), _p(angle2), self.mfNNratio, self.mbCheckOrientation,
                                                _p(out), C.byref(nm)))
        return nm.value, out

    def SearchForTriangulation(self, d1, fv1, has_mp1, kp1, d2, fv2, has_mp2, kp2, F12, ex, ey, scale, sigma2):
        """ORBmatcher.cc:660 (monocular) -> (nmatches, pairs[nmatches,2])."""
        d1 = _u8(d1).reshape(-1, 32); d2 = _u8(d2).reshape(-1, 32)
        f1, f2 = _featvec(fv1), _featvec(fv2)
        has_mp1 = _u8(has_mp1); has_mp2 = _u8(has_mp2)
        kp1 = np.ascontiguousarray(kp1, KEYPOINT_DTYPE); kp2 = np.ascontiguousarray(kp2, KEYPOINT_DTYPE)
        F12 = _f32(F12).reshape(9)
        scale = _f32(scale); sigma2 = _f32(sigma2)
        pairs = np.empty((max(len(d1), 1), 2), np.int32)
        nm = C.c_int()
        _check(lib().sslpl_search_for_triangulation(self.ctx._h, _p(d1), len(d1), _p(d2), len(d2), C.byref(f1), C.byref(f2),
                                                    _p(has_mp1), _p(has_mp2), _p(kp1), _p(kp2), _p(F12), ex, ey, _p(scale), _p(sigma2), len(scale),
                                                    self.mbCheckOrientation, _p(pairs), C.byref(nm)))
        return nm.value, pairs[:nm.value].copy()


class LSDmatcher:
    """Mirror of the knnMatch-based entry points of StructureSLAM::LSDmatcher (include/LSDmatcher.h:36-64)."""

    def __init__(self, ctx=None):
        self.ctx = ctx or Matcher()

    def _run(self, mode, d1, d2, has_ml1, has_ml2):
        d1 = _u8(d1).reshape(-1, 32); d2 = _u8(d2).reshape(-1, 32)
        h1 = _u8(has_ml1 if has_ml1 is not None else np.zeros(len(d1)))
        h2 = _u8(has_ml2 if has_ml2 is not None else np.zeros(len(d2)))
        out = np.full(2 * max(len(d1), len(d2), 1), -1, np.int32)
        k = C.c_int(); nm = C.c_int(); mad = (C.c_double * 2)()
        _check(lib().sslpl_line_match(self.ctx._h, mode, _p(d1), len(d1), _p(d2), len(d2), _p(h1), _p(h2), _p(out),
                                      C.byref(k), C.byref(nm), mad))
        self.last_mad = (mad[0], mad[1])
        if mode == 0:
            return nm.value, out[:len(d2)].copy()
        if mode == 2:
            return nm.value, out[:len(d1)].copy()
        return nm.value, out[:2 * k.value].reshape(-1, 2).copy()

    def SearchByProjection(self, ldescKF, has_mapline_KF, ldescF):      # LSDmatcher.cpp:143 (KeyFrame*, Frame&)
        return self._run(0, ldescKF, ldescF, has_mapline_KF, None)

    SearchByDescriptor = SearchByProjection                             # LSDmatcher.cpp:286 (identical body)

    def SerachForInitialize(self, ldesc1, ldesc2):                      # LSDmatcher.cpp:257 (sic)
        return self._run(1, ldesc1, ldesc2, None, None)

    def SearchByDescriptorKF(self, ldesc1, ldesc2, has_mapline_KF2):    # LSDmatcher.cpp:329
        return self._run(2, ldesc1, ldesc2, None, has_mapline_KF2)

    def SearchForTriangulation(self, ldesc1, has_ml1, ldesc2, has_ml2):  # LSDmatcher.cpp:382 -> (n, pairs[n, 2])
        return self._run(3, ldesc1, ldesc2, has_ml1, has_ml2)

    def DescriptorDistance(self, a, b):                                 # LSDmatcher.cpp:364
        return int(self.ctx.descriptor_distance(a, b)[0])


# =====================================================================================================
# Frame level
# =====================================================================================================
class FrameParams(C.Structure):
    _fields_ = [("orb", OrbParams), ("line", LineParams)]


class Frame(_Handle, kind="frame", lifecycle=("sync", "launch_count")):
    """What StructureSLAM::Frame::Frame(imGray, ...) does with the two extractors (src/Frame.cc:69-131): ONE upload of the frame,
    ORB and LSD+LBD on two streams, optional colour conversion in front (Tracking.cc:148-161) and keypoint undistortion behind
    (Frame.cc:483-513).  `extract(image)` -> dict(keys, keysUn, desc, keylines, ldesc, lineeq)."""

    def __init__(self, nfeatures=1000, scaleFactor=1.2, nlevels=8, iniThFAST=20, minThFAST=7, lsdNFeatures=40,
                 max_width=1280, max_height=960, max_batch=1, device=0):
        self._create(FrameParams(OrbParams(nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST, max_width, max_height, max_batch, device),
                                 LineParams(lsdNFeatures, max_width, max_height, max_batch, device)))
        orb = lib().sslpl_frame_orb(self._h)
        self.cap = lib().sslpl_orb_max_keypoints(orb)
        self.orb = ORBextractor._borrow(orb, nfeatures=nfeatures, scaleFactor=scaleFactor, nlevels=nlevels, max_batch=max_batch, cap=self.cap)
        self.line = LineSegment._borrow(lib().sslpl_frame_line(self._h), cap=lsdNFeatures, max_batch=max_batch)
        self.lcap = lsdNFeatures
        self.max_batch = max_batch

    def stream(self, which):
        """CUDA stream handle of the ORB (0) or line (1) side."""
        return lib().sslpl_frame_stream(self._h, which)

    def extract_batch_begin(self, frames, out):
        """Asynchronous: frames [B, H, W] uint8 in pinned memory (host_alloc); out = dict(keys, desc, n, keylines, ldesc, lineeq, nl) of
        pinned arrays with the handle's capacities.  Finish with sync()."""
        B, h, w = frames.shape[:3]
        cn = 1 if frames.ndim == 3 else frames.shape[3]
        assert out["keys"].shape[1] == self.cap and out["keylines"].shape[1] == self.lcap
        _check(lib().sslpl_frame_extract_batch_begin(self._h, _p(frames), B, w, h, frames.strides[1], frames.strides[0], cn, 0,
                                                     _p(out["keys"]), None, _p(out["desc"]), self.cap, _p(out["n"]),
                                                     _p(out["keylines"]), _p(out["ldesc"]), _p(out["lineeq"]), self.lcap, _p(out["nl"])))

    def device_keypoints_un(self):
        """(device pointer, cap) of the last call's mvKeysUn: undistorted keypoints when k1 != 0, else the ORB keypoints (Frame.cc:485).
        Counts are those of self.orb.device_results(); written on stream(0)."""
        p = C.c_void_p(); cap = C.c_int()
        _check(lib().sslpl_frame_device_keypoints_un(self._h, C.byref(p), C.byref(cap)))
        return p.value, cap.value

    def set_camera(self, fx, fy, cx, cy, dist=()):
        d = _f32(dist)
        _check(lib().sslpl_frame_set_camera(self._h, fx, fy, cx, cy, _p(d) if len(d) else None, len(d)))

    def image_bounds(self, cols, rows):
        b = np.zeros(4, np.float32)
        _check(lib().sslpl_frame_image_bounds(self._h, cols, rows, _p(b)))
        return b

    def debug_undistort(self, xy):
        """The device's mvKeysUn arithmetic (k_undistort with this handle's camera) on float32 points [N, 2] -> float32 [N, 2]."""
        xy = _f32(xy).reshape(-1, 2)
        out = np.empty_like(xy)
        _check(lib().sslpl_frame_debug_undistort(self._h, len(xy), _p(xy), _p(out)))
        return out

    def extract(self, image, rgb_order=False):
        """image: HxW (grey) or HxWx3 / HxWx4 uint8 (BGR[A] unless rgb_order)."""
        assert image.dtype == np.uint8 and image.ndim in (2, 3)
        image = np.ascontiguousarray(image)
        cn = 1 if image.ndim == 2 else image.shape[2]
        h, w = image.shape[:2]
        kps = np.zeros(self.cap, KEYPOINT_DTYPE); un = np.zeros(self.cap, KEYPOINT_DTYPE); desc = np.zeros((self.cap, 32), np.uint8)
        kl = np.zeros(self.lcap, KEYLINE_DTYPE); ld = np.zeros((self.lcap, 32), np.uint8); eq = np.zeros((self.lcap, 3), np.float64)
        n = C.c_int(); nl = C.c_int()
        _check(lib().sslpl_frame_extract(self._h, _p(image), w, h, image.strides[0], cn, int(rgb_order), _p(kps), _p(un), _p(desc), self.cap,
                                         C.byref(n), _p(kl), _p(ld), _p(eq), self.lcap, C.byref(nl)))
        n, nl = n.value, nl.value
        return dict(keys=kps[:n].copy(), keysUn=un[:n].copy(), desc=desc[:n].copy(), keylines=kl[:nl].copy(), ldesc=ld[:nl].copy(), lineeq=eq[:nl].copy())

    def extract_batch(self, frames, rgb_order=False):
        """frames: [B, H, W] or [B, H, W, C] uint8 -> dict of per-frame arrays (padded to the capacities) and counts."""
        frames = np.ascontiguousarray(frames)
        B, h, w = frames.shape[:3]
        cn = 1 if frames.ndim == 3 else frames.shape[3]
        kps = np.zeros((B, self.cap), KEYPOINT_DTYPE); un = np.zeros((B, self.cap), KEYPOINT_DTYPE); desc = np.zeros((B, self.cap, 32), np.uint8)
        kl = np.zeros((B, self.lcap), KEYLINE_DTYPE); ld = np.zeros((B, self.lcap, 32), np.uint8); eq = np.zeros((B, self.lcap, 3), np.float64)
        n = np.zeros(B, np.int32); nl = np.zeros(B, np.int32)
        _check(lib().sslpl_frame_extract_batch(self._h, _p(frames), B, w, h, frames.strides[1], frames.strides[0], cn, int(rgb_order),
                                               _p(kps), _p(un), _p(desc), self.cap, _p(n), _p(kl), _p(ld), _p(eq), self.lcap, _p(nl)))
        return dict(keys=kps, keysUn=un, desc=desc, n=n, keylines=kl, ldesc=ld, lineeq=eq, nl=nl)


# =====================================================================================================
# Lines
# =====================================================================================================
class LineSegment(_Handle, kind="line", lifecycle=("sync", "set_stream", "stream", "launch_count", "set_profiling", "stage_ms")):
    """Mirror of StructureSLAM::LineSegment (include/ExtractLineSegment.h:53-76).  lsdNFeatures is hard-coded to 40
    in the reference (ExtractLineSegment.cpp:42); it is a constructor parameter here (BASELINE.json config 4: 500)."""

    def __init__(self, lsdNFeatures=40, max_width=1280, max_height=960, max_batch=1, device=0):
        self._create(LineParams(lsdNFeatures, max_width, max_height, max_batch, device))
        self.cap = lsdNFeatures
        self.max_batch = max_batch

    def ExtractLineSegment(self, img, scale=1, numOctaves=1):
        """-> (keylines, ldesc, keylineFunctions): ExtractLineSegment.cpp:18-69 (scale / numOctaves as the reference
        passes them: int 1 and 1; other values are not supported)."""
        assert int(scale) == 1 and numOctaves == 1
        assert img.dtype == np.uint8 and img.ndim == 2
        if img.strides[1] != 1:
            img = np.ascontiguousarray(img)
        kl = np.zeros(self.cap, KEYLINE_DTYPE); ld = np.zeros((self.cap, 32), np.uint8); eq = np.zeros((self.cap, 3), np.float64)
        n = C.c_int()
        _check(lib().sslpl_line_extract(self._h, _p(img), img.shape[1], img.shape[0], img.strides[0], _p(kl), _p(ld), _p(eq),
                                        self.cap, C.byref(n)))
        return kl[:n.value].copy(), ld[:n.value].copy(), eq[:n.value].copy()

    def extract_batch(self, frames, out=None):
        assert frames.dtype == np.uint8 and frames.ndim == 3 and frames.strides[2] == 1
        B, H, W = frames.shape
        if out is None:
            out = (np.zeros((B, self.cap), KEYLINE_DTYPE), np.zeros((B, self.cap, 32), np.uint8),
                   np.zeros((B, self.cap, 3), np.float64), np.zeros(B, np.int32))
        kl, ld, eq, n = out
        _check(lib().sslpl_line_extract_batch(self._h, _p(frames), B, W, H, frames.strides[1], frames.strides[0],
                                              _p(kl), _p(ld), _p(eq), self.cap, _p(n)))
        return kl, ld, eq, n

    def extract_batch_begin(self, frames, out):
        B, H, W = frames.shape
        kl, ld, eq, n = out
        _check(lib().sslpl_line_extract_batch_begin(self._h, _p(frames), B, W, H, frames.strides[1], frames.strides[0],
                                                    _p(kl), _p(ld), _p(eq), self.cap, _p(n)))

    def extract_batch_device(self, d_ptr, nframes, width, height, pitch, frame_stride):
        _check(lib().sslpl_line_extract_batch_device(self._h, d_ptr, nframes, width, height, pitch, frame_stride))

    def device_results(self):
        kl = C.c_void_p(); ld = C.c_void_p(); eq = C.c_void_p(); n = C.c_void_p(); cap = C.c_int()
        _check(lib().sslpl_line_device_results(self._h, C.byref(kl), C.byref(ld), C.byref(eq), C.byref(n), C.byref(cap)))
        return kl.value, ld.value, eq.value, n.value, cap.value

    def raw_segments(self, frame=0, cap=1 << 15):
        seg = np.empty((cap, 4), np.float32); n = C.c_int()
        _check(lib().sslpl_line_download_segments(self._h, frame, _p(seg), cap, C.byref(n)))
        return seg[:min(n.value, cap)].copy()

    def prep_planes(self, frame=0):
        """Per-pixel pre-pass of `frame` of the last call: dict(dx, dy [h, w] int16; angdeg [sh, sw] float32 (-1024 = NOTDEF);
        cs, cs0 [sh, sw, 2] float32; modgrad [sh, sw] float64; maxgrad float; seeds uint32 pixel indices y * sw + x)."""
        w, h, sw, sh, ns = C.c_int(), C.c_int(), C.c_int(), C.c_int(), C.c_int()
        _check(lib().sslpl_line_download_prep(self._h, frame, C.byref(w), C.byref(h), C.byref(sw), C.byref(sh), *([None] * 9)))
        W, H, SW, SH = w.value, h.value, sw.value, sh.value
        dx = np.empty((H, W), np.int16); dy = np.empty((H, W), np.int16); ang = np.empty((SH, SW), np.float32)
        cs = np.empty((SH, SW, 2), np.float32); cs0 = np.empty((SH, SW, 2), np.float32); mod = np.empty((SH, SW), np.float64)
        mg = C.c_double(); seeds = np.empty(max(SW * SH, 1), np.uint32)
        _check(lib().sslpl_line_download_prep(self._h, frame, None, None, None, None, _p(dx), _p(dy), _p(ang), _p(cs), _p(cs0), _p(mod),
                                              C.byref(mg), _p(seeds), C.byref(ns)))
        return dict(dx=dx, dy=dy, angdeg=ang, cs=cs, cs0=cs0, modgrad=mod, maxgrad=mg.value, seeds=seeds[:ns.value].copy())

    def ll_table(self):
        """The pre-pass's ll_angle arithmetic on every 2x2 difference pair: arrays [511, 511] indexed [DA + 255, BC + 255]
        (angdeg, modgrad) and [511, 511, 2] (cs, cs0)."""
        n = 511
        ang = np.empty((n, n), np.float32); cs = np.empty((n, n, 2), np.float32); cs0 = np.empty((n, n, 2), np.float32)
        mod = np.empty((n, n), np.float64)
        _check(lib().sslpl_line_debug_ll_table(self._h, _p(ang), _p(cs), _p(cs0), _p(mod)))
        return dict(angdeg=ang, cs=cs, cs0=cs0, modgrad=mod)

    def debug_nfa(self, width, height, n, k, p, plain=False):
        """The NFA kernels' nfa() on arrays (n, k, p) with the log_nt and log-gamma table of a width x height frame -> (log_nfa float64,
        stop int32: loop index of the early stop, n + 1 when the tail loop ran out, -1 for the early returns).  plain=True turns the
        pow skip and the log10 bracket off."""
        n = _i32(n); k = _i32(k); p = _f64(p)
        assert n.shape == k.shape == p.shape and n.ndim == 1
        out = np.empty(len(n), np.float64); stop = np.empty(len(n), np.int32)
        _check(lib().sslpl_line_debug_nfa(self._h, width, height, len(n), _p(n), _p(k), _p(p), int(bool(plain)), _p(out), _p(stop)))
        return out, stop

    def debug_sincos(self, x, full=False):
        """ddtrig::sincos_cr (full=False, region2rect's form) or sincos_cr_full of a float64 array on the device -> (sin, cos)."""
        x = _f64(x).reshape(-1)
        s = np.empty_like(x); c = np.empty_like(x)
        _check(lib().sslpl_line_debug_sincos(self._h, len(x), _p(x), int(bool(full)), _p(s), _p(c)))
        return s, c

    def debug_atan2(self, y, x):
        """The line path's fast_atan2_deg (cv::fastAtan2) of float32 arrays on the device."""
        y = _f32(y).reshape(-1); x = _f32(x).reshape(-1)
        assert y.shape == x.shape
        out = np.empty_like(x)
        _check(lib().sslpl_line_debug_atan2(self._h, len(x), _p(y), _p(x), _p(out)))
        return out

    def set_max_walkers(self, n):
        _check(lib().sslpl_line_set_max_walkers(self._h, n))

    def walker_stats(self):
        out = (C.c_ulonglong * 16)()
        _check(lib().sslpl_line_walker_stats(self._h, out))
        names = ["turn_regions", "turn_cycles", "turn_pixels", "_", "seed_swallowed", "redo_abandoned", "redo_poisoned", "redo_invalid", "redo_presumed",
                 "committed_as_speculated", "speculated_pixels", "commit_lock_cycles", "claim_lock_cycles", "repeated_attempts", "frame_cycles", "claims"]
        return {k: int(out[i]) for i, k in enumerate(names)}

    def debug_trace(self, frame=0, cap=1 << 16):
        out = np.empty((cap, 10), np.float64); n = C.c_int()
        _check(lib().sslpl_line_debug_trace(self._h, frame, _p(out), cap, C.byref(n)))
        return out[:min(n.value, cap)].copy()
