"""GPU parity of the batched, device-resident CreateNewMapPoints (LocalMapping.cc:371-637, monocular): SearchForTriangulation and the
triangulation of every neighbour, neighbour after neighbour, with the KF1 features of the created rows masked for the later neighbours.
Every pair's rows, count, statuses and the bits of every written x3D are compared with tests/create_points_model.py (the NumPy
restatement, matcher rows from the oracle) and cross-checked against the batched matcher under the chain's mask, against shorter
chains and against separate calls.  The device SVD and hypot are compared with cv2.SVDecomp, the model and glibc.

The scene builder below is shared with tests/test_create_points_cpu.py, which checks on the model alone that the gates, the masking and
the shared idx2 occur on these scenes."""
import ctypes
import os

import cv2
import numpy as np
import pytest

import create_points_model as M
from test_kf_triangulation_gpu import LEVELSUP, VOCAB, feature_vectors, vocabulary_arrays

pytestmark = pytest.mark.gpu

NKF = 21
FLAT = 15                      # a keyframe without keypoints, among KF 0's neighbours
NLEVELS, SCALE_FACTOR = 8, 1.2
f32 = np.float32


def _rot(ax, ay, az):
    cx_, sx = np.cos(ax), np.sin(ax); cy_, sy = np.cos(ay), np.sin(ay); cz, sz = np.cos(az), np.sin(az)
    Rx = np.array([[1, 0, 0], [0, cx_, -sx], [0, sx, cx_]]); Ry = np.array([[cy_, 0, sy], [0, 1, 0], [-sy, 0, cy_]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def scene(pkg, oracle, W=640, H=480, nfeat=1000, nkf=NKF, flat=FLAT, seed=0, p_mp=0.15, pose_err=0.004):
    """A synthetic 3D scene seen by nkf keyframes: 3D points in front of KF 0, camera centres along a curve (baselines up to ~0.6 at
    depths 2-9) with small rotations.  Every keyframe gets the projections of the points it sees with 0.3 px noise (2.5 px on 15 %), an octave
    within 3 of the point's own (a few KF 0 octaves outside the pyramid), duplicates of some points (two keypoints of one point: created rows that share
    an idx2) and ~6 % outliers (a point's descriptor at a wrong position).  Descriptors: a per-point base with 0-5 flipped bits.
    The pose table the triangulation reads (`pose`) differs from the true poses (`pose_true`, which F12 is computed from) on some
    keyframes, so that the reprojection and depth tests reject rows.
    Returns the keyframe set in the extractors' layout (cap = nfeat + 64 rows) with poses, camera and pyramid tables."""
    rng = np.random.default_rng(seed)
    fx = fy = f32(0.8 * W); cx, cy = f32(W / 2), f32(H / 2)
    cam = np.array([fx, fy, cx, cy, f32(1) / fx, f32(1) / fy], f32)
    npt = int(nfeat * 1.6)
    z = rng.uniform(2.0, 9.0, npt)
    P = np.stack([(rng.uniform(0, W, npt) - W / 2) * z / fx, (rng.uniform(0, H, npt) - H / 2) * z / fy, z], 1)
    base = rng.integers(0, 256, (npt, 32), dtype=np.uint8)
    poct = rng.integers(0, NLEVELS, npt)
    cap = nfeat + 64
    kps = np.zeros((nkf, cap), pkg.KEYPOINT_DTYPE); desc = np.zeros((nkf, cap, 32), np.uint8); n = np.zeros(nkf, np.int32)
    pose = np.zeros((nkf, 15), f32); pose_true = np.zeros((nkf, 15), f32)
    for k in range(nkf):
        t = k / (nkf - 1)
        C = np.array([0.6 * t * np.cos(3 * t), 0.25 * np.sin(5 * t), 0.3 * t]) if k else np.zeros(3)
        R = _rot(0.03 * np.sin(7 * t), -0.08 * t, 0.05 * np.cos(4 * t)) if k else np.eye(3)
        tcw = -R @ C
        pose_true[k] = np.array([*R[0], tcw[0], *R[1], tcw[1], *R[2], tcw[2], *C], f32)
        # the pose table the triangulation reads carries a pose error on some keyframes (F12 is computed from the true poses):
        # the matcher then accepts rows that the reprojection and depth tests reject (KF 10's table moves it 3 into the scene and
        # turns it: some of its rows land behind it)
        Re = R @ _rot(*(pose_err * rng.standard_normal(3))) if k % 4 == 3 else R @ _rot(0, 0.15, 0) if k == 10 else R
        Ce = C + (pose_err * 20 * rng.standard_normal(3) if k % 4 == 3 else 0) + (np.array([1.5, 0, 3.0]) if k == 10 else 0)
        te = -Re @ Ce
        pose[k] = np.array([*Re[0], te[0], *Re[1], te[1], *Re[2], te[2], *Ce], f32)
        if k == flat:
            continue
        Xc = P @ R.T + tcw
        u = fx * Xc[:, 0] / Xc[:, 2] + cx; v = fy * Xc[:, 1] / Xc[:, 2] + cy
        vis = np.nonzero((Xc[:, 2] > 0.1) & (u >= 0) & (u < W) & (v >= 0) & (v < H))[0]
        vis = rng.permutation(vis)[: int(nfeat * 0.85)]
        dup = vis[rng.random(len(vis)) < 0.05]
        out = rng.choice(npt, int(0.06 * len(vis)))
        ids = np.concatenate([vis, dup, out])[:nfeat]
        m = len(ids)
        kind = np.concatenate([np.zeros(len(vis)), np.ones(len(dup)), 2 * np.ones(len(out))])[:m]
        sd = np.where(rng.random(m) < 0.15, 2.5, 0.3)
        x = u[ids] + rng.normal(0, 1, m) * sd; y = v[ids] + rng.normal(0, 1, m) * sd
        x = np.where(kind == 1, x + rng.normal(0, 0.5, m), x); y = np.where(kind == 1, y + rng.normal(0, 0.5, m), y)
        x = np.where(kind == 2, rng.uniform(0, W, m), x); y = np.where(kind == 2, rng.uniform(0, H, m), y)
        octv = np.clip(poct[ids] + rng.integers(-3, 4, m), 0, NLEVELS - 1)
        if k == 0:
            octv[rng.random(m) < 0.02] = NLEVELS + rng.integers(0, 3)
        kps["x"][k, :m] = np.clip(x, 0, W - 1); kps["y"][k, :m] = np.clip(y, 0, H - 1)
        kps["octave"][k, :m] = octv; kps["angle"][k, :m] = rng.uniform(0, 360, m); kps["size"][k, :m] = 31
        kps["response"][k, :m] = rng.random(m)
        d = base[ids].copy()
        nflip = rng.integers(0, 6, m)
        for r in range(m):
            for b in rng.integers(0, 256, nflip[r]):
                d[r, b >> 3] ^= np.uint8(1 << (b & 7))
        desc[k, :m] = d; n[k] = m
    sf = np.ones(NLEVELS, f32)
    for l in range(1, NLEVELS):                               # ORBextractor: mvScaleFactor[i] = mvScaleFactor[i-1] * scaleFactor
        sf[l] = sf[l - 1] * f32(SCALE_FACTOR)
    s2 = (sf * sf).astype(f32)
    has_mp = (rng.random((nkf, cap)) < p_mp).astype(np.uint8)
    va = vocabulary_arrays(pkg)
    return dict(kps=kps, desc=desc, n=n, cap=cap, pose=pose, pose_true=pose_true, cam=cam, scale=sf, sigma2=s2, scale_factor=f32(SCALE_FACTOR),
                has_mp=has_mp, voc_arrays=va, fv=feature_vectors(pkg, oracle, va, desc, n), W=W, H=H)


def geometry(K, pairs, skew=0.02):
    """d_geom per pair: LocalMapping::ComputeF12 (:1286-1300) and SearchForTriangulation's epipole (ORBmatcher.cc:666-673).  Every
    third pair's F12 is computed with KF2 turned by `skew` radians, as a pose error would give it."""
    fx, fy, cx, cy = [float(v) for v in K["cam"][:4]]
    Km = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]])
    geom = np.zeros((len(pairs), 11), f32)
    for p, (i, j) in enumerate(pairs):
        if not (0 <= i < len(K["n"]) and 0 <= j < len(K["n"])):
            continue
        T1 = K["pose_true"][i, :12].reshape(3, 4).astype(np.float64); T2 = K["pose_true"][j, :12].reshape(3, 4).astype(np.float64)
        R12 = T1[:, :3] @ T2[:, :3].T
        if p % 3 == 2:
            R12 = R12 @ _rot(skew, -skew, 0)
        t12 = -R12 @ T2[:, 3] + T1[:, 3]
        tx = np.array([[0, -t12[2], t12[1]], [t12[2], 0, -t12[0]], [-t12[1], t12[0], 0]])
        F = np.linalg.inv(Km).T @ tx @ R12 @ np.linalg.inv(Km)
        C2 = T2[:, :3] @ K["pose_true"][i, 12:15].astype(np.float64) + T2[:, 3]
        geom[p, :9] = F.reshape(-1); geom[p, 9] = fx * C2[0] / C2[2] + cx; geom[p, 10] = fy * C2[1] / C2[2] + cy
    return geom


def oracle_chain(oracle, K, pairs, geom, trace=None):
    """The model's CreateNewMapPoints over the chains, the matcher rows from the oracle's SearchForTriangulation (checkOrientation false)."""
    def match(p, pr, hm):
        i, j = pr
        n1, n2 = int(K["n"][i]), int(K["n"][j])
        return oracle.search_for_triangulation(K["desc"][i, :n1], K["desc"][j, :n2], K["fv"][i], K["fv"][j], hm[i, :n1], hm[j, :n2],
                                               K["kps"][i, :n1], K["kps"][j, :n2], geom[p, :9].reshape(3, 3), float(geom[p, 9]),
                                               float(geom[p, 10]), K["scale"], K["sigma2"], False)
    return M.create_points(match, K, pairs, K["pose"], K["cam"], K["scale"], K["sigma2"], K["scale_factor"], trace)


def neighbour_pairs(kf=0, count=20):
    return [(kf, k) for k in range(1, count + 1)]


# ------------------------------------------------------------------------------------------------------------------ GPU helpers
@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


def upload(pkg, torch, K):
    D = dict(K)
    D["d_kps_t"] = torch.from_numpy(K["kps"].view(np.uint8).reshape(len(K["n"]), -1).copy()).cuda()
    D["d_desc_t"] = torch.from_numpy(K["desc"]).cuda(); D["d_n_t"] = torch.from_numpy(K["n"]).cuda()
    D["d_has_mp_t"] = torch.from_numpy(K["has_mp"]).cuda(); D["d_pose_t"] = torch.from_numpy(K["pose"]).cuda()
    D["voc"] = pkg.Vocabulary(VOCAB["k"], VOCAB["L"], *K["voc_arrays"])
    return D


def matcher(pkg, D, max_batch=32):
    return pkg.Matcher(max_features=D["cap"] - 64, max_lines=0, max_nodes=D["voc"].level_nodes(LEVELSUP), max_batch=max_batch)


def run(mt, torch, D, pairs, geom, has_mp=None, sync=True):
    P, cap = len(pairs), D["cap"]
    d_pair = torch.tensor(np.array(pairs, np.int32).reshape(-1, 2), device="cuda"); d_geom = torch.from_numpy(geom).cuda()
    out = dict(rows=torch.full((P, cap, 2), 7, dtype=torch.int32, device="cuda"), n=torch.full((P,), -7, dtype=torch.int32, device="cuda"),
               status=torch.full((P, cap), 77, dtype=torch.int32, device="cuda"), x3d=torch.full((P, cap, 3), 7.5, dtype=torch.float32, device="cuda"),
               nnew=torch.full((P,), -7, dtype=torch.int32, device="cuda"))
    hm = D["d_has_mp_t"] if has_mp is None else has_mp
    mt.create_new_map_points_batch_device(D["d_kps_t"].data_ptr(), D["d_desc_t"].data_ptr(), D["d_n_t"].data_ptr(), len(D["n"]), cap,
                                          hm.data_ptr(), D["voc"], LEVELSUP, P, d_pair.data_ptr(), d_geom.data_ptr(), D["d_pose_t"].data_ptr(),
                                          D["cam"], D["scale"], D["sigma2"], D["scale_factor"], out["rows"].data_ptr(), out["n"].data_ptr(),
                                          out["status"].data_ptr(), out["x3d"].data_ptr(), out["nnew"].data_ptr())
    if sync:
        mt.sync()
    out["keep"] = (d_pair, d_geom)
    return {k: (v.cpu().numpy() if k != "keep" else v) for k, v in out.items()}


def check_pair(G, p, exp):
    n = exp["n"]
    assert G["n"][p] == n, (p, int(G["n"][p]), n)
    k = max(n, 0)
    assert np.array_equal(G["rows"][p, :k], exp["rows"]), p
    assert (G["rows"][p, k:] == -1).all() and (G["status"][p, k:] == -1).all(), p
    assert np.array_equal(G["status"][p, :k], exp["status"]), (p, np.nonzero(G["status"][p, :k] != exp["status"])[0][:8])
    w = exp["written"]
    assert np.array_equal(G["x3d"][p, :k][w].view(np.uint32), exp["x3d"][w].view(np.uint32)), p
    assert (G["x3d"][p, :k][~w] == 7.5).all(), p
    assert G["nnew"][p] == exp["nnew"], p


def check_all(G, E):
    for p, e in enumerate(E):
        check_pair(G, p, e)


@pytest.fixture(scope="module")
def small(pkg, oracle, torch):
    K = scene(pkg, oracle)
    assert K["n"][FLAT] == 0 and (np.delete(K["n"], FLAT) > 700).all()
    return upload(pkg, torch, K)


def test_equal_model(pkg, oracle, torch, small):
    """KF 0 against 20 neighbours (FLAT among them), then a second chain (KF 12's), in one call: rows, counts, statuses, x3D bits."""
    D = small
    mt = matcher(pkg, D)
    pairs = neighbour_pairs() + [(12, k) for k in (11, 13, 14, 16, 20, 3, 0)]
    geom = geometry(D, pairs)
    G = run(mt, torch, D, pairs, geom)
    E = oracle_chain(oracle, D, pairs, geom)
    check_all(G, E)
    assert sum(e["nnew"] for e in E) > 500 and G["n"][FLAT - 1] == 0


def test_rows_equal_batched_matcher_under_chain_mask(pkg, torch, small):
    """Each pair's rows equal sslpl_search_for_triangulation_batch_device(checkOrientation = 0) given d_has_mp with the created rows
    of the earlier pairs of its chain set; the masking changes some pair's rows."""
    D = small
    mt = matcher(pkg, D)
    pairs = neighbour_pairs()
    geom = geometry(D, pairs)
    G = run(mt, torch, D, pairs, geom)
    hm = D["has_mp"].copy()
    changed = 0
    for p, (i, j) in enumerate(pairs):
        for h, tag in ((hm, "chain"), (D["has_mp"], "plain")):
            d_h = torch.from_numpy(h).cuda()
            d_pair = torch.tensor([[i, j]], dtype=torch.int32, device="cuda"); d_geom = torch.from_numpy(geom[p:p + 1]).cuda()
            d_rows = torch.full((1, D["cap"], 2), 7, dtype=torch.int32, device="cuda"); d_n = torch.full((1,), -7, dtype=torch.int32, device="cuda")
            mt.search_for_triangulation_batch_device(D["d_kps_t"].data_ptr(), D["d_desc_t"].data_ptr(), D["d_n_t"].data_ptr(), NKF, D["cap"],
                                                     d_h.data_ptr(), D["voc"], LEVELSUP, 1, d_pair.data_ptr(), d_geom.data_ptr(), D["scale"],
                                                     D["sigma2"], False, d_rows.data_ptr(), d_n.data_ptr())
            mt.sync()
            rows, n = d_rows.cpu().numpy()[0], int(d_n.cpu().numpy()[0])
            if tag == "chain":
                assert n == G["n"][p] and np.array_equal(rows, G["rows"][p]), p
            else:
                changed += n != G["n"][p]
        k = G["n"][p]
        hm[i, G["rows"][p, :k][G["status"][p, :k] == 0, 0]] = 1
    assert changed > 0


def test_prefix_and_separate_chains(pkg, torch, small):
    """The first k pairs of a chain give the results of a call with only those pairs; two chains in one call equal two calls."""
    D = small
    mt = matcher(pkg, D)
    a = neighbour_pairs(); b = [(5, k) for k in (4, 6, 7, 0, 9, 3)]
    ga, gb = geometry(D, a), geometry(D, b)
    Gab = run(mt, torch, D, a + b, np.concatenate([ga, gb]))
    Ga, Gb = run(mt, torch, D, a, ga), run(mt, torch, D, b, gb)
    for key in ("rows", "n", "status", "nnew"):
        assert np.array_equal(Gab[key], np.concatenate([Ga[key], Gb[key]])), key
    assert np.array_equal(Gab["x3d"].view(np.uint32), np.concatenate([Ga["x3d"], Gb["x3d"]]).view(np.uint32))
    for k in (1, 5, 13):
        Gk = run(mt, torch, D, a[:k], ga[:k])
        for key in ("rows", "n", "status", "nnew"):
            assert np.array_equal(Gk[key], Ga[key][:k]), (k, key)
        assert np.array_equal(Gk["x3d"].view(np.uint32), Ga["x3d"][:k].view(np.uint32)), k


def test_bad_pairs(pkg, oracle, torch, small):
    """Out-of-range indices, kf2 == kf1 and a repeated kf2 get -1 and no rows, and leave the chain's state alone."""
    D = small
    mt = matcher(pkg, D)
    good = [(0, 1), (0, 2), (0, 3), (0, 4)]
    pairs = [(0, 1), (0, NKF), (0, 2), (0, 0), (0, 1), (0, -3), (0, 3), (0, 2), (0, 4), (NKF, 1), (-1, 2)]
    with np.errstate(invalid="ignore"):                       # (0, 0) has no epipole
        geom = geometry(D, pairs)
    G = run(mt, torch, D, pairs, geom)
    E = oracle_chain(oracle, D, good, geom[[pairs.index(pr) for pr in good]])
    gi = 0
    for p, pr in enumerate(pairs):
        if pr in good and pr not in pairs[:p]:
            check_pair(G, p, E[gi]); gi += 1
        else:
            assert G["n"][p] == -1 and G["nnew"][p] == 0 and (G["rows"][p] == -1).all() and (G["status"][p] == -1).all(), p
            assert (G["x3d"][p] == 7.5).all(), p
    assert gi == 4 and all(e["nnew"] > 0 for e in E)


def test_large_frames(pkg, oracle, torch):
    """1280x960, 4000 features per keyframe, 5 keyframes: KF 0 against 4 neighbours."""
    K = scene(pkg, oracle, 1280, 960, 4000, nkf=5, flat=None, seed=3)
    D = upload(pkg, torch, K)
    mt = matcher(pkg, D, max_batch=8)
    pairs = neighbour_pairs(0, 4) + [(2, 1), (2, 3)]
    geom = geometry(D, pairs)
    G = run(mt, torch, D, pairs, geom)
    E = oracle_chain(oracle, D, pairs, geom)
    check_all(G, E)
    assert min(e["nnew"] for e in E) > 0 and sum(e["nnew"] for e in E) > 1000


def test_caller_stream_and_argument_errors(pkg, oracle, torch, small):
    D = small
    mt = matcher(pkg, D)
    pairs = neighbour_pairs(0, 8)
    geom = geometry(D, pairs)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        mt.set_stream(s.cuda_stream)
        G = run(mt, torch, D, pairs, geom, sync=False)
    s.synchronize()
    mt.set_stream(0)
    check_all(G, oracle_chain(oracle, D, pairs, geom))
    # bad arguments: SSLPL_ERR_ARG, nothing enqueued, nothing written
    P, cap = len(pairs), D["cap"]
    d_pair = torch.tensor(np.array(pairs, np.int32), device="cuda"); d_geom = torch.from_numpy(geom).cuda()
    outs = [torch.full((P, cap, 2), 7, dtype=torch.int32, device="cuda"), torch.full((P,), -7, dtype=torch.int32, device="cuda"),
            torch.full((P, cap), 77, dtype=torch.int32, device="cuda"), torch.full((P, cap, 3), 7.5, dtype=torch.float32, device="cuda"),
            torch.full((P,), -7, dtype=torch.int32, device="cuda")]
    good = dict(d_kps=D["d_kps_t"].data_ptr(), d_desc=D["d_desc_t"].data_ptr(), d_n=D["d_n_t"].data_ptr(), nkf=NKF, cap=cap,
                d_has_mp=D["d_has_mp_t"].data_ptr(), vocab=D["voc"], levelsup=LEVELSUP, npairs=P, d_pair=d_pair.data_ptr(),
                d_geom=d_geom.data_ptr(), d_kfpose=D["d_pose_t"].data_ptr(), cam=D["cam"], scale_factors=D["scale"], level_sigma2=D["sigma2"],
                scale_factor=D["scale_factor"], d_pairs=outs[0].data_ptr(), d_nmatch=outs[1].data_ptr(), d_status=outs[2].data_ptr(),
                d_x3d=outs[3].data_ptr(), d_nnew=outs[4].data_ptr())
    mt_small = pkg.Matcher(max_features=cap - 64, max_lines=0, max_nodes=D["voc"].level_nodes(LEVELSUP), max_batch=8)
    one = np.ones(17, np.float32)
    bad = [dict(d_kps=0), dict(d_desc=0), dict(d_n=0), dict(d_has_mp=0), dict(d_pair=0), dict(d_geom=0), dict(d_kfpose=0), dict(d_pairs=0),
           dict(d_nmatch=0), dict(d_status=0), dict(d_x3d=0), dict(d_nnew=0), dict(nkf=10), dict(npairs=0), dict(npairs=9), dict(cap=0),
           dict(cap=cap + 1), dict(scale_factors=one[:0], level_sigma2=one[:0]), dict(scale_factors=one, level_sigma2=one), dict(levelsup=0),
           dict(scale_factor=0.0), dict(scale_factor=float("nan"))]
    before = mt_small.launch_count
    for b in bad:
        with pytest.raises(pkg.SslplError, match="error -1:"):
            mt_small.create_new_map_points_batch_device(**{**good, **b})
    mt_small.sync()
    assert mt_small.launch_count == before
    assert (outs[0] == 7).all().item() and (outs[1] == -7).all().item() and (outs[2] == 77).all().item() and (outs[3] == 7.5).all().item()
    assert (outs[4] == -7).all().item()
    mt_small.create_new_map_points_batch_device(**{**good, "nkf": 9})
    mt_small.sync()
    assert mt_small.launch_count == before + 5 and (outs[1] > 0).all().item()


# ------------------------------------------------------------------------------------------------------------------ device SVD / hypot
def glibc_version():
    try:
        v = ctypes.CDLL("libc.so.6").gnu_get_libc_version
        v.restype = ctypes.c_char_p
        return tuple(int(x) for x in v().decode().split(".")[:2])
    except (OSError, AttributeError):
        return (0, 0)


def svd_tables(rng, n):
    """Random, rank-2, rank-3, zero-row and triangulation-shaped 4x4 matrices."""
    A = rng.standard_normal((n, 4, 4)).astype(f32)
    q = n // 6
    A[q:2 * q, 3] = A[q:2 * q, 0] * f32(0.5) + A[q:2 * q, 1]                     # rank 3
    A[2 * q:3 * q, 2] = A[2 * q:3 * q, 0]; A[2 * q:3 * q, 3] = A[2 * q:3 * q, 1] * f32(-2)  # rank 2
    A[3 * q:3 * q + q // 2, rng.integers(0, 4)] = 0                               # a zero row
    A[3 * q + q // 2:4 * q, :, 1] = 0                                             # a zero column: W = 0 sorts last, vt(3, 3) = 0
    m = n - 4 * q                                                                  # the point form x * T.row(2) - T.row(0|1)
    R = np.stack([_rot(*a) for a in rng.uniform(-0.3, 0.3, (64, 3))]).astype(f32)
    t = rng.uniform(-1, 1, (64, 3)).astype(f32)
    T = np.concatenate([R, t[:, :, None]], 2)
    a, b = rng.integers(0, 64, m), rng.integers(0, 64, m)
    xn = rng.uniform(-0.6, 0.6, (m, 4)).astype(f32)
    A[4 * q:] = np.stack([M.add_weighted(T[a, 2], xn[:, 0:1].astype(np.float64), T[a, 0], -1.0),
                          M.add_weighted(T[a, 2], xn[:, 1:2].astype(np.float64), T[a, 1], -1.0),
                          M.add_weighted(T[b, 2], xn[:, 2:3].astype(np.float64), T[b, 0], -1.0),
                          M.add_weighted(T[b, 2], xn[:, 3:4].astype(np.float64), T[b, 1], -1.0)], 1)
    return A


def test_device_svd_and_hypot(pkg):
    mt = pkg.Matcher(max_features=64, max_lines=0, max_nodes=16)
    rng = np.random.default_rng(11)
    n = 1 << 20
    A = svd_tables(rng, n)
    hx = rng.standard_normal(n) * np.exp2(rng.integers(-1070, 1020, n)); hy = rng.standard_normal(n) * np.exp2(rng.integers(-1070, 1020, n))
    hy[: n // 2] = hx[: n // 2] * rng.uniform(-3, 3, n // 2)
    W, Vt, h = mt.debug_svd4(A, hx, hy)
    Wm, Vm = M.svd4(A)
    assert np.array_equal(W.view(np.uint32), Wm.view(np.uint32)) and np.array_equal(Vt.view(np.uint32), Vm.view(np.uint32))
    assert np.array_equal(h.view(np.uint64), M.hypot(hx, hy).view(np.uint64))
    assert (Vm[:, 3, 3] == 0).any()                                              # the w == 0 case is reachable through the SVD
    if glibc_version() < (2, 35):
        pytest.skip("cv2 calls this machine's libm hypot, which is glibc's corrected one only from 2.35; the model leg ran")
    assert np.array_equal(h.view(np.uint64), np.hypot(hx, hy).view(np.uint64))
    # Exact everywhere except where the numerical null space is two-dimensional: both of the two smallest singular values below
    # FLT_MIN (exactly rank-2 matrices).  There the last two W and Vt rows are subnormal noise and may differ from cv2 (DESIGN.md);
    # the two leading singular values and Vt rows must still be bit-identical.  Such a matrix never reaches the triangulation
    # (test_create_points_cpu.py::test_scene_is_not_vacuous checks the third singular value of every triangulation).
    tiny = np.finfo(f32).tiny
    for k in range(n):
        w, _, vt = cv2.SVDecomp(A[k].copy(), flags=cv2.SVD_MODIFY_A | cv2.SVD_FULL_UV)
        w = w.ravel()
        if w[2] < tiny and W[k, 2] < tiny:
            assert np.array_equal(w[:2].view(np.uint32), W[k, :2].view(np.uint32)) and np.array_equal(vt[:2].view(np.uint32), Vt[k, :2].view(np.uint32)), k
        else:
            assert np.array_equal(w.view(np.uint32), W[k].view(np.uint32)) and np.array_equal(vt.view(np.uint32), Vt[k].view(np.uint32)), k
