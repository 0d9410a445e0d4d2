"""GPU parity of the batched, device-resident CreateNewMapLines2 (LocalMapping.cc:911-1173, monocular): LSDmatcher::SearchForTriangulation
and the triangulation of both end points of every match, neighbour after neighbour, with the KF1 lines of the created rows masked for
the later neighbours.  Every pair's rows, count, statuses and the bits of every written s3D / e3D are compared with
tests/create_lines_model.py (the NumPy restatement, matcher rows from the oracle) and cross-checked against the batched line matcher
under the chain's mask, against shorter chains and against separate calls.  The device SVD is compared with the model on line-shaped
matrices.

The scene builder below is shared with tests/test_create_lines_cpu.py, which checks on the model alone that the gates, the masking and
the shared tdx occur on this scene, and compares the model's SVD with cv2 on the same kind of matrices."""
import numpy as np
import pytest

import create_lines_model as M

pytestmark = pytest.mark.gpu

NKF = 11                       # KF 0 and its 10 line neighbours (LocalMapping.cc:914-918, monocular nn = 10)
EMPTY, SINGLE = 8, 9           # a keyframe without lines and one with a single line, among KF 0's neighbours
f32 = np.float32


def _rot(ax, ay, az):
    cx_, sx = np.cos(ax), np.sin(ax); cy_, sy = np.cos(ay), np.sin(ay); cz, sz = np.cos(az), np.sin(az)
    Rx = np.array([[1, 0, 0], [0, cx_, -sx], [0, sx, cx_]]); Ry = np.array([[cy_, 0, sy], [0, 1, 0], [-sy, 0, cy_]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def look_at(C, target, roll=0.0):
    """Rcw of a camera at C looking at target (image y down, KF 0 at the origin looking along +z gets the identity)."""
    z = (target - C) / np.linalg.norm(target - C)
    x = np.cross(z, [0.0, -1.0, 0.0]); x /= np.linalg.norm(x)
    R = np.stack([x, np.cross(z, x), z])
    return _rot(0, 0, roll) @ R


def line_function(sx, sy, ex, ey):
    """mvKeyLineFunctions (ExtractLineSegment.cpp:58-67): sp x ep normalised by the length of its first two components."""
    l = np.cross(np.stack([sx, sy, np.ones_like(sx)], -1).astype(np.float64), np.stack([ex, ey, np.ones_like(ex)], -1).astype(np.float64))
    return l / np.sqrt(l[..., 0:1] * l[..., 0:1] + l[..., 1:2] * l[..., 1:2])


def segments(rng, n, Cs):
    """3D segments [n, 2, 3] around the scene centre (0, 0, 4): ordinary ones, long ones along the depth, ones with one end close to a
    camera centre Cs[k] (within 0.7-1.3 of it, in front of it and of KF 0; the other end at least 1.6 from every centre), and ones close
    to the epipolar planes of the cameras, which lie near the y = 0 plane (y ~ 0, direction in the x-z plane)."""
    centre = np.array([0.0, 0.0, 4.0])
    kind = rng.choice(5, n, p=[0.5, 0.1, 0.12, 0.12, 0.16])
    mid = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), rng.uniform(2.5, 7, n)], 1)
    d = rng.standard_normal((n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    length = rng.uniform(0.3, 2.0, n)
    lg = kind == 1                                                             # long: mostly along the depth
    d[lg] = np.stack([rng.uniform(-0.3, 0.3, lg.sum()), rng.uniform(-0.3, 0.3, lg.sum()), np.ones(lg.sum())], 1)
    d[lg] /= np.linalg.norm(d[lg], axis=1, keepdims=True); length[lg] = rng.uniform(2.4, 4.0, lg.sum())
    ep = kind == 4                                                             # near-epipolar: y ~ 0, direction in the x-z plane
    mid[ep, 1] = rng.normal(0, 0.02, ep.sum())
    d[ep, 1] = rng.choice([0.0, 1e-5, 1e-3, 1e-2], ep.sum())
    d[ep] /= np.linalg.norm(d[ep], axis=1, keepdims=True)
    P = np.stack([mid - 0.5 * length[:, None] * d, mid + 0.5 * length[:, None] * d], 1)
    for s in np.nonzero((kind == 2) | (kind == 3))[0]:                         # one end near a camera centre
        C = Cs[0] if rng.random() < 0.5 else Cs[rng.integers(1, len(Cs))]
        ax = (centre - C) / np.linalg.norm(centre - C)
        while True:
            u = rng.standard_normal(3); u /= np.linalg.norm(u)
            near = C + rng.uniform(0.7, 1.3) * u
            far = near + rng.uniform(0.3, 1.2) * d[s]
            if u @ ax > 0.85 and near[2] > 0.6 and far[2] > 0.6 and min(np.linalg.norm(far - c) for c in Cs) >= 1.6:
                break
            d[s] = rng.standard_normal(3); d[s] /= np.linalg.norm(d[s])
        P[s] = (near, far) if kind[s] == 2 else (far, near)
    return P


def scene(pkg, W=640, H=480, nlines=40, nkf=NKF, empty=EMPTY, single=SINGLE, seed=0, p_ml=0.15):
    """A synthetic 3D scene of segments seen by nkf keyframes: KF 0 at the origin, the others on an arc of radius 4 around the scene centre
    (0, 0, 4) at 4-40 degrees, looking at it (parallax up to ~40 degrees; the nearest neighbours stay below the 11.5 degrees of cos 0.98).
    Every keyframe gets the projections of the segments it sees fully (0.3 px noise on each end point, ends sliding a little along the
    segment), at most nlines of them; KF 0 also sees a second, shifted copy of some segments (created rows that share a tdx), and ~5 % of
    the lines get a random descriptor.  Descriptors: a per-segment base with 0-4 flipped bits.  The pose table the triangulation reads
    (`pose`) carries a pose error on KF 3 and KF 7 and moves KF 10 3 into the scene (some triangulations land behind a camera).
    `depth` is the median depth of each keyframe's segment end points (ComputeSceneMedianDepth(2)'s role).
    Returns the keyframe set in the layout of sslpl_line_device_results (capl = nlines + 64 rows)."""
    rng = np.random.default_rng(seed)
    fx = fy = f32(0.55 * W); cx, cy = f32(W / 2), f32(H / 2)
    cam = np.array([fx, fy, cx, cy, f32(1) / fx, f32(1) / fy], f32)
    centre = np.array([0.0, 0.0, 4.0])
    ang = np.deg2rad([0, 4, -9, 14, -18, 22, -26, 30, -34, 12, -40, 24, -7, 36, -20, 28][:nkf]) if nkf <= 16 else \
        np.deg2rad(rng.uniform(-40, 40, nkf))
    ang[0] = 0
    Cs, Rs = [], []
    for k in range(nkf):
        C = centre + _rot(0, ang[k], 0) @ np.array([0.0, 0.0, -4.0]) + (np.array([0, 0.15 * np.sin(3 * k), 0]) if k else 0)
        Cs.append(C); Rs.append(look_at(C, centre + (rng.normal(0, 0.1, 3) if k else 0), 0.02 * np.sin(5 * k) if k else 0))
    nseg = int(nlines * 1.5)
    P = segments(rng, nseg, Cs)
    prio = rng.permutation(nseg)                                               # the segments every keyframe prefers
    base = rng.integers(0, 256, (nseg, 32), dtype=np.uint8)
    capl = nlines + 64
    kl = np.zeros((nkf, capl), pkg.KEYLINE_DTYPE); ldesc = np.zeros((nkf, capl, 32), np.uint8); eq = np.zeros((nkf, capl, 3))
    nl = np.zeros(nkf, np.int32); pose = np.zeros((nkf, 15), f32); pose_true = np.zeros((nkf, 15), f32); depth = np.full(nkf, 4.0, f32)
    for k in range(nkf):
        R, C = Rs[k], Cs[k]
        t = -R @ C
        pose_true[k] = np.array([*R[0], t[0], *R[1], t[1], *R[2], t[2], *C], f32)
        Re, Ce = R, C
        if k in (3, 7):
            Re = R @ _rot(*(0.01 * rng.standard_normal(3))); Ce = C + 0.08 * rng.standard_normal(3)
        if k == 10:
            Re = R @ _rot(0, 0.3, 0); Ce = C + 3.0 * (centre - C) / np.linalg.norm(centre - C)
        te = -Re @ Ce
        pose[k] = np.array([*Re[0], te[0], *Re[1], te[1], *Re[2], te[2], *Ce], f32)
        Xc = P @ R.T + t                                                       # [nseg, 2, 3]
        z = Xc[..., 2]
        u = fx * Xc[..., 0] / np.where(z > 0, z, 1) + cx; v = fy * Xc[..., 1] / np.where(z > 0, z, 1) + cy
        slide = rng.uniform(-0.04, 0.04, (nseg, 2))
        us = u + slide[:, :1] * (u[:, 1:] - u[:, :1]) * [[1, -1]]; vs = v + slide[:, :1] * (v[:, 1:] - v[:, :1]) * [[1, -1]]
        us += rng.normal(0, 0.3, us.shape); vs += rng.normal(0, 0.3, vs.shape)
        inside = (z > 0.1).all(1) & (us >= 0).all(1) & (us < W - 1).all(1) & (vs >= 0).all(1) & (vs < H - 1).all(1)
        inside &= np.hypot(us[:, 1] - us[:, 0], vs[:, 1] - vs[:, 0]) > 8
        vis = prio[inside[prio]]
        if k == 0:                                                             # a second, shifted keyline of some segments
            nd = max(2, min(len(vis), nlines) // 8)
            vis = np.concatenate([vis[: nlines - nd], vis[:nd]])
        vis = vis[: (0 if k == empty else 1 if k == single else nlines)]
        m = len(vis)
        if m:
            sx, sy, ex, ey = us[vis, 0].copy(), vs[vis, 0].copy(), us[vis, 1].copy(), vs[vis, 1].copy()
            if k == 0:
                rep = np.zeros(m, bool); seen = set()
                for r, s in enumerate(vis):
                    rep[r] = s in seen; seen.add(s)
                sx[rep] += 1.5; sy[rep] -= 1.0; ex[rep] += 1.5; ey[rep] -= 1.0
            for f, a in (("startPointX", sx), ("startPointY", sy), ("endPointX", ex), ("endPointY", ey)):
                kl[f][k, :m] = a
            kl["pt_x"][k, :m] = (sx + ex) / 2; kl["pt_y"][k, :m] = (sy + ey) / 2
            kl["lineLength"][k, :m] = np.hypot(ex - sx, ey - sy); kl["angle"][k, :m] = np.arctan2(ey - sy, ex - sx)
            kl["class_id"][k, :m] = np.arange(m); kl["numOfPixels"][k, :m] = kl["lineLength"][k, :m].astype(np.int32)
            eq[k, :m] = line_function(kl["startPointX"][k, :m], kl["startPointY"][k, :m], kl["endPointX"][k, :m], kl["endPointY"][k, :m])
            d = base[vis].copy()
            nflip = rng.integers(0, 5, m)
            for r in range(m):
                for b in rng.integers(0, 256, nflip[r]):
                    d[r, b >> 3] ^= np.uint8(1 << (b & 7))
            d[rng.random(m) < 0.05] = rng.integers(0, 256, 32, dtype=np.uint8)
            ldesc[k, :m] = d
            depth[k] = f32(np.median(z[vis].ravel()))
        nl[k] = m
    has_ml = (rng.random((nkf, capl)) < p_ml).astype(np.uint8)
    return dict(kl=kl, ldesc=ldesc, lineeq=eq, nl=nl, capl=capl, has_ml=has_ml, pose=pose, pose_true=pose_true, depth=depth, cam=cam,
                W=W, H=H)


def oracle_chain(oracle, K, pairs, trace=None):
    """The model's CreateNewMapLines2 over the chains, the matcher rows from the oracle's LSDmatcher::SearchForTriangulation."""
    def match(p, pr, hm):
        i, j = pr
        n1, n2 = int(K["nl"][i]), int(K["nl"][j])
        return oracle.line_match(3, K["ldesc"][i, :n1], K["ldesc"][j, :n2], hm[i, :n1], hm[j, :n2])
    return M.create_lines(match, K, pairs, trace)


def neighbour_pairs(kf=0, count=NKF - 1):
    return [(kf, k) for k in range(count + 1) if k != kf][:count]


_ENDS = np.dtype([("startPointX", "<f4"), ("startPointY", "<f4"), ("endPointX", "<f4"), ("endPointY", "<f4")])   # the fields read


def line_svd_tables(rng, n, K=None, oracle=None):
    """Line-shaped 4x4 matrices (the A and B of :1056-1077): those of every row of K's neighbour loop, then rows of random lines (random
    look-at camera pairs, segments in front of both, end points projected, line functions from them) of which a third lie close to the
    epipolar plane of the two camera centres (direction in the plane plus a normal component of 0, 1e-7 .. 1e-2).  -> [n, 4, 4] f32."""
    out = []
    if K is not None:
        tr = []
        oracle_chain(oracle, K, neighbour_pairs(), tr)
        out += [t[1] for t in tr if isinstance(t[0], str) and t[0] == "A"]
    have = sum(len(a) for a in out)
    cam = np.array([512, 512, 320, 240, 1 / 512, 1 / 512], f32)
    batch = 500
    while have < n:
        C1 = np.zeros(3); C2 = rng.normal(0, 1.0, 3)
        tgt = np.array([0, 0, 4.0]) + rng.normal(0, 0.5, 3)
        poses = []
        for C in (C1, C2):
            R = look_at(C, tgt, rng.normal(0, 0.05)); t = -R @ C
            poses.append(np.array([*R[0], t[0], *R[1], t[1], *R[2], t[2], *C], f32))
        m = batch
        mid = tgt + rng.normal(0, 1.0, (m, 3))
        d = rng.standard_normal((m, 3))
        ep = np.arange(m) < m // 3
        b = (C2 - C1) / np.linalg.norm(C2 - C1)
        w = mid[ep] - C1; w /= np.linalg.norm(w, axis=1, keepdims=True)
        nrm = np.cross(b, w); nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
        a = rng.uniform(-1, 1, (ep.sum(), 1))
        d[ep] = a * b + (1 - np.abs(a)) * w + rng.choice([0.0, 1e-7, 1e-5, 1e-3, 1e-2], (ep.sum(), 1)) * nrm
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        Pw = np.stack([mid - 0.6 * d, mid + 0.6 * d], 1)
        kls = []
        for ps in poses:
            T = ps[:12].reshape(3, 4).astype(np.float64)
            Xc = Pw @ T[:, :3].T + T[:, 3]
            u = 512 * Xc[..., 0] / Xc[..., 2] + 320; v = 512 * Xc[..., 1] / Xc[..., 2] + 240
            kk = np.zeros(m, _ENDS)
            kk["startPointX"], kk["startPointY"], kk["endPointX"], kk["endPointY"] = u[:, 0], v[:, 0], u[:, 1], v[:, 1]
            kls.append(kk)
        eqs = [line_function(k_["startPointX"], k_["startPointY"], k_["endPointX"], k_["endPointY"]) for k_ in kls]
        rows = np.stack([np.arange(m), np.arange(m)], 1)
        with np.errstate(all="ignore"):
            _, A, B = M.line_matrices(kls[0], kls[1], eqs[0], eqs[1], rows, poses[0], poses[1], cam)
        keep = np.isfinite(A).all((1, 2)) & np.isfinite(B).all((1, 2))
        out += [A[keep], B[keep]]
        have += 2 * keep.sum()
    return np.concatenate(out)[:n].astype(f32)


# ------------------------------------------------------------------------------------------------------------------ GPU helpers
@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


def upload(torch, K):
    D = dict(K)
    n = len(K["nl"])
    D["d_kl_t"] = torch.from_numpy(K["kl"].view(np.uint8).reshape(n, -1).copy()).cuda()
    D["d_ldesc_t"] = torch.from_numpy(K["ldesc"]).cuda(); D["d_eq_t"] = torch.from_numpy(K["lineeq"]).cuda()
    D["d_nl_t"] = torch.from_numpy(K["nl"]).cuda(); D["d_has_ml_t"] = torch.from_numpy(K["has_ml"]).cuda()
    D["d_pose_t"] = torch.from_numpy(K["pose"]).cuda(); D["d_depth_t"] = torch.from_numpy(K["depth"]).cuda()
    return D


def matcher(pkg, D, max_batch=32):
    return pkg.Matcher(max_features=64, max_lines=D["capl"] - 64, max_nodes=16, max_batch=max_batch)


def outputs(torch, P, capl):
    return dict(rows=torch.full((P, capl, 2), 7, dtype=torch.int32, device="cuda"), n=torch.full((P,), -7, dtype=torch.int32, device="cuda"),
                status=torch.full((P, capl), 77, dtype=torch.int32, device="cuda"),
                line3d=torch.full((P, capl, 6), 7.5, dtype=torch.float32, device="cuda"), nnew=torch.full((P,), -7, dtype=torch.int32, device="cuda"))


def run(mt, torch, D, pairs, has_ml=None, depth=None, sync=True):
    P, capl = len(pairs), D["capl"]
    d_pair = torch.tensor(np.array(pairs, np.int32).reshape(-1, 2), device="cuda")
    out = outputs(torch, P, capl)
    hm = D["d_has_ml_t"] if has_ml is None else has_ml
    dp = D["d_depth_t"] if depth is None else depth
    mt.create_new_map_lines_batch_device(D["d_kl_t"].data_ptr(), D["d_ldesc_t"].data_ptr(), D["d_eq_t"].data_ptr(), D["d_nl_t"].data_ptr(),
                                         len(D["nl"]), capl, hm.data_ptr(), P, d_pair.data_ptr(), D["d_pose_t"].data_ptr(), dp.data_ptr(),
                                         D["cam"], out["rows"].data_ptr(), out["n"].data_ptr(), out["status"].data_ptr(),
                                         out["line3d"].data_ptr(), out["nnew"].data_ptr())
    if sync:
        mt.sync()
    res = {k: v.cpu().numpy() for k, v in out.items()}
    res["keep"] = d_pair
    return res


def check_pair(G, p, exp):
    n = exp["n"]
    assert G["n"][p] == n, (p, int(G["n"][p]), n)
    k = max(n, 0)
    assert np.array_equal(G["rows"][p, :k], exp["rows"]), p
    assert (G["rows"][p, k:] == -1).all() and (G["status"][p, k:] == -1).all(), p
    assert np.array_equal(G["status"][p, :k], exp["status"]), (p, np.nonzero(G["status"][p, :k] != exp["status"])[0][:8])
    w = exp["written"]
    assert np.array_equal(G["line3d"][p, :k][w].view(np.uint32), exp["line3d"][w].view(np.uint32)), p
    assert (G["line3d"][p, :k][~w] == 7.5).all() and (G["line3d"][p, k:] == 7.5).all(), p
    assert G["nnew"][p] == exp["nnew"], p


def check_all(G, E):
    for p, e in enumerate(E):
        check_pair(G, p, e)


@pytest.fixture(scope="module")
def small(pkg, torch):
    K = scene(pkg)
    assert K["nl"][EMPTY] == 0 and K["nl"][SINGLE] == 1 and (np.delete(K["nl"], [EMPTY, SINGLE]) >= 30).all(), K["nl"]
    return upload(torch, K)


def test_equal_model(pkg, oracle, torch, small):
    """KF 0 against its 10 neighbours (EMPTY and SINGLE among them), a second chain (KF 3's) and a KF1 without lines, in one call."""
    D = small
    mt = matcher(pkg, D)
    pairs = neighbour_pairs() + [(3, k) for k in (2, 4, 5, 0, 7, 10)] + [(EMPTY, 1)]
    G = run(mt, torch, D, pairs)
    E = oracle_chain(oracle, D, pairs)
    check_all(G, E)
    assert sum(e["nnew"] for e in E) > 40 and G["n"][EMPTY - 1] == -1 and G["n"][SINGLE - 1] == -1 and G["n"][-1] == 0


def test_rows_equal_batched_matcher_under_chain_mask(pkg, torch, small):
    """Each pair's rows equal sslpl_line_search_for_triangulation_batch_device given d_has_ml with the created rows of the earlier pairs
    of its chain set; the masking changes some pair's rows."""
    D = small
    mt = matcher(pkg, D)
    pairs = neighbour_pairs()
    G = run(mt, torch, D, pairs)
    hm = D["has_ml"].copy()
    changed = 0
    for p, (i, j) in enumerate(pairs):
        for h, tag in ((hm, "chain"), (D["has_ml"], "plain")):
            d_h = torch.from_numpy(h).cuda()
            d_pair = torch.tensor([[i, j]], dtype=torch.int32, device="cuda")
            d_rows = torch.full((1, D["capl"], 2), 7, dtype=torch.int32, device="cuda"); d_n = torch.full((1,), -7, dtype=torch.int32, device="cuda")
            mt.line_search_for_triangulation_batch_device(D["d_ldesc_t"].data_ptr(), D["d_nl_t"].data_ptr(), NKF, D["capl"], d_h.data_ptr(), 1,
                                                          d_pair.data_ptr(), d_rows.data_ptr(), d_n.data_ptr())
            mt.sync()
            rows, n = d_rows.cpu().numpy()[0], int(d_n.cpu().numpy()[0])
            if tag == "chain":
                assert n == G["n"][p] and np.array_equal(rows, G["rows"][p]), p
            else:
                changed += n != G["n"][p]
        k = max(G["n"][p], 0)
        hm[i, G["rows"][p, :k][G["status"][p, :k] == 0, 0]] = 1
    assert changed > 0


def test_prefix_and_separate_chains(pkg, torch, small):
    """The first k pairs of a chain give the results of a call with only those pairs; two chains in one call equal two calls."""
    D = small
    mt = matcher(pkg, D)
    a = neighbour_pairs(); b = [(5, k) for k in (4, 6, 7, 0, 3, 1)]
    Gab = run(mt, torch, D, a + b)
    Ga, Gb = run(mt, torch, D, a), run(mt, torch, D, b)
    for key in ("rows", "n", "status", "nnew"):
        assert np.array_equal(Gab[key], np.concatenate([Ga[key], Gb[key]])), key
    assert np.array_equal(Gab["line3d"].view(np.uint32), np.concatenate([Ga["line3d"], Gb["line3d"]]).view(np.uint32))
    for k in (1, 4, 7):
        Gk = run(mt, torch, D, a[:k])
        for key in ("rows", "n", "status", "nnew"):
            assert np.array_equal(Gk[key], Ga[key][:k]), (k, key)
        assert np.array_equal(Gk["line3d"].view(np.uint32), Ga["line3d"][:k].view(np.uint32)), k


def test_bad_pairs(pkg, oracle, torch, small):
    """Out-of-range indices, kf2 == kf1, a repeated kf2, a KF2 with one line or none get -1 and no rows and leave the chain's state
    alone; a KF1 without lines gives 0."""
    D = small
    mt = matcher(pkg, D)
    good = [(0, 1), (0, 2), (0, 3), (0, 4)]
    pairs = [(0, 1), (0, NKF), (0, 2), (0, 0), (0, 1), (0, SINGLE), (0, -3), (0, 3), (0, EMPTY), (0, 2), (0, 4), (NKF, 1), (-1, 2),
             (EMPTY, 1), (EMPTY, SINGLE)]
    G = run(mt, torch, D, pairs)
    E = oracle_chain(oracle, D, good)
    gi = 0
    for p, pr in enumerate(pairs):
        if pr in good and pr not in pairs[:p]:
            check_pair(G, p, E[gi]); gi += 1
        else:
            n = 0 if pr[0] == EMPTY else -1
            assert G["n"][p] == n and G["nnew"][p] == 0 and (G["rows"][p] == -1).all() and (G["status"][p] == -1).all(), p
            assert (G["line3d"][p] == 7.5).all(), p
    assert gi == 4 and sum(e["nnew"] for e in E) > 0


def test_depth_zero_negative_inf(pkg, oracle, torch, small):
    """A KF2 median depth of 0, a negative one and +inf follow IEEE through the gates as in the model."""
    D = dict(small)
    mt = matcher(pkg, D)
    depth = D["depth"].copy()
    depth[[4, 5, 6]] = [0.0, -3.0, np.inf]
    D["depth"] = depth
    pairs = neighbour_pairs()
    G = run(mt, torch, D, pairs, depth=torch.from_numpy(depth).cuda())
    E = oracle_chain(oracle, D, pairs)
    check_all(G, E)
    assert all(E[k - 1]["n"] > 0 for k in (4, 5, 6))
    assert (E[3]["status"] == M.LONG).any() and (E[4]["status"] == M.NEAR_S1).any() and (E[5]["status"] == M.NEAR_S1).any()


def test_device_svd_line_matrices(pkg, oracle, small):
    """The device SVD equals the model on line-shaped matrices (the scene's, random lines, near-epipolar lines)."""
    mt = pkg.Matcher(max_features=64, max_lines=0, max_nodes=16)
    A = line_svd_tables(np.random.default_rng(12), 200000, small, oracle)
    W, Vt, _ = mt.debug_svd4(A)
    Wm, Vm = M.svd4(A)
    assert np.array_equal(W.view(np.uint32), Wm.view(np.uint32)) and np.array_equal(Vt.view(np.uint32), Vm.view(np.uint32))


def test_large_frames(pkg, oracle, torch):
    """1280x960, 500 lines per keyframe (capl = 564), nkf = max_batch + 1 and npairs = max_batch."""
    K = scene(pkg, 1280, 960, 500, nkf=11, empty=None, single=None, seed=3)
    D = upload(torch, K)
    assert D["capl"] == 564 and (D["nl"] > 300).all(), D["nl"]
    mt = matcher(pkg, D, max_batch=10)
    pairs = neighbour_pairs()
    assert len(pairs) == 10
    G = run(mt, torch, D, pairs)
    E = oracle_chain(oracle, D, pairs)
    check_all(G, E)
    assert sum(e["nnew"] for e in E) > 200


def test_caller_stream_and_argument_errors(pkg, oracle, torch, small):
    D = small
    mt = matcher(pkg, D)
    pairs = neighbour_pairs()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        mt.set_stream(s.cuda_stream)
        G1 = run(mt, torch, D, pairs, sync=False)
        G2 = run(mt, torch, D, pairs[:5] + [(3, 2), (3, 4)], sync=False)
    s.synchronize()
    mt.set_stream(0)
    check_all(G1, oracle_chain(oracle, D, pairs))
    check_all(G2, oracle_chain(oracle, D, pairs[:5] + [(3, 2), (3, 4)]))
    # bad arguments: SSLPL_ERR_ARG, nothing enqueued, nothing written
    P, capl = len(pairs), D["capl"]
    d_pair = torch.tensor(np.array(pairs, np.int32), device="cuda")
    o = outputs(torch, P, capl)
    good = dict(d_kl=D["d_kl_t"].data_ptr(), d_ldesc=D["d_ldesc_t"].data_ptr(), d_lineeq=D["d_eq_t"].data_ptr(), d_nl=D["d_nl_t"].data_ptr(),
                nkf=NKF, capl=capl, d_has_ml=D["d_has_ml_t"].data_ptr(), npairs=P, d_pair=d_pair.data_ptr(), d_kfpose=D["d_pose_t"].data_ptr(),
                d_kfdepth=D["d_depth_t"].data_ptr(), cam=D["cam"], d_lpairs=o["rows"].data_ptr(), d_nlmatch=o["n"].data_ptr(),
                d_status=o["status"].data_ptr(), d_line3d=o["line3d"].data_ptr(), d_nnew=o["nnew"].data_ptr())
    mt_small = pkg.Matcher(max_features=64, max_lines=capl - 64, max_nodes=16, max_batch=10)
    mt_nolines = pkg.Matcher(max_features=64, max_lines=0, max_nodes=16, max_batch=10)
    bad = [dict(d_kl=0), dict(d_ldesc=0), dict(d_lineeq=0), dict(d_nl=0), dict(d_has_ml=0), dict(d_pair=0), dict(d_kfpose=0),
           dict(d_kfdepth=0), dict(d_lpairs=0), dict(d_nlmatch=0), dict(d_status=0), dict(d_line3d=0), dict(d_nnew=0), dict(nkf=0),
           dict(nkf=12), dict(npairs=0), dict(npairs=11), dict(capl=0), dict(capl=capl + 1)]
    for h, cases in ((mt_small, bad), (mt_nolines, [dict()])):
        before = h.launch_count
        for b in cases:
            with pytest.raises(pkg.SslplError, match="error -1:"):
                h.create_new_map_lines_batch_device(**{**good, **b})
        h.sync()
        assert h.launch_count == before
    assert (o["rows"] == 7).all().item() and (o["n"] == -7).all().item() and (o["status"] == 77).all().item()
    assert (o["line3d"] == 7.5).all().item() and (o["nnew"] == -7).all().item()
    before = mt_small.launch_count
    mt_small.create_new_map_lines_batch_device(**good)
    mt_small.sync()
    assert mt_small.launch_count == before + 3 and (o["n"][[p for p in range(P) if pairs[p][1] not in (EMPTY, SINGLE)]] > 0).all().item()
