"""GPU tests of sslpl_pose_optimization_batch_device (Optimizer::PoseOptimization, Optimizer.cc:666-1022) against tests/pose_model.py.
The parity contract (DESIGN.md, "Pose optimisation"): rotation within 1e-6 rad, translation within 1e-6 (1 + |t|), and identical
outlier flags and return values except for edges whose model chi2 lies within a relative 1e-5 of its threshold in some round (at most
0.5 % of the edges).  Also: bitwise determinism across batch positions, batch sizes and runs; the edge cases of the C ABI; bad
arguments; and an ORB -> pose optimisation -> SearchByProjection chain without a host round trip."""
import math

import numpy as np
import pytest

import pose_model as pm
from test_motion_batch_gpu import BOUNDS, SF, device_batch

pytestmark = pytest.mark.gpu
SENT = 7                                                   # what the flag rows hold before a call


@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


def dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def pack(pkg, scenes, points=True, lines=True, cap=None, capl=None):
    """Host tables of a batch of scenes: one element table for all frames' MapPoints and one for their MapLines."""
    B = len(scenes)
    cap = cap or max(len(s["obs"]) for s in scenes)
    capl = capl or max(1, max(len(s["lineeq"]) for s in scenes))
    kps = np.zeros((B, cap), pkg.KEYPOINT_DTYPE)
    n, nl = np.zeros(B, np.int32), np.zeros(B, np.int32)
    fmp, fml = np.full((B, cap), -1, np.int32), np.full((B, capl), -1, np.int32)
    lineeq = np.zeros((B, capl, 3))
    mp, ml, T = [], [], np.zeros((B, 12), np.float32)
    op = ol = 0
    for f, s in enumerate(scenes):
        k, kl = len(s["obs"]), len(s["lineeq"])
        kps["x"][f, :k], kps["y"][f, :k], kps["octave"][f, :k] = s["obs"][:, 0], s["obs"][:, 1], s["octave"]
        n[f], nl[f] = k, kl
        if points:
            fmp[f, :k] = np.where(s["fmp"] >= 0, s["fmp"] + op, s["fmp"])
        if lines:
            fml[f, :kl] = np.where(s["fml"] >= 0, s["fml"] + ol, s["fml"])
        lineeq[f, :kl] = s["lineeq"]
        mp.append(np.hstack([s["mp"], np.zeros((len(s["mp"]), 6), np.float32)]))
        ml.append(s["mlpos"])
        op, ol = op + len(s["mp"]), ol + len(s["mlpos"])
        T[f] = s["T0"]
    return dict(kps=kps, n=n, fmp=fmp, mp=np.concatenate(mp).astype(np.float32), lineeq=lineeq, nl=nl, fml=fml if lines else None,
                mlpos=np.concatenate(ml).astype(np.float64), T=T, cam=scenes[0]["cam"], inv=scenes[0]["inv"], cap=cap, capl=capl)


def matcher(pkg, P, max_batch=64):
    return pkg.Matcher(max_features=P["cap"], max_lines=P["capl"], max_nodes=16, max_batch=max_batch)


def upload(torch, P):
    U = dict(kps=dev(torch, P["kps"].view(np.uint8)), n=dev(torch, P["n"]), fmp=dev(torch, P["fmp"]), mp=dev(torch, P["mp"]),
             lineeq=dev(torch, P["lineeq"]), nl=dev(torch, P["nl"]), mlpos=dev(torch, P["mlpos"]), T=dev(torch, P["T"]))
    if P["fml"] is not None:
        U["fml"] = dev(torch, P["fml"])
    return U


def run(mt, torch, P, U=None, rows=None, inplace=False, sync=True):
    """The device call on the frames `rows` of a packed batch (all by default) -> host (T, outlier, line_outlier, ninlier)."""
    U = U or upload(torch, P)
    rows = np.arange(len(P["n"])) if rows is None else np.asarray(rows)
    sel = lambda k: U[k] if len(rows) == len(P["n"]) and (rows == np.arange(len(rows))).all() else U[k][torch.as_tensor(rows).cuda()].contiguous()
    B = len(rows)
    kps, n, fmp, lq, nl, T = sel("kps"), sel("n"), sel("fmp"), sel("lineeq"), sel("nl"), sel("T").clone()
    fml = sel("fml") if P["fml"] is not None else None
    Tout = T if inplace else torch.zeros((B, 12), dtype=torch.float32, device="cuda")
    out = torch.full((B, P["cap"]), SENT, dtype=torch.uint8, device="cuda")
    lout = torch.full((B, P["capl"]), SENT, dtype=torch.uint8, device="cuda")
    ninl = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    mt.pose_optimization_batch_device(kps.data_ptr(), n.data_ptr(), B, P["cap"], fmp.data_ptr(), len(P["mp"]), U["mp"].data_ptr(),
                                      lq.data_ptr(), nl.data_ptr(), P["capl"], fml.data_ptr() if fml is not None else 0,
                                      len(P["mlpos"]), U["mlpos"].data_ptr(), T.data_ptr(), P["cam"], P["inv"], Tout.data_ptr(),
                                      out.data_ptr(), lout.data_ptr(), ninl.data_ptr())
    if not sync:
        return Tout, out, lout, ninl
    mt.sync()
    return Tout.cpu().numpy(), out.cpu().numpy(), lout.cpu().numpy(), ninl.cpu().numpy()


def model(P, f):
    k = min(max(int(P["n"][f]), 0), P["cap"])
    kl = min(max(int(P["nl"][f]), 0), P["capl"])
    kp = P["kps"][f, :k]
    return pm.pose_optimization(np.stack([kp["x"], kp["y"]], 1), kp["octave"], P["fmp"][f, :k], P["mp"][:, :3], P["T"][f], P["cam"],
                                P["inv"], lineeq=P["lineeq"][f, :kl], fml=None if P["fml"] is None else P["fml"][f, :kl],
                                mlpos=P["mlpos"], outlier=np.full(k, SENT, np.uint8), line_outlier=np.full(kl, SENT, np.uint8))


def check_parity(P, got, frames=None):
    """The parity contract frame by frame; returns (edges, edges in the band)."""
    T, out, lout, ninl = got
    edges = band = 0
    for f in (range(len(P["n"])) if frames is None else frames):
        r = model(P, f)
        k, kl = len(r["outlier"]), len(r["line_outlier"])
        bp, bl = pm.in_band(r) if r["rounds"] else (np.zeros(0, bool), np.zeros(0, bool))
        ip = np.nonzero((P["fmp"][f, :k] >= 0) & (P["fmp"][f, :k] < len(P["mp"])))[0]
        il = np.nonzero((P["fml"][f, :kl] >= 0) & (P["fml"][f, :kl] < len(P["mlpos"])))[0] if P["fml"] is not None else np.zeros(0, int)
        nb = int(bp.sum() + bl.sum()) if r["rounds"] else 0
        edges += len(ip) + 2 * len(il)
        band += nb
        okp = np.ones(k, bool)
        okl = np.ones(kl, bool)
        if nb:
            okp[ip[bp]] = False
            okl[il[bl]] = False
        assert np.array_equal(out[f, :k][okp], r["outlier"][okp]), f
        assert (out[f, k:] == SENT).all()
        if P["fml"] is not None:
            assert np.array_equal(lout[f, :kl][okl], r["line_outlier"][okl]), f
        assert abs(int(ninl[f]) - r["ninlier"]) <= nb, (f, int(ninl[f]), r["ninlier"])
        if r["pose"] is None:
            assert np.array_equal(T[f], r["T"]), f
        elif nb == 0:
            Rg, Rm = T[f].reshape(3, 4)[:, :3].astype(np.float64), pm.quat_to_matrix(r["pose"][0])
            # the device result is narrowed to float: compare its rotation with the model's double one
            assert pm.rot_angle(Rg, Rm) < 1e-6, f
            tm = r["pose"][1]
            assert np.abs(T[f].reshape(3, 4)[:, 3] - tm).max() < 1e-6 * (1 + np.linalg.norm(tm)), f
    assert band <= 0.005 * max(edges, 1), (band, edges)
    return edges, band


SIZES = {"640": (640, 480, 1000, 40), "1280": (1280, 960, 4000, 500)}


def scenes(size, frac, nframes, seed):
    W, H, npts, nlines = SIZES[size]
    rng = np.random.default_rng(seed)
    return [pm.make_scene(rng, W, H, npts, nlines, outlier_frac=frac) for _ in range(nframes)]


@pytest.mark.parametrize("size", ["640", "1280"])
@pytest.mark.parametrize("frac", [0.0, 0.2, 0.5])
@pytest.mark.parametrize("kind", ["points", "lines", "both"])
def test_parity_with_the_model(pkg, torch, size, frac, kind):
    S = scenes(size, frac, 6, seed=100 + int(10 * frac))
    P = pack(pkg, S, points=kind != "lines", lines=kind != "points")
    mt = matcher(pkg, P)
    got = run(mt, torch, P)
    edges, band = check_parity(P, got)
    print(f"{size} frac {frac} {kind}: {edges} edges, {band} in the 1e-5 band")
    if kind != "lines":                                               # the optimised pose is near the ground truth
        for f, s in enumerate(S):
            assert math.degrees(pm.rot_angle(got[0][f].reshape(3, 4)[:, :3].astype(np.float64), s["R"])) < 0.1


def test_deterministic_across_positions_batch_sizes_and_runs(pkg, torch):
    S = scenes("640", 0.2, 12, seed=7)
    P = pack(pkg, S)
    mt = matcher(pkg, P)
    U = upload(torch, P)
    a = run(mt, torch, P, U)
    b = run(mt, torch, P, U)
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()
    rev = np.arange(12)[::-1].copy()
    c = run(mt, torch, P, U, rows=rev)
    for x, y in zip(a, c):
        assert x[rev].tobytes() == y.tobytes()
    for f in (0, 5, 11):
        d = run(mt, torch, P, U, rows=[f])
        for x, y in zip(a, d):
            assert x[f].tobytes() == y[0].tobytes()


def test_edge_cases(pkg, torch):
    rng = np.random.default_rng(9)
    S = [pm.make_scene(rng, 640, 480, 200, 20, outlier_frac=0.1) for _ in range(7)]
    S[0]["fmp"][2:] = -1                                               # 2 points + 0 lines: fewer than 3 correspondences
    S[0]["fml"][:] = -1
    S[1]["fmp"][3:] = -1                                               # 3 points + 3 lines = 9 edges: one round
    S[1]["fml"][3:] = -1
    S[2] = pm.make_scene(rng, 640, 480, 200, 20, outlier_frac=1.0, noise=100.0)   # every edge an outlier after round 0
    S[3]["octave"][17] = -1                                            # an octave outside the pyramid
    S[4]["fmp"][::3] = 10 ** 6                                         # element indices outside the tables: NULL
    S[4]["fml"][::2] = -5
    P = pack(pkg, S, cap=256, capl=32)
    P["n"][5], P["nl"][5] = 10 ** 6, 10 ** 6                           # counts above cap / capl: clamped
    P["n"][6], P["nl"][6] = -4, 0                                      # negative count: no features
    mt = matcher(pkg, P)
    got = run(mt, torch, P)
    check_parity(P, got)
    T, out, lout, ninl = got
    assert ninl[0] == 0 and np.array_equal(T[0], P["T"][0]) and out[0, :2].tolist() == [0, 0] and (out[0, 2:] == SENT).all()
    assert [rd["ran"] for rd in model(P, 2)["rounds"]] == [True, False, False, False]
    assert ninl[2] == 0 and np.array_equal(T[2], pm.se3_to_f32(pm.se3_from_f32(P["T"][2])))
    assert ninl[3] == -1 and np.array_equal(T[3], P["T"][3]) and (out[3] == SENT).all() and (lout[3] == SENT).all()
    assert (out[4, ::3][:67] == SENT).all()
    assert ninl[6] == 0 and np.array_equal(T[6], P["T"][6])
    # in place: d_Tcw_out = d_Tcw
    g2 = run(mt, torch, P, inplace=True)
    for x, y in zip(got, g2):
        assert x.tobytes() == y.tobytes()


def test_caller_stream_and_argument_errors(pkg, torch):
    S = scenes("640", 0.2, 4, seed=13)
    P = pack(pkg, S)
    mt = matcher(pkg, P, max_batch=4)
    U = upload(torch, P)
    ref = run(mt, torch, P, U)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        mt.set_stream(s.cuda_stream)
        o = run(mt, torch, P, U, sync=False)
    s.synchronize()
    mt.set_stream(0)
    for x, y in zip(ref, o):
        assert x.tobytes() == y.cpu().numpy().tobytes()
    Tout = torch.zeros((5, 12), dtype=torch.float32, device="cuda")
    out = torch.full((5, P["cap"]), SENT, dtype=torch.uint8, device="cuda")
    lout = torch.full((5, P["capl"]), SENT, dtype=torch.uint8, device="cuda")
    ninl = torch.full((5,), -7, dtype=torch.int32, device="cuda")
    good = dict(d_kps=U["kps"].data_ptr(), d_n=U["n"].data_ptr(), nframes=4, cap=P["cap"], d_fmp=U["fmp"].data_ptr(), nmp=len(P["mp"]),
                d_mp=U["mp"].data_ptr(), d_lineeq=U["lineeq"].data_ptr(), d_nl=U["nl"].data_ptr(), capl=P["capl"],
                d_fml=U["fml"].data_ptr(), nml=len(P["mlpos"]), d_mlpos=U["mlpos"].data_ptr(), d_Tcw=U["T"].data_ptr(), cam=P["cam"],
                inv_level_sigma2=P["inv"], d_Tcw_out=Tout.data_ptr(), d_outlier=out.data_ptr(), d_line_outlier=lout.data_ptr(),
                d_ninlier=ninl.data_ptr())
    torch.cuda.synchronize()
    before = mt.launch_count
    for kw in (dict(nframes=0), dict(nframes=5), dict(cap=0), dict(cap=P["cap"] + 65), dict(nmp=-1), dict(d_mp=0),
               dict(capl=0), dict(capl=P["capl"] + 65), dict(nml=-1), dict(d_mlpos=0), dict(d_lineeq=0), dict(d_nl=0),
               dict(d_line_outlier=0), dict(inv_level_sigma2=np.ones(17, np.float32)), dict(inv_level_sigma2=np.ones(0, np.float32)),
               dict(d_kps=0), dict(d_n=0), dict(d_fmp=0), dict(d_Tcw=0), dict(d_Tcw_out=0), dict(d_outlier=0), dict(d_ninlier=0)):
        with pytest.raises(pkg.SslplError):
            mt.pose_optimization_batch_device(**dict(good, **kw))
    torch.cuda.synchronize()
    assert mt.launch_count == before
    assert (Tout == 0).all() and (out == SENT).all() and (lout == SENT).all() and (ninl == -7).all()
    # without lines the line arguments are not read
    mt.pose_optimization_batch_device(**dict(good, d_fml=0, d_lineeq=0, d_nl=0, capl=0, nml=-1, d_mlpos=0, d_line_outlier=0))
    mt.sync()
    assert mt.launch_count == before + 1 and (lout == SENT).all() and (ninl[:4] >= 0).all() and ninl[4] == -7


def test_chain_from_orb_to_search_by_projection_without_the_host(pkg, synth, torch):
    """ORB keypoints of synthetic frames, MapPoints back-projected from them under a known pose, a perturbed pose, the batched
    optimisation, then d_Tcw_out straight into sslpl_search_by_projection_frame_batch_device; the same chain with the poses staged
    through the host gives the same tables."""
    B = 6
    D = device_batch(pkg, torch, synth.batch(640, 480, B), 1000)
    cap, kps, n = D["cap"], D["kps"], D["n"]
    cam = np.array([481.2, 480.0, 319.5, 239.5], np.float32)
    inv = (np.float32(1) / SF.astype(np.float32) ** 2).astype(np.float32)
    rng = np.random.default_rng(17)
    Xw = np.zeros((B, cap, 3), np.float32)
    T0 = np.zeros((B, 12), np.float32)
    R, t = pm.random_pose(rng, 10.0, 0.3)                             # one pose for the whole (nearly static) sequence
    for f in range(B):
        z = rng.uniform(1.0, 6.0, cap)
        Xc = np.stack([(kps["x"][f] - cam[2]) / cam[0] * z, (kps["y"][f] - cam[3]) / cam[1] * z, z], 1)
        Xw[f] = ((Xc - t) @ R).astype(np.float32)
        R0, t0 = pm.perturb(R, t, rng, 2.0, 0.05)
        T0[f] = pm.pose12(R0, t0)
    fmp = np.where(np.arange(cap)[None] < n[:, None], np.arange(B)[:, None] * cap + np.arange(cap)[None], -1).astype(np.int32)
    mp = np.hstack([Xw.reshape(-1, 3), np.zeros((B * cap, 6), np.float32)])
    mt = pkg.Matcher(max_features=cap, max_lines=64, max_nodes=3072, max_batch=B)
    d_fmp, d_mp, d_T = dev(torch, fmp), dev(torch, mp), dev(torch, T0)
    d_out = torch.zeros((B, 12), dtype=torch.float32, device="cuda")
    d_ol = torch.full((B, cap), SENT, dtype=torch.uint8, device="cuda")
    d_ni = torch.zeros(B, dtype=torch.int32, device="cuda")
    d_Xw = dev(torch, Xw)
    d_flag = dev(torch, np.where(np.arange(cap)[None] < n[:, None], 3, 0).astype(np.uint8))

    def search(d_pose):
        a = torch.full((B - 1, cap), 7, dtype=torch.int32, device="cuda")
        m = torch.full((B - 1,), -7, dtype=torch.int32, device="cuda")
        mt.search_by_projection_frame_batch_device(D["d_kps"], D["d_desc"], D["d_n"], B, cap, d_Xw.data_ptr(), d_flag.data_ptr(), 0,
                                                   d_pose.data_ptr(), cam, BOUNDS, SF, 15.0, True, 20, a.data_ptr(), m.data_ptr())
        return a, m

    mt.pose_optimization_batch_device(D["d_kps"], D["d_n"], B, cap, d_fmp.data_ptr(), len(mp), d_mp.data_ptr(), 0, 0, 0, 0, 0, 0,
                                      d_T.data_ptr(), cam, inv, d_out.data_ptr(), d_ol.data_ptr(), 0, d_ni.data_ptr())
    a_dev, m_dev = search(d_out)                                       # no host synchronisation in between
    mt.sync()
    T_host = d_out.cpu().numpy()
    a_host, m_host = search(dev(torch, T_host))
    mt.sync()
    assert np.array_equal(a_dev.cpu().numpy(), a_host.cpu().numpy()) and np.array_equal(m_dev.cpu().numpy(), m_host.cpu().numpy())
    assert (m_dev.cpu().numpy() > 0).all()
    ni = d_ni.cpu().numpy()
    assert (ni == n).all()
    for f in range(B):
        assert math.degrees(pm.rot_angle(T_host[f].reshape(3, 4)[:, :3].astype(np.float64), R)) < 0.01
    # and the device chain's poses are the model's
    P = dict(kps=kps, n=n, fmp=fmp, mp=mp, lineeq=np.zeros((B, 1, 3)), nl=np.zeros(B, np.int32), fml=None, mlpos=np.zeros((0, 6)),
             T=T0, cam=cam, inv=inv, cap=cap, capl=1)
    check_parity(P, (T_host, d_ol.cpu().numpy(), np.zeros((B, 1), np.uint8), ni))
