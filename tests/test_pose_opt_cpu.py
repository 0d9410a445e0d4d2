"""CPU tests of tests/pose_model.py, the restatement of Optimizer::PoseOptimization (Optimizer.cc:666-1022) that
sslpl_pose_optimization_batch_device is held to: the edges' Jacobians, the SE3 exp map and quaternion conversions, pose recovery on
synthetic scenes, the final unrobust round against scipy's least squares, and each rule of the reference's four-round loop."""
import math

import numpy as np
import pytest
from scipy.optimize import least_squares
from scipy.spatial.transform import Rotation

import pose_model as pm


def scene(seed, npts=300, nlines=40, **kw):
    return pm.make_scene(np.random.default_rng(seed), 640, 480, npts, nlines, **kw)


def pose_err(P, R, t):
    return math.degrees(pm.rot_angle(pm.quat_to_matrix(P[0]), R)), float(np.abs(P[1] - t).max())


@pytest.mark.parametrize("kind", ["mono", "line"])
def test_jacobians_match_central_differences(kind):
    sc = scene(3, npts=50, nlines=50, dtype=np.float64)
    P = pm.se3_from_f32(sc["T0"])
    cam = sc["cam"]
    if kind == "mono":
        f = lambda Q: pm.mono_edge(Q, sc["mp"], sc["obs"], cam)
        J = pm.mono_edge(P, sc["mp"], sc["obs"], cam, jac=True)[1]
    else:
        f = lambda Q: pm.line_edge(Q, sc["mlpos"][:, :3], sc["lineeq"], cam)[:, None]
        J = pm.line_edge(P, sc["mlpos"][:, :3], sc["lineeq"], cam, jac=True)[1][:, None, :]
    h = 1e-6
    for k in range(6):
        d = np.zeros(6)
        d[k] = h
        num = (f(pm.se3_exp_mul(d, P)) - f(pm.se3_exp_mul(-d, P))) / (2 * h)
        scale = np.abs(J[:, :, k]).max() + 1.0
        assert np.abs(num - J[:, :, k]).max() < 1e-5 * scale, (kind, k)


def test_exp_map_matches_scipy():
    rng = np.random.default_rng(5)
    for theta in (1e-4, 1e-3, 0.1, 1.0, 2.5, 3.1):
        for _ in range(5):
            w = rng.normal(size=3)
            w *= theta / np.linalg.norm(w)
            R, V, (q, t) = pm.se3_exp(np.concatenate([w, [0.3, -0.2, 0.5]]))
            ref = Rotation.from_rotvec(w)
            assert np.abs(R - ref.as_matrix()).max() < 1e-12
            assert np.abs(pm.quat_to_matrix(q) - ref.as_matrix()).max() < 1e-12
            qs = ref.as_quat()                                    # (x, y, z, w)
            qs = qs if qs[3] >= 0 else -qs
            assert np.abs(q - np.array([qs[3], qs[0], qs[1], qs[2]])).max() < 1e-12
    # below theta = 1e-5 the reference uses R = V = I + Omega + Omega^2 (se3quat.h: exp), not the series
    w = np.array([3e-6, -2e-6, 1e-6])
    R, V, _ = pm.se3_exp(np.concatenate([w, np.zeros(3)]))
    O = pm.skew(w)
    assert np.array_equal(R, np.eye(3) + O + O @ O) and np.array_equal(V, R)


def test_quaternion_from_matrix_every_branch():
    rng = np.random.default_rng(6)
    mats = [Rotation.from_rotvec(v).as_matrix() for v in rng.normal(size=(50, 3)) * 1.5]
    mats += [Rotation.from_rotvec(np.pi * np.eye(3)[i] * 0.999).as_matrix() for i in range(3)]    # trace < 0, each largest diagonal
    for M in mats:
        q = pm.quat_from_matrix(M)
        assert q[0] >= 0 and abs(np.linalg.norm(q) - 1) < 1e-15
        assert np.abs(pm.quat_to_matrix(q) - M).max() < 1e-12


@pytest.mark.parametrize("points,lines", [(True, True), (True, False), (False, True)])
def test_noise_free_scene_recovers_the_pose(points, lines):
    sc = scene(11, npts=400, nlines=60, noise=0.0, dtype=np.float64)
    r = pm.run_scene(sc, points=points, lines=lines)
    rot, tr = pose_err(r["pose"], sc["R"], sc["t"])
    assert math.radians(rot) < 1e-9 and tr < 1e-9
    assert r["ninlier"] == 400 * points + 60 * lines
    assert not r["outlier"].any() and not r["line_outlier"].any()


@pytest.mark.parametrize("frac", [0.2, 0.5])
def test_noisy_scene_flags_gross_outliers(frac):
    for seed in range(3):
        sc = scene(20 + seed, npts=1000, nlines=40, outlier_frac=frac)
        r = pm.run_scene(sc)
        rot, tr = pose_err(r["pose"], sc["R"], sc["t"])
        assert rot < 0.1 and tr < 0.01
        assert r["outlier"][sc["bad_p"]].all() and r["line_outlier"][sc["bad_l"]].all()
        # every gross outlier is counted, plus the noise tail of chi2(2) above 5.991 (about 5 % of the good points)
        good = ~sc["bad_p"]
        assert r["outlier"][good].mean() < 0.1
        assert r["ninlier"] == len(sc["obs"]) + len(sc["lineeq"]) - int(r["outlier"].sum()) - int(r["line_outlier"].sum())


def test_final_round_is_the_least_squares_optimum_of_its_inliers():
    sc = scene(31, npts=600, nlines=40, outlier_frac=0.2)
    r = pm.run_scene(sc)
    last = r["rounds"][-1]
    assert len(r["rounds"]) == 4 and not last["robust"]
    ap, al = last["active_p"], last["active_l"]
    P0 = pm.se3_from_f32(sc["T0"])
    obs, X, inv = sc["obs"].astype(np.float64)[ap], sc["mp"].astype(np.float64)[ap], sc["inv"][sc["octave"]].astype(np.float64)[ap]
    lq, S, E = sc["lineeq"][al], sc["mlpos"][al, :3], sc["mlpos"][al, 3:]

    def res(d):
        P = pm.se3_exp_mul(d, P0)
        e = pm.mono_edge(P, X, obs, sc["cam"]) * np.sqrt(inv)[:, None]
        return np.concatenate([e.reshape(-1), pm.line_edge(P, S, lq, sc["cam"]), pm.line_edge(P, E, lq, sc["cam"])])

    sol = least_squares(res, np.zeros(6), method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15)
    P = pm.se3_exp_mul(sol.x, P0)
    rot = pm.rot_angle(pm.quat_to_matrix(P[0]), pm.quat_to_matrix(r["pose"][0]))
    assert rot < 1e-7 and np.abs(P[1] - r["pose"][1]).max() < 1e-7


def test_every_round_restarts_from_the_input_pose_and_round_3_drops_the_kernels():
    sc = scene(41, npts=500, nlines=40, outlier_frac=0.3)
    r = pm.run_scene(sc)
    P0 = pm.se3_from_f32(sc["T0"])
    assert [x["robust"] for x in r["rounds"]] == [True, True, True, False]
    ip = np.arange(len(sc["obs"]))
    edges = pm._Edges(sc["obs"].astype(np.float64), sc["inv"][sc["octave"]].astype(np.float64), sc["mp"].astype(np.float64),
                      sc["lineeq"], sc["mlpos"][:, :3], sc["mlpos"][:, 3:], sc["cam"])
    for k, rd in enumerate(r["rounds"]):
        assert rd["start"][0].tobytes() == P0[0].tobytes() and rd["start"][1].tobytes() == P0[1].tobytes()
        # the round is one optimize() from the input pose on its level-0 edges, whatever the previous round reached
        P = pm.levenberg(edges, P0, ~rd["active_p"][ip], ~rd["active_l"], rd["robust"])[0]
        assert np.array_equal(P[0], rd["est"][0]) and np.array_equal(P[1], rd["est"][1])
    # with its kernels round 3 would end elsewhere: they are gone
    rd = r["rounds"][3]
    P = pm.levenberg(edges, P0, ~rd["active_p"], ~rd["active_l"], True)[0]
    assert not np.array_equal(P[1], rd["est"][1])


def test_active_points_are_classified_with_the_last_trial_error():
    sc = scene(43, npts=400, nlines=0, outlier_frac=0.3)
    r = pm.run_scene(sc, lines=False)
    for rd in r["rounds"]:
        a = rd["active_p"]
        e_last = pm.mono_edge(rd["last"], sc["mp"], sc["obs"], sc["cam"])
        e_est = pm.mono_edge(rd["est"], sc["mp"], sc["obs"], sc["cam"])
        inv = sc["inv"][sc["octave"]].astype(np.float64)
        c = lambda e: (e[:, 0] * (inv * e[:, 0]) + e[:, 1] * (inv * e[:, 1])).astype(np.float32)
        assert np.array_equal(rd["chi2_p"][a], c(e_last)[a]) and np.array_equal(rd["chi2_p"][~a], c(e_est)[~a])


def test_fewer_than_three_correspondences_return_zero_and_clear_the_flags():
    sc = scene(51, npts=8, nlines=4)
    fmp = np.full(8, -1, np.int32)
    fmp[[2, 5]] = [2, 5]
    fml = np.full(4, -1, np.int32)
    r = pm.pose_optimization(sc["obs"], sc["octave"], fmp, sc["mp"], sc["T0"], sc["cam"], sc["inv"], lineeq=sc["lineeq"], fml=fml,
                             mlpos=sc["mlpos"], outlier=np.full(8, 9, np.uint8), line_outlier=np.full(4, 9, np.uint8))
    assert r["ninlier"] == 0 and r["rounds"] == [] and np.array_equal(r["T"], sc["T0"])
    assert r["outlier"].tolist() == [9, 9, 0, 9, 9, 0, 9, 9] and r["line_outlier"].tolist() == [9] * 4


@pytest.mark.parametrize("npts,nlines,rounds", [(3, 3, 1), (9, 0, 1), (10, 0, 4), (4, 3, 4)])
def test_fewer_than_ten_edges_stop_after_the_first_round(npts, nlines, rounds):
    sc = scene(61, npts=npts, nlines=nlines)
    r = pm.run_scene(sc)
    assert len(r["rounds"]) == rounds


def test_points_only_form_ignores_the_line_tables():
    sc = scene(71, npts=300, nlines=30)
    a = pm.pose_optimization(sc["obs"], sc["octave"], sc["fmp"], sc["mp"], sc["T0"], sc["cam"], sc["inv"], lineeq=np.full((30, 3), np.nan),
                             fml=None, mlpos=None)
    b = pm.run_scene(dict(sc, lineeq=np.zeros((0, 3)), fml=np.zeros(0, np.int32), mlpos=np.zeros((0, 6))))
    assert np.array_equal(a["T"], b["T"]) and a["ninlier"] == b["ninlier"] and np.array_equal(a["outlier"], b["outlier"])
    assert len(a["line_outlier"]) == 0


def test_round_without_level0_edges_keeps_the_reset_pose():
    # every observation far from where any pose near the start puts it: all edges are outliers after round 0
    sc = scene(81, npts=40, nlines=6, outlier_frac=1.0)
    r = pm.run_scene(sc)
    assert r["ninlier"] == 0 and len(r["rounds"]) == 4
    P0 = pm.se3_from_f32(sc["T0"])
    for rd in r["rounds"][1:]:
        assert not rd["ran"] and rd["iters"] == 0
        assert np.array_equal(rd["est"][0], P0[0]) and np.array_equal(rd["est"][1], P0[1])
    assert np.array_equal(r["T"], pm.se3_to_f32(P0))


def test_octave_outside_the_pyramid_rejects_the_frame():
    sc = scene(91, npts=50, nlines=5)
    for bad in (-1, 8):
        octv = sc["octave"].copy()
        octv[7] = bad
        r = pm.pose_optimization(sc["obs"], octv, sc["fmp"], sc["mp"], sc["T0"], sc["cam"], sc["inv"], lineeq=sc["lineeq"],
                                 fml=sc["fml"], mlpos=sc["mlpos"], outlier=np.full(50, 3, np.uint8))
        assert r["ninlier"] == -1 and np.array_equal(r["T"], sc["T0"]) and (r["outlier"] == 3).all()
    # the octave of a feature without a MapPoint is never read
    octv = sc["octave"].copy()
    octv[7] = -1
    fmp = sc["fmp"].copy()
    fmp[7] = 50                                                     # outside the element table: NULL
    assert pm.pose_optimization(sc["obs"], octv, fmp, sc["mp"], sc["T0"], sc["cam"], sc["inv"])["ninlier"] >= 0
