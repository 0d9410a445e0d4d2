"""GPU parity, SURVEY.md 8(f) row 3: the search stages of the line projection matchers (LSDmatcher.cpp:22-141, :185-255) and of
Fuse (ORBmatcher.cc:828-973, LSDmatcher.cpp:417-548) against the oracle restatement (itself pinned to the reference in
tests/test_ref_parity_cpu.py) on the same projection-stage outputs."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mt(pkg):
    return pkg.Matcher(max_features=2048, max_lines=512, max_nodes=3072)


@pytest.mark.parametrize("seed,th,mono,sign,ratio", [(1, 20.0, True, 0, 0.8), (2, 20.0, False, 1, 0.8), (3, 40.0, False, -1, 0.9), (4, 10.0, True, 0, 0.6)])
def test_line_search_by_projection_frame(mt, oracle, synth, seed, th, mono, sign, ratio):
    from scenarios import line_scenario
    sc = line_scenario(oracle, synth, seed, f0=seed, stereo_sign=sign)
    last, cur = sc["last"], sc["cur"]
    q = oracle.line_project_frame(last["state"] == 1, last["Pw"], last["oct"], sc["Tcw"][:3], sc["Tlw"][:3], sc["cam5"], sc["bounds"], sc["sf"], th, mono)
    n_o, a_o = oracle.line_window_search(q, last["obs"], last["dml"], cur["ld"], cur["kl"], cur["oct"], cur["held"], ratio)
    n_g, a_g = mt.line_search_by_projection(q, last["obs"], last["dml"], cur["ld"], cur["kl"], cur["oct"], cur["held"], ratio)
    assert n_g == n_o and np.array_equal(a_g, a_o), (n_g, n_o, int((a_g != a_o).sum()))
    assert n_o > 5


@pytest.mark.parametrize("seed,th,ratio", [(1, 1.0, 0.8), (2, 3.0, 0.8), (3, 1.0, 0.6), (4, 0.5, 0.9)])
def test_line_search_by_projection_map_lines(mt, oracle, synth, seed, th, ratio):
    from scenarios import local_lines_scenario
    ml, cur, sf = local_lines_scenario(oracle, synth, seed, f0=seed)
    for mod in ("plain", "none_in_view", "all_held", "no_obs") if seed == 1 else ("plain",):
        m2, c2 = dict(ml), dict(cur)
        if mod == "none_in_view": m2["inview"] = np.zeros_like(ml["inview"])
        if mod == "all_held": c2["held"] = np.ones(len(cur["oct"]), np.uint8)
        if mod == "no_obs": m2["obs"] = np.zeros_like(ml["obs"])
        q = oracle.line_project_mls(m2["inview"], m2["bad"], m2["level"], m2["viewcos"], sf, th); q["proj"] = m2["proj"]
        n_o, a_o = oracle.line_window_search(q, m2["obs"], m2["desc"], c2["ld"], c2["kl"], c2["oct"], c2["held"], ratio)
        n_g, a_g = mt.line_search_by_projection(q, m2["obs"], m2["desc"], c2["ld"], c2["kl"], c2["oct"], c2["held"], ratio)
        assert n_g == n_o and np.array_equal(a_g, a_o), (mod, n_g, n_o)
        if mod == "plain":
            assert n_o > 30


@pytest.mark.parametrize("seed,th,stereo", [(1, 3.0, False), (2, 3.0, True), (3, 5.0, False), (4, 1.5, True), (5, 30.0, False)])
def test_fuse_points_search(mt, oracle, synth, seed, th, stereo):
    from scenarios import fuse_points_scenario
    sc = fuse_points_scenario(oracle, synth, seed, f0=seed, stereo=stereo)
    mp, kf = sc["mp"], sc["kf"]
    Tcw = sc["Tcw"]
    Ow = (-(Tcw[:3, :3].astype(np.float64).T @ Tcw[:3, 3].astype(np.float64))).astype(np.float32)
    q = oracle.fuse_project_points(mp["state"] != 1, mp["Xw"], mp["normal"], mp["min_raw"] * np.float32(0.8), mp["max_raw"] * np.float32(1.2), mp["max_raw"],
                                   Tcw[:3], Ow, sc["cam5"], sc["bounds"], 8, np.log(np.float32(1.2)))
    bi_o, bd_o = oracle.fuse_points_search(q, mp["desc"], kf["desc"], kf["x"], kf["y"], kf["oct"], kf["uright"], sc["bounds"], sc["sf"], sc["inv_sigma2"], th)
    bi_g, bd_g = mt.fuse_points_search(q, mp["desc"], kf["desc"], kf["x"], kf["y"], kf["oct"], kf["uright"], sc["bounds"], sc["sf"], sc["inv_sigma2"], th)
    assert np.array_equal(bi_g, bi_o) and np.array_equal(bd_g, bd_o), (int((bi_g != bi_o).sum()), int((bd_g != bd_o).sum()))
    assert ((bd_o <= 50) & (bi_o >= 0)).sum() > 150


@pytest.mark.parametrize("seed,th", [(1, 3.0), (2, 5.0), (3, 10.0), (4, 40.0)])
def test_fuse_lines_search(mt, oracle, synth, seed, th):
    from scenarios import fuse_lines_scenario
    sc = fuse_lines_scenario(oracle, synth, seed, f0=seed)
    ml, kf = sc["ml"], sc["kf"]
    Tcw = sc["Tcw"]
    Ow = (-(Tcw[:3, :3].astype(np.float64).T @ Tcw[:3, 3].astype(np.float64))).astype(np.float32)
    q = oracle.fuse_project_lines(ml["state"] != 1, ml["Pw"], ml["normal"], ml["min_raw"] * np.float32(0.8), ml["max_raw"] * np.float32(1.2), ml["max_raw"],
                                  Tcw[:3], Ow, sc["cam5"], sc["bounds"], 8, np.log(np.float32(1.2)))
    bi_o, bd_o = oracle.fuse_lines_search(q, ml["desc"], kf["ld"], kf["kl"], kf["oct"], sc["sf"], th)
    bi_g, bd_g = mt.fuse_lines_search(q, ml["desc"], kf["ld"], kf["kl"], kf["oct"], sc["sf"], th)
    assert np.array_equal(bi_g, bi_o) and np.array_equal(bd_g, bd_o), (int((bi_g != bi_o).sum()), int((bd_g != bd_o).sum()))
    assert ((bd_o <= 50) & (bi_o >= 0)).sum() > 10


def test_row3_edge_cases(mt, oracle, pkg):
    """Empty inputs on either side; a MapLine level outside the pyramid is dropped; a MapPoint level outside it is an argument error."""
    z = np.zeros(0)
    q = dict(active=np.zeros(0, np.uint8), proj=np.zeros((0, 4), np.float32), radius=z, min_level=z, max_level=z, level=z, u=z, v=z, ur=z)
    n, a = mt.line_search_by_projection(q, z, np.zeros((0, 32), np.uint8), np.zeros((3, 32), np.uint8), np.zeros((3, 3), np.float32), np.zeros(3, np.int32))
    assert n == 0 and np.array_equal(a, [-1, -1, -1])
    sf = (np.float32(1.2) ** np.arange(8)).astype(np.float32)
    bi, bd = mt.fuse_lines_search(q, np.zeros((0, 32), np.uint8), np.zeros((3, 32), np.uint8), np.zeros((3, 3), np.float32), np.zeros(3, np.int32), sf)
    assert len(bi) == 0
    q1 = dict(active=np.ones(2, np.uint8), proj=np.array([[10, 10, 30, 12], [10, 10, 30, 12]], np.float32), level=np.array([9, 0], np.int32))
    kl = np.array([[20, 11, 0.1]], np.float32)
    bi, bd = mt.fuse_lines_search(q1, np.zeros((2, 32), np.uint8), np.zeros((1, 32), np.uint8), kl, np.zeros(1, np.int32), sf, 3.0)
    assert list(bi) == [-1, 0] and bd[1] == 0
    bi, bd = mt.fuse_lines_search(q1, np.zeros((2, 32), np.uint8), np.zeros((0, 32), np.uint8), np.zeros((0, 3), np.float32), np.zeros(0, np.int32), sf, 3.0)
    assert list(bi) == [-1, -1]
    qp = dict(active=np.ones(1, np.uint8), u=np.array([100.], np.float32), v=np.array([100.], np.float32), ur=np.array([90.], np.float32), level=np.array([8], np.int32))
    with pytest.raises(pkg.SslplError):
        mt.fuse_points_search(qp, np.zeros((1, 32), np.uint8), np.zeros((1, 32), np.uint8), [100.], [100.], [0], None, (0, 640, 0, 480), sf, 1 / (sf * sf), 3.0)
    qp["level"] = np.array([0], np.int32)
    bi, bd = mt.fuse_points_search(qp, np.zeros((1, 32), np.uint8), np.zeros((1, 32), np.uint8), [100.], [100.], [0], None, (0, 640, 0, 480), sf, 1 / (sf * sf), 3.0)
    assert list(bi) == [0] and list(bd) == [0]
    for bad in ((640, 640, 0, 480), (0, 640, 480, 0)):                          # degenerate image bounds: rejected before any launch
        before = mt.launch_count
        with pytest.raises(pkg.SslplError):
            mt.fuse_points_search(qp, np.zeros((1, 32), np.uint8), np.zeros((1, 32), np.uint8), [100.], [100.], [0], None, bad, sf, 1 / (sf * sf), 3.0)
        assert mt.launch_count == before, bad
