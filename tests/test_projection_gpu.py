"""GPU parity: ORBmatcher::SearchByProjection(Frame&, const Frame&, th, bMono) (ORBmatcher.cc:1331-1473) with the 64 x 48
feature grid (Frame.cc:133-148, 368-421) — SURVEY.md 8(f) row 2 — against the oracle restatement."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


from scenarios import projection_scenario as scenario


@pytest.mark.parametrize("seed,th,mono,ori,claimed", [(1, 15.0, True, True, 0.05), (2, 7.0, True, True, 0.0), (3, 30.0, True, False, 0.2),
                                                       (4, 15.0, False, True, 0.05), (5, 15.0, False, True, 0.0), (6, 100.0, True, True, 0.0)])
def test_search_by_projection_frame(pkg, oracle, synth, seed, th, mono, ori, claimed):
    last, cur, Tcw, Tlw, cam, bounds, sf = scenario(oracle, synth, seed, n_claimed=claimed, stereo=not mono, f0=seed)
    n_o, a_o = oracle.search_by_projection_frame(last, cur, Tcw, Tlw, cam, bounds, sf, th, mono, ori)
    mt = pkg.Matcher(max_features=2048, max_lines=64, max_nodes=3072)
    n_g, a_g = mt.search_by_projection_frame(last, cur, Tcw, Tlw, cam, bounds, sf, th, mono, ori)
    assert n_g == n_o and np.array_equal(a_g, a_o), (seed, n_g, n_o, int((a_g != a_o).sum()))
    assert n_o > 50 or th < 10


def test_projection_edge_cases(pkg, oracle, synth):
    last, cur, Tcw, Tlw, cam, bounds, sf = scenario(oracle, synth, 9)
    mt = pkg.Matcher(max_features=2048, max_lines=64, max_nodes=3072)
    # nothing valid / everything claimed / observations all zero (later points may overwrite earlier ones: counted twice, as the reference does)
    for mod in ("novalid", "allclaimed", "noobs"):
        l2, c2 = dict(last), dict(cur)
        if mod == "novalid": l2["valid"] = np.zeros_like(last["valid"])
        if mod == "allclaimed": c2["claimed"] = np.ones(len(cur["x"]), np.uint8)
        if mod == "noobs": l2["obs"] = np.zeros_like(last["obs"]); l2["valid"] = np.ones_like(last["valid"])
        n_o, a_o = oracle.search_by_projection_frame(l2, c2, Tcw, Tlw, cam, bounds, sf, 20.0, True, True)
        n_g, a_g = mt.search_by_projection_frame(l2, c2, Tcw, Tlw, cam, bounds, sf, 20.0, True, True)
        assert n_g == n_o and np.array_equal(a_g, a_o), mod
    with pytest.raises(pkg.SslplError):                                         # needs the 3072-cell grid
        pkg.Matcher(max_features=2048, max_nodes=100).search_by_projection_frame(last, cur, Tcw, Tlw, cam, bounds, sf, 15.0)
    # degenerate image bounds (zero width, negative height) would give an infinite or negative grid cell: rejected before any launch
    z32 = np.zeros((1, 32), np.uint8)
    mp = dict(inview=[1], bad=[0], obs=[0], projx=[100.], projy=[100.], level=[0], viewcos=[1.], desc=z32)
    one = dict(desc=z32, x=[100.], y=[100.], oct=[0], octave=[0], angle=[0.])
    for bad in ((640., 640., 0., 480.), (0., 640., 480., 0.)):
        for call in (lambda: mt.search_by_projection_frame(last, cur, Tcw, Tlw, cam, bad, sf, 15.0),
                     lambda: mt.search_by_projection_mps(mp, one, bad, sf),
                     lambda: mt.search_for_initialization(z32, one, z32, one, [[100., 100.]], bad)):
            before = mt.launch_count
            with pytest.raises(pkg.SslplError):
                call()
            assert mt.launch_count == before, bad


@pytest.mark.parametrize("seed,th,ratio", [(1, 1.0, 0.8), (2, 3.0, 0.8), (3, 1.0, 0.6), (4, 5.0, 0.9)])
def test_search_by_projection_map_points(pkg, oracle, synth, seed, th, ratio):
    """ORBmatcher::SearchByProjection(Frame&, const vector<MapPoint*>&, th) (ORBmatcher.cc:45-129) — the oracle of this matcher is
    pinned to the reference itself in tests/test_ref_parity_cpu.py."""
    from scenarios import local_map_scenario
    mp, cur, bounds, sf = local_map_scenario(oracle, synth, seed, f0=seed)
    mt = pkg.Matcher(max_features=2048, max_lines=64, max_nodes=3072)
    n_o, a_o = oracle.search_by_projection_mps(mp, cur, bounds, sf, ratio, th)
    n_g, a_g = mt.search_by_projection_mps(mp, cur, bounds, sf, ratio, th)
    assert n_g == n_o and np.array_equal(a_g, a_o), (n_g, n_o, int((a_g != a_o).sum()))
    for mod in ("none_in_view", "all_held", "no_obs"):
        m2, c2 = dict(mp), dict(cur)
        if mod == "none_in_view": m2["inview"] = np.zeros_like(mp["inview"])
        if mod == "all_held": c2["held"] = np.ones(len(cur["x"]), np.uint8)
        if mod == "no_obs": m2["obs"] = np.zeros_like(mp["obs"])
        n_o, a_o = oracle.search_by_projection_mps(m2, c2, bounds, sf, ratio, th)
        n_g, a_g = mt.search_by_projection_mps(m2, c2, bounds, sf, ratio, th)
        assert n_g == n_o and np.array_equal(a_g, a_o), mod


@pytest.mark.parametrize("f0,window,ratio,ori,nf", [(0, 100, 0.9, True, 2000), (8, 50, 0.9, True, 1000), (16, 100, 0.7, False, 2000), (3, 10, 0.9, True, 1000)])
def test_search_for_initialization(pkg, oracle, synth, f0, window, ratio, ori, nf):
    """ORBmatcher::SearchForInitialization (ORBmatcher.cc:408-523)."""
    orc = oracle.OrbOracle(nf, 1.2, 8, 20, 7)
    k1, d1 = orc.extract(synth.frame(640, 480, f0)); k2, d2 = orc.extract(synth.frame(640, 480, f0 + 2))
    prev = np.stack([k1["x"], k1["y"]], 1)
    bounds = (0.0, 640.0, 0.0, 480.0)
    mt = pkg.Matcher(max_features=4096, max_lines=64, max_nodes=3072)
    n_o, m_o, p_o = oracle.search_for_initialization(d1, k1, d2, k2, prev, bounds, ratio, ori, window)
    n_g, m_g, p_g = mt.search_for_initialization(d1, k1, d2, k2, prev, bounds, ratio, ori, window)
    assert n_g == n_o and np.array_equal(m_g, m_o) and np.array_equal(p_g, p_o)
    n_o2, m_o2, _ = oracle.search_for_initialization(d1, k1, d2, k2, p_o, bounds, ratio, ori, window)
    n_g2, m_g2, _ = mt.search_for_initialization(d1, k1, d2, k2, p_g, bounds, ratio, ori, window)
    assert n_g2 == n_o2 and np.array_equal(m_g2, m_o2)
