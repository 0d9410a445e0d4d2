"""GPU parity of the relocalisation matchers (include/sslpl.h): SearchByProjection(Frame &F, KeyFrame *pKF, sAlreadyFound, th, ORBdist)
single and batched over (keyframe row, frame row) pairs in HBM, and the candidate table as a pair list, against tests/reloc_model.py bit
for bit.  tests/test_reloc_match_cpu.py holds that model to the reference's own matcher."""
import numpy as np
import pytest

import reloc_model as rm

pytestmark = pytest.mark.gpu
f32 = np.float32
SETTINGS = [(10, 100), (3, 64)]                          # Tracking.cc:2071, :2085


@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


@pytest.fixture(scope="module")
def mt(pkg):
    return pkg.Matcher(max_features=1100, max_lines=64, max_nodes=1024, max_batch=576)


@pytest.fixture(scope="module")
def scenes(oracle, synth):
    return [rm.reloc_scene(oracle, synth, s, f0=2 * s) for s in range(4)] + [rm.reloc_scene(oracle, synth, 11, identity=True)]


def single_args(S):
    e = np.maximum(S["kfmp"], 0)
    el = rm.element_table(S["Xw"], S["mindist"], S["maxdist"])
    flag = (S["kfmp"] >= 0) & (S["bad"][e] == 0) & (S["found_el"][e] == 0)
    kf = dict(flag=flag.astype(np.uint8), Xw=el[e, :3], dmp=S["eldesc"][e], dist3=el[e, 6:9], angle=S["kf_kps"]["angle"])
    k = S["kps"]
    cur = dict(desc=S["desc"], x=k["x"], y=k["y"], oct=k["octave"].astype(np.int32), angle=k["angle"], held=S["held"])
    return kf, cur


@pytest.mark.parametrize("th,orb_dist", SETTINGS)
@pytest.mark.parametrize("check_ori", [True, False])
def test_single_equals_model(oracle, mt, scenes, th, orb_dist, check_ori):
    for S in scenes:
        kf, cur = single_args(S)
        n_g, a_g = mt.search_by_projection_kf(kf, cur, S["Tcw"], rm.CAM, rm.BOUNDS, rm.SF, rm.LOG_SF, th, orb_dist, check_ori)
        n_m, a_m = rm.scene_model(oracle, S, th, orb_dist, check_ori)
        assert n_g == n_m and np.array_equal(a_g, a_m)


def _perturb(rng, T, k):
    if k == 0:
        return T.copy()
    R = rm._rot(rng.normal(0, 0.004, 3)).astype(f32)
    out = np.empty((3, 4), f32); out[:, :3] = (R @ T[:, :3]).astype(f32); out[:, 3] = T[:, 3] + rng.normal(0, 0.01, 3).astype(f32)
    return out


@pytest.mark.parametrize("th,orb_dist,check_ori,masks", [(10, 100, True, True), (3, 64, True, True), (10, 100, False, False)])
def test_batch_equals_model(torch, oracle, pkg, mt, scenes, th, orb_dist, check_ori, masks):
    """576 pairs at 1000 features: 4 scenes x 4 poses (plus the camera-plane scene) repeated, found and held masks per pair (or NULL
    masks), two pairs with a row outside the set, and pairs whose frame is their own keyframe row (the keyframe's keypoints with zero
    descriptors)."""
    rng = np.random.default_rng(7)
    cap = 1000 + 64
    R = rm.DeviceRows(torch, scenes, cap)
    combos, want = [], []
    for s, S in enumerate(scenes):
        for k in range(4 if s < 4 else 1):
            T = _perturb(rng, S["Tcw"], k)
            found = np.where(S["kfmp"] >= 0, S["found_el"][np.maximum(S["kfmp"], 0)], 0).astype(np.uint8)
            if k == 3:
                found = (rng.random(len(found)) < 0.3).astype(np.uint8)
            if not masks:
                found = np.zeros_like(found)
            el = rm.element_table(S["Xw"], S["mindist"], S["maxdist"])
            held = S["held"] if masks else None
            want.append(rm.search_by_projection_kf(oracle, S["kf_kps"], S["kfmp"], el, S["eldesc"], S["bad"], found, S["kps"], S["desc"],
                                                   held, T, rm.CAM, rm.BOUNDS, rm.SF, rm.LOG_SF, th, orb_dist, check_ori))
            combos.append((2 * s, 2 * s + 1, T, found, held))
    S = scenes[0]                                                   # a keyframe row against itself
    el = rm.element_table(S["Xw"], S["mindist"], S["maxdist"])
    want.append(rm.search_by_projection_kf(oracle, S["kf_kps"], S["kfmp"], el, S["eldesc"], S["bad"], None, S["kf_kps"],
                                           np.zeros((len(S["kf_kps"]), 32), np.uint8), None, S["Tcw"], rm.CAM, rm.BOUNDS, rm.SF, rm.LOG_SF,
                                           th, orb_dist, check_ori))
    combos.append((0, 0, S["Tcw"], np.zeros(0, np.uint8), None))
    npairs = 576
    pair = np.zeros((npairs, 2), np.int32); Tcw = np.zeros((npairs, 12), f32)
    found = np.zeros((npairs, cap), np.uint8); held = np.zeros((npairs, cap), np.uint8)
    which = rng.integers(0, len(combos), npairs)
    which[7] = which[8] = len(combos) - 1
    for p, c in enumerate(which):
        kr, fr, T, fd, hd = combos[c]
        pair[p] = (kr, fr); Tcw[p] = T.reshape(-1); found[p, :len(fd)] = fd
        if hd is not None:
            held[p, :len(hd)] = hd
    pair[5] = (R.nrows, 1); pair[6] = (0, -1)                      # rows outside the set
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d_pair, d_T, d_found, d_held = dev(pair), dev(Tcw), dev(found), dev(held)
    p_found, p_held = (d_found.data_ptr(), d_held.data_ptr()) if masks else (0, 0)
    d_assign = torch.full((npairs, cap), 7, dtype=torch.int32, device="cuda"); d_nm = torch.zeros(npairs, dtype=torch.int32, device="cuda")
    mt.search_by_projection_kf_batch_device(R.kps.data_ptr(), R.desc.data_ptr(), R.n.data_ptr(), R.nrows, cap, R.kfmp.data_ptr(),
                                            R.bad.data_ptr(), R.nel, R.el.data_ptr(), R.eldesc.data_ptr(), npairs, d_pair.data_ptr(),
                                            d_T.data_ptr(), p_found, p_held, rm.CAM, rm.BOUNDS, rm.SF, rm.LOG_SF, th,
                                            orb_dist, check_ori, d_assign.data_ptr(), d_nm.data_ptr())
    mt.sync()
    A = d_assign.cpu().numpy(); NM = d_nm.cpu().numpy()
    for p, c in enumerate(which):
        if p in (5, 6):
            assert NM[p] == -1 and (A[p] == -1).all()
            continue
        n_m, a_m = want[c]
        n2 = len(a_m)
        assert NM[p] == n_m, p
        assert np.array_equal(A[p, :n2], a_m), p
        assert (A[p, n2:] == -1).all()
    assert NM.max() > 10


def test_reloc_pairs(torch, mt):
    rng = np.random.default_rng(3)
    nq, ndb, kmax = 40, 30, 8
    cand = np.full((nq, ndb), -1, np.int32); ncand = rng.integers(0, 14, nq).astype(np.int32)
    ncand[0], ncand[1], ncand[2] = -1, 0, kmax
    for q in range(nq):
        if ncand[q] > 0:
            cand[q, :ncand[q]] = rng.permutation(500)[:ncand[q]]
    query = rng.integers(0, 1000, nq).astype(np.int32)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d_query, d_cand, d_ncand = dev(query), dev(cand), dev(ncand)
    d_pair = torch.full((nq * kmax, 2), 5, dtype=torch.int32, device="cuda")
    mt.reloc_pairs_batch_device(d_query.data_ptr(), d_cand.data_ptr(), d_ncand.data_ptr(), nq, ndb, kmax, d_pair.data_ptr())
    mt.sync()
    assert np.array_equal(d_pair.cpu().numpy(), rm.reloc_pairs(query, cand, ncand, kmax))
    assert (ncand > kmax).any()                                          # truncation
    # a count beyond the table's width (kmax > ndb) reads no further than the query's own row
    nd2 = 5
    cand2 = np.ascontiguousarray(cand[:, :nd2]); d_cand2 = dev(cand2)
    mt.reloc_pairs_batch_device(d_query.data_ptr(), d_cand2.data_ptr(), d_ncand.data_ptr(), nq, nd2, kmax, d_pair.data_ptr())
    mt.sync()
    assert np.array_equal(d_pair.cpu().numpy(), rm.reloc_pairs(query, cand2, ncand, kmax))


def test_bad_arguments(torch, pkg, mt, scenes):
    S = scenes[0]
    kf, cur = single_args(S)
    before = mt.launch_count
    for kw in (dict(orb_dist=256), dict(th=0.0), dict(bounds=(0.0, 0.0, 0.0, 480.0)), dict(scale_factors=np.zeros(0, f32))):
        a = dict(th=10, orb_dist=100, bounds=rm.BOUNDS, scale_factors=rm.SF); a.update(kw)
        with pytest.raises(pkg.SslplError):
            mt.search_by_projection_kf(kf, cur, S["Tcw"], rm.CAM, a["bounds"], a["scale_factors"], rm.LOG_SF, a["th"], a["orb_dist"])
    buf = torch.zeros(1 << 16, dtype=torch.int32, device="cuda")
    x = buf.data_ptr()
    args = lambda npairs=1, cap=64, nrows=2, orb=100: (x, x, x, nrows, cap, x, 0, 0, 0, 0, npairs, x, x, 0, 0, rm.CAM, rm.BOUNDS, rm.SF,
                                                      rm.LOG_SF, 10.0, orb, True, x, x)
    for kw in (dict(npairs=577), dict(npairs=0), dict(cap=1100 + 65), dict(nrows=0), dict(orb=256)):
        with pytest.raises(pkg.SslplError):
            mt.search_by_projection_kf_batch_device(*args(**kw))
    for bad in ((x, x, x, 73, 8, 8, x), (x, x, x, 0, 8, 8, x), (x, x, x, 4, 8, 0, x), (0, x, x, 4, 8, 8, x)):
        with pytest.raises(pkg.SslplError):
            mt.reloc_pairs_batch_device(*bad)
    assert mt.launch_count == before
