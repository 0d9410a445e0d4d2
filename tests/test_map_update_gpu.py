"""GPU parity of the batched, device-resident map-element refresh (include/sslpl_map.h): MapPoint::ComputeDistinctiveDescriptors /
UpdateNormalAndDepth and MapLine::ComputeDistinctiveDescriptors / UpdateAverageDir over keyframes the extractors left in HBM.  Every row,
descriptor and status is compared bit for bit with tests/map_update_model.py, with sentinels in every field a call may leave alone; the
device medoid with sslpl_descriptor_medoid_batch; and the chain CreateNewMapPoints -> refresh -> Fuse (phase A), all in HBM, with the
model chain create_points_model -> map_update_model -> the oracle's Fuse stages."""
import importlib

import numpy as np
import pytest

import fuse_model as fm
import map_update_model as mu
from test_kf_fuse_gpu import device_keyframes, matcher
from test_kf_triangulation_gpu import FLAT, keyframe_frames

pytestmark = pytest.mark.gpu
f32 = np.float32


@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


@pytest.fixture(scope="module")
def mapping(pkg):
    return importlib.import_module(pkg.__name__ + ".mapping")


def _patched(torch, K):
    """Keyframe 3's features 0..2 get the octaves -1, 8 and 99 (outside the pyramid), keylines 0..1 -1 and 8; uploaded copies."""
    kps = K["kps"].copy(); kps["octave"][3, :3] = (-1, 8, 99)
    kl = K["kl"].copy(); kl["octave"][3, :2] = (-1, 8)
    dk = torch.from_numpy(kps.view(np.uint8).reshape(len(kps), -1).copy()).cuda()
    dl = torch.from_numpy(kl.view(np.uint8).reshape(len(kl), -1).copy()).cuda()
    return dict(K, kps=kps, kl=kl, d_kps_t=dk, d_kl_t=dl)


@pytest.fixture(scope="module")
def small(pkg, synth, torch):
    K = device_keyframes(pkg, torch, keyframe_frames(synth))
    assert K["n"][FLAT] == 0 and K["nl"][FLAT] == 0
    return _patched(torch, K)


@pytest.fixture(scope="module")
def large(pkg, synth, torch):
    K = device_keyframes(pkg, torch, keyframe_frames(synth, W=1280, H=960, flat=None), nfeatures=4000, nlines=500)
    assert (K["n"] > 1000).all() and (K["nl"] > 100).all()
    return _patched(torch, K)


def _entries(rng, n, nel, all_kf=0):
    """One entry per element 0 .. nel - 10 (1 .. nkf observations, reference keyframe mostly one of them), then the special cases on the
    last 9 elements, out-of-range elements and a repeated element."""
    nkf = len(n)
    ok = [k for k in range(nkf) if n[k] > 0]
    E = []
    for e in range(nel - 9):
        ks = ok if e < all_kf else sorted(rng.choice(ok, min(int(rng.geometric(0.25)), len(ok)), replace=False).tolist())
        obs = [(int(k), int(rng.integers(0, n[k]))) for k in ks]
        r = rng.random()
        rk = int(rng.choice(ks)) if r < 0.85 else int(rng.choice(ok))
        E.append((e, rk, obs))
    s = nel - 9
    flat = [k for k in range(nkf) if n[k] == 0]
    E += [(s, 0, []),                                         # NO_OBS
          (s + 1, 0, [(0, 0), (0, 1)]),                       # a keyframe twice: BAD
          (s + 2, 0, [(0, 0), (nkf, 0)]),                     # keyframe out of range: BAD
          (s + 3, 0, [(0, int(n[0]))]),                       # feature out of range: BAD
          (s + 4, -1, [(1, 0)]),                              # reference keyframe out of range: BAD with GEOM
          (s + 5, 3, [(1, 5), (3, 0)]),                       # reference octave -1: REF_OCTAVE
          (s + 6, 3, [(0, 7)]),                               # refkf not in the list: its feature 0, octave -1
          (s + 7, 3, [(3, 2), (4, 1)]),                       # reference octave 99
          (s + 8, flat[0] if flat else 3, [(0, 3)] if flat else [(3, 1)]),   # refkf without features (BAD) / octave 8
          (nel, 0, [(0, 0)]), (-1, 0, [(0, 0)]), (5, 0, [(0, 0)])]          # element out of range twice, element 5 again
    return E


def _sources(E, nel, n):
    """The feature each element's position is made from: its first observation, (0, 0) when that one is not a feature."""
    first = [o[0] if o else (0, 0) for _, _, o in E[:nel]]
    return [(k, i) if 0 <= k < len(n) and 0 <= i < n[k] else (0, 0) for k, i in first]


def _point_case(K, seed, all_kf=0):
    rng = np.random.default_rng(seed)
    nkf = len(K["n"])
    E = _entries(rng, K["n"], min(int(K["n"].sum()) // 8, 6000), all_kf)
    nel = E[-3][0]
    src = _sources(E, nel, K["n"])
    mp = fm.point_table(rng, src, K["kps"], K["desc"], K["pose"], nkf, K["W"], K["H"], p_gate=0)["mp"]
    mp[:, 3:] = rng.standard_normal((nel, 6)).astype(f32)                 # sentinels
    mpdesc = rng.integers(0, 256, (nel, 32), dtype=np.uint8)
    bad = (rng.random(nkf) < 0.25).astype(np.uint8)
    return E, mp, mpdesc, bad


def _line_case(K, seed, all_kf=0):
    rng = np.random.default_rng(seed)
    nkf = len(K["nl"])
    E = _entries(rng, K["nl"], max(int(K["nl"].sum()) // 4, 40), all_kf)
    nel = E[-3][0]
    src = _sources(E, nel, K["nl"])
    ml = fm.line_table(rng, src, K["kl"], K["ldesc"], K["pose"], nkf, K["W"], K["H"], p_gate=0)["ml"]
    pos = ml[:, :6].astype(np.float64) * (1 + rng.uniform(-1e-6, 1e-6, (nel, 6)))
    ml[:, :6] = pos; ml[:, 6:] = rng.standard_normal((nel, 6)).astype(f32)
    mldesc = rng.integers(0, 256, (nel, 32), dtype=np.uint8)
    bad = (rng.random(nkf) < 0.25).astype(np.uint8)
    return E, pos, ml, mldesc, bad


def _dev(torch, a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


def _csr(torch, E):
    return [_dev(torch, a, np.int32) for a in mu.csr(E)]


def run_points(mapping, mt, torch, K, E, mp, mpdesc, bad, what, sf=fm.SF):
    d_mp, d_md, d_bad = _dev(torch, mp, f32), _dev(torch, mpdesc, np.uint8), _dev(torch, bad, np.uint8)
    elem, refkf, off, obs = _csr(torch, E)
    st = torch.full((len(E),), 77, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()                                              # the matcher runs on its own stream
    mapping.update_map_points(mt, K["d_kps_t"].data_ptr(), K["d_desc"], K["d_n"], len(K["n"]), K["cap"], K["d_pose"].data_ptr(), d_bad.data_ptr(),
                              len(mp), d_mp.data_ptr(), d_md.data_ptr(), len(E), elem.data_ptr(), refkf.data_ptr(), off.data_ptr(), obs.data_ptr(),
                              sf, what, st.data_ptr())
    mt.sync()
    return d_mp.cpu().numpy(), d_md.cpu().numpy(), st.cpu().numpy()


def run_lines(mapping, mt, torch, K, E, pos, ml, mldesc, bad, what, normal=True, sf=fm.SF):
    d_pos, d_ml, d_md, d_bad = _dev(torch, pos, np.float64), _dev(torch, ml, f32), _dev(torch, mldesc, np.uint8), _dev(torch, bad, np.uint8)
    d_nrm = torch.full((len(ml), 3), 7.5, dtype=torch.float64, device="cuda") if normal else None
    elem, refkf, off, obs = _csr(torch, E)
    st = torch.full((len(E),), 77, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    mapping.update_map_lines(mt, K["d_kl_t"].data_ptr(), K["d_ldesc"], K["d_nl"], len(K["nl"]), K["capl"], K["d_pose"].data_ptr(), d_bad.data_ptr(),
                             len(ml), d_pos.data_ptr(), d_ml.data_ptr(), d_md.data_ptr(), d_nrm.data_ptr() if normal else 0, len(E), elem.data_ptr(),
                             refkf.data_ptr(), off.data_ptr(), obs.data_ptr(), sf, what, st.data_ptr())
    mt.sync()
    return d_ml.cpu().numpy(), d_md.cpu().numpy(), (d_nrm.cpu().numpy() if normal else None), st.cpu().numpy()


def _same(a, b):
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def check_points(mapping, mt, torch, K, E, mp, mpdesc, bad, what):
    got = run_points(mapping, mt, torch, K, E, mp, mpdesc, bad, what)
    exp = mu.update_points(K["kps"], K["desc"], K["n"], K["pose"], bad, mp, mpdesc, E, fm.SF, what)
    assert np.array_equal(got[2], exp[2]), np.nonzero(got[2] != exp[2])[0][:8]
    rows = np.nonzero(~(got[0].view(np.uint32) == exp[0].view(np.uint32)).all(1))[0]
    assert len(rows) == 0, (what, rows[:5], got[0][rows[:2]], exp[0][rows[:2]])
    assert _same(got[1], exp[1]), what
    return exp


def check_lines(mapping, mt, torch, K, E, pos, ml, mldesc, bad, what, normal=True):
    got = run_lines(mapping, mt, torch, K, E, pos, ml, mldesc, bad, what, normal)
    nrm = np.full((len(ml), 3), 7.5) if normal else None
    exp = mu.update_lines(K["kl"], K["ldesc"], K["nl"], K["pose"], bad, pos, ml, mldesc, nrm, E, fm.SF, what)
    assert np.array_equal(got[3], exp[3]), np.nonzero(got[3] != exp[3])[0][:8]
    rows = np.nonzero(~(got[0].view(np.uint32) == exp[0].view(np.uint32)).all(1))[0]
    assert len(rows) == 0, (what, rows[:5], got[0][rows[:2]], exp[0][rows[:2]])
    assert _same(got[1], exp[1]), what
    if normal:
        assert _same(got[2], exp[2]), what
    return exp


def _reached(st):
    return {mu.OK, mu.NO_OBS, mu.NO_GOOD_KF, mu.REF_OCTAVE, mu.BAD} <= set(st.tolist())


@pytest.mark.parametrize("what", [mu.DESC, mu.GEOM, mu.DESC | mu.GEOM])
def test_points_equal_model(pkg, mapping, torch, small, what):
    mt = matcher(pkg, small)
    E, mp, mpdesc, bad = _point_case(small, 1)
    _, _, st = check_points(mapping, mt, torch, small, E, mp, mpdesc, bad, what)
    if what == mu.DESC | mu.GEOM:
        assert _reached(st)
    assert (st[-3:] == mu.BAD).all() and st[-9 - 3] == mu.NO_OBS


@pytest.mark.parametrize("what", [mu.DESC, mu.GEOM, mu.DESC | mu.GEOM])
def test_lines_equal_model(pkg, mapping, torch, small, what):
    mt = matcher(pkg, small)
    E, pos, ml, mldesc, bad = _line_case(small, 2)
    st = check_lines(mapping, mt, torch, small, E, pos, ml, mldesc, bad, what)[3]
    if what == mu.DESC | mu.GEOM:
        assert _reached(st)
    check_lines(mapping, mt, torch, small, E, pos, ml, mldesc, bad, what, normal=False)


def test_large_frames_all_keyframes(pkg, mapping, torch, large):
    """1280x960, 4000 features and 500 lines per keyframe; the first elements are observed by all 21 keyframes."""
    mt = matcher(pkg, large)
    E, mp, mpdesc, bad = _point_case(large, 3, all_kf=40)
    assert len(E[0][2]) == len(large["n"]) == 21
    assert _reached(check_points(mapping, mt, torch, large, E, mp, mpdesc, bad, mu.DESC | mu.GEOM)[2])
    E, pos, ml, mldesc, bad = _line_case(large, 4, all_kf=40)
    assert _reached(check_lines(mapping, mt, torch, large, E, pos, ml, mldesc, bad, mu.DESC | mu.GEOM)[3])


def test_medoid_equals_descriptor_medoid_batch(pkg, mapping, torch, large):
    mt = matcher(pkg, large)
    E, mp, mpdesc, bad = _point_case(large, 5, all_kf=40)
    _, md, st = run_points(mapping, mt, torch, large, E, mp, mpdesc, bad, mu.DESC)
    sel = [u for u, s in enumerate(st) if s == mu.OK]
    groups = [np.array([large["desc"][k, i] for k, i in E[u][2] if not bad[k]], np.uint8) for u in sel]
    off = np.concatenate([[0], np.cumsum([len(g) for g in groups])]).astype(np.int32)
    bi, _ = mt.descriptor_medoid(np.concatenate(groups), off)
    assert len(sel) > 1000
    assert all(np.array_equal(md[E[u][0]], groups[j][bi[j]]) for j, u in enumerate(sel))


def test_replace_flow_desc_refresh(pkg, mapping, torch, small):
    """The elements fuse_model.MapModel.replace recomputed: a DESC-only refresh of their observations equals MapModel.compute_desc."""
    K = small
    rng = np.random.default_rng(6)
    n = [int(c) for c in K["n"]]
    kf_desc = [K["desc"][k] for k in range(len(n))]
    M, _ = fm.replay_map(rng, kf_desc, n, [k for k in range(len(n)) if n[k] > 0], p_own=0.2, p_extra=0.6)
    nel = len(M.obs)
    for _ in range(200):
        a, b = (int(x) for x in rng.integers(0, nel, 2))
        if not M.bad[a] and not M.bad[b]:
            M.replace(a, b)
    touched = [e for e in range(nel) if not M.bad[e] and M.ver[e] > 1]
    assert len(touched) > 50
    E = [(e, 0, sorted(M.obs[e].items())) for e in touched]
    mt = matcher(pkg, K)
    start = rng.integers(0, 256, (nel, 32), dtype=np.uint8)
    _, md, st = run_points(mapping, mt, torch, K, E, np.zeros((nel, 9), f32), start, np.zeros(len(n), np.uint8), mu.DESC)
    assert (st == mu.OK).all()
    assert all(np.array_equal(md[e], M.desc[e]) for e in touched)
    others = np.setdiff1d(np.arange(nel), touched)
    assert np.array_equal(md[others], start[others])


def test_argument_errors(pkg, mapping, torch, small):
    K = small
    mt = matcher(pkg, K)
    E, mp, mpdesc, bad = _point_case(K, 1)
    before = mt.launch_count
    for kw in (dict(what=0), dict(what=4), dict(sf=np.ones(17, f32)), dict(sf=np.zeros(0, f32))):
        with pytest.raises(pkg.SslplError):
            run_points(mapping, mt, torch, K, E, mp, mpdesc, bad, kw.get("what", 3), kw.get("sf", fm.SF))
    got = run_points(mapping, mt, torch, K, [], mp, mpdesc, bad, 3)
    assert mt.launch_count == before and _same(got[0], mp) and _same(got[1], mpdesc)
    # d_obs is read as int2 pairs: an observation list 4 bytes into an int32 buffer is refused before anything is enqueued
    elem, refkf, off, obs = _csr(torch, E)
    shifted = torch.zeros(obs.numel() + 1, dtype=torch.int32, device="cuda"); shifted[1:] = obs.reshape(-1)
    d_mp, d_md, st = _dev(torch, mp, f32), _dev(torch, mpdesc, np.uint8), torch.zeros(len(E), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    with pytest.raises(pkg.SslplError, match="aligned"):
        mapping.update_map_points(mt, K["d_kps_t"].data_ptr(), K["d_desc"], K["d_n"], len(K["n"]), K["cap"], K["d_pose"].data_ptr(), 0, len(mp),
                                  d_mp.data_ptr(), d_md.data_ptr(), len(E), elem.data_ptr(), refkf.data_ptr(), off.data_ptr(),
                                  shifted.data_ptr() + 4, fm.SF, 3, st.data_ptr())
    assert mt.launch_count == before


# ---------------------------------------------------------------------------------------------------------------- the chain
def test_chain_create_refresh_fuse(pkg, oracle, mapping, torch):
    """CreateNewMapPoints over KF 0's 20 neighbours, the refresh of every created MapPoint (observations (kf1, idx1), (kf2, idx2),
    reference keyframe kf1, CSR built on the device from the call's rows and statuses) and phase A of Fuse (every created MapPoint into
    every neighbour), with nothing downloaded in between, equal the model chain."""
    import test_kf_create_points_gpu as cp
    K = cp.upload(pkg, torch, cp.scene(pkg, oracle))
    pairs = cp.neighbour_pairs(); geom = cp.geometry(K, pairs)
    mt = cp.matcher(pkg, K)
    stream = torch.cuda.Stream()                                          # the matcher and the torch steps in between share it
    torch.cuda.synchronize()
    mt.set_stream(stream.cuda_stream)
    with torch.cuda.stream(stream):
        P, cap = len(pairs), K["cap"]
        d_pair = torch.tensor(np.array(pairs, np.int32), device="cuda"); d_geom = torch.from_numpy(geom).cuda()
        rows = torch.empty((P, cap, 2), dtype=torch.int32, device="cuda"); cnt = torch.empty(P, dtype=torch.int32, device="cuda")
        status = torch.empty((P, cap), dtype=torch.int32, device="cuda"); x3d = torch.zeros((P, cap, 3), dtype=torch.float32, device="cuda")
        nnew = torch.empty(P, dtype=torch.int32, device="cuda")
        mt.create_new_map_points_batch_device(K["d_kps_t"].data_ptr(), K["d_desc_t"].data_ptr(), K["d_n_t"].data_ptr(), len(K["n"]), cap,
                                              K["d_has_mp_t"].data_ptr(), K["voc"], cp.LEVELSUP, P, d_pair.data_ptr(), d_geom.data_ptr(),
                                              K["d_pose_t"].data_ptr(), K["cam"], K["scale"], K["sigma2"], K["scale_factor"], rows.data_ptr(),
                                              cnt.data_ptr(), status.data_ptr(), x3d.data_ptr(), nnew.data_ptr())
        # the created rows in (pair, row) order, on the device
        sel = (status == 0).nonzero()
        p, r = sel[:, 0], sel[:, 1]
        kf1, kf2 = d_pair[p, 0], d_pair[p, 1]
        i1, i2 = rows[p, r, 0], rows[p, r, 1]
        lo = kf1 < kf2
        obs = torch.stack([torch.stack([torch.where(lo, kf1, kf2), torch.where(lo, i1, i2)], 1),
                           torch.stack([torch.where(lo, kf2, kf1), torch.where(lo, i2, i1)], 1)], 1).reshape(-1, 2).contiguous()
        nel = len(sel)
        off = torch.arange(0, 2 * nel + 1, 2, dtype=torch.int32, device="cuda")
        elem = torch.arange(nel, dtype=torch.int32, device="cuda"); refkf = kf1.contiguous()
        d_mp = torch.zeros((nel, 9), dtype=torch.float32, device="cuda"); d_mp[:, :3] = x3d[p, r]
        d_md = torch.zeros((nel, 32), dtype=torch.uint8, device="cuda")
        st = torch.empty(nel, dtype=torch.int32, device="cuda")
        mapping.update_map_points(mt, K["d_kps_t"].data_ptr(), K["d_desc_t"].data_ptr(), K["d_n_t"].data_ptr(), len(K["n"]), cap, K["d_pose_t"].data_ptr(),
                                  0, nel, d_mp.data_ptr(), d_md.data_ptr(), nel, elem.data_ptr(), refkf.data_ptr(), off.data_ptr(), obs.data_ptr(),
                                  fm.SF, mu.DESC | mu.GEOM, st.data_ptr())
        # phase A: every created MapPoint into every neighbour; skip = IsInKeyFrame
        tg = torch.arange(1, len(pairs) + 1, dtype=torch.int32, device="cuda")
        ent = torch.stack([tg[:, None].expand(-1, nel), elem[None].expand(len(tg), -1)], 2).reshape(-1, 2).contiguous()
        skip = ((ent[:, 0] == kf1[ent[:, 1].long()]) | (ent[:, 0] == kf2[ent[:, 1].long()])).to(torch.uint8)
        bi = torch.empty(len(ent), dtype=torch.int32, device="cuda"); bd = torch.empty(len(ent), dtype=torch.int32, device="cuda")
        cam, bounds = K["cam"][:4], np.array([0, 640, 0, 480], f32)
        mt.fuse_points_batch_device(K["d_kps_t"].data_ptr(), K["d_desc_t"].data_ptr(), K["d_n_t"].data_ptr(), len(K["n"]), cap, K["d_pose_t"].data_ptr(),
                                    nel, d_mp.data_ptr(), d_md.data_ptr(), len(ent), ent.data_ptr(), skip.data_ptr(), cam, bounds, fm.SF, fm.INV_SIGMA2,
                                    fm.LOGS, fm.TH, bi.data_ptr(), bd.data_ptr())
        mt.sync()
    mt.set_stream(0)
    # the model chain
    exp = cp.oracle_chain(oracle, K, pairs, geom)
    E = []
    for (a, b), x in zip(pairs, exp):
        for row, s, X in zip(x["rows"], x["status"], x["x3d"]):
            if s == 0:
                E.append((len(E), a, sorted([(a, int(row[0])), (b, int(row[1]))])))
    assert len(E) == nel > 500
    X = np.concatenate([x["x3d"][x["status"] == 0] for x in exp]).astype(f32)
    mp0 = np.zeros((nel, 9), f32); mp0[:, :3] = X
    mp, md, mst = mu.update_points(K["kps"], K["desc"], K["n"], K["pose"], None, mp0, np.zeros((nel, 32), np.uint8), E, fm.SF, mu.DESC | mu.GEOM)
    assert (mst == mu.OK).all() and (st.cpu().numpy() == mst).all()
    assert _same(d_mp.cpu().numpy(), mp) and _same(d_md.cpu().numpy(), md)
    ent_h = ent.cpu().numpy(); skip_h = skip.cpu().numpy()
    Kf = dict(kps=K["kps"], desc=K["desc"], n=K["n"], cam=cam, bounds=bounds)
    ebi, ebd, _ = fm.oracle_points(oracle, Kf, K["pose"], mp, md, ent_h, skip_h)
    assert np.array_equal(bi.cpu().numpy(), ebi) and np.array_equal(bd.cpu().numpy(), ebd)
    assert ((ebd <= fm.TH_LOW) & (ebi >= 0)).sum() > 100
