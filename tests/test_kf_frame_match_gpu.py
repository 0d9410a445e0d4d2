"""GPU parity of the batched keyframe-to-frame matchers over (keyframe row, frame row) pairs in HBM: sslpl_search_by_bow_batch_device
(ORBmatcher::SearchByBoW(KeyFrame*, Frame&), ORBmatcher.cc:159-291) and sslpl_match_lines_kf_batch_device
(LSDmatcher::SearchByProjection(KeyFrame*, Frame&), LSDmatcher.cpp:143-183), pair by pair against tests/kf_frame_match_model.py (held to
the reference in tests/test_kf_frame_match_cpu.py), against the single-pair entry points, and, where oracle/_ref/libref.so is present,
against the reference directly.  All results are integer tables: every comparison is exact."""
import os

import numpy as np
import pytest

import kf_frame_match_model as km
from test_kf_triangulation_gpu import device_lines
from test_motion_batch_gpu import device_batch

pytestmark = pytest.mark.gpu
FLAT = 5                       # a flat grey frame: no keypoints, no lines


@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


def dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def row_set(pkg, torch, frames, nfeatures, nlines=40, seed=0, nmp=3000, nml=200):
    """Host row set (tests/kf_frame_match_model.py's layout) of the device extractors' results, with element maps drawn from shared pools,
    8 % of the MapPoints bad."""
    B, H, W = frames.shape
    D = device_batch(pkg, torch, frames, nfeatures)
    L = device_lines(pkg, torch, D["dfr"], B, W, H, nlines)
    rng = np.random.default_rng(seed)
    R = dict(kps=D["kps"].copy(), desc=D["desc"].copy(), n=D["n"].copy(), ldesc=L["ldesc"].copy(), nl=L["nl"].copy(), nmp=nmp, nml=nml)
    R["kfmp"] = km.element_maps(rng, R["n"], D["cap"], nmp)
    R["bad"] = (rng.random(nmp) < 0.08).astype(np.uint8)
    R["kfml"] = km.element_maps(rng, R["nl"], L["capl"], nml, p_null=0.3, twice=False)
    return R


def with_fv(oracle, R, va):
    cap = R["desc"].shape[1]
    cache = {}
    R["fv"] = lambda r: cache.setdefault(r, km.feature_vector(oracle, va, R["desc"][r, :km.clamp(R["n"][r], cap)]))
    return R


def upload(torch, R):
    return dict(kps=dev(torch, R["kps"].view(np.uint8)), desc=dev(torch, R["desc"]), n=dev(torch, R["n"]), kfmp=dev(torch, R["kfmp"]),
                bad=dev(torch, R["bad"]), ldesc=dev(torch, R["ldesc"]), nl=dev(torch, R["nl"]), kfml=dev(torch, R["kfml"]))


def vocabulary(pkg):
    va = km.vocabulary_arrays(pkg)
    return va, pkg.Vocabulary(km.VOCAB["k"], km.VOCAB["L"], *va)


def run_points(mt, torch, R, U, voc, pairs, nnratio, check_ori, bad=True):
    P, cap = len(pairs), R["desc"].shape[1]
    d_pair = dev(torch, np.array(pairs, np.int32).reshape(-1, 2))
    d_match = torch.full((P, cap), 7, dtype=torch.int32, device="cuda"); d_nm = torch.full((P,), -7, dtype=torch.int32, device="cuda")
    mt.search_by_bow_batch_device(U["kps"].data_ptr(), U["desc"].data_ptr(), U["n"].data_ptr(), len(R["n"]), cap, U["kfmp"].data_ptr(),
                                  U["bad"].data_ptr() if bad else 0, R["nmp"], voc, km.LEVELSUP, P, d_pair.data_ptr(), nnratio, check_ori,
                                  d_match.data_ptr(), d_nm.data_ptr())
    mt.sync()
    return d_match.cpu().numpy(), d_nm.cpu().numpy()


def run_lines(mt, torch, R, U, pairs, d_nl=None, d_kfml=None):
    P, capl = len(pairs), R["ldesc"].shape[1]
    d_pair = dev(torch, np.array(pairs, np.int32).reshape(-1, 2))
    d_lm = torch.full((P, capl), 7, dtype=torch.int32, device="cuda"); d_nm = torch.full((P,), -7, dtype=torch.int32, device="cuda")
    mt.match_lines_kf_batch_device(U["ldesc"].data_ptr(), (d_nl if d_nl is not None else U["nl"]).data_ptr(), len(R["nl"]), capl,
                                   (d_kfml if d_kfml is not None else U["kfml"]).data_ptr(), R["nml"], P, d_pair.data_ptr(), d_lm.data_ptr(),
                                   d_nm.data_ptr())
    mt.sync()
    return d_lm.cpu().numpy(), d_nm.cpu().numpy()


def check_points(oracle, R, pairs, got, nm, nnratio, check_ori):
    for p, pr in enumerate(pairs):
        n, want = km.search_by_bow(oracle, R, R["fv"], pr, nnratio, check_ori)
        assert nm[p] == n, (p, pr, int(nm[p]), n)
        assert np.array_equal(got[p], want), (p, pr)


def check_lines(oracle, R, pairs, got, nm):
    for p, pr in enumerate(pairs):
        n, want = km.line_match(oracle, R, pr)
        assert nm[p] == n, (p, pr, int(nm[p]), n)
        assert np.array_equal(got[p], want), (p, pr)


@pytest.fixture(scope="module")
def scene(pkg, oracle, synth, torch):
    """16 rows of 640x480 frames at 1000 features / 40 lines (two scenes of 8, row FLAT flat).  Row 9 has a count above cap (its rows
    past the extractor's count are copies of row 0's, so every feature read is a real one)."""
    frames = synth.batch(640, 480, 16, group=8)
    frames[FLAT] = 128
    R = row_set(pkg, torch, frames, 1000)
    cap = R["desc"].shape[1]
    k = int(R["n"][9])
    R["kps"][9, k:] = R["kps"][0, :cap - k]; R["desc"][9, k:] = R["desc"][0, :cap - k]
    R["n"][9] = cap + 100
    va, voc = vocabulary(pkg)
    with_fv(oracle, R, va)
    assert R["n"][FLAT] == 0 and R["nl"][FLAT] == 0 and (np.delete(R["n"], FLAT) > 500).all()
    return R, upload(torch, R), voc


def matcher(pkg, R, voc, max_batch):
    return pkg.Matcher(max_features=R["desc"].shape[1], max_lines=R["ldesc"].shape[1], max_nodes=voc.level_nodes(km.LEVELSUP),
                       max_batch=max_batch)


def point_pairs(rng, nrows, npairs):
    """npairs pairs: keyframe row 2 in many pairs, frame row 11 in many pairs, a row against itself, FLAT in both roles, row 9 (count above
    cap) in both roles, and rows outside the set, the (-1, -1) slots of the reloc pair list among them."""
    pairs = [tuple(int(x) for x in rng.integers(0, nrows, 2)) for _ in range(npairs)]
    fixed = [(2, 11), (2, 3), (2, 12), (7, 11), (0, 11), (4, 4), (FLAT, 1), (1, FLAT), (9, 10), (10, 9), (-1, -1), (-1, -1), (nrows, 0),
             (0, -3), (2, 1), (13, 11)]
    pairs[:len(fixed)] = fixed
    return pairs


@pytest.mark.parametrize("nnratio,check_ori,bad", [(0.75, True, True), (0.9, True, True), (0.75, False, True), (0.9, True, False)])
def test_points_equal_model(pkg, oracle, torch, scene, nnratio, check_ori, bad):
    R, U, voc = scene
    mt = matcher(pkg, R, voc, 64)
    pairs = point_pairs(np.random.default_rng(1), len(R["n"]), 64)
    got, nm = run_points(mt, torch, R, U, voc, pairs, nnratio, check_ori, bad)
    Rm = R if bad else dict(R, bad=None)
    check_points(oracle, Rm, pairs, got, nm, nnratio, check_ori)
    assert (nm[10:14] == -1).all() and nm[6] == 0 and nm[7] == 0 and nm.max() > 50


def test_points_4000_features(pkg, oracle, synth, torch):
    frames = synth.batch(1280, 960, 6, group=6)
    R = row_set(pkg, torch, frames, 4000, nlines=100, seed=3, nmp=12000)
    va, voc = vocabulary(pkg)
    with_fv(oracle, R, va)
    U = upload(torch, R)
    mt = matcher(pkg, R, voc, 16)
    pairs = [(0, 5), (1, 5), (2, 5), (3, 5), (4, 5), (0, 1), (5, 0), (3, 3), (-1, -1), (0, 2), (4, 2), (1, 5)]
    for check_ori in (True, False):
        got, nm = run_points(mt, torch, R, U, voc, pairs, 0.75, check_ori)
        check_points(oracle, R, pairs, got, nm, 0.75, check_ori)
        assert nm.max() > 200
    lg, lnm = run_lines(mt, torch, R, U, pairs)
    check_lines(oracle, R, pairs, lg, lnm)


@pytest.mark.parametrize("check_ori", [True, False])
def test_points_equal_single_pair(pkg, torch, scene, check_ori):
    """Every pair equals sslpl_search_by_bow on the same handle, and where the reference library is present a subset equals the reference."""
    R, U, voc = scene
    mt = matcher(pkg, R, voc, 64)
    pairs = [p for p in point_pairs(np.random.default_rng(2), len(R["n"]), 40) if min(p) >= 0 and max(p) < len(R["n"]) and 9 not in p]
    got, nm = run_points(mt, torch, R, U, voc, pairs, 0.75, check_ori)
    om = pkg.ORBmatcher(0.75, check_ori, mt)
    ref = None
    from oracle import ref as REF
    if os.path.exists(REF._LIB):
        ref = REF
    for p, (kr, fr) in enumerate(pairs):
        n1, n2 = int(R["n"][kr]), int(R["n"][fr])
        state = km.element_state(R["kfmp"][kr, :n1], R["nmp"], R["bad"])
        n, m = om.SearchByBoW(R["desc"][kr, :n1], R["fv"](kr), (state == 1).astype(np.uint8), R["kps"][kr, :n1]["angle"], R["desc"][fr, :n2],
                              R["fv"](fr), R["kps"][fr, :n2]["angle"])
        assert nm[p] == n and np.array_equal(got[p, :n2], m) and (got[p, n2:] == -1).all(), (p, kr, fr)
        if ref is not None and p < 8:
            n_r, m_r = ref.search_by_bow(R["desc"][kr, :n1], R["kps"][kr, :n1], R["desc"][fr, :n2], R["kps"][fr, :n2], R["fv"](kr),
                                         R["fv"](fr), state, 0.75, check_ori)
            assert nm[p] == n_r and np.array_equal(got[p, :n2], m_r), (p, kr, fr)


def test_lines_equal_model(pkg, oracle, torch, scene):
    """Frames with 0 and 1 lines, keyframes with 0 lines, two keyframe lines with the same best frame line (the last one wins and both
    count), all MapLines NULL, rows outside the set; and every defined pair equals sslpl_line_match(mode 0)."""
    R, U, voc = scene
    mt = matcher(pkg, R, voc, 64)
    R = dict(R, ldesc=R["ldesc"].copy(), nl=R["nl"].copy(), kfml=R["kfml"].copy())
    R["nl"][9] = 1                                                            # a frame with one line
    # keyframe row 2: its last line j a copy of the first accepted line i0 of the pair (2, 3), both with MapLines
    n0, m0 = km.line_match(oracle, R, (2, 3))
    i0, j = int(m0[m0 >= 0].min()), int(R["nl"][2]) - 1
    assert i0 < j
    R["ldesc"][2, j] = R["ldesc"][2, i0]; R["kfml"][2, [i0, j]] = (1, 2)
    U = dict(U, ldesc=dev(torch, R["ldesc"]), nl=dev(torch, R["nl"]), kfml=dev(torch, R["kfml"]))
    pairs = [(2, 3), (0, 1), (1, 0), (0, FLAT), (FLAT, 0), (FLAT, 9), (0, 9), (4, 4), (12, 13), (8, 15), (-1, -1), (0, len(R["nl"]))]
    pairs += [tuple(int(x) for x in r) for r in np.random.default_rng(4).integers(0, len(R["nl"]), (52, 2))]
    got, nm = run_lines(mt, torch, R, U, pairs)
    check_lines(oracle, R, pairs, got, nm)
    assert list(nm[3:7]) == [-1, 0, 0, -1] and nm[10] == nm[11] == -1
    assert j in got[0].tolist() and i0 not in got[0].tolist()                          # the last writer
    assert nm[0] > len(set(got[0][got[0] >= 0].tolist()))                              # the overwritten acceptance counts
    lm = pkg.LSDmatcher(mt)
    for p, (kr, fr) in enumerate(pairs):
        if min(kr, fr) < 0 or max(kr, fr) >= len(R["nl"]) or nm[p] == -1:
            continue
        n1, n2 = int(R["nl"][kr]), int(R["nl"][fr])
        has = (km.element_state(R["kfml"][kr, :n1], R["nml"]) != 0).astype(np.uint8)
        n, m = lm.SearchByProjection(R["ldesc"][kr, :n1], has, R["ldesc"][fr, :n2])
        assert nm[p] == n and np.array_equal(got[p, :n2], m), (p, kr, fr)
    # all MapLines NULL
    none = torch.full_like(U["kfml"], -1)
    got, nm2 = run_lines(mt, torch, R, U, pairs, d_kfml=none)
    assert (nm2[nm >= 0] == 0).all() and (nm2[nm < 0] == -1).all() and (got == -1).all()


def test_reloc_chain_in_hbm(pkg, oracle, torch):
    """BowVectors -> DetectRelocalizationCandidates -> the pair list -> SearchByBoW, all on the stream with nothing downloaded until the
    end: 64 frames against a database of 300 keyframes, up to 8 candidates each; equal to the model on the downloaded pair list."""
    from test_kfdb_gpu import rows
    rng = np.random.default_rng(11)
    ndb, nq, kmax, nfeat = 300, 64, 8, 1000
    cap = nfeat + 64
    nrows = ndb + nq
    desc, n, _ = rows(rng, nrows, nfeat, cap)
    n[ndb] = 0                                                      # a frame with no features: no candidate, its slots (-1, -1)
    kps = np.zeros((nrows, cap), pkg.KEYPOINT_DTYPE)
    kps["angle"] = rng.uniform(0, 360, (nrows, cap)).astype(np.float32)
    nmp = 20000
    R = dict(kps=kps, desc=desc, n=n, kfmp=km.element_maps(rng, n, cap, nmp), bad=(rng.random(nmp) < 0.08).astype(np.uint8), nmp=nmp)
    va, voc = vocabulary(pkg)
    with_fv(oracle, R, va)
    db = np.arange(ndb, dtype=np.int32); query = np.arange(ndb, nrows, dtype=np.int32)
    covis = np.full((nrows, 10), -1, np.int32)
    mt = pkg.Matcher(max_features=nfeat, max_lines=64, max_nodes=max(voc.level_nodes(km.LEVELSUP), 16), max_batch=nq * kmax)
    d_desc, d_n, d_kps, d_kfmp, d_bad = dev(torch, desc), dev(torch, n), dev(torch, kps.view(np.uint8)), dev(torch, R["kfmp"]), dev(torch, R["bad"])
    word = torch.empty((nrows, cap), dtype=torch.int32, device="cuda"); val = torch.empty((nrows, cap), dtype=torch.float64, device="cuda")
    bn = torch.empty(nrows, dtype=torch.int32, device="cuda")
    d_db, d_query, d_covis = dev(torch, db), dev(torch, query), dev(torch, covis)
    rs = torch.zeros(nrows, dtype=torch.float32, device="cuda")
    cand = torch.empty((nq, ndb), dtype=torch.int32, device="cuda"); ncand = torch.empty(nq, dtype=torch.int32, device="cuda")
    words = torch.empty((nq, ndb), dtype=torch.int32, device="cuda"); score = torch.empty((nq, ndb), dtype=torch.float32, device="cuda")
    d_pair = torch.empty((nq * kmax, 2), dtype=torch.int32, device="cuda")
    d_match = torch.empty((nq * kmax, cap), dtype=torch.int32, device="cuda"); d_nm = torch.empty(nq * kmax, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    mt.bow_vectors_batch_device(voc, d_desc.data_ptr(), d_n.data_ptr(), nrows, cap, word.data_ptr(), val.data_ptr(), bn.data_ptr())
    mt.detect_relocalization_candidates_batch_device(word.data_ptr(), val.data_ptr(), bn.data_ptr(), nrows, cap, d_db.data_ptr(), ndb,
                                                     d_query.data_ptr(), nq, d_covis.data_ptr(), rs.data_ptr(), cand.data_ptr(),
                                                     ncand.data_ptr(), words.data_ptr(), score.data_ptr())
    mt.reloc_pairs_batch_device(d_query.data_ptr(), cand.data_ptr(), ncand.data_ptr(), nq, ndb, kmax, d_pair.data_ptr())
    mt.search_by_bow_batch_device(d_kps.data_ptr(), d_desc.data_ptr(), d_n.data_ptr(), nrows, cap, d_kfmp.data_ptr(), d_bad.data_ptr(), nmp,
                                  voc, km.LEVELSUP, nq * kmax, d_pair.data_ptr(), 0.75, True, d_match.data_ptr(), d_nm.data_ptr())
    mt.sync()
    pairs, got, nm = d_pair.cpu().numpy(), d_match.cpu().numpy(), d_nm.cpu().numpy()
    check_points(oracle, R, [tuple(p) for p in pairs], got, nm, 0.75, True)
    empty = (pairs == -1).all(1)
    assert empty.any() and (~empty).sum() >= nq // 2 and (nm[empty] == -1).all() and nm.max() > 15


def test_argument_errors_enqueue_nothing(pkg, torch, scene):
    R, U, voc = scene
    mt = matcher(pkg, R, voc, 8)
    cap, capl, nrows = R["desc"].shape[1], R["ldesc"].shape[1], len(R["n"])
    x = torch.zeros(1 << 20, dtype=torch.int32, device="cuda").data_ptr()
    good = dict(d_kps=x, d_desc=x, d_n=x, nrows=nrows, cap=cap, d_kfmp=x, d_mpbad=x, nmp=10, vocab=voc, levelsup=km.LEVELSUP, npairs=8,
                d_pair=x, nnratio=0.75, check_ori=True, d_match=x, d_nmatch=x)
    lgood = dict(d_ldesc=x, d_nl=x, nrows=nrows, capl=capl, d_kfml=x, nml=10, npairs=8, d_pair=x, d_lmatch=x, d_nlmatch=x)
    before = mt.launch_count
    for kw in (dict(npairs=0), dict(npairs=9), dict(nrows=0), dict(nrows=65536), dict(cap=0), dict(cap=cap + 65), dict(nmp=-1),
               dict(levelsup=0), dict(d_pair=0), dict(d_kfmp=0), dict(d_match=0), dict(d_nmatch=0), dict(d_kps=0), dict(d_desc=0), dict(d_n=0)):
        with pytest.raises(pkg.SslplError):
            mt.search_by_bow_batch_device(**dict(good, **kw))
    for kw in (dict(npairs=0), dict(npairs=9), dict(nrows=0), dict(nrows=65536), dict(capl=0), dict(capl=capl + 65), dict(nml=-1),
               dict(d_kfml=0), dict(d_pair=0), dict(d_lmatch=0), dict(d_nlmatch=0), dict(d_ldesc=0), dict(d_nl=0)):
        with pytest.raises(pkg.SslplError):
            mt.match_lines_kf_batch_device(**dict(lgood, **kw))
    assert mt.launch_count == before
