"""GPU parity of the batched initialisation matchers over (init row, current row) pairs in HBM: sslpl_search_for_initialization_batch_device
(ORBmatcher::SearchForInitialization, ORBmatcher.cc:408-523, chained through vbPrevMatched) and sslpl_line_search_for_initialize_batch_device
(LSDmatcher::SerachForInitialize, LSDmatcher.cpp:257-284).  Every pair equals the single calls (sslpl_search_for_initialization with prev
carried on the host, sslpl_line_match(mode 1)), tests/init_match_model.py on the oracle and, where oracle/_ref/libref.so is present, the
reference.  Frames come from the device extractors at 2 x nFeatures.  All results are integer tables or copied keypoint coordinates: every
comparison is exact."""
import os

import numpy as np
import pytest

import init_match_model as im
from test_kf_triangulation_gpu import device_lines
from test_motion_batch_gpu import device_batch

pytestmark = pytest.mark.gpu
SENT_M, SENT_P, SENT_N = 7, 12345.0, -7          # what the outputs hold before a call: a row left alone keeps it


@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


def dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def pan(img, nframes, step):
    return np.stack([np.pad(img[:, step * k:], ((0, 0), (0, step * k)), mode="edge") for k in range(nframes)])


def row_set(pkg, torch, frames, nfeatures, nlines):
    B, H, W = frames.shape
    D = device_batch(pkg, torch, frames, nfeatures)
    L = device_lines(pkg, torch, D["dfr"], B, W, H, nlines)
    R = dict(kps=D["kps"].copy(), desc=D["desc"].copy(), n=D["n"].copy(), ldesc=L["ldesc"].copy(), nl=L["nl"].copy(),
             bounds=(0.0, float(W), 0.0, float(H)), W=W, H=H)
    R["U"] = dict(kps=dev(torch, R["kps"].view(np.uint8)), desc=dev(torch, R["desc"]), n=dev(torch, R["n"]), ldesc=dev(torch, R["ldesc"]),
                  nl=dev(torch, R["nl"]))
    return R


@pytest.fixture(scope="module")
def scene(pkg, synth, torch):
    """18 rows at 640x480 from the 2 x 1000-feature extractor: rows 0-8 one moving synthetic sequence, rows 9-17 a frame panned 14 px per
    frame (its carried windows reach the left border)."""
    frames = np.concatenate([synth.batch(640, 480, 9, start=32, group=16), pan(synth.frame(640, 480, 3), 9, 14)])
    return row_set(pkg, torch, frames, 2000, 40)


def matcher(pkg, R, max_batch=64):
    return pkg.Matcher(max_features=R["desc"].shape[1], max_lines=R["ldesc"].shape[1], max_nodes=3072, max_batch=max_batch)


def outputs(torch, P, cap):
    return dict(m12=torch.full((P, cap), SENT_M, dtype=torch.int32, device="cuda"),
                prev=torch.full((P, cap, 2), SENT_P, dtype=torch.float32, device="cuda"),
                n=torch.full((P,), SENT_N, dtype=torch.int32, device="cuda"))


def run_points(mt, torch, R, pairs, nnratio=0.9, check_ori=True, window=100, d_prev0=None, sync=True, o=None):
    P, cap = len(pairs), R["desc"].shape[1]
    d_pair = dev(torch, np.array(pairs, np.int32).reshape(-1, 2))
    o = o or outputs(torch, P, cap)
    U = R["U"]
    mt.search_for_initialization_batch_device(U["kps"].data_ptr(), U["desc"].data_ptr(), U["n"].data_ptr(), len(R["n"]), cap, P,
                                              d_pair.data_ptr(), d_prev0.data_ptr() if d_prev0 is not None else 0, R["bounds"], nnratio,
                                              check_ori, window, o["m12"].data_ptr(), o["prev"].data_ptr(), o["n"].data_ptr())
    o["pair"] = d_pair
    if sync:
        mt.sync()
    return o


def host(o):
    return o["m12"].cpu().numpy(), o["prev"].cpu().numpy(), o["n"].cpu().numpy()


def check_points(R, got, want):
    m12, prev, nm = got
    cap = R["desc"].shape[1]
    for p, (n, row, state) in enumerate(want):
        assert nm[p] == n, (p, int(nm[p]), n)
        if n == -1:
            assert (m12[p] == SENT_M).all() and (prev[p] == SENT_P).all(), p        # a bad pair writes no rows
            continue
        n1 = len(state)
        assert np.array_equal(m12[p], row), p
        assert np.array_equal(prev[p, :n1], state) and (prev[p, n1:] == SENT_P).all(), p
        assert n1 <= cap


def run_lines(mt, torch, R, pairs, d_nl=None):
    P, capl = len(pairs), R["ldesc"].shape[1]
    d_pair = dev(torch, np.array(pairs, np.int32).reshape(-1, 2))
    d_lp = torch.full((P, capl, 2), SENT_M, dtype=torch.int32, device="cuda"); d_nm = torch.full((P,), SENT_N, dtype=torch.int32, device="cuda")
    mt.line_search_for_initialize_batch_device(R["U"]["ldesc"].data_ptr(), (d_nl if d_nl is not None else R["U"]["nl"]).data_ptr(),
                                               len(R["nl"]), capl, P, d_pair.data_ptr(), d_lp.data_ptr(), d_nm.data_ptr())
    mt.sync()
    return d_lp.cpu().numpy(), d_nm.cpu().numpy()


def chains(nrows, base=0, span=9):
    """Chains of length 1 .. 8 inside rows [base, base + span), each on its own init row, current rows the following ones (cyclically)."""
    pairs = []
    for L in range(1, 9):
        r1 = (L - 1) % span
        pairs += [(base + r1, base + (r1 + k) % span) for k in range(1, L + 1)]
    return pairs


def ref_lib():
    from oracle import ref as REF
    return REF if os.path.exists(REF._LIB) else None


@pytest.mark.parametrize("window,nnratio,check_ori", [(100, 0.9, True), (50, 0.9, False), (100, 0.7, False), (50, 0.7, True)])
def test_points_equal_single_calls_and_oracle(pkg, oracle, torch, scene, window, nnratio, check_ori):
    R = scene
    mt = matcher(pkg, R)
    pairs = chains(len(R["n"])) + chains(len(R["n"]), base=9)[:28]
    assert len(pairs) <= 64
    got = host(run_points(mt, torch, R, pairs, nnratio, check_ori, window))
    single = im.points(mt.search_for_initialization, R, pairs, R["bounds"], nnratio, check_ori, window)
    check_points(R, got, single)
    check_points(R, got, im.points(oracle.search_for_initialization, R, pairs, R["bounds"], nnratio, check_ori, window))
    ref = ref_lib()
    if ref is not None:
        call = lambda d1, k1, d2, k2, prev, b, r, o, w: ref.search_for_initialization(d1, k1, d2, k2, prev, ref.cam(500, 500, 320, 240, *b),
                                                                                      8, 1.2, r, o, w)
        check_points(R, got, im.points(call, R, pairs[:20], R["bounds"], nnratio, check_ori, window) + single[20:])
    assert got[2].min() >= 0 and got[2].sum() > 50 * len(pairs)


def test_lines_equal_single_calls_and_oracle(pkg, oracle, torch, scene):
    R = dict(scene, nl=scene["nl"].copy())
    R["nl"][4] = 1; R["nl"][5] = 0; R["nl"][6] = R["ldesc"].shape[1] + 50                # one line, none, a count above capl
    d_nl = dev(torch, R["nl"])
    mt = matcher(pkg, R)
    pairs = chains(len(R["nl"]))[:30] + [(4, 0), (0, 4), (5, 0), (0, 5), (5, 4), (6, 1), (1, 6), (-1, 0), (0, len(R["nl"])), (3, 3)]
    pairs += [tuple(int(x) for x in r) for r in np.random.default_rng(5).integers(0, len(R["nl"]), (64 - len(pairs), 2))]
    lp, nm = run_lines(mt, torch, R, pairs, d_nl)
    lm = pkg.LSDmatcher(mt)
    ref = ref_lib()
    capl = R["ldesc"].shape[1]
    for p, pr in enumerate(pairs):
        n, rows = im.lines(oracle, R, pr)
        assert nm[p] == n and np.array_equal(lp[p], rows), (p, pr, int(nm[p]), n)
        n1, n2 = (im.clamp(R["nl"][r], capl) if 0 <= r < len(R["nl"]) else 0 for r in pr)
        if n >= 0 and n1 > 0:                                                 # where the single call is defined
            ns, ms = lm.SerachForInitialize(R["ldesc"][pr[0], :n1], R["ldesc"][pr[1], :n2])
            assert ns == n and np.array_equal(lp[p, :n], ms), (p, pr)
            if ref is not None and p < 16:
                n_r, m_r, _ = ref.line_match(1, R["ldesc"][pr[0], :n1], R["ldesc"][pr[1], :n2])
                assert n_r == n and np.array_equal(lp[p, :n], m_r), (p, pr)
    assert nm[31] == -1 and nm[32] == 0 and nm[33] == -1 and nm[34] == 0 and nm[37] == nm[38] == -1 and nm[39] > 0 and nm.max() > 5


def test_1280x960_8000_features(pkg, oracle, torch, synth):
    """The 2 x 4000-feature extractor at 1280x960 with 500 lines; chains of 3, 2 and 1 pairs."""
    R = row_set(pkg, torch, synth.batch(1280, 960, 6, start=40, group=16), 8000, 500)
    assert R["n"].min() > 4000
    mt = matcher(pkg, R, max_batch=8)
    pairs = [(0, 1), (0, 2), (0, 3), (4, 5), (4, 3), (1, 2)]
    for window, check_ori in ((100, True), (50, False)):
        got = host(run_points(mt, torch, R, pairs, 0.9, check_ori, window))
        check_points(R, got, im.points(mt.search_for_initialization, R, pairs, R["bounds"], 0.9, check_ori, window))
        check_points(R, got, im.points(oracle.search_for_initialization, R, pairs, R["bounds"], 0.9, check_ori, window))
        assert got[2].min() > 500
    lp, nm = run_lines(mt, torch, R, pairs)
    lm = pkg.LSDmatcher(mt)
    for p, (r1, r2) in enumerate(pairs):
        n, rows = im.lines(oracle, R, (r1, r2))
        ns, ms = lm.SerachForInitialize(R["ldesc"][r1, :R["nl"][r1]], R["ldesc"][r2, :R["nl"][r2]])
        assert nm[p] == n == ns and np.array_equal(lp[p], rows) and np.array_equal(lp[p, :n], ms), p
    assert nm.min() > 20


def test_chain_semantics(pkg, oracle, torch, scene):
    R = scene
    mt = matcher(pkg, R)
    cap = R["desc"].shape[1]
    A = [(9, 10), (9, 11), (9, 12), (9, 13), (9, 14), (9, 15)]
    B = [(1, 2), (1, 3), (1, 4)]
    whole = host(run_points(mt, torch, R, A + B))
    want = im.points(oracle.search_for_initialization, R, A + B, R["bounds"])
    check_points(R, whole, want)
    # the prefix property: the first k pairs of a chain alone give the same rows
    for k in (1, 3, 5):
        check_points(R, host(run_points(mt, torch, R, A[:k])), want[:k])
    # chains do not affect one another: each alone, and in the other order
    check_points(R, host(run_points(mt, torch, R, B)), want[len(A):])
    check_points(R, host(run_points(mt, torch, R, B + A)), want[len(A):] + want[:len(A)])
    # bad pairs: -1, no rows, and the chain's state left alone (the good pairs equal the chain without them)
    bad = [(9, 10), (9, -1), (9, 11), (9, 9), (9, len(R["n"])), (9, 12)]
    good = [pr for pr in bad if 0 <= pr[1] < len(R["n"]) and pr[1] != 9]
    g = host(run_points(mt, torch, R, bad + [(-2, 3), (-2, 4)]))
    assert list(g[2][[1, 3, 4, 6, 7]]) == [-1] * 5
    wg = im.points(oracle.search_for_initialization, R, good, R["bounds"])
    check_points(R, tuple(x[[0, 2, 5]] for x in g), wg)
    check_points(R, g, im.points(oracle.search_for_initialization, R, bad + [(-2, 3), (-2, 4)], R["bounds"]))
    # d_prev0 = NULL equals passing the init row's keypoint positions
    prev0 = np.full((len(A + B), cap, 2), -1.0, np.float32)
    for p in im.chain_starts(A + B):
        r1 = (A + B)[p][0]
        prev0[p, :, 0] = R["kps"][r1]["x"]; prev0[p, :, 1] = R["kps"][r1]["y"]
    check_points(R, host(run_points(mt, torch, R, A + B, d_prev0=dev(torch, prev0))), want)
    # a moved prev0 changes the result, and equals the model started from it
    moved = prev0.copy(); moved[..., 0] -= 40.0
    mv = host(run_points(mt, torch, R, A + B, d_prev0=dev(torch, moved)))
    check_points(R, mv, im.points(oracle.search_for_initialization, R, A + B, R["bounds"], prev0=moved))
    assert not np.array_equal(mv[0], whole[0])
    # a chain continued across two calls through d_prev equals one call
    first = run_points(mt, torch, R, A[:2])
    cont = torch.full((4, cap, 2), SENT_P, dtype=torch.float32, device="cuda")
    cont[0] = first["prev"][1]
    second = host(run_points(mt, torch, R, A[2:], d_prev0=cont))
    check_points(R, second, want[2:len(A)])
    # a repeated current row: each pair is simply the next call
    rep = [(9, 12), (9, 12), (9, 13), (9, 12)]
    check_points(R, host(run_points(mt, torch, R, rep)), im.points(mt.search_for_initialization, R, rep, R["bounds"]))
    # the inputs are never modified
    for key in ("kps", "desc", "n"):
        assert np.array_equal(R["U"][key].cpu().numpy().reshape(-1), R[key].view(np.uint8).reshape(-1) if key == "kps" else R[key].reshape(-1))


def test_caller_stream_and_argument_errors(pkg, oracle, torch, scene):
    R = scene
    mt = matcher(pkg, R, max_batch=20)
    cap, capl, nrows = R["desc"].shape[1], R["ldesc"].shape[1], len(R["n"])
    A = [(9, 10), (9, 11), (9, 12), (0, 1), (0, 2)]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        mt.set_stream(s.cuda_stream)
        o = run_points(mt, torch, R, A, sync=False)
    s.synchronize()
    mt.set_stream(0)
    check_points(R, host(o), im.points(oracle.search_for_initialization, R, A, R["bounds"]))
    # bad arguments: SSLPL_ERR_ARG, nothing enqueued, nothing written
    U = R["U"]
    o = outputs(torch, 21, cap)
    d_pair = dev(torch, np.zeros((21, 2), np.int32))
    good = dict(d_kps=U["kps"].data_ptr(), d_desc=U["desc"].data_ptr(), d_n=U["n"].data_ptr(), nrows=nrows, cap=cap, npairs=4,
                d_pair=d_pair.data_ptr(), d_prev0=0, bounds=R["bounds"], nnratio=0.9, check_ori=True, window=100,
                d_match12=o["m12"].data_ptr(), d_prev=o["prev"].data_ptr(), d_nmatch=o["n"].data_ptr())
    d_lp = torch.full((21, capl, 2), SENT_M, dtype=torch.int32, device="cuda")
    lgood = dict(d_ldesc=U["ldesc"].data_ptr(), d_nl=U["nl"].data_ptr(), nrows=nrows, capl=capl, npairs=4, d_pair=d_pair.data_ptr(),
                 d_lpairs=d_lp.data_ptr(), d_nlmatch=o["n"].data_ptr())
    torch.cuda.synchronize()
    before = mt.launch_count
    small = pkg.Matcher(max_features=64, max_lines=64, max_nodes=16, max_batch=20)
    for kw in (dict(npairs=0), dict(npairs=21), dict(nrows=1), dict(nrows=22), dict(cap=0), dict(cap=cap + 65), dict(d_pair=0),
               dict(d_kps=0), dict(d_desc=0), dict(d_n=0), dict(d_match12=0), dict(d_prev=0), dict(d_nmatch=0),
               dict(bounds=(640.0, 640.0, 0.0, 480.0)), dict(bounds=(0.0, 640.0, 480.0, 0.0))):
        with pytest.raises(pkg.SslplError):
            mt.search_for_initialization_batch_device(**dict(good, **kw))
    with pytest.raises(pkg.SslplError):                                   # cap above this handle's max_features + 64
        small.search_for_initialization_batch_device(**good)
    for kw in (dict(npairs=0), dict(npairs=21), dict(nrows=0), dict(nrows=22), dict(capl=0), dict(capl=capl + 65), dict(d_pair=0),
               dict(d_ldesc=0), dict(d_nl=0), dict(d_lpairs=0), dict(d_nlmatch=0)):
        with pytest.raises(pkg.SslplError):
            mt.line_search_for_initialize_batch_device(**dict(lgood, **kw))
    torch.cuda.synchronize()
    assert mt.launch_count == before and small.launch_count == 0
    assert (o["m12"] == SENT_M).all() and (o["prev"] == SENT_P).all() and (o["n"] == SENT_N).all() and (d_lp == SENT_M).all()
