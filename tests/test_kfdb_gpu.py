"""GPU parity of the batched, device-resident keyframe database (include/sslpl.h): the BowVector build, the L1 score and
KeyFrameDatabase::DetectLoopCandidates / DetectRelocalizationCandidates over rows in HBM, against tests/kfdb_model.py, bit for bit.
tests/test_kfdb_cpu.py holds that model to the reference's own KeyFrameDatabase and DBoW2 code."""
import numpy as np
import pytest

import kfdb_model as km

pytestmark = pytest.mark.gpu
f32 = np.float32


@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


@pytest.fixture(scope="module")
def mt(pkg):
    return pkg.Matcher(max_features=4096, max_lines=64, max_nodes=1024, max_batch=1)


@pytest.fixture(scope="module")
def voc(pkg):
    """k = 10, L = 3 (1000 words, so that rows share many): some words stopped, some leaves above the last level."""
    return pkg.Vocabulary.random(10, 3, seed=3, stop_fraction=0.05, early_leaf_fraction=0.1)


def rows(rng, nrows, nfeat, cap, nplaces=4, flip=0.03):
    """Descriptors of rows drawn from a few places: [nrows, cap, 32] and counts; row 0 is empty, row 1 repeats one descriptor 60 times,
    row 2 is a copy of row 1 (equal BowVectors)."""
    base = rng.integers(0, 256, (nplaces, 400, 32), dtype=np.uint8)
    place = rng.integers(0, nplaces, nrows)
    desc = np.zeros((nrows, cap, 32), np.uint8)
    n = np.full(nrows, nfeat, np.int32)
    for r in range(nrows):
        d = base[place[r]][rng.integers(0, 400, nfeat)] ^ np.packbits(rng.random((nfeat, 256)) < flip, axis=-1, bitorder="little")
        desc[r, :nfeat] = d
    n[0] = 0
    desc[1, :60] = desc[1, 0]
    desc[2] = desc[1]
    return desc, n, place


class RowSet:
    """A row set in HBM and its BowVector tables after sslpl_bow_vectors_batch_device."""

    def __init__(self, torch, mt, voc, desc, n):
        self.nrows, self.cap = desc.shape[0], desc.shape[1]
        self.d_desc = torch.from_numpy(desc).cuda(); self.d_n = torch.from_numpy(n).cuda()
        self.word = torch.full((self.nrows, self.cap), 7, dtype=torch.int32, device="cuda")
        self.val = torch.full((self.nrows, self.cap), 7.0, dtype=torch.float64, device="cuda")
        self.bn = torch.full((self.nrows,), -7, dtype=torch.int32, device="cuda")
        mt.bow_vectors_batch_device(voc, self.d_desc.data_ptr(), self.d_n.data_ptr(), self.nrows, self.cap, self.word.data_ptr(),
                                    self.val.data_ptr(), self.bn.data_ptr())
        mt.sync()
        self.tables = (self.word.data_ptr(), self.val.data_ptr(), self.bn.data_ptr(), self.nrows, self.cap)

    def bows(self):
        w, v, n = self.word.cpu().numpy(), self.val.cpu().numpy(), self.bn.cpu().numpy()
        return [(w[r, :n[r]].copy(), v[r, :n[r]].copy()) for r in range(self.nrows)]


@pytest.mark.parametrize("nfeat", [1000, 4000])
def test_bow_vectors_equal_model(torch, mt, voc, nfeat):
    rng = np.random.default_rng(nfeat)
    desc, n, _ = rows(rng, 24, nfeat, nfeat + 64)
    S = RowSet(torch, mt, voc, desc, n)
    word, val, bn = S.word.cpu().numpy(), S.val.cpu().numpy(), S.bn.cpu().numpy()
    stopped = repeated = 0
    for r in range(S.nrows):
        fw, _, fv = mt.bow_transform(voc, desc[r, :n[r]]) if n[r] else (np.zeros(0, np.int32), None, np.zeros(0))
        mw, mv = km.bow_vector(fw, fv)
        hw, hv = voc.bow_vector(fw, fv)
        assert bn[r] == len(mw)
        assert np.array_equal(word[r, :bn[r]], mw) and np.array_equal(val[r, :bn[r]].view(np.uint64), mv.view(np.uint64)), r
        assert np.array_equal(hw, mw) and np.array_equal(hv.view(np.uint64), mv.view(np.uint64))
        assert (word[r, bn[r]:] == -1).all() and (val[r, bn[r]:].view(np.uint64) == 0).all()
        stopped += int((fv <= 0).sum())
        if n[r]:
            repeated = max(repeated, int(np.bincount(fw[fv > 0]).max()))
    assert bn[0] == 0 and stopped > 0 and repeated >= 60


def scene(torch, mt, voc, ndb, nq, nfeat=1000, seed=0):
    """ndb + nq + 8 rows: ndb + 8 keyframes are added in a random order and 8 of them erased, leaving a database of ndb; the queries are
    rows of the database and rows outside it.  Returns the row set, its model BowVectors, the database, queries, covisibility table,
    each query's connected rows, and (add order, erased rows, connected rows of every row) for the reference."""
    rng = np.random.default_rng(seed)
    nrows = ndb + nq + 8
    desc, n, place = rows(rng, nrows, nfeat, nfeat + 64)
    S = RowSet(torch, mt, voc, desc, n)
    bows = S.bows()
    add = rng.permutation(ndb + 8).astype(np.int32)
    erase = rng.choice(add, 8, replace=False).astype(np.int32)
    db = np.array([r for r in add if r not in set(erase.tolist())], np.int32)
    query = np.concatenate([rng.choice(db, min(nq // 2, ndb), replace=False), ndb + 8 + np.arange(nq - min(nq // 2, ndb))]).astype(np.int32)
    query[0] = 0                                                    # the empty row
    covis = np.full((nrows, 10), -1, np.int32)
    for r in range(nrows):
        same = np.nonzero(place == place[r])[0]
        k = min(int(rng.integers(0, 11)), len(same))
        covis[r, :k] = rng.choice(same, k, replace=False)
    covis[5, 3] = nrows + 7                                          # out of range: outside the database
    conn_rows = [sorted(set(rng.choice(nrows, int(rng.integers(0, min(30, nrows))), replace=False).tolist()) - {r}) for r in range(nrows)]
    conn = [conn_rows[r] for r in query]
    return S, bows, db, query, covis, conn, (add, erase, conn_rows)


def covis_lists(covis):
    return [[int(c) for c in row if c != -1] for row in covis]


def dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def run_loop(torch, mt, S, db, query, covis, conn, minscore, off=None):
    nq, ndb = len(query), len(db)
    if off is None:
        off = np.zeros(nq + 1, np.int32); off[1:] = np.cumsum([len(c) for c in conn])
    flat = np.array(sum(conn, []) + [0], np.int32)
    t = [dev(torch, a) for a in (db, query, covis, off, flat, np.asarray(minscore, f32))]
    cand = torch.full((nq, ndb), 9, dtype=torch.int32, device="cuda"); ncand = torch.full((nq,), 9, dtype=torch.int32, device="cuda")
    words = torch.full((nq, ndb), 9, dtype=torch.int32, device="cuda"); score = torch.full((nq, ndb), 9.0, dtype=torch.float32, device="cuda")
    mt.detect_loop_candidates_batch_device(*S.tables, t[0].data_ptr(), ndb, t[1].data_ptr(), nq, t[2].data_ptr(), t[3].data_ptr(),
                                           t[4].data_ptr(), len(flat) - 1, t[5].data_ptr(), cand.data_ptr(), ncand.data_ptr(), words.data_ptr(), score.data_ptr())
    mt.sync()
    return cand.cpu().numpy(), ncand.cpu().numpy(), words.cpu().numpy(), score.cpu().numpy()


def run_reloc(torch, mt, S, db, query, covis, relocscore):
    nq, ndb = len(query), len(db)
    t = [dev(torch, a) for a in (db, query, covis)]
    rs = dev(torch, np.asarray(relocscore, f32))
    cand = torch.full((nq, ndb), 9, dtype=torch.int32, device="cuda"); ncand = torch.full((nq,), 9, dtype=torch.int32, device="cuda")
    words = torch.full((nq, ndb), 9, dtype=torch.int32, device="cuda"); score = torch.full((nq, ndb), 9.0, dtype=torch.float32, device="cuda")
    mt.detect_relocalization_candidates_batch_device(*S.tables, t[0].data_ptr(), ndb, t[1].data_ptr(), nq, t[2].data_ptr(), rs.data_ptr(),
                                                     cand.data_ptr(), ncand.data_ptr(), words.data_ptr(), score.data_ptr())
    mt.sync()
    return cand.cpu().numpy(), ncand.cpu().numpy(), words.cpu().numpy(), score.cpu().numpy(), rs.cpu().numpy()


def same_as_model(got, model):
    cand, ncand, words, score = got[:4]
    mc, mw, ms, _ = model
    for q, c in enumerate(mc):
        if c is None:
            assert ncand[q] == -1 and (cand[q] == -1).all()
        else:
            assert ncand[q] == len(c) and cand[q, :len(c)].tolist() == c and (cand[q, len(c):] == -1).all(), q
    assert np.array_equal(words, mw)
    assert np.array_equal(score.view(np.uint32), ms.view(np.uint32))


@pytest.fixture(scope="module")
def ref_kfdb(voc, tmp_path_factory):
    """The reference's own KeyFrameDatabase (oracle/_ref/libref_kfdb.so) and the vocabulary loaded by its loadFromTextFile, or None where
    the library is absent."""
    from test_kfdb_cpu import load_ref_kfdb
    from test_ref_parity_cpu import write_vocab_text
    L = load_ref_kfdb()
    if L is None:
        return None
    from oracle import ref as R
    path = str(tmp_path_factory.mktemp("kfdb_gpu") / "voc.txt")
    write_vocab_text(path, voc.k, voc.L, voc.parent, voc.desc, voc.weight, voc.is_leaf)
    return L, R.Vocabulary(path)


def same_as_reference(ref_kfdb, got, bows, db, covis, extra, loop, query, minscore=None, relocscore=None):
    """The device results against the reference's own KeyFrameDatabase, run on the same BowVectors, add / erase sequence and graph."""
    from test_kfdb_cpu import check_against_ref, run_ref
    L, V = ref_kfdb
    add, erase, conn_rows = extra
    nrows = len(bows)
    lists = [[int(c) if 0 <= c < nrows else int(erase[0]) for c in row if c != -1] for row in covis]   # out of range: an erased keyframe
    rcov = np.full((nrows, 10), -1, np.int32); ncov = np.array([len(c) for c in lists], np.int32)
    for r, c in enumerate(lists):
        rcov[r, :len(c)] = c
    out = run_ref(L, V, bows, rcov, ncov, conn_rows, relocscore if relocscore is not None else np.zeros(nrows, f32), add, erase, loop,
                  query, minscore)
    cand, ncand, words, score = got[:4]
    check_against_ref(out, ([cand[q, :ncand[q]].tolist() for q in range(len(query))], words, score, None), db, relocscore, loop)


@pytest.mark.parametrize("ndb", [1, 50, 2000])
def test_detect_loop_candidates_equal_model(torch, mt, voc, ref_kfdb, ndb):
    S, bows, db, query, covis, conn, extra = scene(torch, mt, voc, ndb, 12, seed=ndb)
    rng = np.random.default_rng(ndb + 1)
    minscore = rng.uniform(0, 0.2, len(query)).astype(f32); minscore[3] = 2.0
    got = run_loop(torch, mt, S, db, query, covis, conn, minscore)
    model = km.detect(bows, db, query, covis_lists(covis), True, conn=conn, minscore=minscore)
    same_as_model(got, model)
    if ref_kfdb is not None:
        same_as_reference(ref_kfdb, got, bows, db, covis, extra, True, query, minscore=minscore)
    assert got[1][0] == 0 and got[1][3] == 0
    if ndb > 1:
        assert (got[1] > 0).sum() >= 4


@pytest.mark.parametrize("ndb", [1, 50, 2000])
def test_detect_relocalization_candidates_equal_model(torch, mt, voc, ref_kfdb, ndb):
    S, bows, db, query, covis, _, extra = scene(torch, mt, voc, ndb, 12, seed=ndb + 10)
    rs0 = np.random.default_rng(ndb).uniform(0, 1, S.nrows).astype(f32)
    got = run_reloc(torch, mt, S, db, query, covis, rs0)
    model = km.detect(bows, db, query, covis_lists(covis), False, relocscore=rs0)
    same_as_model(got, model)
    assert np.array_equal(got[4].view(np.uint32), model[3].view(np.uint32))
    if ref_kfdb is not None:
        same_as_reference(ref_kfdb, got, bows, db, covis, extra, False, query, relocscore=rs0)
    if ndb > 1:
        assert (got[1] > 0).sum() >= 4


def test_one_call_equals_single_calls(torch, mt, voc):
    """nq queries in one call equal nq one-query calls with the reloc scores chained through them."""
    S, bows, db, query, covis, conn, _ = scene(torch, mt, voc, 300, 10, seed=5)
    rs = np.zeros(S.nrows, f32)
    whole = run_reloc(torch, mt, S, db, query, covis, rs)
    for q in range(len(query)):
        one = run_reloc(torch, mt, S, db, query[q:q + 1], covis, rs)
        for a, b in zip(whole[:4], one[:4]):
            assert np.array_equal(a[q:q + 1].view(np.uint32), b.view(np.uint32))
        rs = one[4]
    assert np.array_equal(rs.view(np.uint32), whole[4].view(np.uint32))
    minscore = np.full(len(query), 0.05, f32)
    whole = run_loop(torch, mt, S, db, query, covis, conn, minscore)
    for q in range(len(query)):
        one = run_loop(torch, mt, S, db, query[q:q + 1], covis, conn[q:q + 1], minscore[q:q + 1])
        for a, b in zip(whole, one):
            assert np.array_equal(a[q:q + 1].view(np.uint32), b.view(np.uint32))


def test_scores_equal_model(torch, mt, voc):
    """>= 10^5 pairs, bit for bit as float64; pairs with a row out of range get NaN."""
    rng = np.random.default_rng(9)
    desc, n, _ = rows(rng, 400, 300, 364)
    S = RowSet(torch, mt, voc, desc, n)
    bows = S.bows()
    pair = rng.integers(0, 400, (100000, 2)).astype(np.int32)
    pair[:400, 0] = np.arange(400); pair[:400, 1] = np.arange(400)
    pair[-3:] = [(-1, 0), (0, 400), (5, 1 << 30)]
    d_pair = dev(torch, pair); d_score = torch.zeros(len(pair), dtype=torch.float64, device="cuda")
    mt.bow_score_batch_device(*S.tables, len(pair), d_pair.data_ptr(), d_score.data_ptr())
    mt.sync()
    got = d_score.cpu().numpy()
    want = np.array([km.score(bows[a], bows[b]) for a, b in pair[:-3].tolist()])
    assert np.array_equal(got[:-3].view(np.uint64), want.view(np.uint64))
    assert np.isnan(got[-3:]).all()


def test_validation(torch, mt, voc, pkg, tmp_path):
    """Bad host arguments return their status and enqueue nothing; malformed device lists give -1 counts."""
    S, bows, db, query, covis, conn, _ = scene(torch, mt, voc, 20, 4, seed=1)
    w, v, bn, nrows, cap = S.tables
    d = [dev(torch, a) for a in (db, query, covis, np.zeros(5, np.int32), np.zeros(1, np.int32), np.zeros(4, f32), np.zeros(nrows, f32))]
    out = [torch.zeros((4, 20), dtype=torch.int32, device="cuda"), torch.zeros(4, dtype=torch.int32, device="cuda"),
           torch.zeros((4, 20), dtype=torch.int32, device="cuda"), torch.zeros((4, 20), dtype=torch.float32, device="cuda")]
    o = [t.data_ptr() for t in out]
    L = pkg.lib()
    loop_ok = [mt._h, w, v, bn, nrows, cap, d[0].data_ptr(), 20, d[1].data_ptr(), 4, d[2].data_ptr(), d[3].data_ptr(), d[4].data_ptr(), 1,
               d[5].data_ptr()] + o
    reloc_ok = [mt._h, w, v, bn, nrows, cap, d[0].data_ptr(), 20, d[1].data_ptr(), 4, d[2].data_ptr(), d[6].data_ptr()] + o
    before = mt.launch_count
    bad = []
    for i in (0, 1, 6, 8, 10, 11, 12, 14, 15, 16, 17, 18):
        bad.append(("loop", i, None))
    bad.append(("loop", 13, -1))
    for i, val in ((4, 0), (5, 0), (5, 4096 + 65), (7, 0), (7, 25601), (9, 0), (9, 65536)):
        bad.append(("loop", i, val)); bad.append(("reloc", i, val))
    for kind, i, val in bad:
        a = list(loop_ok if kind == "loop" else reloc_ok)
        a[i] = val
        fn = L.sslpl_detect_loop_candidates_batch_device if kind == "loop" else L.sslpl_detect_relocalization_candidates_batch_device
        assert fn(*a) == -1, (kind, i, val)
    assert L.sslpl_bow_score_batch_device(mt._h, w, v, bn, nrows, cap, 0, d[0].data_ptr(), d[5].data_ptr()) == -1
    assert L.sslpl_bow_score_batch_device(mt._h, w, v, bn, 0, cap, 1, d[0].data_ptr(), d[5].data_ptr()) == -1
    assert L.sslpl_bow_score_batch_device(mt._h, w, v, bn, nrows, cap, 1, None, d[5].data_ptr()) == -1
    assert L.sslpl_bow_vectors_batch_device(mt._h, voc._h, S.d_desc.data_ptr(), S.d_n.data_ptr(), 0, cap, w, v, bn) == -1
    assert L.sslpl_bow_vectors_batch_device(mt._h, voc._h, S.d_desc.data_ptr(), S.d_n.data_ptr(), nrows, 4096 + 65, w, v, bn) == -1
    assert L.sslpl_bow_vectors_batch_device(mt._h, None, S.d_desc.data_ptr(), S.d_n.data_ptr(), nrows, cap, w, v, bn) == -1
    parent, nd, wt, leaf = pkg.Vocabulary.random_arrays(10, 2, seed=1)
    lines = ["10 2 1 0"] + [f"{int(parent[i])} {int(leaf[i])} " + " ".join(str(int(x)) for x in nd[i]) + f" {float(wt[i])!r}"
                            for i in range(1, len(parent))]
    (tmp_path / "l2.txt").write_text("\n".join(lines))
    l2 = pkg.Vocabulary.load_text(str(tmp_path / "l2.txt"))
    assert L.sslpl_bow_vectors_batch_device(mt._h, l2._h, S.d_desc.data_ptr(), S.d_n.data_ptr(), nrows, cap, w, v, bn) == -4
    with pytest.raises(pkg.SslplError):
        mt.bow_vectors_batch_device(l2, S.d_desc.data_ptr(), S.d_n.data_ptr(), nrows, cap, w, v, bn)
    assert mt.launch_count == before
    # malformed device lists
    q_bad = query.copy(); q_bad[1] = nrows + 3
    got = run_reloc(torch, mt, S, db, q_bad, covis, np.zeros(nrows, f32))
    assert got[1][1] == -1 and (got[1][[0, 2, 3]] >= 0).all() and (got[2][1] == 0).all() and np.isnan(got[3][1]).all()
    conn_n = sum(len(c) for c in conn)
    for bad_off in ([0, 0, 1, 1, conn_n + 1], [0, 5, 3, 5, conn_n], [-1, 0, 0, 0, conn_n]):      # beyond nconn, decreasing, negative
        got = run_loop(torch, mt, S, db, query, covis, conn, np.zeros(4, f32), off=np.array(bad_off, np.int32))
        bad_q = [q for q in range(4) if not 0 <= bad_off[q] <= bad_off[q + 1] <= conn_n]
        assert all(got[1][q] == -1 for q in bad_q) and all(got[1][q] >= 0 for q in range(4) if q not in bad_q), (bad_off, got[1])
    for db_bad in (np.concatenate([db[:-1], db[:1]]), np.concatenate([db[:-1], [-2]])):
        got = run_loop(torch, mt, S, db_bad.astype(np.int32), query, covis, conn, np.zeros(4, f32))
        assert (got[1] == -1).all() and (got[0] == -1).all()
        rs = np.full(nrows, 0.5, f32)
        got = run_reloc(torch, mt, S, db_bad.astype(np.int32), query, covis, rs)
        assert (got[1] == -1).all() and (got[4] == 0.5).all()
