"""CPU tests (no GPU): tests/kfdb_model.py against the reference's own DBoW2 BowVector / L1Scoring and KeyFrameDatabase, bit for bit.
The database entry points are those of tests/ref_kfdb.cpp, which oracle/ref_kfdb_build.sh compiles against the reference's headers into
oracle/_ref/libref_kfdb.so, linked with oracle/_ref/libref.so (the reference's sources as oracle/ref_build.sh compiles them).  Skipped
when that library is absent."""
import ctypes as C
import os

import numpy as np
import pytest

import kfdb_model as km
from test_ref_parity_cpu import write_vocab_text

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle")
f32 = np.float32


@pytest.fixture(scope="module")
def ref():
    if not os.path.exists(os.path.join(ORACLE, "_ref", "libref.so")):
        pytest.skip("oracle/_ref/libref.so is not present")
    from oracle import ref as R
    return R


def load_ref_kfdb():
    """oracle/_ref/libref_kfdb.so (oracle/ref_kfdb_build.sh, run by build() where the reference's sources are present), or None."""
    path = os.path.join(ORACLE, "_ref", "libref_kfdb.so")
    if not os.path.exists(path):
        return None
    L = C.CDLL(path)
    L.ref_kfdb_query.restype = None; L.ref_bow_score.restype = None
    return L


@pytest.fixture(scope="module")
def kfdb_lib(ref):
    L = load_ref_kfdb()
    if L is None:
        pytest.skip("oracle/_ref/libref_kfdb.so is not present")
    return L


@pytest.fixture(scope="module")
def voc(ref, pkg, tmp_path_factory):
    """A random k = 10, L = 3 tree (1000 words, some stopped) loaded by DBoW2's own loadFromTextFile."""
    parent, desc, w, leaf = pkg.Vocabulary.random_arrays(10, 3, seed=7, stop_fraction=0.05)
    path = str(tmp_path_factory.mktemp("kfdb") / "voc.txt")
    write_vocab_text(path, 10, 3, parent, desc, w, leaf)
    return ref.Vocabulary(path), (parent, desc, w, leaf)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def place_descriptors(rng, nplaces, nbase=300):
    return rng.integers(0, 256, (nplaces, nbase, 32), dtype=np.uint8)


def row_descriptors(rng, base, place, n, flip=0.02):
    idx = rng.integers(0, base.shape[1], n)
    return base[place][idx] ^ np.packbits(rng.random((n, 256)) < flip, axis=-1, bitorder="little")


def scene(rng, V, nrows, nplaces, nfeat):
    """Rows drawn from a few places, so that many share words: (bows, place of each row).  Row 0 is empty; rows 1 and 2 have the same
    BowVector (score ties); row 3 has one word no other row has (a query sharing nothing)."""
    base = place_descriptors(rng, nplaces)
    place = rng.integers(0, nplaces, nrows)
    bows = []
    for r in range(nrows):
        n = 0 if r == 0 else int(rng.integers(nfeat[0], nfeat[1] + 1))
        _, w, v = V.transform(row_descriptors(rng, base, place[r], n))
        bows.append((w, v))
    bows[2] = (bows[1][0].copy(), bows[1][1].copy())
    used = set(np.concatenate([b[0] for b in bows]).tolist())
    free = next(w for w in range(len(V)) if w not in used)
    bows[3] = (np.array([free], np.int32), np.array([1.0]))
    return bows, place


def graph(rng, nrows, place):
    """covis[r]: up to 10 rows of the same place (some lists shorter, some entries outside the database); conn[r]: a few rows."""
    covis = np.full((nrows, 10), -1, np.int32); ncov = np.zeros(nrows, np.int32); conn = []
    for r in range(nrows):
        same = [s for s in np.nonzero(place == place[r])[0].tolist() if s != r]
        k = min(len(same), int(rng.integers(0, 11)))
        nb = rng.permutation(same)[:k]
        covis[r, :k] = nb; ncov[r] = k
        conn.append(sorted(set(rng.choice(nrows, int(rng.integers(0, 6)), replace=False).tolist()) - {r}))
    return covis, ncov, conn


def database(rng, nrows, frac=0.8, nerase=5):
    """(add order, erased rows, the database rows in add order): row 3, the row sharing nothing, is never added."""
    rows = np.array([r for r in rng.permutation(nrows)[:int(frac * nrows)] if r != 3])
    erase = rng.choice(rows, nerase, replace=False)
    return rows, erase, np.array([r for r in rows if r not in set(erase.tolist())], np.int32)


def run_ref(lib, V, bows, covis, ncov, conn, relocscore, add, erase, loop, query, minscore):
    nrows, nq = len(bows), len(query)
    off, word, val = flat(bows)
    coff = np.zeros(nrows + 1, np.int32); coff[1:] = np.cumsum([len(c) for c in conn])
    cflat = np.array(sum(conn, []) + [0], np.int32)
    add = np.ascontiguousarray(add, np.int32); erase = np.ascontiguousarray(erase, np.int32); query = np.ascontiguousarray(query, np.int32)
    ms = np.ascontiguousarray(minscore if minscore is not None else np.zeros(nq), f32); rs = np.ascontiguousarray(relocscore, f32)
    cand = np.full((nq, nrows), -1, np.int32); ncand = np.zeros(nq, np.int32)
    words = np.zeros((nq, nrows), np.int32); score = np.zeros((nq, nrows), f32)
    lib.ref_kfdb_query(C.c_void_p(V.h), nrows, _p(off), _p(word), _p(val), _p(covis), _p(ncov), _p(coff), _p(cflat), _p(rs), len(add), _p(add),
                       len(erase), _p(erase), int(loop), nq, _p(query), _p(ms), _p(cand), _p(ncand), _p(words), _p(score), None)
    return [cand[q, :ncand[q]].tolist() for q in range(nq)], words, score


def check_against_ref(ref_out, model_out, db, relocscore, loop):
    """Candidates equal; every keyframe's words field as the model's table (0 off the database); every score field is the model's where
    the query scored the keyframe and unchanged elsewhere."""
    rc, rw, rsc = ref_out
    mc, mw, msc, _ = model_out
    nq, nrows = rw.shape
    assert rc == mc
    want_w = np.zeros((nq, nrows), np.int32); want_w[:, db] = mw
    assert np.array_equal(rw, want_w)
    prev = np.zeros(nrows, f32) if loop else np.array(relocscore, f32)
    for q in range(nq):
        want = prev.copy()
        scored = ~np.isnan(msc[q])
        want[db[scored]] = msc[q][scored]
        assert np.array_equal(rsc[q].view(np.uint32), want.view(np.uint32)), q
        prev = rsc[q]


def test_bow_vector_equals_dbow2_transform(voc):
    """The model's BowVector equals DBoW2's transform bit for bit: stopped words, one word repeated 50 times, an empty row."""
    V, _ = voc
    rng = np.random.default_rng(1)
    base = place_descriptors(rng, 2)
    for n in (0, 1, 7, 300, 1000):
        d = row_descriptors(rng, base, n % 2, n)
        if n == 300:
            d[:50] = d[0]                                            # one word 50 times
        w, v = V.words(d)
        mw, mv = km.bow_vector(w, v)
        _, rw, rv = V.transform(d)
        assert np.array_equal(mw, rw) and np.array_equal(mv.view(np.uint64), rv.view(np.uint64)), n
        if n == 300:
            assert (w == w[0]).sum() >= 50 and (v[w == w[0]] > 0).all()
    assert (V.words(row_descriptors(rng, base, 0, 1000))[1] <= 0).any()   # the tree has stopped words


def test_score_equals_l1_scoring(kfdb_lib, voc):
    """The model's score equals TemplatedVocabulary::score (L1Scoring) bit for bit, on rows with ties, an empty row and no common word."""
    V, _ = voc
    rng = np.random.default_rng(2)
    bows, _ = scene(rng, V, 40, 2, (50, 400))
    off, word, val = flat(bows)
    pair = np.array([(a, b) for a in range(40) for b in range(40)], np.int32)
    out = np.zeros(len(pair))
    kfdb_lib.ref_bow_score(C.c_void_p(V.h), _p(off), _p(word), _p(val), len(pair), _p(pair), _p(out))
    want = np.array([km.score(bows[a], bows[b]) for a, b in pair.tolist()])
    assert np.array_equal(out.view(np.uint64), want.view(np.uint64))
    S = want.reshape(40, 40)
    assert np.array_equal(S[1], S[2]) and (S[0] == 0).all() and (np.delete(S[3], 3) == 0).all() and (S[4:] > 0).sum() > 100   # ties, nothing shared


def flat(bows):
    off = np.zeros(len(bows) + 1, np.int32); off[1:] = np.cumsum([len(b[0]) for b in bows])
    word = np.concatenate([b[0] for b in bows] + [np.zeros(1, np.int32)]).astype(np.int32)
    val = np.concatenate([b[1] for b in bows] + [np.zeros(1)]).astype(np.float64)
    return off, word, val


SCENES = [  # seed, nrows, nplaces, feature range
    (11, 60, 3, (5, 40)),
    (12, 120, 4, (20, 120)),
    (13, 200, 6, (3, 15)),
]


@pytest.mark.parametrize("seed,nrows,nplaces,nfeat", SCENES)
def test_detect_loop_candidates_equal_reference(kfdb_lib, voc, seed, nrows, nplaces, nfeat):
    V, _ = voc
    rng = np.random.default_rng(seed)
    bows, place = scene(rng, V, nrows, nplaces, nfeat)
    covis, ncov, conn = graph(rng, nrows, place)
    add, erase, db = database(rng, nrows)
    query = np.array([0, 1, 3] + rng.integers(4, nrows, 15).tolist(), np.int32)
    minscore = rng.uniform(0, 0.05, len(query)).astype(f32)
    minscore[5] = 2.0                                                # rejects everything
    out = run_ref(kfdb_lib, V, bows, covis, ncov, conn, np.zeros(nrows, f32), add, erase, True, query, minscore)
    covl = [covis[r, :ncov[r]].tolist() for r in range(nrows)]
    model = km.detect(bows, db, query, covl, True, conn=[conn[q] for q in query], minscore=minscore)
    check_against_ref(out, model, db, None, True)
    assert model[0][0] == [] and model[0][2] == [] and model[0][5] == []          # empty row, nothing shared, minScore too high
    assert sum(len(c) for c in model[0]) >= 10


@pytest.mark.parametrize("seed,nrows,nplaces,nfeat", SCENES)
def test_detect_relocalization_candidates_equal_reference(kfdb_lib, voc, seed, nrows, nplaces, nfeat):
    """Sequences of 16 queries, started from two mRelocScore tables: both equal the reference, and the stale scores change the output."""
    V, _ = voc
    rng = np.random.default_rng(seed + 100)
    bows, place = scene(rng, V, nrows, nplaces, nfeat)
    covis, ncov, conn = graph(rng, nrows, place)
    add, erase, db = database(rng, nrows)
    query = np.array([0, 3] + rng.integers(4, nrows, 14).tolist(), np.int32)
    covl = [covis[r, :ncov[r]].tolist() for r in range(nrows)]
    cands = []
    for init in (np.zeros(nrows, f32), rng.uniform(0, 2, nrows).astype(f32)):
        out = run_ref(kfdb_lib, V, bows, covis, ncov, conn, init, add, erase, False, query, None)
        model = km.detect(bows, db, query, covl, False, relocscore=init)
        check_against_ref(out, model, db, init, False)
        cands.append(model[0])
    assert cands[0] != cands[1]                                      # stale scores decide candidates


def test_scenes_cover_the_edges(voc):
    """maxCommonWords * 0.8f on an integer (a multiple of 5) and keyframes listed below minCommonWords occur in the scenes above."""
    V, _ = voc
    on_integer = below = 0
    for seed, nrows, nplaces, nfeat in SCENES:
        rng = np.random.default_rng(seed + 100)
        bows, place = scene(rng, V, nrows, nplaces, nfeat)
        covis, ncov, conn = graph(rng, nrows, place)
        add, erase, db = database(rng, nrows)
        query = np.array([0, 3] + rng.integers(4, nrows, 14).tolist(), np.int32)
        _, W, S, _ = km.detect(bows, db, query, [covis[r, :ncov[r]].tolist() for r in range(nrows)], False, relocscore=np.zeros(nrows, f32))
        mx = W.max(1)
        on_integer += int(((mx % 5 == 0) & (mx > 0)).sum())
        below += int(((W > 0) & np.isnan(S)).sum())
    assert on_integer >= 1 and below >= 1
