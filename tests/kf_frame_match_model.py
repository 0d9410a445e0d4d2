"""Per-pair model of the batched keyframe-to-frame matchers of include/sslpl.h, on the oracle (itself pinned to the reference in
tests/test_ref_parity_cpu.py):

- sslpl_search_by_bow_batch_device: ORBmatcher::SearchByBoW(KeyFrame* pKF, Frame& F, vector<MapPoint*>&) (ORBmatcher.cc:159-291) for a
  (keyframe row, frame row) pair of a row set, the keyframe's MapPoints given as element indices with isBad() flags;
- sslpl_match_lines_kf_batch_device: LSDmatcher::SearchByProjection(KeyFrame* pKF, Frame& F, vector<MapLine*>&) (LSDmatcher.cpp:143-183),
  the keyframe's MapLines given as element indices.

A row set is a dict of host arrays padded to the row capacity: points kps [nrows, cap] (KEYPOINT_DTYPE, mvKeysUn), desc [nrows, cap, 32],
n [nrows], kfmp [nrows, cap] i32, bad [nmp] u8 or None; lines ldesc [nrows, capl, 32], nl [nrows], kfml [nrows, capl] i32, nml."""
import numpy as np

LEVELSUP = 1                   # k = 10, L = 3 tree: FeatureVector nodes at level 2
VOCAB = dict(k=10, L=3, seed=21, stop_fraction=0.05, early_leaf_fraction=0.1)


def vocabulary_arrays(pkg):
    return pkg.Vocabulary.random_arrays(VOCAB["k"], VOCAB["L"], seed=VOCAB["seed"], stop_fraction=VOCAB["stop_fraction"],
                                        early_leaf_fraction=VOCAB["early_leaf_fraction"])


def feature_vector(oracle, voc_arrays, desc, levelsup=LEVELSUP, L=VOCAB["L"]):
    """Frame::ComputeBoW's FeatureVector of one row's descriptors: the node at level L - levelsup of each feature, stopped words (weight
    <= 0) left out (TemplatedVocabulary.h:1162-1166), as CSR (node ids, offsets, ascending feature indices)."""
    parent, nd, w, leaf = voc_arrays
    _, node, wt = oracle.vocab_transform(L, parent, nd, w, leaf, desc, levelsup)
    keep = np.nonzero(wt > 0)[0].astype(np.int32)
    ids, off, order = oracle.feature_vector_csr(node[keep])
    return ids, off, keep[order].astype(np.int32)


def clamp(n, cap):
    return int(min(max(int(n), 0), cap))


def element_state(kfmp_row, nmp, bad=None):
    """Per keyframe feature: 0 NULL (index outside [0, nmp)), 1 a good MapPoint, 2 a bad one (the state1 of oracle/ref.py)."""
    e = np.asarray(kfmp_row, np.int64)
    inside = (e >= 0) & (e < nmp)
    isbad = np.zeros(len(e), bool)
    if bad is not None and nmp > 0:
        isbad = np.asarray(bad, bool)[np.where(inside, e, 0)]
    return np.where(inside, np.where(isbad, 2, 1), 0).astype(np.uint8)


def pair_rows(pair, nrows):
    kr, fr = int(pair[0]), int(pair[1])
    return (kr, fr) if 0 <= kr < nrows and 0 <= fr < nrows else None


def search_by_bow(oracle, R, fv, pair, nnratio, check_ori):
    """(count, match[cap]) of one pair: match[j] = the keyframe feature matched to frame feature j or -1; (-1, all -1) for a pair with a
    row outside the set.  fv(row) gives the row's FeatureVector."""
    cap = R["desc"].shape[1]
    out = np.full(cap, -1, np.int32)
    rows = pair_rows(pair, len(R["n"]))
    if rows is None:
        return -1, out
    kr, fr = rows
    n1, n2 = clamp(R["n"][kr], cap), clamp(R["n"][fr], cap)
    valid1 = element_state(R["kfmp"][kr, :n1], R["nmp"], R["bad"]) == 1
    n, m = oracle.search_by_bow(R["desc"][kr, :n1], R["desc"][fr, :n2], fv(kr), fv(fr), valid1.astype(np.uint8), R["kps"][kr, :n1]["angle"],
                                R["kps"][fr, :n2]["angle"], nnratio, check_ori)
    out[:n2] = m
    return int(n), out


def line_match(oracle, R, pair):
    """(count, lmatch[capl]) of one pair: lmatch[tdx] = the last accepted qdx or -1; -1 and all -1 for a pair with a row outside the set
    and where the keyframe has lines and the frame fewer than 2."""
    capl = R["ldesc"].shape[1]
    out = np.full(capl, -1, np.int32)
    rows = pair_rows(pair, len(R["nl"]))
    if rows is None:
        return -1, out
    kr, fr = rows
    n1, n2 = clamp(R["nl"][kr], capl), clamp(R["nl"][fr], capl)
    if n1 == 0:
        return 0, out
    if n2 < 2:
        return -1, out
    has_ml1 = element_state(R["kfml"][kr, :n1], R["nml"]) != 0
    n, m = oracle.line_match(0, R["ldesc"][kr, :n1], R["ldesc"][fr, :n2], has_ml1.astype(np.uint8))
    out[:n2] = m
    return int(n), out


def element_maps(rng, n, cap, nel, p_null=0.15, p_out=0.03, twice=True):
    """A map [nrows, cap] of element indices drawn from a pool of nel shared by all rows (so rows share elements), with NULLs as -1 and as
    indices >= nel, and (twice) one element at two feature indices of each row."""
    nrows = len(n)
    M = rng.integers(0, nel, (nrows, cap)).astype(np.int32)
    u = rng.random((nrows, cap))
    M[u < p_null] = -1
    M[(u >= p_null) & (u < p_null + p_out)] = nel + rng.integers(0, 50)
    if twice:
        for r in range(nrows):
            if n[r] >= 8:
                M[r, 7] = M[r, 3] = abs(int(M[r, 3])) % nel
    return M
