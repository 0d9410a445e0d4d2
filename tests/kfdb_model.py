"""NumPy restatement of the keyframe database calls of include/sslpl.h (sslpl_bow_vectors_batch_device, sslpl_bow_score_batch_device,
sslpl_detect_loop_candidates_batch_device, sslpl_detect_relocalization_candidates_batch_device): DBoW2's BowVector build with TF_IDF
weighting and L1 scoring, L1Scoring::score, and KeyFrameDatabase::DetectLoopCandidates / DetectRelocalizationCandidates
(src/KeyFrameDatabase.cc:81-314) over rows.  Doubles are summed sequentially (np.cumsum runs left to right), floats in float32."""
import numpy as np

f32 = np.float32
NAN32 = f32(np.nan)


def bow_vector(word, weight):
    """TemplatedVocabulary::transform's BowVector (TF_IDF, L1): stopped words (weight <= 0) left out, the weights of a word added in
    feature order, then every value divided by the sequential sum of |value| in ascending word order.  -> (words, values)."""
    acc = {}
    for w, v in zip(np.asarray(word).tolist(), np.asarray(weight, np.float64).tolist()):
        if v > 0:
            acc[w] = acc[w] + v if w in acc else v
    keys = np.array(sorted(acc), np.int32)
    vals = np.array([acc[k] for k in keys.tolist()], np.float64)
    if len(vals):
        norm = np.cumsum(np.abs(vals))[-1]
        if norm > 0:
            vals = vals / norm
    return keys, vals


def score(a, b):
    """L1Scoring::score(a, b) of two (words, values) BowVectors."""
    _, ia, ib = np.intersect1d(a[0], b[0], assume_unique=True, return_indices=True)
    if len(ia) == 0:
        return -0.0                                              # -score / 2.0 of score = 0
    vi, wi = a[1][ia], b[1][ib]
    t = (np.abs(vi - wi) - np.abs(vi)) - np.abs(wi)
    return -float(np.cumsum(t)[-1]) / 2.0


def _common(a, b):
    """(number of common words, index in a of the first common word)."""
    c, ia, _ = np.intersect1d(a[0], b[0], assume_unique=True, return_indices=True)
    return len(c), (int(ia.min()) if len(c) else -1)


def detect(bows, db, queries, covis, loop, conn=None, minscore=None, relocscore=None):
    """Both queries over rows.  bows[r] = (words, values); db = database rows in add order (erased ones left out); covis[r] = up to 10 rows
    (-1 / out of range: outside the database); loop: conn[q] = connected rows of query q, minscore[q]; reloc: relocscore[nrows] float32,
    the keyframes' mRelocScore before the first query.  -> (cand lists of rows, words [nq, ndb] i32, score [nq, ndb] f32 (NaN: not scored),
    relocscore after the last query)."""
    nrows, ndb, nq = len(bows), len(db), len(queries)
    pos = {int(r): p for p, r in enumerate(db)}
    state = None if loop else np.array(relocscore, f32).copy()
    cands, W, S = [], np.zeros((nq, ndb), np.int32), np.full((nq, ndb), NAN32, f32)
    if len(pos) != ndb or any(not 0 <= int(r) < nrows for r in db):
        return [None] * nq, W, S, state
    for q, qr in enumerate(queries):
        if not 0 <= int(qr) < nrows:
            cands.append(None)
            continue
        qb = bows[int(qr)]
        connected = {pos[int(r)] for r in (conn[q] if loop else ()) if int(r) in pos}
        listed = []                                              # (first common word, position)
        for p, r in enumerate(db):
            if p in connected:
                continue
            n, first = _common(qb, bows[int(r)])
            if n:
                W[q, p] = n
                listed.append((first, p))
        listed.sort()
        if not listed:
            cands.append([])
            continue
        minw = int(f32(W[q].max()) * f32(0.8))
        ms = f32(minscore[q]) if loop else f32(0)
        entries = []
        for _, p in listed:
            if W[q, p] > minw:
                si = f32(score(qb, bows[int(db[p])]))
                S[q, p] = si
                if not loop or si >= ms:
                    entries.append((si, p))

        def neighbour_score(p2):
            if W[q, p2] > minw:
                return S[q, p2]
            return state[int(db[p2])]

        acc_list, best_acc = [], ms
        for si, p in entries:
            acc, best_s, best_p = si, si, p
            for r2 in covis[int(db[p])]:
                p2 = pos.get(int(r2), -1) if 0 <= int(r2) < nrows else -1
                if p2 < 0 or W[q, p2] == 0 or (loop and W[q, p2] <= minw):
                    continue
                s2 = neighbour_score(p2)
                acc = f32(acc + s2)
                if s2 > best_s:
                    best_s, best_p = s2, p2
            acc_list.append((acc, best_p))
            if acc > best_acc:
                best_acc = acc
        keep = f32(f32(0.75) * best_acc)
        out, seen = [], set()
        for acc, bp in acc_list:
            if acc > keep and bp not in seen:
                seen.add(bp)
                out.append(int(db[bp]))
        cands.append(out)
        if not loop:
            for p in range(ndb):
                if not np.isnan(S[q, p]):
                    state[int(db[p])] = S[q, p]
    return cands, W, S, state
