"""The batched initialisation matchers (sslpl_search_for_initialization_batch_device, sslpl_line_search_for_initialize_batch_device) as a
per-pair model over a host row set: R = dict(kps [nrows, cap] KEYPOINT_DTYPE, desc [nrows, cap, 32], n [nrows], ldesc [nrows, capl, 32],
nl [nrows]).  A chain (a maximal run of consecutive pairs with the same init row) calls SearchForInitialization pair after pair with
vbPrevMatched carried, starting from prev0 or the init row's keypoints; a bad pair (a row outside the set, or current row == init row)
gives -1 and leaves the chain's state alone.  Lines are LSDmatcher::SerachForInitialize per pair with the batched call's -1 / 0
conventions.  `call` is any function with the signature of oracle.search_for_initialization (the oracle, the reference, the single
device call)."""
import numpy as np


def clamp(n, cap):
    return max(0, min(int(n), cap))


def chain_starts(pairs):
    return [p for p in range(len(pairs)) if p == 0 or pairs[p - 1][0] != pairs[p][0]]


def points(call, R, pairs, bounds, nnratio=0.9, check_ori=True, window=100, prev0=None):
    """-> list over pairs of (nmatch, match12 [cap] (-1 past n1), prev [n1, 2] after the pair); (-1, None, None) for a bad pair."""
    nrows, cap = R["desc"].shape[:2]
    out = []
    for p, (r1, r2) in enumerate(pairs):
        if p == 0 or pairs[p - 1][0] != r1:
            ok1 = 0 <= r1 < nrows
            n1 = clamp(R["n"][r1], cap) if ok1 else 0
            if ok1:
                k1 = R["kps"][r1, :n1]
                state = (np.asarray(prev0[p], np.float32)[:n1] if prev0 is not None else np.stack([k1["x"], k1["y"]], 1)).copy()
        if not ok1 or not 0 <= r2 < nrows or r2 == r1:
            out.append((-1, None, None))
            continue
        n2 = clamp(R["n"][r2], cap)
        n, m12, state = call(R["desc"][r1, :n1], R["kps"][r1, :n1], R["desc"][r2, :n2], R["kps"][r2, :n2], state, bounds, nnratio,
                             check_ori, window)
        row = np.full(cap, -1, np.int32)
        row[:n1] = m12
        state = np.asarray(state, np.float32).reshape(-1, 2).copy()
        out.append((int(n), row, state))
    return out


def lines(oracle, R, pair):
    """-> (nlmatch, lpairs [capl, 2] with (-1, -1) after the count)."""
    nrows, capl = R["ldesc"].shape[:2]
    rows = np.full((capl, 2), -1, np.int32)
    r1, r2 = pair
    if not (0 <= r1 < nrows and 0 <= r2 < nrows):
        return -1, rows
    n1, n2 = clamp(R["nl"][r1], capl), clamp(R["nl"][r2], capl)
    if n1 == 0:
        return 0, rows
    if n2 < 2:                                  # knnMatch would leave lmatches[i][1] undefined (LSDmatcher.cpp:276)
        return -1, rows
    n, m = oracle.line_match(1, R["ldesc"][r1, :n1], R["ldesc"][r2, :n2])
    rows[:len(m)] = m
    return int(n), rows
