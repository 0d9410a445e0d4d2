"""CPU: the sequence builder of tests/test_motion_batch_gpu.py, run on the oracle alone, yields frame pairs on both sides of
TrackWithMotionModel's retry threshold (Tracking.cc:1240-1244), so the GPU tests exercise both the first pass and the 2 * th rerun."""
import numpy as np

from test_motion_batch_gpu import RETRY, motion_sequence, oracle_motion_model, sequence_frames


def test_sequence_covers_both_sides_of_the_retry_threshold(oracle, synth):
    frames = sequence_frames(synth)
    orc = oracle.OrbOracle(1000, 1.2, 8, 20, 7)
    ex = [orc.extract(f) for f in frames]
    n = np.array([len(k) for k, _ in ex], np.int32)
    cap = int(n.max())
    kps = np.zeros((len(frames), cap), ex[0][0].dtype); desc = np.zeros((len(frames), cap, 32), np.uint8)
    for f, (k, d) in enumerate(ex):
        kps[f, :len(k)] = k; desc[f, :len(k)] = d
    assert n[4] == 0 and (np.delete(n, 4) > 500).all()
    seq = motion_sequence(kps, desc, n, seed=11)
    live = [p for p in range(len(frames) - 1) if p not in (3, 4)]                  # pairs 3 and 4 touch the flat frame
    for check_ori in (True, False):
        res = [oracle_motion_model(oracle, kps, desc, n, seq, p, 15.0, check_ori, RETRY) for p in range(len(frames) - 1)]
        final, first = np.array([r[0] for r in res]), np.array([r[2] for r in res])
        assert (final[[3, 4]] == 0).all()
        retried = [p for p in live if first[p] < RETRY]
        assert retried and len(retried) < len(live), first
        assert (final[retried] != first[retried]).all(), (first, final)         # the wider window changes those pairs' results
