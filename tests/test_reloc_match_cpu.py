"""CPU tests (no GPU): tests/reloc_model.py's SearchByProjection(Frame &F, KeyFrame *pKF, sAlreadyFound, th, ORBdist) against the
reference's own (ORBmatcher.cc:1475-1602), bit for bit, through tests/ref_reloc.cpp, which oracle/ref_reloc_build.sh compiles into
oracle/_ref/libref_reloc.so.  Skipped when that library is absent."""
import numpy as np
import pytest

import reloc_model as rm

SETTINGS = [(10, 100), (3, 64)]                          # Tracking.cc:2071, :2085


@pytest.fixture(scope="module")
def ref():
    if not rm.ref_available():
        pytest.skip("oracle/_ref/libref_reloc.so is not present")
    return rm


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("th,orb_dist", SETTINGS)
@pytest.mark.parametrize("check_ori", [True, False])
def test_model_equals_reference(oracle, synth, ref, seed, th, orb_dist, check_ori):
    S = rm.reloc_scene(oracle, synth, seed, f0=2 * seed)
    n_m, a_m = rm.scene_model(oracle, S, th, orb_dist, check_ori)
    n_r, a_r = rm.scene_ref(S, th, orb_dist, check_ori)
    assert n_m == n_r
    assert np.array_equal(rm.as_elements(S, a_m), a_r)
    assert n_m == int((a_m >= 0).sum()) and n_m > 10
    if check_ori:
        assert (a_m == -2).any() or seed > 0                  # the rotation check drops matches on this scene


def test_scene_covers_the_edges(oracle, synth, ref):
    """The scene reaches what the issue lists: bad / NULL / found, held, points behind the camera that are searched, both invariance
    edges, levels 0 and nlevels - 1 and the MapPoint shared by two keyframe indices."""
    S = rm.reloc_scene(oracle, synth, 0)
    el = rm.element_table(S["Xw"], S["mindist"], S["maxdist"])
    n, a = rm.scene_model(oracle, S, 10, 100, False)
    used = S["kfmp"][a[a >= 0]]
    assert (S["Xw"][used, 2] < 0).any()                      # behind the camera, matched
    e = S["kfmp"]
    assert len(e) - len(np.unique(e[e >= 0])) - (e < 0).sum() >= 1
    ratio = S["maxdist"] / np.linalg.norm(S["Xw"], axis=1)             # the frame moved by a few cm: close to the measured ratio
    assert (ratio < 0.95).any() and (ratio > 1.05 * rm.f32(1.2) ** 7).any()     # levels 0 and nlevels - 1
    assert (el[:, 7] > 0).all() and S["bad"].any() and S["found_el"].any() and S["held"].any()


@pytest.mark.parametrize("th,orb_dist", SETTINGS)
def test_camera_plane_points(oracle, synth, ref, th, orb_dist):
    """z = 0 in the frame: the projection is NaN (point at the centre) or inf; the reference finds no feature for either."""
    S = rm.reloc_scene(oracle, synth, 11, identity=True)
    n_m, a_m = rm.scene_model(oracle, S, th, orb_dist)
    n_r, a_r = rm.scene_ref(S, th, orb_dist)
    assert n_m == n_r and np.array_equal(rm.as_elements(S, a_m), a_r)
    assert not np.isin(S["kfmp"][a_m[a_m >= 0]], [0, 1]).any()


def test_reloc_pairs_model():
    cand = np.array([[5, 7, 9, -1], [3, -1, -1, -1], [-1, -1, -1, -1]], np.int32)
    P = rm.reloc_pairs(np.array([10, 11, 12], np.int32), cand, np.array([3, 1, -1], np.int32), 2)
    assert P.tolist() == [[5, 10], [7, 10], [3, 11], [-1, -1], [-1, -1], [-1, -1]]
