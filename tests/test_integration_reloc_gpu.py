"""GPU: ORBmatcher::SearchByProjection(Frame&, KeyFrame*, sAlreadyFound, th, ORBdist) inside the linked reference build.
oracle/_ref/ref_link_reloc_test (oracle/ref_link_reloc_build.sh, run by build() where the reference's sources are present) links the
reference's own objects, with ORBmatcher.cc's symbols weak, the adapters of structure-slam-pointline_b200/host/ and libsslpl_b200.so.  It
builds the reference's Frame, KeyFrame and MapPoints of a scene (tests/ref_reloc.cpp), calls the overload, which runs the adapter of
host/matcher_b200.cc on the GPU (flags from isBad() and sAlreadyFound, fields from the MapPoint accessors, mvpMapPoints written back), and
reports which MapPoint each frame feature holds.  That must equal tests/reloc_model.py and, where oracle/_ref/libref_reloc.so is present,
the reference's own matcher on the same scene."""
import os
import subprocess

import numpy as np
import pytest

import reloc_model as rm

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "oracle", "_ref", "ref_link_reloc_test")


def write_scene(path, S, th, orb_dist, check_ori):
    n1, nel, n2 = len(S["kfmp"]), len(S["Xw"]), len(S["kps"])
    cam8 = list(rm.CAM) + list(rm.BOUNDS)
    with open(path, "wb") as f:
        np.array([n1, nel, n2, len(rm.SF), orb_dist, int(check_ori)], np.int32).tofile(f)
        np.array([th, 1.2] + cam8 + list(np.asarray(S["Tcw"], np.float32).reshape(-1)[:12]), np.float32).tofile(f)
        np.ascontiguousarray(S["kf_kps"]).tofile(f)
        for a, t in ((S["kfmp"], np.int32), (S["Xw"], np.float32), (S["mindist"], np.float32), (S["maxdist"], np.float32),
                     (S["eldesc"], np.uint8), (S["bad"], np.uint8), (S["found_el"], np.uint8), (S["held"], np.uint8)):
            np.ascontiguousarray(a, t).tofile(f)
        np.ascontiguousarray(S["kps"]).tofile(f)
        np.ascontiguousarray(S["desc"], np.uint8).tofile(f)


@pytest.mark.parametrize("seed,identity", [(0, False), (1, False), (11, True)])
@pytest.mark.parametrize("th,orb_dist,check_ori", [(10, 100, True), (3, 64, True), (10, 100, False)])
def test_adapter_inside_the_reference_build(oracle, synth, tmp_path, seed, identity, th, orb_dist, check_ori):
    if not os.path.exists(BIN):
        pytest.skip("oracle/_ref/ref_link_reloc_test not built (build() builds it where the reference's sources are present)")
    S = rm.reloc_scene(oracle, synth, seed, f0=2 * seed, identity=identity)
    write_scene(tmp_path / "scene.bin", S, th, orb_dist, check_ori)
    r = subprocess.run([BIN, str(tmp_path / "scene.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    out = np.fromfile(tmp_path / "out.bin", np.int32)
    n_g, a_g = int(out[0]), out[1:]
    n_m, a_m = rm.scene_model(oracle, S, th, orb_dist, check_ori)
    assert n_g == n_m and np.array_equal(a_g, rm.as_elements(S, a_m))
    assert (a_g == -3).sum() == int(S["held"].sum())              # what the frame held on entry stays
    if rm.ref_available():
        n_r, a_r = rm.scene_ref(S, th, orb_dist, check_ori)
        assert n_g == n_r and np.array_equal(a_g, a_r)
