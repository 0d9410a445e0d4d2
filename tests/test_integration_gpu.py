"""GPU: the drop-in claim, end to end.  oracle/_ref/ref_link_test (built by build(), oracle/ref_link_build.sh) is linked from the reference's OWN unmodified translation
units (Frame.cc, KeyFrame.cc, MapPoint.cc, MapLine.cpp, Map.cc, KeyFrameDatabase.cc, ORBmatcher.cc, LSDmatcher.cpp, DBoW2), the
adapters of structure-slam-pointline_b200/host/ (tests/integration/ref_link_test.cpp) and libsslpl_b200.so.  It runs Frame::Frame,
ComputeBoW, KeyFrame, ORBmatcher::SearchByBoW / SearchByProjection and LSDmatcher::SearchByProjection the way Tracking does; what it
produced through the GPU is compared here with the fixtures frozen from the reference and with oracle/_ref (the reference on the CPU)."""
import os
import subprocess
import numpy as np
import pytest

from conftest import ROOT
from test_ref_golden_cpu import load
from test_ref_parity_cpu import write_vocab_text

pytestmark = pytest.mark.gpu
BIN = os.path.join(ROOT, "oracle", "_ref", "ref_link_test")


def test_reference_objects_plus_adapters_on_the_gpu(pkg, oracle, icl_gray, tmp_path):
    if not os.path.exists(BIN):
        pytest.skip("oracle/_ref/ref_link_test not built (build() builds it where the reference's sources are present)")
    from oracle import ref as R
    if not R.available():
        pytest.skip("oracle/_ref not built")
    img2 = np.ascontiguousarray(np.roll(icl_gray, 2, axis=1))
    icl_gray.tofile(tmp_path / "a.raw"); img2.tofile(tmp_path / "b.raw")
    parent, nd, w, leaf = pkg.Vocabulary.random_arrays(10, 3, seed=5)
    voc_path = str(tmp_path / "voc.txt")
    write_vocab_text(voc_path, 10, 3, parent, nd, w, leaf)
    out = tmp_path / "out"; out.mkdir()
    r = subprocess.run([BIN, str(tmp_path / "a.raw"), str(tmp_path / "b.raw"), "640", "480", voc_path, str(out)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    L = lambda n: np.load(out / f"{n}.npy")
    KP = pkg.KEYPOINT_DTYPE
    k1 = L("f1_keys").view(KP); d1 = L("f1_desc"); k2 = L("f2_keys").view(KP); d2 = L("f2_desc")
    # Frame::Frame through the adapters == the reference's own Frame constructor (fixtures from oracle/_ref)
    g = load("ref_orb.npz"); gf = load("ref_frame.npz")
    assert k1.tobytes() == g["orb_icl1000_kps"].tobytes() and np.array_equal(d1, g["orb_icl1000_desc"])
    assert L("f1_keysun").tobytes() == L("f1_keys").tobytes()
    assert np.array_equal(L("f1_ldesc"), gf["ldesc"]) and np.allclose(L("f1_lineeq"), gf["lineeq"], rtol=1e-9, atol=1e-9)
    kl = L("f1_keylines").view(pkg.KEYLINE_DTYPE)
    assert np.array_equal(kl["numOfPixels"], gf["keylines"]["numOfPixels"]) and np.max(np.abs(kl["startPointX"] - gf["keylines"]["startPointX"])) <= 1e-4
    # Frame::ComputeBoW == DBoW2 on the CPU
    voc = R.Vocabulary(voc_path)
    node1, _, _ = voc.transform(d1, 4); node2, _, _ = voc.transform(d2, 4)
    assert np.array_equal(L("f1_node"), node1) and np.array_equal(L("f2_node"), node2)
    # ORBmatcher::SearchByBoW(KeyFrame*, Frame&) through the adapter == the reference's body
    fv1 = oracle.feature_vector_csr(node1); fv2 = oracle.feature_vector_csr(node2)
    state1 = L("state1")
    n_r, m_r = R.search_by_bow(d1, k1, d2, k2, fv1, fv2, state1, 0.7, True)
    got = L("bow_match2")
    assert got[-1] == n_r and np.array_equal(got[:-1], m_r) and n_r > 100
    # ORBmatcher::SearchByProjection(Frame&, const Frame&) through the adapter
    valid = (state1 > 0).astype(np.uint8)           # bad MapPoints are still projected (the reference does not test isBad here)
    last = dict(valid=valid, obs=valid, Xw=L("proj_Xw"), dmp=d1, kps=k1)
    cur = dict(desc=d2, kps=k2, claimed=None)
    Tcw = L("proj_Tcw").reshape(3, 4); Tlw = np.eye(4, dtype=np.float32)[:3]
    camv = R.cam(481.2, 480.0, 319.5, 239.5, 0, 640, 0, 480)
    n_r, a_r = R.search_by_projection_frame(last, cur, Tcw, Tlw, camv, 8, 1.2, 15.0, True, True)
    got = L("proj_assign2")
    assert got[-1] == n_r and np.array_equal(got[:-1], np.where(a_r == -2, -1, a_r)) and n_r > 100
    # LSDmatcher::SearchByProjection(KeyFrame*, Frame&) through the adapter
    n_r, m_r, _ = R.line_match(0, L("f1_ldesc"), L("f2_ldesc"), L("has_ml1"), None)
    got = L("line_match2")
    assert got[-1] == n_r and np.array_equal(got[:-1], m_r)
    # ---- SURVEY.md 8(f) row 3 through the adapters, against the reference's own bodies (oracle/_ref) on the inputs the program dumped
    state = L("state1")
    mp = dict(state=state, nobs=np.ones(len(state), np.int32), Xw=L("proj_Xw"), normal=L("fuse_normal"), min_raw=L("fuse_dmin"), max_raw=L("fuse_dmax"), desc=d1)
    kf = dict(desc=d2, kps=k2, uright=None, kfobs=L("fuse_kfobs"))
    n_r, f_r, _ = R.fuse_points(mp, kf, np.vstack([Tcw, [0, 0, 0, 1]]).astype(np.float32), camv, 0.0, 8, 1.2, 3.0)
    got = L("fuse_idx")
    assert got[-1] == n_r and np.array_equal(got[:-1], f_r) and n_r > 300, (got[-1], n_r, int((got[:-1] != f_r).sum()))
    kl2 = L("f2_keylines").view(pkg.KEYLINE_DTYPE)
    cur = dict(ld=L("f2_ldesc"), kl=np.stack([kl2["pt_x"], kl2["pt_y"], kl2["angle"]], 1), oct=kl2["octave"].astype(np.int32), held=None)
    ls = L("lfuse_state")
    ml = dict(inview=np.array([(i % 11 != 7) for i in range(len(ls))], np.uint8) * (ls > 0), bad=(ls == 2).astype(np.uint8), obs=(ls > 0).astype(np.uint8),
              proj=L("lproj"), level=np.zeros(len(ls), np.int32), viewcos=np.where(np.arange(len(ls)) % 2, 0.9999, 0.9).astype(np.float32), desc=L("f1_ldesc"))
    keep = np.nonzero(ls > 0)[0]                                       # the program passes NULL for the others; the harness has no NULL entries
    mlk = {k: v[keep] for k, v in ml.items()}
    n_r, a_r = R.line_projection_mls(mlk, cur, camv, 8, 1.2, 0.8, 3.0)
    got = L("lproj_assign2")
    assert got[-1] == n_r and np.array_equal(got[:-1], np.where(a_r >= 0, keep[np.maximum(a_r, 0)], -1)) and n_r > 5, (got[-1], n_r)
    mlf = dict(state=np.where(ls == 1, 1, np.where(ls == 2, 2, 0)).astype(np.uint8), nobs=np.ones(len(ls), np.int32), Pw=L("lfuse_pw"), normal=L("lfuse_normal"),
               min_raw=L("lfuse_dmin"), max_raw=L("lfuse_dmax"), desc=L("f1_ldesc"))
    kfl = dict(ld=cur["ld"], kl=cur["kl"], oct=cur["oct"], kfobs=L("lfuse_kfobs"))
    n_r, f_r, _ = R.fuse_lines(mlf, kfl, np.vstack([Tcw, [0, 0, 0, 1]]).astype(np.float32), camv, 8, 1.2, 10.0)
    got = L("lfuse_idx")
    assert got[-1] == n_r and np.array_equal(got[:-1], f_r) and n_r > 5, (got[-1], n_r, int((got[:-1] != f_r).sum()))
