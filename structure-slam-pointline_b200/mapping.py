"""LocalMapping's map-element refresh over keyframes in HBM (include/sslpl_map.h): MapPoint::ComputeDistinctiveDescriptors /
UpdateNormalAndDepth and MapLine::ComputeDistinctiveDescriptors / UpdateAverageDir, batched.  Like the Matcher's *_batch_device methods,
these take a Matcher and raw device pointers and enqueue on the matcher's stream."""
from . import _check, _f32, _p, lib

DESC, GEOM = 1, 2                                       # `what`: SSLPL_MAPUPD_DESC, SSLPL_MAPUPD_GEOM (both = 3)
OK, NO_OBS, NO_GOOD_KF, REF_OCTAVE, BAD = 0, 1, 2, 3, -1  # d_status: SSLPL_MAPUPD_*


def update_map_points(mt, d_kps, d_desc, d_n, nkf, cap, d_kfpose, d_kfbad, nmp, d_mp, d_mpdesc, nupd, d_elem, d_refkf, d_obs_off, d_obs,
                      scale_factors, what, d_status):
    """sslpl_update_map_points_batch_device.  The keyframe set d_kps / d_desc / d_n (mvKeysUn, cap rows each), d_kfpose [nkf, 15] f32
    (Tcw 3x4, Ow), d_kfbad [nkf] u8 or 0; the Fuse tables d_mp [nmp, 9] f32 and d_mpdesc [nmp, 32] u8, rewritten in place; per entry
    d_elem [nupd], d_refkf [nupd] (0 allowed with what = DESC), d_obs_off [nupd + 1] and d_obs [.., 2] (keyframe, feature) i32;
    scale_factors a host array (nlevels = len) -> d_status [nupd] i32."""
    sf = _f32(scale_factors)
    _check(lib().sslpl_update_map_points_batch_device(
        mt._h, d_kps, d_desc, d_n, nkf, cap, d_kfpose, d_kfbad or None, nmp, d_mp, d_mpdesc, nupd, d_elem, d_refkf or None, d_obs_off,
        d_obs, _p(sf), len(sf), what, d_status))


def update_map_lines(mt, d_kl, d_ldesc, d_nl, nkf, capl, d_kfpose, d_kfbad, nml, d_mlpos, d_ml, d_mldesc, d_mlnormal, nupd, d_elem,
                     d_refkf, d_obs_off, d_obs, scale_factors, what, d_status):
    """sslpl_update_map_lines_batch_device.  As update_map_points over the line keyframe set (d_kl / d_ldesc / d_nl as
    sslpl_line_device_results gives them), with mWorldPos d_mlpos [nml, 6] f64 (read only), d_ml [nml, 12] f32, d_mldesc [nml, 32] u8
    and d_mlnormal [nml, 3] f64 or 0 for the double normal."""
    sf = _f32(scale_factors)
    _check(lib().sslpl_update_map_lines_batch_device(
        mt._h, d_kl, d_ldesc, d_nl, nkf, capl, d_kfpose, d_kfbad or None, nml, d_mlpos, d_ml, d_mldesc, d_mlnormal or None, nupd, d_elem,
        d_refkf or None, d_obs_off, d_obs, _p(sf), len(sf), what, d_status))
