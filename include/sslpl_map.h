/*
 * include/sslpl_map.h — map-element refresh of LocalMapping over keyframes resident in HBM (libsslpl_b200.so, csrc/match.cu).
 *
 * MapPoint::ComputeDistinctiveDescriptors / UpdateNormalAndDepth (MapPoint.cc:247-312, 335-376) and MapLine::ComputeDistinctiveDescriptors /
 * UpdateAverageDir (MapLine.cpp:246-317, 325-372), batched: one call rewrites in place the element rows that the batched Fuse calls of
 * sslpl.h read (d_mp[m][9] / d_ml[m][12] and the element descriptors), from the keyframe set and pose table the other batched LocalMapping
 * calls use.  So CreateNewMapPoints / CreateNewMapLines2 -> refresh -> Fuse needs no host round trip.  Conventions as in sslpl.h.
 */
#ifndef SSLPL_MAP_H
#define SSLPL_MAP_H
#include "sslpl.h"
#ifdef __cplusplus
extern "C" {
#endif

/* `what`: which of the two member functions an entry runs (both = 3) */
enum { SSLPL_MAPUPD_DESC = 1, SSLPL_MAPUPD_GEOM = 2 };
/* d_status[u] of entry u */
enum {
    SSLPL_MAPUPD_OK = 0,           /* everything requested was written */
    SSLPL_MAPUPD_NO_OBS = 1,       /* empty observation list: nothing written (MapPoint.cc:261, :350) */
    SSLPL_MAPUPD_NO_GOOD_KF = 2,   /* every observing keyframe is bad: descriptor left as it was (:274); geometry still written */
    SSLPL_MAPUPD_REF_OCTAVE = 3,   /* reference keyframe's feature octave outside [0, nlevels) (the reference reads mvScaleFactors out of
                                      bounds): normal written, the three distance fields left as they were.  Takes precedence over
                                      NO_GOOD_KF when both hold. */
    SSLPL_MAPUPD_BAD = -1          /* element / keyframe / feature index out of range, a keyframe twice in one list, or the element
                                      already listed earlier in this call: nothing written by this entry */
};

/* ---- The refresh of nupd elements.  Entry u names the element row d_elem[u], its mpRefKF d_refkf[u] (read only for GEOM; may be NULL
   for what = DESC) and its observations d_obs[2 * j] = (keyframe, feature index) for j in [d_obs_off[u], d_obs_off[u + 1]), int32;
   d_obs is read as 8-byte pairs and must be 8-byte aligned (SSLPL_ERR_ARG otherwise).
   The keyframe set is that of the batched Fuse calls (d_kps[k][cap] = mvKeysUn, d_desc[k][cap][32], d_n[k] clamped to cap; lines
   d_kl[k][capl] = mvKeyLines, d_ldesc, d_nl), d_kfpose[k][15] = Tcw then Ow (f32), d_kfbad[k] = KeyFrame::isBad() (NULL: none is bad).
   scaleFactors = mvScaleFactors (HOST, nlevels entries).

   Observation order is the caller's and stands for the order of mObservations (std::map<KeyFrame*, size_t>): keyframe creation order
   under a bump allocator.  It decides the medoid's tie-break and the summation order of the normal.
     Descriptor (DESC): the medoid of the rows of the observing keyframes that are not bad; row median = sorted[int(0.5 (N - 1))] of the
       N distances, the self-distance 0 included; the first least median wins (as sslpl_descriptor_medoid_batch).
     Geometry (GEOM), over every observation, bad keyframes included (UpdateNormalAndDepth does not skip them): the normal is the mean of
       the unit rays from each camera centre; mfMaxDistance = dist * scaleFactors[level] with dist = |Pos - Ow(refkf)| and level the
       octave of the reference keyframe's observed feature (feature 0 when refkf is not in the list: observations[pRefKF] default-inserts
       0); mfMinDistance = mfMaxDistance / scaleFactors[nlevels - 1].
   Points write d_mp[m][3..8] = normal, 0.8f * mfMinDistance, 1.2f * mfMaxDistance, mfMaxDistance, and d_mpdesc[m][32]; Xw (columns
   0..2) is read, never written.  Lines read mWorldPos from d_mlpos[m][6] (f64: UpdateAverageDir uses the double position for the normal
   and its float narrowing for the distances) and write d_ml[m][6..11] = the normal narrowed to float, the three distance fields, and
   d_mlnormal[m][3] = the double normal when d_mlnormal is not NULL; d_mldesc[m][32].
   An element listed again is written once, by its first entry; the later ones get SSLPL_MAPUPD_BAD.  A keyframe listed twice in one
   observation list is SSLPL_MAPUPD_BAD (mObservations cannot hold it), so a list has at most nkf entries.
   Numerics are those of the reference with cv2 4.13 (DESIGN.md): normal + normali / cv::norm(normali) is scaleAdd, one fused
   multiply-add with the scale narrowed to float; normal / n is convertTo with the scale 1.0 / n narrowed to float; the line normal is
   Eigen's double arithmetic without contraction.
   Asynchronous on the matcher's stream.  The first-entry table of the call (nmp / nml int32) lives in the handle's grow-only scratch
   and is freed with it.  nupd = 0 enqueues nothing.  Needs nkf in [1, max_batch + 1], cap in [1, max_features + 64] (capl in
   [1, max_lines + 64]), nlevels in [1, SSLPL_MAX_LEVELS], what in {1, 2, 3} and the pointers `what` reads; bad arguments return
   SSLPL_ERR_ARG and enqueue nothing. ---- */
int  sslpl_update_map_points_batch_device(sslpl_matcher* m,
        const sslpl_keypoint* d_kps, const uint8_t* d_desc, const int* d_n, int nkf, int cap,
        const float* d_kfpose, const uint8_t* d_kfbad,
        int nmp, float* d_mp, uint8_t* d_mpdesc,
        int nupd, const int32_t* d_elem, const int32_t* d_refkf, const int32_t* d_obs_off, const int32_t* d_obs,
        const float* scaleFactors, int nlevels, int what, int32_t* d_status);
int  sslpl_update_map_lines_batch_device(sslpl_matcher* m,
        const sslpl_keyline* d_kl, const uint8_t* d_ldesc, const int* d_nl, int nkf, int capl,
        const float* d_kfpose, const uint8_t* d_kfbad,
        int nml, const double* d_mlpos, float* d_ml, uint8_t* d_mldesc, double* d_mlnormal,
        int nupd, const int32_t* d_elem, const int32_t* d_refkf, const int32_t* d_obs_off, const int32_t* d_obs,
        const float* scaleFactors, int nlevels, int what, int32_t* d_status);

#ifdef __cplusplus
}
#endif
#endif /* SSLPL_MAP_H */
