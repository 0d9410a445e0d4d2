// tests/ref_map_update.cpp — TEST INFRASTRUCTURE ONLY.
//
// C entry points over the reference's own MapPoint::ComputeDistinctiveDescriptors / UpdateNormalAndDepth and MapLine::
// ComputeDistinctiveDescriptors / UpdateAverageDir, as compiled into oracle/_ref/libref.so.  tests/test_map_update_ref_cpu.py compiles
// this file against the reference's headers and the stand-ins of oracle/refshim/ with the flags of oracle/ref_build.sh, links it with
// libref.so, and holds tests/map_update_model.py (with the stand-in's rounding) to it.
//
// Every call builds the keyframes as the reference would hold them (a Frame of the given features, then KeyFrame(F, map, db)), with the
// given camera centre as Ow.  mObservations is a std::map keyed by KeyFrame*: the keyframes are constructed in one block in index
// order, so that index order is the map's order, as under the bump allocator of the canonical definition.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>
#include "refshim/minicv.hpp"

#define private public
#define protected public
#include "Frame.h"
#include "KeyFrame.h"
#include "MapPoint.h"
#include "MapLine.h"
#include "Map.h"
#include "KeyFrameDatabase.h"
#include "ORBVocabulary.h"
#undef private
#undef protected

using namespace StructureSLAM;

namespace {

struct Scene {
    Map map; ORBVocabulary voc; KeyFrameDatabase db;
    std::vector<Frame*> frames; std::vector<KeyFrame*> kfs;
    char* slab;                                       // the keyframes, one after the other
    explicit Scene(int nkf) : db(voc), slab(static_cast<char*>(::operator new((size_t)nkf * sizeof(KeyFrame)))) {}
    ~Scene() { for (auto p : kfs) p->~KeyFrame(); ::operator delete(slab); for (auto p : frames) delete p; }
};

cv::Mat desc_mat(const uint8_t* d, int n) { cv::Mat m(std::max(n, 0), 32, CV_8UC1); if (n > 0) memcpy(m.data, d, (size_t)n * 32); return m; }

// keyframe k: n[k] features (points: mvKeysUn octaves and mDescriptors; lines: mvKeyLines octaves and mLineDescriptors), the pyramid
// table, pose[k][15] = Tcw (3x4), Ow (set as KeyFrame::Ow after construction), bad[k] = mbBad.  Keyframe k lies at a lower address
// than keyframe k + 1, so mObservations iterates in index order.
std::vector<KeyFrame*> keyframes(Scene& S, int nkf, int cap, const int32_t* n, const int32_t* octave, const uint8_t* desc, bool lines,
                                 const float* pose, const uint8_t* bad, const float* scale, int nlevels) {
    Frame::fx = 500.f; Frame::fy = 500.f; Frame::cx = 320.f; Frame::cy = 240.f; Frame::invfx = 1.f / 500.f; Frame::invfy = 1.f / 500.f;
    Frame::mnMinX = 0.f; Frame::mnMaxX = 640.f; Frame::mnMinY = 0.f; Frame::mnMaxY = 480.f;
    Frame::mfGridElementWidthInv = FRAME_GRID_COLS / 640.f; Frame::mfGridElementHeightInv = FRAME_GRID_ROWS / 480.f;
    Frame::mbInitialComputations = false;
    for (int k = 0; k < nkf; k++) {
        Frame* F = new Frame();
        S.frames.push_back(F);
        F->mpORBvocabulary = &S.voc; F->mpORBextractorLeft = nullptr; F->mpORBextractorRight = nullptr; F->mpLineSegment = nullptr;
        F->mTimeStamp = 0; F->mbf = 0; F->mb = 0; F->mThDepth = 0; F->mpReferenceKF = nullptr; F->dealWithLine = true; F->blurNumber = 0;
        F->mnId = Frame::nNextId++;
        F->mnScaleLevels = nlevels; F->mfScaleFactor = nlevels > 1 ? scale[1] : 1.f; F->mfLogScaleFactor = log(F->mfScaleFactor);
        F->mvScaleFactors.assign(scale, scale + nlevels);
        F->mvInvScaleFactors.resize(nlevels); F->mvLevelSigma2.resize(nlevels); F->mvInvLevelSigma2.resize(nlevels);
        for (int l = 0; l < nlevels; l++) {
            F->mvInvScaleFactors[l] = 1.f / scale[l]; F->mvLevelSigma2[l] = scale[l] * scale[l]; F->mvInvLevelSigma2[l] = 1.f / F->mvLevelSigma2[l];
        }
        const int np = lines ? 0 : n[k], nl = lines ? n[k] : 0;
        F->N = np;
        F->mvKeys.assign(np, cv::KeyPoint());
        for (int i = 0; i < np; i++) { F->mvKeys[i].pt.x = 10.f; F->mvKeys[i].pt.y = 10.f; F->mvKeys[i].octave = octave[(size_t)k * cap + i]; }
        F->mvKeysUn = F->mvKeys;
        F->mvuRight = std::vector<float>(np, -1); F->mvDepth = std::vector<float>(np, -1);
        F->mDescriptors = desc_mat(lines ? nullptr : desc + (size_t)k * cap * 32, np);
        F->mvpMapPoints = std::vector<MapPoint*>(np, static_cast<MapPoint*>(NULL));
        F->mvbOutlier = std::vector<bool>(np, false);
        F->NL = nl;
        F->mLdesc = desc_mat(lines ? desc + (size_t)k * cap * 32 : nullptr, nl);
        F->mvKeylinesUn.resize(nl); F->mvKeyLineFunctions.resize(nl);
        for (int i = 0; i < nl; i++) F->mvKeylinesUn[i].octave = octave[(size_t)k * cap + i];
        F->mvpMapLines = std::vector<MapLine*>(nl, static_cast<MapLine*>(NULL));
        F->mvbLineOutlier = std::vector<bool>(nl, false);
        F->mK = cv::Mat::eye(3, 3, CV_32F);
        F->mK.at<float>(0, 0) = 500.f; F->mK.at<float>(1, 1) = 500.f; F->mK.at<float>(0, 2) = 320.f; F->mK.at<float>(1, 2) = 240.f;
        F->mDistCoef = cv::Mat::zeros(4, 1, CV_32F);
        cv::Mat T = cv::Mat::eye(4, 4, CV_32F);
        for (int i = 0; i < 3; i++) for (int j = 0; j < 4; j++) T.at<float>(i, j) = pose[15 * k + 4 * i + j];
        F->SetPose(T);
        KeyFrame* K = new (S.slab + (size_t)k * sizeof(KeyFrame)) KeyFrame(*F, &S.map, &S.db);   // ascending addresses
        S.kfs.push_back(K);
        for (int c = 0; c < 3; c++) K->Ow.at<float>(c) = pose[15 * k + 12 + c];   // the camera centre as given
        K->mbBad = bad && bad[k];
    }
    return S.kfs;
}

}  // namespace

extern "C" {

/* MapPoint::ComputeDistinctiveDescriptors (what & 1) and UpdateNormalAndDepth (what & 2) of nel MapPoints: element e at X[e][3], mpRefKF
   refkf[e], observations obs[2 j] = (kf, idx) for j in [off[e], off[e + 1]).  Out: desc[e][32] and has_desc[e] (mDescriptor set),
   geom[e][6] = mNormalVector, GetMinDistanceInvariance(), GetMaxDistanceInvariance(), mfMaxDistance. */
void ref_update_map_points(int nkf, int cap, const int32_t* n, const int32_t* octave, const uint8_t* desc, const float* pose, const uint8_t* bad,
                           const float* scale, int nlevels, int nel, const float* X, const int32_t* refkf, const int32_t* off, const int32_t* obs,
                           int what, uint8_t* out_desc, uint8_t* has_desc, float* geom) {
    Scene S(nkf);
    std::vector<KeyFrame*> K = keyframes(S, nkf, cap, n, octave, desc, false, pose, bad, scale, nlevels);
    for (int e = 0; e < nel; e++) {
        cv::Mat P(3, 1, CV_32F);
        for (int c = 0; c < 3; c++) P.at<float>(c) = X[3 * e + c];
        MapPoint* p = new MapPoint(P, K[refkf[e]], &S.map);
        for (int j = off[e]; j < off[e + 1]; j++) p->AddObservation(K[obs[2 * j]], obs[2 * j + 1]);
        if (what & 1) p->ComputeDistinctiveDescriptors();
        if (what & 2) p->UpdateNormalAndDepth();
        has_desc[e] = !p->mDescriptor.empty();
        if (has_desc[e]) memcpy(out_desc + 32 * (size_t)e, p->mDescriptor.data, 32);
        for (int c = 0; c < 3; c++) geom[6 * e + c] = p->mNormalVector.at<float>(c);
        geom[6 * e + 3] = p->GetMinDistanceInvariance(); geom[6 * e + 4] = p->GetMaxDistanceInvariance(); geom[6 * e + 5] = p->mfMaxDistance;
        delete p;
    }
}

/* MapLine::ComputeDistinctiveDescriptors and UpdateAverageDir of nel MapLines at pos[e][6] (double).  Out as for points, plus
   normal[e][3] = the double mNormalVector (geom holds it narrowed to float). */
void ref_update_map_lines(int nkf, int cap, const int32_t* n, const int32_t* octave, const uint8_t* desc, const float* pose, const uint8_t* bad,
                          const float* scale, int nlevels, int nel, const double* pos, const int32_t* refkf, const int32_t* off, const int32_t* obs,
                          int what, uint8_t* out_desc, uint8_t* has_desc, float* geom, double* normal) {
    Scene S(nkf);
    std::vector<KeyFrame*> K = keyframes(S, nkf, cap, n, octave, desc, true, pose, bad, scale, nlevels);
    for (int e = 0; e < nel; e++) {
        Vector6d P;
        for (int c = 0; c < 6; c++) P(c) = pos[6 * e + c];
        MapLine* l = new MapLine(P, K[refkf[e]], &S.map);
        for (int j = off[e]; j < off[e + 1]; j++) l->AddObservation(K[obs[2 * j]], obs[2 * j + 1]);
        if (what & 1) l->ComputeDistinctiveDescriptors();
        if (what & 2) l->UpdateAverageDir();
        has_desc[e] = !l->mLDescriptor.empty();
        if (has_desc[e]) memcpy(out_desc + 32 * (size_t)e, l->mLDescriptor.data, 32);
        for (int c = 0; c < 3; c++) { normal[3 * e + c] = l->mNormalVector(c); geom[6 * e + c] = (float)l->mNormalVector(c); }
        geom[6 * e + 3] = l->GetMinDistanceInvariance(); geom[6 * e + 4] = l->GetMaxDistanceInvariance(); geom[6 * e + 5] = l->mfMaxDistance;
        delete l;
    }
}

}  // extern "C"
