// tests/ref_reloc.cpp — TEST INFRASTRUCTURE ONLY.
//
// A C entry point over the reference's own ORBmatcher::SearchByProjection(Frame &F, KeyFrame *pKF, sAlreadyFound, th, ORBdist)
// (src/ORBmatcher.cc:1475-1602), as compiled into oracle/_ref/libref.so.  oracle/ref_reloc_build.sh compiles this file against the
// reference's headers and the stand-ins of oracle/refshim/ with the flags of oracle/ref_build.sh and links it with libref.so;
// tests/test_reloc_match_cpu.py holds tests/reloc_model.py to it.
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <set>
#include <vector>
#include "refshim/minicv.hpp"

#define private public
#define protected public
#include "ORBextractor.h"
#include "ORBmatcher.h"
#include "Frame.h"
#include "KeyFrame.h"
#include "MapPoint.h"
#include "Map.h"
#include "KeyFrameDatabase.h"
#include "ORBVocabulary.h"
#undef private
#undef protected

using namespace StructureSLAM;

namespace {

cv::Mat desc_mat(const uint8_t* d, int n) { cv::Mat m(std::max(n, 0), 32, CV_8UC1); if (n > 0) memcpy(m.data, d, (size_t)n * 32); return m; }

// A Frame as the reference's constructor leaves it (Frame.cc:69-131) from already undistorted keypoints (cv::KeyPoint layout, 28 B each)
Frame* make_frame(ORBVocabulary* voc, int nlevels, float scaleFactor, const void* kps, int n, const uint8_t* desc, const float* Tcw12) {
    Frame* F = new Frame();
    ORBextractor ext(1000, scaleFactor, nlevels, 20, 7);          // the pyramid tables of the reference's own constructor (Frame.cc:77-83)
    F->mpORBvocabulary = voc; F->mpORBextractorLeft = nullptr; F->mpORBextractorRight = nullptr; F->mpLineSegment = nullptr;
    F->mTimeStamp = 0; F->mbf = 0; F->mb = 0; F->mThDepth = 0; F->mpReferenceKF = nullptr; F->dealWithLine = false; F->blurNumber = 0;
    F->mnId = Frame::nNextId++;
    F->mnScaleLevels = ext.GetLevels(); F->mfScaleFactor = ext.GetScaleFactor(); F->mfLogScaleFactor = log(F->mfScaleFactor);
    F->mvScaleFactors = ext.GetScaleFactors(); F->mvInvScaleFactors = ext.GetInverseScaleFactors();
    F->mvLevelSigma2 = ext.GetScaleSigmaSquares(); F->mvInvLevelSigma2 = ext.GetInverseScaleSigmaSquares();
    F->N = n;
    F->mvKeys.resize(n);
    if (n) memcpy((void*)F->mvKeys.data(), kps, (size_t)n * sizeof(cv::KeyPoint));
    F->mvKeysUn = F->mvKeys;
    F->mvuRight = std::vector<float>(n, -1); F->mvDepth = std::vector<float>(n, -1);
    F->mDescriptors = desc_mat(desc, n);
    F->mvpMapPoints = std::vector<MapPoint*>(n, static_cast<MapPoint*>(NULL));
    F->mvbOutlier = std::vector<bool>(n, false);
    F->NL = 0;
    F->mK = cv::Mat::eye(3, 3, CV_32F);
    F->mK.at<float>(0, 0) = Frame::fx; F->mK.at<float>(1, 1) = Frame::fy; F->mK.at<float>(0, 2) = Frame::cx; F->mK.at<float>(1, 2) = Frame::cy;
    F->mDistCoef = cv::Mat::zeros(4, 1, CV_32F);
    F->AssignFeaturesToGrid();                                     // Frame.cc:133-148
    cv::Mat T = cv::Mat::eye(4, 4, CV_32F);
    if (Tcw12) for (int i = 0; i < 3; i++) for (int j = 0; j < 4; j++) T.at<float>(i, j) = Tcw12[i * 4 + j];
    F->SetPose(T);                                                 // Frame.cc:217-233
    return F;
}

}  // namespace

extern "C" {

/* SearchByProjection(F, pKF, sAlreadyFound, th, ORBdist) with ORBmatcher(0.9, checkOri).  cam8 = fx, fy, cx, cy, mnMinX, mnMaxX, mnMinY,
   mnMaxY.  The keyframe has n1 features with keypoints kp1 (its mvKeysUn); feature i holds element kfmp[i] (-1: NULL).  Element m is a
   MapPoint with GetWorldPos() = Xw[m], mfMinDistance = mindist[m], mfMaxDistance = maxdist[m], descriptor eldesc[m], isBad() = bad[m],
   in sAlreadyFound when found[m].  The frame has n2 features (kp2, d2) with pose Tcw; held2[j] gives feature j a MapPoint of its own on
   entry (NULL = none).  assign2[j] = the element whose MapPoint ends in mvpMapPoints[j] (-1: none, -3: the held one); *seconds (may be
   NULL) = the wall time of the matcher call alone.  Returns the reference's return value. */
int ref_search_by_projection_kf(int n1, const void* kp1, const int32_t* kfmp, int nel, const float* Xw, const float* mindist,
                                const float* maxdist, const uint8_t* eldesc, const uint8_t* bad, const uint8_t* found,
                                int n2, const void* kp2, const uint8_t* d2, const uint8_t* held2, const float* Tcw, const float* cam8,
                                int nlevels, float scaleFactor, float th, int ORBdist, int checkOri, int32_t* assign2, double* seconds) {
    Frame::fx = cam8[0]; Frame::fy = cam8[1]; Frame::cx = cam8[2]; Frame::cy = cam8[3];
    Frame::invfx = 1.0f / cam8[0]; Frame::invfy = 1.0f / cam8[1];
    Frame::mnMinX = cam8[4]; Frame::mnMaxX = cam8[5]; Frame::mnMinY = cam8[6]; Frame::mnMaxY = cam8[7];
    Frame::mfGridElementWidthInv = static_cast<float>(FRAME_GRID_COLS) / static_cast<float>(Frame::mnMaxX - Frame::mnMinX);   // Frame.cc:96-97
    Frame::mfGridElementHeightInv = static_cast<float>(FRAME_GRID_ROWS) / static_cast<float>(Frame::mnMaxY - Frame::mnMinY);
    Frame::mbInitialComputations = false;
    ORBVocabulary voc;
    Map map;
    KeyFrameDatabase db(voc);
    std::vector<uint8_t> zero((size_t)std::max(n1, 1) * 32, 0);
    Frame* Fk = make_frame(&voc, nlevels, scaleFactor, kp1, n1, zero.data(), nullptr);
    KeyFrame* KF = new KeyFrame(*Fk, &map, &db);
    Frame* F = make_frame(&voc, nlevels, scaleFactor, kp2, n2, d2, Tcw);
    std::vector<MapPoint*> el(nel);
    std::set<MapPoint*> sFound;
    for (int m = 0; m < nel; m++) {
        cv::Mat P(3, 1, CV_32F);
        for (int c = 0; c < 3; c++) P.at<float>(c) = Xw[3 * m + c];
        MapPoint* p = new MapPoint(P, KF, &map);
        p->mfMinDistance = mindist[m]; p->mfMaxDistance = maxdist[m];
        desc_mat(eldesc + 32 * (size_t)m, 1).copyTo(p->mDescriptor);
        p->mbBad = bad[m] != 0;
        if (found[m]) sFound.insert(p);
        el[m] = p;
    }
    for (int i = 0; i < n1; i++) KF->mvpMapPoints[i] = kfmp[i] >= 0 ? el[kfmp[i]] : nullptr;
    const float far[3] = {0, 0, 100};
    cv::Mat Pf(3, 1, CV_32F);
    for (int c = 0; c < 3; c++) Pf.at<float>(c) = far[c];
    MapPoint* other = new MapPoint(Pf, KF, &map);
    if (held2) for (int j = 0; j < n2; j++) if (held2[j]) F->mvpMapPoints[j] = other;
    ORBmatcher matcher(0.9f, checkOri != 0);
    const auto t0 = std::chrono::steady_clock::now();
    const int n = matcher.SearchByProjection(*F, KF, sFound, th, ORBdist);
    if (seconds) *seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    for (int j = 0; j < n2; j++) {
        MapPoint* p = F->mvpMapPoints[j];
        assign2[j] = -1;
        if (p == other) assign2[j] = -3;
        else if (p) for (int m = 0; m < nel; m++) if (el[m] == p) { assign2[j] = m; break; }
    }
    for (MapPoint* p : el) delete p;
    delete other; delete KF; delete Fk; delete F;
    return n;
}

}  // extern "C"
