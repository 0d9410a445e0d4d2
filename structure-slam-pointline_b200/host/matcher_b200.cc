// host/matcher_b200.cc — GPU-backed bodies for the Hamming entry points of the reference's matchers.  Compiled inside
// the reference tree against ITS headers (ORBmatcher.h, LSDmatcher.h, Frame.h, KeyFrame.h, MapPoint.h, MapLine.h):
// the class declarations stay untouched; in src/ORBmatcher.cc and src/LSDmatcher.cpp the bodies of the functions
// below are deleted (or #if 0'ed) and this file is added to the source list (INTEGRATION.md).
//
// The GPU side works on indices + validity masks; this adapter maps KeyFrame*/MapPoint* data to flat arrays and the
// index tables back to pointers.  The matchers are constructed on the stack and called concurrently from the Tracking
// and LocalMapping threads (Tracking.cc:1323, LocalMapping.cc:91): one sslpl_matcher per thread (thread_local).
#include "ORBmatcher.h"
#include "LSDmatcher.h"
#include "sslpl.h"
#include <mutex>
#include <set>
#include <stdexcept>
#include <string>

namespace StructureSLAM
{
namespace {
struct MatcherCtx {
    sslpl_matcher* h;
    MatcherCtx(): h(NULL) {
        sslpl_matcher_params p; p.max_features = 8192; p.max_lines = 1024; p.max_nodes = 100000; p.max_batch = 1; p.device = sslpl_default_device();
        if(sslpl_matcher_create(&p, &h) != SSLPL_OK) throw std::runtime_error(std::string("sslpl_matcher_create: ") + sslpl_last_error());
    }
    ~MatcherCtx() { sslpl_matcher_destroy(h); }
};
sslpl_matcher* Ctx() { static thread_local MatcherCtx c; return c.h; }

// DBoW2::FeatureVector (std::map<NodeId, std::vector<unsigned int>>) -> CSR
struct Csr {
    std::vector<int32_t> nodes, off, idx; sslpl_featvec fv;
    explicit Csr(const DBoW2::FeatureVector &v) {
        off.push_back(0);
        for(DBoW2::FeatureVector::const_iterator it=v.begin(); it!=v.end(); ++it) {
            nodes.push_back((int32_t)it->first);
            for(size_t k=0; k<it->second.size(); k++) idx.push_back((int32_t)it->second[k]);
            off.push_back((int32_t)idx.size());
        }
        fv.nodes = nodes.empty() ? NULL : &nodes[0]; fv.off = &off[0]; fv.idx = idx.empty() ? NULL : &idx[0]; fv.nn = (int)nodes.size();
    }
};
void Check(int rc, const char* what) { if(rc != SSLPL_OK) throw std::runtime_error(std::string(what) + ": " + sslpl_last_error()); }
}

// ORBmatcher::DescriptorDistance (ORBmatcher.cc:1650) and LSDmatcher::DescriptorDistance (LSDmatcher.cpp:364) are NOT replaced: the
// matchers that keep their CPU bodies (SearchByProjection x3, Fuse, SearchBySim3, MapPoint::ComputeDistinctiveDescriptors) call them
// per descriptor pair inside inner loops, where the reference's 8-word popcount costs nanoseconds and a device round trip would
// cost tens of microseconds.  The GPU distance exists in batched form only (sslpl_descriptor_distance with n >> 1, the medoid batch).

// ORBmatcher::SearchByProjection(Frame&, const Frame&, th, bMono) — ORBmatcher.cc:1331-1473, the matcher of
// Tracking::TrackWithMotionModel (Tracking.cc:1227, :1243).  Both call sites fill CurrentFrame.mvpMapPoints with NULL first;
// features the kernel never touched keep what they held, features removed by the rotation check are set to NULL (:1461).
int ORBmatcher::SearchByProjection(Frame &CurrentFrame, const Frame &LastFrame, const float th, const bool bMono)
{
    const int n1 = LastFrame.N, n2 = CurrentFrame.N;
    if(n1 == 0 || n2 == 0) return 0;
    std::vector<uint8_t> valid1(n1, 0), obs1(n1, 0), dmp((size_t)n1*32, 0), claimed2(n2, 0), d2((size_t)n2*32);
    std::vector<float> Xw((size_t)3*n1, 0.f), a1(n1), x2(n2), y2(n2), a2(n2), ur2(n2);
    std::vector<int32_t> o1(n1), o2(n2), assign(n2);
    for(int i=0; i<n1; i++) {
        a1[i] = LastFrame.mvKeysUn[i].angle; o1[i] = LastFrame.mvKeys[i].octave;
        MapPoint* p = LastFrame.mvpMapPoints[i];
        if(p && !LastFrame.mvbOutlier[i]) {
            valid1[i] = 1; obs1[i] = p->Observations() > 0 ? 1 : 0;
            const cv::Mat X = p->GetWorldPos();
            for(int k=0; k<3; k++) Xw[3*i+k] = X.at<float>(k);
            const cv::Mat d = p->GetDescriptor();
            std::copy(d.ptr<uchar>(), d.ptr<uchar>() + 32, &dmp[(size_t)32*i]);
        }
    }
    for(int j=0; j<n2; j++) {
        const cv::KeyPoint &kp = CurrentFrame.mvKeysUn[j];
        x2[j] = kp.pt.x; y2[j] = kp.pt.y; a2[j] = kp.angle; o2[j] = kp.octave; ur2[j] = CurrentFrame.mvuRight[j];
        MapPoint* q = CurrentFrame.mvpMapPoints[j];
        claimed2[j] = (q && q->Observations() > 0) ? 1 : 0;
        std::copy(CurrentFrame.mDescriptors.ptr<uchar>(j), CurrentFrame.mDescriptors.ptr<uchar>(j) + 32, &d2[(size_t)32*j]);
    }
    float Tcw[12], Tlw[12];
    for(int r=0; r<3; r++) for(int c=0; c<4; c++) { Tcw[4*r+c] = CurrentFrame.mTcw.at<float>(r,c); Tlw[4*r+c] = LastFrame.mTcw.at<float>(r,c); }
    const float cam[6] = {CurrentFrame.fx, CurrentFrame.fy, CurrentFrame.cx, CurrentFrame.cy, CurrentFrame.mbf, CurrentFrame.mb};
    const float bounds[4] = {CurrentFrame.mnMinX, CurrentFrame.mnMaxX, CurrentFrame.mnMinY, CurrentFrame.mnMaxY};
    int nmatches = 0;
    Check(sslpl_search_by_projection_frame(Ctx(), n1, &valid1[0], &obs1[0], &Xw[0], &dmp[0], &o1[0], &a1[0],
                                           n2, &d2[0], &x2[0], &y2[0], &o2[0], &a2[0], &ur2[0], &claimed2[0], Tcw, Tlw, cam, bounds,
                                           &CurrentFrame.mvScaleFactors[0], (int)CurrentFrame.mvScaleFactors.size(), th, bMono ? 1 : 0,
                                           mbCheckOrientation ? 1 : 0, &assign[0], &nmatches), "sslpl_search_by_projection_frame");
    for(int j=0; j<n2; j++)
    {
        if(assign[j] >= 0) CurrentFrame.mvpMapPoints[j] = LastFrame.mvpMapPoints[assign[j]];
        else if(assign[j] == -2) CurrentFrame.mvpMapPoints[j] = static_cast<MapPoint*>(NULL);   // removed by the rotation check, ORBmatcher.cc:1461
    }
    return nmatches;
}

// MapPoint::PredictScale(dist, Frame*) reads mfMaxDistance under mMutexPos (MapPoint.cc:407-422); both are protected and have no accessor,
// so they are reached through member pointers formed in a derived class (never instantiated).
struct MapPointFields : MapPoint {
    static float MapPoint::* MaxDistance() { return &MapPointFields::mfMaxDistance; }
    static std::mutex MapPoint::* MutexPos() { return &MapPointFields::mMutexPos; }
};

// ORBmatcher::SearchByProjection(Frame &CurrentFrame, KeyFrame *pKF, sAlreadyFound, th, ORBdist) — ORBmatcher.cc:1475-1602, run by
// Tracking::Relocalization (Tracking.cc:2071, :2085) after PnP and PoseOptimization.  Frame features the kernel never touched keep what
// they held; features removed by the rotation check are set to NULL (:1595).
int ORBmatcher::SearchByProjection(Frame &CurrentFrame, KeyFrame *pKF, const set<MapPoint*> &sAlreadyFound, const float th, const int ORBdist)
{
    const vector<MapPoint*> vpMPs = pKF->GetMapPointMatches();
    const int n1 = (int)vpMPs.size(), n2 = CurrentFrame.N;
    if(n1 == 0 || n2 == 0) return 0;
    std::vector<uint8_t> flag1(n1, 0), dmp((size_t)n1*32, 0), held2(n2, 0), d2((size_t)n2*32);
    std::vector<float> Xw((size_t)3*n1, 0.f), dist3((size_t)3*n1, 0.f), a1(n1), x2(n2), y2(n2), a2(n2);
    std::vector<int32_t> o2(n2), assign(n2);
    for(int i=0; i<n1; i++) {
        a1[i] = pKF->mvKeysUn[i].angle;
        MapPoint* p = vpMPs[i];
        if(!p || p->isBad() || sAlreadyFound.count(p)) continue;
        flag1[i] = 1;
        const cv::Mat X = p->GetWorldPos();
        for(int k=0; k<3; k++) Xw[3*i+k] = X.at<float>(k);
        const cv::Mat d = p->GetDescriptor();
        std::copy(d.ptr<uchar>(), d.ptr<uchar>() + 32, &dmp[(size_t)32*i]);
        dist3[3*i] = p->GetMinDistanceInvariance(); dist3[3*i+1] = p->GetMaxDistanceInvariance();
        unique_lock<mutex> lock(p->*MapPointFields::MutexPos());
        dist3[3*i+2] = p->*MapPointFields::MaxDistance();
    }
    for(int j=0; j<n2; j++) {
        const cv::KeyPoint &kp = CurrentFrame.mvKeysUn[j];
        x2[j] = kp.pt.x; y2[j] = kp.pt.y; a2[j] = kp.angle; o2[j] = kp.octave;
        held2[j] = CurrentFrame.mvpMapPoints[j] ? 1 : 0;
        std::copy(CurrentFrame.mDescriptors.ptr<uchar>(j), CurrentFrame.mDescriptors.ptr<uchar>(j) + 32, &d2[(size_t)32*j]);
    }
    float Tcw[12];
    for(int r=0; r<3; r++) for(int c=0; c<4; c++) Tcw[4*r+c] = CurrentFrame.mTcw.at<float>(r,c);
    const float cam[4] = {CurrentFrame.fx, CurrentFrame.fy, CurrentFrame.cx, CurrentFrame.cy};
    const float bounds[4] = {CurrentFrame.mnMinX, CurrentFrame.mnMaxX, CurrentFrame.mnMinY, CurrentFrame.mnMaxY};
    int nmatches = 0;
    Check(sslpl_search_by_projection_kf(Ctx(), n1, &flag1[0], &Xw[0], &dmp[0], &dist3[0], &a1[0], n2, &d2[0], &x2[0], &y2[0], &o2[0], &a2[0],
                                        &held2[0], Tcw, cam, bounds, &CurrentFrame.mvScaleFactors[0], CurrentFrame.mnScaleLevels,
                                        CurrentFrame.mfLogScaleFactor, th, ORBdist, mbCheckOrientation ? 1 : 0, &assign[0], &nmatches),
          "sslpl_search_by_projection_kf");
    for(int j=0; j<n2; j++)
    {
        if(assign[j] >= 0) CurrentFrame.mvpMapPoints[j] = vpMPs[assign[j]];
        else if(assign[j] == -2) CurrentFrame.mvpMapPoints[j] = static_cast<MapPoint*>(NULL);
    }
    return nmatches;
}

// ORBmatcher::SearchByProjection(Frame &F, const vector<MapPoint*> &vpMapPoints, th) — ORBmatcher.cc:45-129, called on every frame by
// Tracking::SearchLocalPoints (Tracking.cc:1736) with the tracking fields Frame::isInFrustum left on each MapPoint.
int ORBmatcher::SearchByProjection(Frame &F, const vector<MapPoint*> &vpMapPoints, const float th)
{
    const int nmp = (int)vpMapPoints.size(), n2 = F.N;
    if(nmp == 0 || n2 == 0) return 0;
    std::vector<uint8_t> inview(nmp), bad(nmp), obs(nmp), dmp((size_t)nmp*32, 0), held(n2, 0), d2((size_t)n2*32);
    std::vector<float> px(nmp), py(nmp), pxr(nmp), vc(nmp), x2(n2), y2(n2), ur2(n2);
    std::vector<int32_t> lvl(nmp), o2(n2), assign(n2);
    for(int i=0; i<nmp; i++) {
        MapPoint* p = vpMapPoints[i];
        inview[i] = p->mbTrackInView ? 1 : 0; bad[i] = p->isBad() ? 1 : 0; obs[i] = p->Observations() > 0 ? 1 : 0;
        px[i] = p->mTrackProjX; py[i] = p->mTrackProjY; pxr[i] = p->mTrackProjXR; vc[i] = p->mTrackViewCos;
        lvl[i] = inview[i] ? p->mnTrackScaleLevel : 0;
        if(inview[i] && !bad[i]) { const cv::Mat d = p->GetDescriptor(); std::copy(d.ptr<uchar>(), d.ptr<uchar>() + 32, &dmp[(size_t)32*i]); }
    }
    bool stereo = false;
    for(int j=0; j<n2; j++) {
        const cv::KeyPoint &kp = F.mvKeysUn[j];
        x2[j] = kp.pt.x; y2[j] = kp.pt.y; o2[j] = kp.octave; ur2[j] = F.mvuRight[j]; stereo = stereo || ur2[j] > 0;
        MapPoint* q = F.mvpMapPoints[j];
        held[j] = q ? (q->Observations() > 0 ? 1 : 2) : 0;
        std::copy(F.mDescriptors.ptr<uchar>(j), F.mDescriptors.ptr<uchar>(j) + 32, &d2[(size_t)32*j]);
    }
    const float bounds[4] = {F.mnMinX, F.mnMaxX, F.mnMinY, F.mnMaxY};
    int nmatches = 0;
    Check(sslpl_search_by_projection_mps(Ctx(), nmp, &inview[0], &bad[0], &obs[0], &px[0], &py[0], &pxr[0], &lvl[0], &vc[0], &dmp[0],
                                         n2, &d2[0], &x2[0], &y2[0], &o2[0], stereo ? &ur2[0] : NULL, &held[0], bounds,
                                         &F.mvScaleFactors[0], (int)F.mvScaleFactors.size(), mfNNratio, th, &assign[0], &nmatches), "sslpl_search_by_projection_mps");
    for(int j=0; j<n2; j++) if(assign[j] >= 0) F.mvpMapPoints[j] = vpMapPoints[assign[j]];
    return nmatches;
}

// ORBmatcher::SearchForInitialization — ORBmatcher.cc:408-523 (Tracking::MonocularInitialization, Tracking.cc:366)
int ORBmatcher::SearchForInitialization(Frame &F1, Frame &F2, vector<cv::Point2f> &vbPrevMatched, vector<int> &vnMatches12, int windowSize)
{
    const int n1 = (int)F1.mvKeysUn.size(), n2 = (int)F2.mvKeysUn.size();
    vnMatches12 = vector<int>(n1,-1);
    if(n1 == 0 || n2 == 0) return 0;
    std::vector<float> a1(n1), prev((size_t)2*n1), x2(n2), y2(n2), a2(n2);
    std::vector<int32_t> o1(n1), o2(n2), m12(n1);
    for(int i=0; i<n1; i++) { a1[i] = F1.mvKeysUn[i].angle; o1[i] = F1.mvKeysUn[i].octave; prev[2*i] = vbPrevMatched[i].x; prev[2*i+1] = vbPrevMatched[i].y; }
    for(int j=0; j<n2; j++) { const cv::KeyPoint &kp = F2.mvKeysUn[j]; x2[j] = kp.pt.x; y2[j] = kp.pt.y; a2[j] = kp.angle; o2[j] = kp.octave; }
    const float bounds[4] = {F2.mnMinX, F2.mnMaxX, F2.mnMinY, F2.mnMaxY};
    int nmatches = 0;
    Check(sslpl_search_for_initialization(Ctx(), n1, F1.mDescriptors.ptr<uchar>(), &o1[0], &a1[0], &prev[0], n2, F2.mDescriptors.ptr<uchar>(),
                                          &x2[0], &y2[0], &o2[0], &a2[0], bounds, mfNNratio, mbCheckOrientation ? 1 : 0, windowSize, &m12[0], &nmatches), "sslpl_search_for_initialization");
    for(int i=0; i<n1; i++) { vnMatches12[i] = m12[i]; vbPrevMatched[i] = cv::Point2f(prev[2*i], prev[2*i+1]); }
    return nmatches;
}

int ORBmatcher::SearchByBoW(KeyFrame* pKF,Frame &F, vector<MapPoint*> &vpMapPointMatches)   // ORBmatcher.cc:159
{
    const vector<MapPoint*> vpMapPointsKF = pKF->GetMapPointMatches();
    vpMapPointMatches = vector<MapPoint*>(F.N,static_cast<MapPoint*>(NULL));
    const int n1 = pKF->mDescriptors.rows, n2 = F.N;
    if(n1 == 0 || n2 == 0) return 0;
    std::vector<uint8_t> valid1(n1);
    std::vector<float> a1(n1), a2(n2);
    for(int i=0; i<n1; i++) { MapPoint* p = vpMapPointsKF[i]; valid1[i] = (p && !p->isBad()) ? 1 : 0; a1[i] = pKF->mvKeysUn[i].angle; }
    for(int i=0; i<n2; i++) a2[i] = F.mvKeys[i].angle;
    Csr f1(pKF->mFeatVec), f2(F.mFeatVec);
    std::vector<int32_t> match2(n2);
    int nmatches = 0;
    Check(sslpl_search_by_bow(Ctx(), pKF->mDescriptors.ptr<uchar>(), n1, F.mDescriptors.ptr<uchar>(), n2, &f1.fv, &f2.fv,
                              &valid1[0], &a1[0], &a2[0], mfNNratio, mbCheckOrientation ? 1 : 0, &match2[0], &nmatches), "sslpl_search_by_bow");
    for(int j=0; j<n2; j++) if(match2[j] >= 0) vpMapPointMatches[j] = vpMapPointsKF[match2[j]];
    return nmatches;
}

int ORBmatcher::SearchByBoW(KeyFrame *pKF1, KeyFrame *pKF2, vector<MapPoint *> &vpMatches12)   // ORBmatcher.cc:525
{
    const vector<MapPoint*> vpMapPoints1 = pKF1->GetMapPointMatches();
    const vector<MapPoint*> vpMapPoints2 = pKF2->GetMapPointMatches();
    vpMatches12 = vector<MapPoint*>(vpMapPoints1.size(),static_cast<MapPoint*>(NULL));
    const int n1 = pKF1->mDescriptors.rows, n2 = pKF2->mDescriptors.rows;
    if(n1 == 0 || n2 == 0) return 0;
    std::vector<uint8_t> v1(n1), v2(n2);
    std::vector<float> a1(n1), a2(n2);
    for(int i=0; i<n1; i++) { MapPoint* p = vpMapPoints1[i]; v1[i] = (p && !p->isBad()) ? 1 : 0; a1[i] = pKF1->mvKeysUn[i].angle; }
    for(int i=0; i<n2; i++) { MapPoint* p = vpMapPoints2[i]; v2[i] = (p && !p->isBad()) ? 1 : 0; a2[i] = pKF2->mvKeysUn[i].angle; }
    Csr f1(pKF1->mFeatVec), f2(pKF2->mFeatVec);
    std::vector<int32_t> m12(n1);
    int nmatches = 0;
    Check(sslpl_search_by_bow_kf(Ctx(), pKF1->mDescriptors.ptr<uchar>(), n1, pKF2->mDescriptors.ptr<uchar>(), n2, &f1.fv, &f2.fv,
                                 &v1[0], &v2[0], &a1[0], &a2[0], mfNNratio, mbCheckOrientation ? 1 : 0, &m12[0], &nmatches), "sslpl_search_by_bow_kf");
    for(int i=0; i<n1; i++) if(m12[i] >= 0) vpMatches12[i] = vpMapPoints2[m12[i]];
    return nmatches;
}

int ORBmatcher::SearchForTriangulation(KeyFrame *pKF1, KeyFrame *pKF2, cv::Mat F12,
                                       vector<pair<size_t, size_t> > &vMatchedPairs, const bool bOnlyStereo)   // ORBmatcher.cc:660
{
    (void)bOnlyStereo;                                      // monocular pipeline: mvuRight < 0 everywhere
    // epipole in the second image, ORBmatcher.cc:666-672
    cv::Mat Cw = pKF1->GetCameraCenter();
    cv::Mat R2w = pKF2->GetRotation();
    cv::Mat t2w = pKF2->GetTranslation();
    cv::Mat C2 = R2w*Cw+t2w;
    const float invz = 1.0f/C2.at<float>(2);
    const float ex =pKF2->fx*C2.at<float>(0)*invz+pKF2->cx;
    const float ey =pKF2->fy*C2.at<float>(1)*invz+pKF2->cy;

    const int n1 = pKF1->N, n2 = pKF2->N;
    vMatchedPairs.clear();
    if(n1 == 0 || n2 == 0) return 0;
    std::vector<uint8_t> h1(n1), h2(n2);
    std::vector<sslpl_keypoint> k1(n1), k2(n2);
    for(int i=0; i<n1; i++) { h1[i] = pKF1->GetMapPoint(i) ? 1 : 0; const cv::KeyPoint &k = pKF1->mvKeysUn[i];
        k1[i].x = k.pt.x; k1[i].y = k.pt.y; k1[i].size = k.size; k1[i].angle = k.angle; k1[i].response = k.response; k1[i].octave = k.octave; k1[i].class_id = k.class_id; }
    for(int i=0; i<n2; i++) { h2[i] = pKF2->GetMapPoint(i) ? 1 : 0; const cv::KeyPoint &k = pKF2->mvKeysUn[i];
        k2[i].x = k.pt.x; k2[i].y = k.pt.y; k2[i].size = k.size; k2[i].angle = k.angle; k2[i].response = k.response; k2[i].octave = k.octave; k2[i].class_id = k.class_id; }
    float F[9];
    for(int r=0; r<3; r++) for(int c=0; c<3; c++) F[3*r+c] = F12.at<float>(r,c);
    Csr f1(pKF1->mFeatVec), f2(pKF2->mFeatVec);
    std::vector<int32_t> pairs(2*(size_t)n1);
    int nmatches = 0;
    Check(sslpl_search_for_triangulation(Ctx(), pKF1->mDescriptors.ptr<uchar>(), n1, pKF2->mDescriptors.ptr<uchar>(), n2, &f1.fv, &f2.fv,
                                         &h1[0], &h2[0], &k1[0], &k2[0], F, ex, ey, &pKF2->mvScaleFactors[0], &pKF2->mvLevelSigma2[0],
                                         (int)pKF2->mvScaleFactors.size(), mbCheckOrientation ? 1 : 0, &pairs[0], &nmatches), "sslpl_search_for_triangulation");
    vMatchedPairs.reserve(nmatches);
    for(int k=0; k<nmatches; k++) vMatchedPairs.push_back(make_pair((size_t)pairs[2*k], (size_t)pairs[2*k+1]));
    return nmatches;
}

// ---- LSDmatcher: the knnMatch-based entry points (LSDmatcher.cpp:143, 257, 286, 329, 382) ----
// (With fewer than two train lines cv::knnMatch returns fewer than two neighbours and the reference reads past the end; these
// bodies return 0 matches then instead of failing.)
static int LineMatchKF_F(KeyFrame* pKF, Frame &currentF, vector<MapLine*> &vpMapLineMatches)
{
    const vector<MapLine*> vpMapLinesKF = pKF->GetMapLineMatches();
    vpMapLineMatches = vector<MapLine*>(currentF.NL,static_cast<MapLine*>(NULL));
    const int n1 = pKF->mLineDescriptors.rows, n2 = currentF.mLdesc.rows;
    if(n1 == 0 || n2 < 2) return 0;
    std::vector<uint8_t> has1(n1);
    for(int i=0; i<n1; i++) has1[i] = vpMapLinesKF[i] ? 1 : 0;
    std::vector<int32_t> out(std::max(n1, n2)*2);
    int nout = 0, nmatches = 0;
    Check(sslpl_line_match(Ctx(), 0, pKF->mLineDescriptors.ptr<uchar>(), n1, currentF.mLdesc.ptr<uchar>(), n2, &has1[0], NULL, &out[0], &nout, &nmatches, NULL), "sslpl_line_match");
    for(int t=0; t<n2; t++) if(out[t] >= 0) vpMapLineMatches[t] = vpMapLinesKF[out[t]];
    return nmatches;
}
int LSDmatcher::SearchByProjection(KeyFrame* pKF,Frame &currentF, vector<MapLine*> &vpMapLineMatches) { return LineMatchKF_F(pKF, currentF, vpMapLineMatches); }   // :143
int LSDmatcher::SearchByDescriptor(KeyFrame* pKF, Frame &currentF, vector<MapLine*> &vpMapLineMatches) { return LineMatchKF_F(pKF, currentF, vpMapLineMatches); }  // :286

int LSDmatcher::SerachForInitialize(Frame &InitialFrame, Frame &CurrentFrame, vector<pair<int, int>> &LineMatches)   // :257
{
    LineMatches.clear();
    const int n1 = InitialFrame.mLdesc.rows, n2 = CurrentFrame.mLdesc.rows;
    if(n1 == 0 || n2 < 2) return 0;
    std::vector<int32_t> out(std::max(n1, n2)*2);
    int nout = 0, nmatches = 0;
    Check(sslpl_line_match(Ctx(), 1, InitialFrame.mLdesc.ptr<uchar>(), n1, CurrentFrame.mLdesc.ptr<uchar>(), n2, NULL, NULL, &out[0], &nout, &nmatches, NULL), "sslpl_line_match");
    for(int k=0; k<nout; k++) LineMatches.push_back(make_pair(out[2*k], out[2*k+1]));
    return nmatches;
}

int LSDmatcher::SearchByDescriptor(KeyFrame* pKF, KeyFrame *pKF2, vector<MapLine*> &vpMapLineMatches)   // :329
{
    const vector<MapLine*> vpMapLinesKF = pKF->GetMapLineMatches();
    const vector<MapLine*> vpMapLinesKF2 = pKF2->GetMapLineMatches();
    vpMapLineMatches = vector<MapLine*>(vpMapLinesKF.size(),static_cast<MapLine*>(NULL));
    const int n1 = pKF->mLineDescriptors.rows, n2 = pKF2->mLineDescriptors.rows;
    if(n1 == 0 || n2 < 2) return 0;
    std::vector<uint8_t> has2(std::max(n2, 1));
    for(int i=0; i<n2; i++) has2[i] = vpMapLinesKF2[i] ? 1 : 0;
    std::vector<int32_t> out(std::max(n1, n2)*2);
    int nout = 0, nmatches = 0;
    Check(sslpl_line_match(Ctx(), 2, pKF->mLineDescriptors.ptr<uchar>(), n1, pKF2->mLineDescriptors.ptr<uchar>(), n2, NULL, &has2[0], &out[0], &nout, &nmatches, NULL), "sslpl_line_match");
    for(int q=0; q<n1; q++) if(out[q] >= 0) vpMapLineMatches[q] = vpMapLinesKF2[out[q]];
    return nmatches;
}

int LSDmatcher::SearchForTriangulation(KeyFrame *pKF1, KeyFrame *pKF2, vector<pair<size_t, size_t>> &vMatchedPairs)   // :382
{
    vMatchedPairs.clear();
    const int n1 = pKF1->mLineDescriptors.rows, n2 = pKF2->mLineDescriptors.rows;
    if(n1 == 0 || n2 < 2) return 0;
    std::vector<uint8_t> has1(n1), has2(std::max(n2, 1));
    for(int i=0; i<n1; i++) has1[i] = pKF1->GetMapLine(i) ? 1 : 0;
    for(int i=0; i<n2; i++) has2[i] = pKF2->GetMapLine(i) ? 1 : 0;
    std::vector<int32_t> out(std::max(n1, n2)*2);
    int nout = 0, nmatches = 0;
    Check(sslpl_line_match(Ctx(), 3, pKF1->mLineDescriptors.ptr<uchar>(), n1, pKF2->mLineDescriptors.ptr<uchar>(), n2, &has1[0], &has2[0], &out[0], &nout, &nmatches, NULL), "sslpl_line_match");
    for(int k=0; k<nout; k++) vMatchedPairs.push_back(make_pair((size_t)out[2*k], (size_t)out[2*k+1]));
    return nmatches;
}


// ---- SURVEY.md 8(f) row 3: line projection matchers and Fuse ----
// Each of these reference functions is a projection stage (per map element: gates + projected quantities) followed by a Hamming search over
// the frame's features.  The projection stage stays here, written with the reference's own cv::Mat / Eigen expressions and accessors (so its
// arithmetic IS the reference's: cv::gemm, cv::norm, Mat::dot, MapPoint::PredictScale); the search stage runs on the device
// (sslpl_line_search_by_projection, sslpl_fuse_lines_search, sslpl_fuse_points_search); Fuse's bookkeeping (Replace / AddObservation) is
// applied afterwards in vector order, re-testing isBad() / IsInKeyFrame() as the reference's loop would see them at that point.
namespace {
struct FlatLines {
    int n; std::vector<uint8_t> desc, held; std::vector<float> kl; std::vector<int32_t> oct;
    FlatLines(const std::vector<KeyLine> &v, const cv::Mat &d): n((int)v.size()), desc((size_t)v.size()*32 + 32), held(v.size() + 1, 0), kl(3*v.size() + 3), oct(v.size() + 1) {
        for(int j=0; j<n; j++) {
            kl[3*j] = v[j].pt.x; kl[3*j+1] = v[j].pt.y; kl[3*j+2] = v[j].angle; oct[j] = v[j].octave;
            std::copy(d.ptr<uchar>(j), d.ptr<uchar>(j) + 32, &desc[(size_t)32*j]);
        }
    }
};
struct LineQueries {
    std::vector<uint8_t> active, obs, desc; std::vector<float> proj, radius; std::vector<int32_t> minLevel, maxLevel, level;
    explicit LineQueries(int n): active(n + 1, 0), obs(n + 1, 0), desc((size_t)n*32 + 32, 0), proj(4*(size_t)n + 4, 0.f), radius(n + 1, 0.f), minLevel(n + 1, -1), maxLevel(n + 1, -1), level(n + 1, 0) {}
    void Set(int i, MapLine* pML, float u1, float v1, float u2, float v2) {
        active[i] = 1; obs[i] = pML->Observations() > 0 ? 1 : 0;
        proj[4*i] = u1; proj[4*i+1] = v1; proj[4*i+2] = u2; proj[4*i+3] = v2;
        const cv::Mat d = pML->GetDescriptor();
        std::copy(d.ptr<uchar>(), d.ptr<uchar>() + 32, &desc[(size_t)32*i]);
    }
};
// Both end points of a MapLine through Rcw, tcw and the pinhole model; false when either lies behind the camera or outside the image bounds
// (LSDmatcher.cpp:45-82 = :439-476)
bool ProjectLine(MapLine* pML, const cv::Mat &Rcw, const cv::Mat &tcw, float fx, float fy, float cx, float cy, float minX, float maxX, float minY, float maxY,
                 cv::Mat &SP, cv::Mat &EP, float &u1, float &v1, float &u2, float &v2)
{
    const Vector6d P = pML->GetWorldPos();
    SP = (cv::Mat_<float>(3, 1) << P(0), P(1), P(2));
    EP = (cv::Mat_<float>(3, 1) << P(3), P(4), P(5));
    const cv::Mat SPc = Rcw * SP + tcw, EPc = Rcw * EP + tcw;
    const float z1 = SPc.at<float>(2), z2 = EPc.at<float>(2);
    if(z1 < 0.0f || z2 < 0.0f) return false;
    const float invz1 = 1.0f / z1;
    u1 = fx * SPc.at<float>(0) * invz1 + cx; v1 = fy * SPc.at<float>(1) * invz1 + cy;
    if(u1 < minX || u1 > maxX || v1 < minY || v1 > maxY) return false;
    const float invz2 = 1.0f / z2;
    u2 = fx * EPc.at<float>(0) * invz2 + cx; v2 = fy * EPc.at<float>(1) * invz2 + cy;
    if(u2 < minX || u2 > maxX || v2 < minY || v2 > maxY) return false;
    return true;
}
int RunLineSearch(const LineQueries &Q, int nml, FlatLines &L, float nnratio, std::vector<int32_t> &assign)
{
    int nmatches = 0;
    assign.assign(L.n + 1, -1);
    Check(sslpl_line_search_by_projection(Ctx(), nml, &Q.active[0], &Q.obs[0], &Q.proj[0], &Q.radius[0], &Q.minLevel[0], &Q.maxLevel[0], &Q.desc[0],
                                          L.n, &L.desc[0], &L.kl[0], &L.oct[0], &L.held[0], nnratio, &assign[0], &nmatches), "sslpl_line_search_by_projection");
    return nmatches;
}
}

// LSDmatcher::SearchByProjection(Frame&, const Frame&, th, bMono) — LSDmatcher.cpp:22-141
int LSDmatcher::SearchByProjection(Frame &CurrentFrame, const Frame &LastFrame, const float th, const bool bMono)
{
    const int nl1 = LastFrame.NL;
    if(nl1 == 0 || CurrentFrame.NL == 0) return 0;
    const cv::Mat Rcw = CurrentFrame.mTcw.rowRange(0, 3).colRange(0, 3), tcw = CurrentFrame.mTcw.rowRange(0, 3).col(3);
    const cv::Mat twc = -Rcw.t()*tcw;
    const cv::Mat Rlw = LastFrame.mTcw.rowRange(0, 3).colRange(0, 3), tlw = LastFrame.mTcw.rowRange(0, 3).col(3);
    const cv::Mat tlc = Rlw*twc+tlw;
    const bool bForward = tlc.at<float>(2)>CurrentFrame.mb && !bMono;
    const bool bBackward = -tlc.at<float>(2)>CurrentFrame.mb && !bMono;
    LineQueries Q(nl1);
    for(int i=0; i<nl1; i++) {
        MapLine* pML = LastFrame.mvpMapLines[i];
        if(!pML || pML->isBad() || LastFrame.mvbLineOutlier[i]) continue;
        cv::Mat SP, EP; float u1, v1, u2, v2;
        if(!ProjectLine(pML, Rcw, tcw, CurrentFrame.fx, CurrentFrame.fy, CurrentFrame.cx, CurrentFrame.cy,
                        CurrentFrame.mnMinX, CurrentFrame.mnMaxX, CurrentFrame.mnMinY, CurrentFrame.mnMaxY, SP, EP, u1, v1, u2, v2)) continue;
        const int nLastOctave = LastFrame.mvKeys[i].octave;            // the POINT keypoint of the same index, as the reference reads it (:84)
        Q.Set(i, pML, u1, v1, u2, v2);
        Q.radius[i] = th*CurrentFrame.mvScaleFactors[nLastOctave];
        if(bForward) { Q.minLevel[i] = nLastOctave; Q.maxLevel[i] = -1; }
        else if(bBackward) { Q.minLevel[i] = 0; Q.maxLevel[i] = nLastOctave; }
        else { Q.minLevel[i] = nLastOctave-1; Q.maxLevel[i] = nLastOctave+1; }
    }
    FlatLines L(CurrentFrame.mvKeylinesUn, CurrentFrame.mLdesc);
    for(int j=0; j<L.n; j++) { MapLine* q = CurrentFrame.mvpMapLines[j]; L.held[j] = q ? (q->Observations() > 0 ? 1 : 2) : 0; }
    std::vector<int32_t> assign;
    const int nmatches = RunLineSearch(Q, nl1, L, mfNNratio, assign);
    for(int j=0; j<L.n; j++) if(assign[j] >= 0) CurrentFrame.mvpMapLines[j] = LastFrame.mvpMapLines[assign[j]];
    return nmatches;
}

// LSDmatcher::SearchByProjection(Frame&, const vector<MapLine*>&, th) — LSDmatcher.cpp:185-255 (Tracking::SearchLocalLines, Tracking.cc:1783)
int LSDmatcher::SearchByProjection(Frame &F, const std::vector<MapLine *> &vpMapLines, const float th)
{
    const int nml = (int)vpMapLines.size();
    if(nml == 0 || F.NL == 0) return 0;
    const bool bFactor = th!=1.0;
    LineQueries Q(nml);
    for(int i=0; i<nml; i++) {
        MapLine* pML = vpMapLines[i];
        if(!pML || pML->isBad() || !pML->mbTrackInView) continue;
        const int nPredictLevel = pML->mnTrackScaleLevel;
        float r = RadiusByViewingCos(pML->mTrackViewCos);
        if(bFactor) r*=th;
        Q.Set(i, pML, pML->mTrackProjX1, pML->mTrackProjY1, pML->mTrackProjX2, pML->mTrackProjY2);
        Q.radius[i] = r*F.mvScaleFactors[nPredictLevel];
        Q.minLevel[i] = nPredictLevel-1; Q.maxLevel[i] = nPredictLevel;
    }
    FlatLines L(F.mvKeylinesUn, F.mLdesc);
    for(int j=0; j<L.n; j++) { MapLine* q = F.mvpMapLines[j]; L.held[j] = q ? (q->Observations() > 0 ? 1 : 2) : 0; }
    std::vector<int32_t> assign;
    const int nmatches = RunLineSearch(Q, nml, L, mfNNratio, assign);
    for(int j=0; j<L.n; j++) if(assign[j] >= 0) F.mvpMapLines[j] = vpMapLines[assign[j]];
    return nmatches;
}

// LSDmatcher::Fuse(KeyFrame*, const vector<MapLine*>&, th) — LSDmatcher.cpp:417-548 (LocalMapping::SearchInNeighbors, LocalMapping.cc:1243, :1264)
int LSDmatcher::Fuse(KeyFrame *pKF, const vector<MapLine *> &vpMapLines, const float th)
{
    const int nml = (int)vpMapLines.size();
    if(nml == 0 || pKF->NL == 0) return 0;
    const cv::Mat Rcw = pKF->GetRotation(), tcw = pKF->GetTranslation(), Ow = pKF->GetCameraCenter();
    LineQueries Q(nml);
    for(int i=0; i<nml; i++) {
        MapLine* pML = vpMapLines[i];
        if(!pML || pML->isBad()) continue;
        cv::Mat SP, EP; float u1, v1, u2, v2;
        if(!ProjectLine(pML, Rcw, tcw, pKF->fx, pKF->fy, pKF->cx, pKF->cy, pKF->mnMinX, pKF->mnMaxX, pKF->mnMinY, pKF->mnMaxY, SP, EP, u1, v1, u2, v2)) continue;
        const float maxDistance = pML->GetMaxDistanceInvariance(), minDistance = pML->GetMinDistanceInvariance();
        const cv::Mat OM = 0.5 * (SP + EP) - Ow;
        const float dist = cv::norm(OM);
        if(dist < minDistance || dist > maxDistance) continue;
        const Vector3d Pn = pML->GetNormal();
        const cv::Mat pn = (cv::Mat_<float>(3, 1) << Pn(0), Pn(1), Pn(2));
        if(OM.dot(pn)<0.5*dist) continue;
        Q.Set(i, pML, u1, v1, u2, v2);
        Q.level[i] = pML->PredictScale(dist, pKF->mfLogScaleFactor);   // not clamped by the reference: levels outside the pyramid are dropped by the search
    }
    FlatLines L(pKF->mvKeyLines, pKF->mLineDescriptors);
    std::vector<int32_t> bestIdx(nml + 1, -1), bestDist(nml + 1, 0x7fffffff);
    Check(sslpl_fuse_lines_search(Ctx(), nml, &Q.active[0], &Q.proj[0], &Q.level[0], &Q.desc[0], L.n, &L.desc[0], &L.kl[0], &L.oct[0],
                                  &pKF->mvScaleFactors[0], (int)pKF->mvScaleFactors.size(), th, &bestIdx[0], &bestDist[0]), "sslpl_fuse_lines_search");
    int nFused=0;
    std::set<MapLine*> recomputed;       // MapLines whose descriptor a Replace() of this loop recomputed (MapLine.cpp:216)
    for(int i=0; i<nml; i++) {
        MapLine* pML = vpMapLines[i];
        if(!Q.active[i] || pML->isBad()) continue;                     // isBad(): an earlier iteration may have replaced it
        if(recomputed.count(pML)) {                                    // (no IsInKeyFrame test in this function: such a line is searched again, with its new descriptor)
            const cv::Mat d = pML->GetDescriptor();
            std::copy(d.ptr<uchar>(), d.ptr<uchar>() + 32, &Q.desc[(size_t)32*i]);
            Check(sslpl_fuse_lines_search(Ctx(), 1, &Q.active[i], &Q.proj[4*i], &Q.level[i], &Q.desc[(size_t)32*i], L.n, &L.desc[0], &L.kl[0], &L.oct[0],
                                          &pKF->mvScaleFactors[0], (int)pKF->mvScaleFactors.size(), th, &bestIdx[i], &bestDist[i]), "sslpl_fuse_lines_search");
        }
        if(bestIdx[i] < 0 || bestDist[i] > TH_LOW) continue;
        MapLine* pMLinKF = pKF->GetMapLine(bestIdx[i]);
        if(pMLinKF) {
            if(!pMLinKF->isBad()) {
                if(pMLinKF->Observations()>pML->Observations()) { pML->Replace(pMLinKF); recomputed.insert(pMLinKF); }
                else { pMLinKF->Replace(pML); recomputed.insert(pML); }
            }
        } else {
            pML->AddObservation(pKF,bestIdx[i]);
            pKF->AddMapLine(pML,bestIdx[i]);
        }
        nFused++;
    }
    return nFused;
}

// ORBmatcher::Fuse(KeyFrame*, const vector<MapPoint*>&, th) — ORBmatcher.cc:828-973 (LocalMapping::SearchInNeighbors, LocalMapping.cc:1206, :1226)
int ORBmatcher::Fuse(KeyFrame *pKF, const vector<MapPoint *> &vpMapPoints, const float th)
{
    const int nMPs = (int)vpMapPoints.size(), n2 = pKF->N;
    if(nMPs == 0 || n2 == 0) return 0;
    const cv::Mat Rcw = pKF->GetRotation(), tcw = pKF->GetTranslation(), Ow = pKF->GetCameraCenter();
    const float &fx = pKF->fx, &fy = pKF->fy, &cx = pKF->cx, &cy = pKF->cy, &bf = pKF->mbf;
    std::vector<uint8_t> active(nMPs, 0), dmp((size_t)nMPs*32, 0), d2((size_t)n2*32);
    std::vector<float> pu(nMPs, 0.f), pv(nMPs, 0.f), pur(nMPs, 0.f), x2(n2), y2(n2), ur2(n2);
    std::vector<int32_t> lvl(nMPs, 0), o2(n2), bestIdx(nMPs, -1), bestDist(nMPs, 256);
    for(int i=0; i<nMPs; i++) {
        MapPoint* pMP = vpMapPoints[i];
        if(!pMP || pMP->isBad() || pMP->IsInKeyFrame(pKF)) continue;
        const cv::Mat p3Dw = pMP->GetWorldPos();
        const cv::Mat p3Dc = Rcw*p3Dw + tcw;
        if(p3Dc.at<float>(2)<0.0f) continue;
        const float invz = 1/p3Dc.at<float>(2);
        const float x = p3Dc.at<float>(0)*invz, y = p3Dc.at<float>(1)*invz;
        const float u = fx*x+cx, v = fy*y+cy;
        if(!pKF->IsInImage(u,v)) continue;
        const float maxDistance = pMP->GetMaxDistanceInvariance(), minDistance = pMP->GetMinDistanceInvariance();
        const cv::Mat PO = p3Dw-Ow;
        const float dist3D = cv::norm(PO);
        if(dist3D<minDistance || dist3D>maxDistance) continue;
        const cv::Mat Pn = pMP->GetNormal();
        if(PO.dot(Pn)<0.5*dist3D) continue;
        active[i] = 1; pu[i] = u; pv[i] = v; pur[i] = u-bf*invz; lvl[i] = pMP->PredictScale(dist3D,pKF);
        const cv::Mat d = pMP->GetDescriptor();
        std::copy(d.ptr<uchar>(), d.ptr<uchar>() + 32, &dmp[(size_t)32*i]);
    }
    bool stereo = false;
    for(int j=0; j<n2; j++) {
        const cv::KeyPoint &kp = pKF->mvKeysUn[j];
        x2[j] = kp.pt.x; y2[j] = kp.pt.y; o2[j] = kp.octave; ur2[j] = pKF->mvuRight[j]; stereo = stereo || ur2[j] >= 0;
        std::copy(pKF->mDescriptors.ptr<uchar>(j), pKF->mDescriptors.ptr<uchar>(j) + 32, &d2[(size_t)32*j]);
    }
    const float bounds[4] = {(float)pKF->mnMinX, (float)pKF->mnMaxX, (float)pKF->mnMinY, (float)pKF->mnMaxY};
    Check(sslpl_fuse_points_search(Ctx(), nMPs, &active[0], &pu[0], &pv[0], &pur[0], &lvl[0], &dmp[0], n2, &d2[0], &x2[0], &y2[0], &o2[0], stereo ? &ur2[0] : NULL,
                                   bounds, &pKF->mvScaleFactors[0], &pKF->mvInvLevelSigma2[0], (int)pKF->mvScaleFactors.size(), th, &bestIdx[0], &bestDist[0]),
          "sslpl_fuse_points_search");
    int nFused=0;
    for(int i=0; i<nMPs; i++) {
        MapPoint* pMP = vpMapPoints[i];
        // re-test what an earlier iteration may have changed (a duplicate entry fused, or this point replaced): the reference tests it at :847
        if(!active[i] || bestIdx[i] < 0 || bestDist[i] > TH_LOW || pMP->isBad() || pMP->IsInKeyFrame(pKF)) continue;
        MapPoint* pMPinKF = pKF->GetMapPoint(bestIdx[i]);
        if(pMPinKF) {
            if(!pMPinKF->isBad()) {
                if(pMPinKF->Observations()>pMP->Observations()) pMP->Replace(pMPinKF);
                else pMPinKF->Replace(pMP);
            }
        } else {
            pMP->AddObservation(pKF,bestIdx[i]);
            pKF->AddMapPoint(pMP,bestIdx[i]);
        }
        nFused++;
    }
    return nFused;
}

} // namespace StructureSLAM
