// oracle/ref_harness.cpp — TEST INFRASTRUCTURE ONLY.
//
// C entry points over the REFERENCE ITSELF.  oracle/ref_build.sh compiles, unmodified and read in place from
// /root/reference, src/{ORBextractor.cc, ORBmatcher.cc, LSDmatcher.cpp, ExtractLineSegment.cpp, Frame.cc, KeyFrame.cc,
// MapPoint.cc, MapLine.cpp, Map.cc, KeyFrameDatabase.cc} and Thirdparty/DBoW2/{DBoW2/*.cpp, DUtils/*.cpp} against the
// OpenCV / Eigen stand-ins of oracle/refshim/, and links them with this file into oracle/_ref/libref.so.  Every function
// below builds the reference's own objects (Frame, KeyFrame, MapPoint, MapLine, ORBVocabulary) from plain arrays, calls the
// reference's own member function, and flattens the result, so that tests/test_ref_parity_cpu.py can hold the oracle's
// restatement (oracle/*.cpp) against what the reference code really does.  Not shipped, not linked by the product.
//
// Allocation: ORBextractor::DistributeOctTree breaks ties between equal-sized nodes by the ADDRESS of the std::list node
// (ORBextractor.cc:684), and MapPoint::ComputeDistinctiveDescriptors walks a std::map keyed by KeyFrame* (MapPoint.cc:262),
// so results depend on the allocator.  The canonical definition (SURVEY.md 7.3 item 3) is "under a monotonic, never-reusing
// allocator": inside a BumpScope, operator new of this library hands out increasing addresses from a per-thread arena.
#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <new>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>
#include "refshim/minicv.hpp"

// ------------------------------------------------------------------------------------------------
// bump allocator (this library only: linked with -Bsymbolic-functions; outside a BumpScope it is plain malloc/free)
// ------------------------------------------------------------------------------------------------
namespace {
struct Arena { char* base = nullptr; size_t cap = 0, off = 0; int depth = 0; };
thread_local Arena g_arena;
const size_t ARENA_BYTES = (size_t)1 << 31;       // virtual; touched lazily
inline bool in_arena(const void* p) { const Arena& a = g_arena; return a.base && (const char*)p >= a.base && (const char*)p < a.base + a.cap; }
void* bump(size_t n) {
    Arena& a = g_arena;
    n = (n + 15) & ~(size_t)15;
    if (a.off + n > a.cap) { fprintf(stderr, "ref_harness: bump arena exhausted\n"); abort(); }
    void* p = a.base + a.off; a.off += n; return p;
}
struct BumpScope {
    BumpScope() {
        Arena& a = g_arena;
        if (!a.base) { a.base = (char*)aligned_alloc(4096, ARENA_BYTES); a.cap = ARENA_BYTES; if (!a.base) abort(); }
        if (a.depth++ == 0) a.off = 0;
    }
    ~BumpScope() { g_arena.depth--; }
};
}  // namespace
void* operator new(size_t n) { if (g_arena.depth > 0) return bump(n); void* p = malloc(n ? n : 1); if (!p) throw std::bad_alloc(); return p; }
void* operator new[](size_t n) { return operator new(n); }
void operator delete(void* p) noexcept { if (p && !in_arena(p)) free(p); }
void operator delete[](void* p) noexcept { operator delete(p); }
void operator delete(void* p, size_t) noexcept { operator delete(p); }
void operator delete[](void* p, size_t) noexcept { operator delete(p); }

// the reference's classes, with their private parts reachable (layout is unaffected by access specifiers)
#define private public
#define protected public
#include "ORBextractor.h"
#include "ORBmatcher.h"
#include "LSDmatcher.h"
#include "ExtractLineSegment.h"
#include "Frame.h"
#include "KeyFrame.h"
#include "MapPoint.h"
#include "MapLine.h"
#include "Map.h"
#include "KeyFrameDatabase.h"
#include "ORBVocabulary.h"
#include "Converter.h"
#undef private
#undef protected
#include "oracle.h"

using namespace StructureSLAM;

// include/Converter.h:37 — src/Converter.cc needs g2o and is not compiled; this one function is all Frame.cc / KeyFrame.cc use
// (Converter.cc:30-38: one cv::Mat header per descriptor row)
std::vector<cv::Mat> StructureSLAM::Converter::toDescriptorVector(const cv::Mat& Descriptors) {
    std::vector<cv::Mat> v; v.reserve(Descriptors.rows);
    for (int j = 0; j < Descriptors.rows; j++) v.push_back(Descriptors.row(j));
    return v;
}

namespace {

struct Cam { float fx, fy, cx, cy, minx, maxx, miny, maxy; };

cv::Mat mat_from(const float* p, int r, int c) { cv::Mat m(r, c, CV_32F); for (int i = 0; i < r; i++) for (int j = 0; j < c; j++) m.at<float>(i, j) = p[i * c + j]; return m; }
cv::Mat pose44(const float* T12) {         // 3x4 row-major [R|t] -> 4x4
    cv::Mat m = cv::Mat::eye(4, 4, CV_32F);
    if (T12) for (int i = 0; i < 3; i++) for (int j = 0; j < 4; j++) m.at<float>(i, j) = T12[i * 4 + j];
    return m;
}
cv::Mat desc_mat(const uint8_t* d, int n) { cv::Mat m(std::max(n, 0), 32, CV_8UC1); if (n > 0) memcpy(m.data, d, (size_t)n * 32); return m; }

// everything a call creates, deleted when the call returns
struct Scene {
    Map map; ORBVocabulary voc; KeyFrameDatabase db;
    std::vector<Frame*> frames; std::vector<KeyFrame*> kfs; std::vector<MapPoint*> mps; std::vector<MapLine*> mls;
    Scene() : db(voc) {}
    ~Scene() { for (auto p : mps) delete p; for (auto p : mls) delete p; for (auto p : kfs) delete p; for (auto p : frames) delete p; }
};

void set_camera(const Cam& c) {
    Frame::fx = c.fx; Frame::fy = c.fy; Frame::cx = c.cx; Frame::cy = c.cy; Frame::invfx = 1.0f / c.fx; Frame::invfy = 1.0f / c.fy;
    Frame::mnMinX = c.minx; Frame::mnMaxX = c.maxx; Frame::mnMinY = c.miny; Frame::mnMaxY = c.maxy;
    // Frame.cc:96-97
    Frame::mfGridElementWidthInv = static_cast<float>(FRAME_GRID_COLS) / static_cast<float>(Frame::mnMaxX - Frame::mnMinX);
    Frame::mfGridElementHeightInv = static_cast<float>(FRAME_GRID_ROWS) / static_cast<float>(Frame::mnMaxY - Frame::mnMinY);
    Frame::mbInitialComputations = false;
}

// A Frame as the reference's constructor would leave it (Frame.cc:69-131), from already extracted features
Frame* make_frame(Scene& S, const Cam& cam, int nlevels, float scaleFactor, const orc_keypoint* kps, int n, const uint8_t* desc,
                  const int32_t* fv_nodes, const int32_t* fv_off, const int32_t* fv_idx, int fv_n, const float* Tcw12,
                  const uint8_t* ldesc = nullptr, int nl = 0) {
    set_camera(cam);
    Frame* F = new Frame();
    S.frames.push_back(F);
    ORBextractor ext(1000, scaleFactor, nlevels, 20, 7);      // the pyramid tables are the reference constructor's own (Frame.cc:77-83)
    F->mpORBvocabulary = &S.voc; F->mpORBextractorLeft = nullptr; F->mpORBextractorRight = nullptr; F->mpLineSegment = nullptr;
    F->mTimeStamp = 0; F->mbf = 0; F->mb = 0; F->mThDepth = 0; F->mpReferenceKF = nullptr; F->dealWithLine = true; F->blurNumber = 0;
    F->mnId = Frame::nNextId++;
    F->mnScaleLevels = ext.GetLevels(); F->mfScaleFactor = ext.GetScaleFactor(); F->mfLogScaleFactor = log(F->mfScaleFactor);
    F->mvScaleFactors = ext.GetScaleFactors(); F->mvInvScaleFactors = ext.GetInverseScaleFactors();
    F->mvLevelSigma2 = ext.GetScaleSigmaSquares(); F->mvInvLevelSigma2 = ext.GetInverseScaleSigmaSquares();
    F->N = n;
    F->mvKeys.resize(n);
    static_assert(sizeof(orc_keypoint) == sizeof(cv::KeyPoint), "layout");
    if (n) memcpy((void*)F->mvKeys.data(), kps, (size_t)n * sizeof(cv::KeyPoint));
    F->mvKeysUn = F->mvKeys;
    F->mvuRight = std::vector<float>(n, -1); F->mvDepth = std::vector<float>(n, -1);
    F->mDescriptors = desc_mat(desc, n);
    F->mvpMapPoints = std::vector<MapPoint*>(n, static_cast<MapPoint*>(NULL));
    F->mvbOutlier = std::vector<bool>(n, false);
    for (int k = 0; k < fv_n; k++) for (int j = fv_off[k]; j < fv_off[k + 1]; j++) F->mFeatVec.addFeature((unsigned)fv_nodes[k], (unsigned)fv_idx[j]);
    F->NL = nl;
    F->mLdesc = desc_mat(ldesc, nl);
    F->mvKeylinesUn.resize(nl); F->mvKeyLineFunctions.resize(nl);
    F->mvpMapLines = std::vector<MapLine*>(nl, static_cast<MapLine*>(NULL));
    F->mvbLineOutlier = std::vector<bool>(nl, false);
    F->mK = cv::Mat::eye(3, 3, CV_32F);
    F->mK.at<float>(0, 0) = cam.fx; F->mK.at<float>(1, 1) = cam.fy; F->mK.at<float>(0, 2) = cam.cx; F->mK.at<float>(1, 2) = cam.cy;
    F->mDistCoef = cv::Mat::zeros(4, 1, CV_32F);
    F->AssignFeaturesToGrid();                                   // Frame.cc:133-148
    F->SetPose(pose44(Tcw12));                                   // Frame.cc:217-233
    return F;
}
KeyFrame* make_kf(Scene& S, Frame* F) { KeyFrame* k = new KeyFrame(*F, &S.map, &S.db); S.kfs.push_back(k); return k; }   // KeyFrame.cc:41-72
MapPoint* make_mp(Scene& S, KeyFrame* kf, const float* Xw3) {
    const float z[3] = {0, 0, 1};
    MapPoint* p = new MapPoint(mat_from(Xw3 ? Xw3 : z, 3, 1), kf, &S.map);       // MapPoint.cc:36-50
    S.mps.push_back(p); return p;
}

}  // namespace

extern "C" {

// ------------------------------------------------------------------------------------------------
// ORBextractor (src/ORBextractor.cc, unmodified)
// ------------------------------------------------------------------------------------------------
/* ORBextractor::operator() :1043-1105 under the bump allocator; level_counts[nlevels] (may be NULL) = keypoints per level */
int ref_orb_extract(int nfeatures, float scaleFactor, int nlevels, int iniThFAST, int minThFAST,
                    const uint8_t* img, int w, int h, int pitch, orc_keypoint* kps, uint8_t* desc, int cap, int* level_counts) {
    BumpScope scope;
    ORBextractor ext(nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST);
    cv::Mat image(h, w, CV_8UC1, (void*)img, (size_t)pitch);
    std::vector<cv::KeyPoint> keys; cv::Mat descriptors;
    ext(image, cv::Mat(), keys, descriptors);
    const int n = (int)keys.size();
    if (level_counts) { for (int l = 0; l < nlevels; l++) level_counts[l] = 0; for (auto& k : keys) level_counts[k.octave]++; }
    for (int i = 0; i < n && i < cap; i++) { memcpy(&kps[i], &keys[i], sizeof(cv::KeyPoint)); memcpy(desc + 32 * (size_t)i, descriptors.ptr(i), 32); }
    return n;
}
/* constructor tables :410-470 */
void ref_orb_tables(int nfeatures, float scaleFactor, int nlevels, float* scale, float* invscale, float* sigma2, float* invsigma2,
                    int* nfeat_per_level, int* umax16) {
    ORBextractor ext(nfeatures, scaleFactor, nlevels, 20, 7);
    for (int l = 0; l < nlevels; l++) {
        scale[l] = ext.mvScaleFactor[l]; invscale[l] = ext.mvInvScaleFactor[l]; sigma2[l] = ext.mvLevelSigma2[l]; invsigma2[l] = ext.mvInvLevelSigma2[l];
        nfeat_per_level[l] = ext.mnFeaturesPerLevel[l];
    }
    for (int i = 0; i < 16; i++) umax16[i] = ext.umax[i];
}
/* ComputePyramid :1107-1132 — level l of the last pyramid, with or without the 19-px border */
int ref_orb_pyramid_level(const uint8_t* img, int w, int h, int pitch, float scaleFactor, int nlevels, int level, int bordered,
                          uint8_t* dst, int dcap, int* lw, int* lh) {
    ORBextractor ext(1000, scaleFactor, nlevels, 20, 7);
    cv::Mat image(h, w, CV_8UC1, (void*)img, (size_t)pitch);
    ext.ComputePyramid(image);
    cv::Mat m = ext.mvImagePyramid[level];
    const int b = bordered ? 19 : 0;
    *lw = m.cols + 2 * b; *lh = m.rows + 2 * b;
    if ((*lw) * (*lh) > dcap) return -1;
    for (int y = 0; y < *lh; y++) memcpy(dst + (size_t)y * (*lw), m.data + (ptrdiff_t)(y - b) * (ptrdiff_t)m.step - b, *lw);
    return 0;
}
/* DistributeOctTree :539-763 alone, under the bump allocator: indices of the chosen candidates, result order */
int ref_octree(const int* xs, const int* ys, const int* resp, int n, int minX, int maxX, int minY, int maxY, int N, int* out_idx, int cap) {
    BumpScope scope;
    ORBextractor ext(1000, 1.2f, 8, 20, 7);
    std::vector<cv::KeyPoint> v(n);
    for (int i = 0; i < n; i++) { v[i] = cv::KeyPoint((float)xs[i], (float)ys[i], 7.f, -1.f, (float)resp[i]); v[i].class_id = i; }
    std::vector<cv::KeyPoint> r = ext.DistributeOctTree(v, minX, maxX, minY, maxY, N, 0);
    for (int i = 0; i < (int)r.size() && i < cap; i++) out_idx[i] = r[i].class_id;
    return (int)r.size();
}

// ------------------------------------------------------------------------------------------------
// ORBmatcher (src/ORBmatcher.cc, unmodified)
// ------------------------------------------------------------------------------------------------
int ref_descriptor_distance(const uint8_t* a, const uint8_t* b) { return ORBmatcher::DescriptorDistance(desc_mat(a, 1), desc_mat(b, 1)); }   // :1650
int ref_line_descriptor_distance(const uint8_t* a, const uint8_t* b) { return LSDmatcher::DescriptorDistance(desc_mat(a, 1), desc_mat(b, 1)); }   // LSDmatcher.cpp:364

static const Cam kCam640 = {500.f, 500.f, 320.f, 240.f, 0.f, 640.f, 0.f, 480.f};

/* SearchByBoW(KeyFrame*, Frame&, vector<MapPoint*>&) :159-291.  state1[i]: 0 = no MapPoint, 1 = good MapPoint, 2 = bad MapPoint */
int ref_search_by_bow(const uint8_t* d1, int n1, const orc_keypoint* k1, const uint8_t* d2, int n2, const orc_keypoint* k2,
                      const int32_t* nodes1, const int32_t* off1, const int32_t* idx1, int nn1,
                      const int32_t* nodes2, const int32_t* off2, const int32_t* idx2, int nn2,
                      const uint8_t* state1, float nnratio, int checkOri, int32_t* match2) {
    Scene S;
    Frame* F1 = make_frame(S, kCam640, 8, 1.2f, k1, n1, d1, nodes1, off1, idx1, nn1, nullptr);
    KeyFrame* KF = make_kf(S, F1);
    std::map<MapPoint*, int> index;
    for (int i = 0; i < n1; i++) if (state1[i]) { MapPoint* p = make_mp(S, KF, nullptr); KF->AddMapPoint(p, i); if (state1[i] == 2) p->mbBad = true; index[p] = i; }
    Frame* F2 = make_frame(S, kCam640, 8, 1.2f, k2, n2, d2, nodes2, off2, idx2, nn2, nullptr);
    std::vector<MapPoint*> matches;
    ORBmatcher matcher(nnratio, checkOri != 0);
    const int n = matcher.SearchByBoW(KF, *F2, matches);
    for (int j = 0; j < n2; j++) match2[j] = matches[j] ? index[matches[j]] : -1;
    return n;
}
/* SearchByBoW(KeyFrame*, KeyFrame*, vector<MapPoint*>&) :525-658: match12[i] = index in KF2 */
int ref_search_by_bow_kf(const uint8_t* d1, int n1, const orc_keypoint* k1, const uint8_t* d2, int n2, const orc_keypoint* k2,
                         const int32_t* nodes1, const int32_t* off1, const int32_t* idx1, int nn1,
                         const int32_t* nodes2, const int32_t* off2, const int32_t* idx2, int nn2,
                         const uint8_t* state1, const uint8_t* state2, float nnratio, int checkOri, int32_t* match12) {
    Scene S;
    KeyFrame* KF1 = make_kf(S, make_frame(S, kCam640, 8, 1.2f, k1, n1, d1, nodes1, off1, idx1, nn1, nullptr));
    KeyFrame* KF2 = make_kf(S, make_frame(S, kCam640, 8, 1.2f, k2, n2, d2, nodes2, off2, idx2, nn2, nullptr));
    std::map<MapPoint*, int> index2;
    for (int i = 0; i < n1; i++) if (state1[i]) { MapPoint* p = make_mp(S, KF1, nullptr); KF1->AddMapPoint(p, i); if (state1[i] == 2) p->mbBad = true; }
    for (int i = 0; i < n2; i++) if (state2[i]) { MapPoint* p = make_mp(S, KF2, nullptr); KF2->AddMapPoint(p, i); if (state2[i] == 2) p->mbBad = true; index2[p] = i; }
    std::vector<MapPoint*> matches;
    ORBmatcher matcher(nnratio, checkOri != 0);
    const int n = matcher.SearchByBoW(KF1, KF2, matches);
    for (int i = 0; i < n1; i++) match12[i] = matches[i] ? index2[matches[i]] : -1;
    return n;
}
/* SearchForTriangulation :660-826 (bOnlyStereo=false).  Tcw1/Tcw2: 3x4 poses; the epipole is computed by the reference from them.
   pairs: 2 ints per match.  epi[2] receives the same epipole evaluated with the same KeyFrame accessors (for the oracle's input). */
int ref_search_for_triangulation(const uint8_t* d1, int n1, const orc_keypoint* k1, const uint8_t* d2, int n2, const orc_keypoint* k2,
                                 const int32_t* nodes1, const int32_t* off1, const int32_t* idx1, int nn1,
                                 const int32_t* nodes2, const int32_t* off2, const int32_t* idx2, int nn2,
                                 const uint8_t* has_mp1, const uint8_t* has_mp2, const float* cam8, const float* Tcw1, const float* Tcw2,
                                 const float* F12, int checkOri, int32_t* pairs, float* epi) {
    Scene S;
    Cam cam; memcpy(&cam, cam8, sizeof(cam));
    KeyFrame* KF1 = make_kf(S, make_frame(S, cam, 8, 1.2f, k1, n1, d1, nodes1, off1, idx1, nn1, Tcw1));
    KeyFrame* KF2 = make_kf(S, make_frame(S, cam, 8, 1.2f, k2, n2, d2, nodes2, off2, idx2, nn2, Tcw2));
    for (int i = 0; i < n1; i++) if (has_mp1[i]) KF1->AddMapPoint(make_mp(S, KF1, nullptr), i);
    for (int i = 0; i < n2; i++) if (has_mp2[i]) KF2->AddMapPoint(make_mp(S, KF2, nullptr), i);
    if (epi) {   // ORBmatcher.cc:667-673, same accessors
        cv::Mat Cw = KF1->GetCameraCenter(), R2w = KF2->GetRotation(), t2w = KF2->GetTranslation();
        cv::Mat C2 = R2w * Cw + t2w;
        const float invz = 1.0f / C2.at<float>(2);
        epi[0] = KF2->fx * C2.at<float>(0) * invz + KF2->cx; epi[1] = KF2->fy * C2.at<float>(1) * invz + KF2->cy;
    }
    std::vector<std::pair<size_t, size_t> > vp;
    ORBmatcher matcher(0.6f, checkOri != 0);
    const int n = matcher.SearchForTriangulation(KF1, KF2, mat_from(F12, 3, 3), vp, false);
    for (size_t i = 0; i < vp.size(); i++) { pairs[2 * i] = (int32_t)vp[i].first; pairs[2 * i + 1] = (int32_t)vp[i].second; }
    return n;
}

/* SearchByProjection(Frame& Current, const Frame& Last, th, bMono) :1331-1473.  Last frame: valid1 (has MapPoint), obs1 (the MapPoint has
   observations), outlier... as the oracle's orc_search_by_projection_frame takes them.  claimed2[j] != 0: current feature j already
   holds a MapPoint with observations.  assign2[j] = index of the last-frame feature whose MapPoint was assigned, -1 none. */
int ref_search_by_projection_frame(int n1, const uint8_t* valid1, const uint8_t* obs1, const float* Xw, const uint8_t* dmp,
                                   const orc_keypoint* k1, int n2, const uint8_t* d2, const orc_keypoint* k2, const uint8_t* claimed2,
                                   const float* uright2, float mbf,
                                   const float* Tcw, const float* Tlw, const float* cam8, int nlevels, float scaleFactor, float th, int mono, int checkOri,
                                   int32_t* assign2) {
    Scene S;
    Cam cam; memcpy(&cam, cam8, sizeof(cam));
    std::vector<uint8_t> zero((size_t)std::max(n1, 1) * 32, 0);
    Frame* L = make_frame(S, cam, nlevels, scaleFactor, k1, n1, zero.data(), nullptr, nullptr, nullptr, 0, Tlw);
    KeyFrame* KFl = make_kf(S, L);
    Frame* Cf = make_frame(S, cam, nlevels, scaleFactor, k2, n2, d2, nullptr, nullptr, nullptr, 0, Tcw);
    Cf->mbf = mbf; Cf->mb = Cf->mbf / Frame::fx;                 // Frame.cc:128
    if (uright2) for (int j = 0; j < n2; j++) Cf->mvuRight[j] = uright2[j];
    std::map<MapPoint*, int> index;
    for (int i = 0; i < n1; i++) if (valid1[i]) {
        MapPoint* p = make_mp(S, KFl, Xw + 3 * i);
        desc_mat(dmp + 32 * (size_t)i, 1).copyTo(p->mDescriptor);
        if (obs1 == nullptr || obs1[i]) p->AddObservation(KFl, i);
        L->mvpMapPoints[i] = p; index[p] = i;
    }
    std::vector<MapPoint*> claimers;
    if (claimed2) for (int j = 0; j < n2; j++) if (claimed2[j]) {
        const float far[3] = {0, 0, 100};
        MapPoint* p = make_mp(S, KFl, far); p->AddObservation(KFl, 0); Cf->mvpMapPoints[j] = p; index[p] = -2;
    }
    ORBmatcher matcher(0.9f, checkOri != 0);
    const int n = matcher.SearchByProjection(*Cf, *L, th, mono != 0);
    for (int j = 0; j < n2; j++) { MapPoint* p = Cf->mvpMapPoints[j]; assign2[j] = p ? index[p] : -1; }
    return n;
}

/* SearchByProjection(Frame& F, const vector<MapPoint*>&, th) :45-129 (TrackLocalMap).  Per MapPoint: the tracking fields
   Frame::isInFrustum would have filled (mbTrackInView, mTrackProjX/Y, mnTrackScaleLevel, mTrackViewCos), its descriptor, bad flag.
   claimed2[j]: 0 free, 1 holds a MapPoint WITH observations (skipped), 2 holds a MapPoint without observations (may be overwritten).
   assign2[j] = index of the MapPoint assigned to frame feature j (-1 none, -2 a pre-existing one). */
int ref_search_by_projection_mps(int nmp, const uint8_t* inview, const uint8_t* bad, const uint8_t* obs, const float* projx, const float* projy,
                                 const int32_t* level, const float* viewcos, const uint8_t* dmp,
                                 int n2, const uint8_t* d2, const orc_keypoint* k2, const uint8_t* claimed2,
                                 const float* cam8, int nlevels, float scaleFactor, float nnratio, float th, int32_t* assign2) {
    Scene S;
    Cam cam; memcpy(&cam, cam8, sizeof(cam));
    Frame* F = make_frame(S, cam, nlevels, scaleFactor, k2, n2, d2, nullptr, nullptr, nullptr, 0, nullptr);
    orc_keypoint one; memset(&one, 0, sizeof(one)); one.x = one.y = 10.f;
    const uint8_t zero32[32] = {0};
    KeyFrame* KF = make_kf(S, make_frame(S, cam, nlevels, scaleFactor, &one, 1, zero32, nullptr, nullptr, nullptr, 0, nullptr));   // the observer (AddObservation reads mvuRight[idx])
    std::map<MapPoint*, int> index;
    std::vector<MapPoint*> mps;
    for (int i = 0; i < nmp; i++) {
        MapPoint* p = make_mp(S, KF, nullptr);
        p->mbTrackInView = inview[i] != 0; p->mbBad = bad && bad[i]; p->mTrackProjX = projx[i]; p->mTrackProjY = projy[i]; p->mTrackProjXR = -1;
        p->mnTrackScaleLevel = level[i]; p->mTrackViewCos = viewcos[i];
        desc_mat(dmp + 32 * (size_t)i, 1).copyTo(p->mDescriptor);
        if (obs && obs[i]) p->AddObservation(KF, 0);
        mps.push_back(p); index[p] = i;
    }
    if (claimed2) for (int j = 0; j < n2; j++) if (claimed2[j]) {
        MapPoint* p = make_mp(S, KF, nullptr); if (claimed2[j] == 1) p->AddObservation(KF, 0); F->mvpMapPoints[j] = p; index[p] = -2;
    }
    ORBmatcher matcher(nnratio, true);
    const int n = matcher.SearchByProjection(*F, mps, th);
    for (int j = 0; j < n2; j++) { MapPoint* p = F->mvpMapPoints[j]; assign2[j] = p ? index[p] : -1; }
    return n;
}

/* SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize) :408-523.  prev[2*n1] in/out, matches12[n1] out */
int ref_search_for_initialization(int n1, const uint8_t* d1, const orc_keypoint* k1, int n2, const uint8_t* d2, const orc_keypoint* k2,
                                  float* prev, const float* cam8, int nlevels, float scaleFactor, float nnratio, int checkOri, int windowSize,
                                  int32_t* matches12) {
    Scene S;
    Cam cam; memcpy(&cam, cam8, sizeof(cam));
    Frame* F1 = make_frame(S, cam, nlevels, scaleFactor, k1, n1, d1, nullptr, nullptr, nullptr, 0, nullptr);
    Frame* F2 = make_frame(S, cam, nlevels, scaleFactor, k2, n2, d2, nullptr, nullptr, nullptr, 0, nullptr);
    std::vector<cv::Point2f> vprev(n1);
    for (int i = 0; i < n1; i++) vprev[i] = cv::Point2f(prev[2 * i], prev[2 * i + 1]);
    std::vector<int> m12;
    ORBmatcher matcher(nnratio, checkOri != 0);
    const int n = matcher.SearchForInitialization(*F1, *F2, vprev, m12, windowSize);
    for (int i = 0; i < n1; i++) { matches12[i] = m12[i]; prev[2 * i] = vprev[i].x; prev[2 * i + 1] = vprev[i].y; }
    return n;
}

/* Frame::GetFeaturesInArea :368-421 over Frame::AssignFeaturesToGrid :133-148 */
int ref_features_in_area(int n, const orc_keypoint* kps, const float* cam8, float x, float y, float r, int minLevel, int maxLevel, int32_t* out, int cap) {
    Scene S;
    Cam cam; memcpy(&cam, cam8, sizeof(cam));
    std::vector<uint8_t> zero((size_t)std::max(n, 1) * 32, 0);
    Frame* F = make_frame(S, cam, 8, 1.2f, kps, n, zero.data(), nullptr, nullptr, nullptr, 0, nullptr);
    std::vector<size_t> v = F->GetFeaturesInArea(x, y, r, minLevel, maxLevel);
    for (int i = 0; i < (int)v.size() && i < cap; i++) out[i] = (int32_t)v[i];
    return (int)v.size();
}

/* MapPoint::ComputeDistinctiveDescriptors MapPoint.cc:247-312 for CSR groups: one MapPoint per group, one KeyFrame per descriptor,
   created in order under the bump allocator (the reference walks a std::map keyed by KeyFrame*) */
void ref_descriptor_medoid(const uint8_t* desc, const int32_t* off, int ngroups, int32_t* best_idx) {
    for (int g = 0; g < ngroups; g++) {
        BumpScope scope;
        Scene* S = new Scene();
        const int n = off[g + 1] - off[g];
        orc_keypoint kp; memset(&kp, 0, sizeof(kp)); kp.x = 10; kp.y = 10;
        std::vector<KeyFrame*> kfs;
        for (int i = 0; i < n; i++) kfs.push_back(make_kf(*S, make_frame(*S, kCam640, 8, 1.2f, &kp, 1, desc + 32 * (size_t)(off[g] + i), nullptr, nullptr, nullptr, 0, nullptr)));
        best_idx[g] = -1;
        if (n > 0) {
            MapPoint* p = make_mp(*S, kfs[0], nullptr);
            for (int i = 0; i < n; i++) p->AddObservation(kfs[i], 0);
            p->ComputeDistinctiveDescriptors();
            cv::Mat d = p->GetDescriptor();
            for (int i = 0; i < n; i++) if (memcmp(d.data, desc + 32 * (size_t)(off[g] + i), 32) == 0) { best_idx[g] = i; break; }
        }
        delete S;
    }
}

// ------------------------------------------------------------------------------------------------
// LSDmatcher (src/LSDmatcher.cpp, unmodified) — the five knnMatch entry points; same modes/outputs as orc_line_match
// ------------------------------------------------------------------------------------------------
int ref_line_match(int mode, const uint8_t* d1, int n1, const uint8_t* d2, int n2, const uint8_t* has_ml1, const uint8_t* has_ml2,
                   int32_t* out, int* nout, double* mad2) {
    Scene S;
    orc_keypoint kp; memset(&kp, 0, sizeof(kp));
    Frame* F1 = make_frame(S, kCam640, 8, 1.2f, &kp, 0, nullptr, nullptr, nullptr, nullptr, 0, nullptr, d1, n1);
    Frame* F2 = make_frame(S, kCam640, 8, 1.2f, &kp, 0, nullptr, nullptr, nullptr, nullptr, 0, nullptr, d2, n2);
    KeyFrame* K1 = make_kf(S, F1); KeyFrame* K2 = make_kf(S, F2);
    std::map<MapLine*, int> i1, i2;
    Vector6d P; P << 0.0, 0.0, 1.0, 1.0, 0.0, 1.0;
    for (int i = 0; i < n1; i++) if (has_ml1 && has_ml1[i]) { MapLine* l = new MapLine(P, K1, &S.map); S.mls.push_back(l); K1->AddMapLine(l, i); i1[l] = i; }
    for (int i = 0; i < n2; i++) if (has_ml2 && has_ml2[i]) { MapLine* l = new MapLine(P, K2, &S.map); S.mls.push_back(l); K2->AddMapLine(l, i); i2[l] = i; }
    LSDmatcher lm;
    int n = 0, k = 0;
    if (mode == 0) {            // SearchByProjection(KF, F, vpMapLineMatches) :143-183 (== SearchByDescriptor(KF,F) :286-327)
        std::vector<MapLine*> m; n = lm.SearchByProjection(K1, *F2, m);
        for (int j = 0; j < n2; j++) out[j] = m[j] ? i1[m[j]] : -1;
    } else if (mode == 4) {     // SearchByDescriptor(KF, F) :286-327 (prints one line to stdout)
        std::cout.setstate(std::ios_base::badbit);          // the function prints a progress line (:300)
        std::vector<MapLine*> m; n = lm.SearchByDescriptor(K1, *F2, m);
        std::cout.clear();
        for (int j = 0; j < n2; j++) out[j] = m[j] ? i1[m[j]] : -1;
    } else if (mode == 1) {     // SerachForInitialize :257-284
        std::vector<std::pair<int, int> > m; n = lm.SerachForInitialize(*F1, *F2, m);
        for (auto& p : m) { out[2 * k] = p.first; out[2 * k + 1] = p.second; k++; }
    } else if (mode == 2) {     // SearchByDescriptor(KF, KF2) :329-362
        std::vector<MapLine*> m; n = lm.SearchByDescriptor(K1, K2, m);
        for (int i = 0; i < n1; i++) out[i] = m[i] ? i2[m[i]] : -1;
    } else {                    // SearchForTriangulation :382-415
        std::vector<std::pair<size_t, size_t> > m; n = lm.SearchForTriangulation(K1, K2, m);
        for (auto& p : m) { out[2 * k] = (int32_t)p.first; out[2 * k + 1] = (int32_t)p.second; k++; }
    }
    if (nout) *nout = k;
    if (mad2) {                 // Frame::lineDescriptorMAD Frame.cc:190-215 on the same knn table
        cv::BFMatcher bfm(cv::NORM_HAMMING, false);
        std::vector<std::vector<cv::DMatch> > lm2;
        bfm.knnMatch(F1->mLdesc, F2->mLdesc, lm2, 2);
        F2->lineDescriptorMAD(lm2, mad2[0], mad2[1]);
    }
    return n;
}

// ------------------------------------------------------------------------------------------------
// DBoW2 (Thirdparty/DBoW2, unmodified): vocabulary text loader + transform
// ------------------------------------------------------------------------------------------------
void* ref_vocab_load_text(const char* path) {
    ORBVocabulary* v = new ORBVocabulary();
    if (!v->loadFromTextFile(path)) { delete v; return nullptr; }
    return v;
}
void ref_vocab_destroy(void* v) { delete (ORBVocabulary*)v; }
int ref_vocab_size(void* v) { return (int)((ORBVocabulary*)v)->size(); }
/* TemplatedVocabulary::transform(features, BowVector&, FeatureVector&, levelsup) :1127-1197 + per-feature transform :1218-1259.
   word[i], weight[i] per feature (the word the feature descends to; -1/0 when it is a stopped word); node[i] = FeatureVector node;
   bow_ids/bow_w: the normalised BowVector (ascending word id), returns its size */
int ref_vocab_transform(void* voc, const uint8_t* desc, int n, int levelsup, int32_t* node, int32_t* bow_ids, double* bow_w, int cap) {
    ORBVocabulary* v = (ORBVocabulary*)voc;
    cv::Mat D = desc_mat(desc, n);
    std::vector<cv::Mat> feats = Converter::toDescriptorVector(D);
    DBoW2::BowVector bv; DBoW2::FeatureVector fv;
    v->transform(feats, bv, fv, levelsup);
    for (int i = 0; i < n; i++) node[i] = -1;
    for (auto& kv : fv) for (unsigned i : kv.second) node[i] = (int32_t)kv.first;
    int k = 0;
    for (auto& kv : bv) { if (k < cap) { bow_ids[k] = (int32_t)kv.first; bow_w[k] = kv.second; } k++; }
    return k;
}
/* single-feature transform (word id + weight), TemplatedVocabulary.h:1218-1259 via the public overload :1200-1210 */
void ref_vocab_words(void* voc, const uint8_t* desc, int n, int32_t* word, double* weight) {
    ORBVocabulary* v = (ORBVocabulary*)voc;
    cv::Mat D = desc_mat(desc, n);
    for (int i = 0; i < n; i++) {
        DBoW2::WordId id; DBoW2::WordValue w;
        v->transform(D.row(i), id, w);
        word[i] = (int32_t)id; weight[i] = w;
    }
}

// ------------------------------------------------------------------------------------------------
// LineSegment::ExtractLineSegment (src/ExtractLineSegment.cpp:18-69, unmodified; lsdNFeatures is hard-coded to 40 there)
// ------------------------------------------------------------------------------------------------
int ref_line_extract(const uint8_t* img, int w, int h, int pitch, orc_keyline* kl, uint8_t* ldesc, double* lineeq3, int cap) {
    cv::Mat image(h, w, CV_8UC1, (void*)img, (size_t)pitch);
    std::vector<KeyLine> keylines; cv::Mat desc; std::vector<Eigen::Vector3d> fn;
    LineSegment ls;
    ls.ExtractLineSegment(image, keylines, desc, fn);
    const int n = (int)keylines.size();
    for (int i = 0; i < n && i < cap; i++) {
        memcpy(&kl[i], &keylines[i], sizeof(KeyLine)); memcpy(ldesc + 32 * (size_t)i, desc.ptr(i), 32);
        for (int k = 0; k < 3; k++) lineeq3[3 * i + k] = fn[i](k);
    }
    return n;
}

// ------------------------------------------------------------------------------------------------
// Frame::Frame(imGray, ...) src/Frame.cc:69-131 — ORB then LSD, UndistortKeyPoints, grid.  dist4: k1 k2 p1 p2.
// Outputs: keys (raw), keysUn, descriptors, keylines, line descriptors, line equations, and the 64x48 grid as CSR.
// ------------------------------------------------------------------------------------------------
int ref_frame_from_image(const uint8_t* img, int w, int h, int pitch, int nfeatures, float scaleFactor, int nlevels, int iniTh, int minTh,
                         const float* K4, const float* dist, int ndist, orc_keypoint* keys, orc_keypoint* keysUn, uint8_t* desc, int cap,
                         orc_keyline* kl, uint8_t* ldesc, double* lineeq3, int lcap, int* NL,
                         int32_t* grid_off /*64*48+1*/, int32_t* grid_idx /*cap*/, float* bounds4) {
    BumpScope scope;
    ORBextractor ext(nfeatures, scaleFactor, nlevels, iniTh, minTh);
    ORBVocabulary voc;
    cv::Mat K = cv::Mat::eye(3, 3, CV_32F);
    K.at<float>(0, 0) = K4[0]; K.at<float>(1, 1) = K4[1]; K.at<float>(0, 2) = K4[2]; K.at<float>(1, 2) = K4[3];
    cv::Mat D(ndist == 5 ? 5 : 4, 1, CV_32F); for (int i = 0; i < D.rows; i++) D.at<float>(i) = dist[i];   // mDistCoef (Tracking.cc:61-72)
    Frame::mbInitialComputations = true;
    cv::Mat image(h, w, CV_8UC1, (void*)img, (size_t)pitch);
    Frame F(image, 0.0, &ext, &voc, K, D, 0.f, 0.f);
    const int n = F.N;
    for (int i = 0; i < n && i < cap; i++) {
        memcpy(&keys[i], &F.mvKeys[i], 28); memcpy(&keysUn[i], &F.mvKeysUn[i], 28); memcpy(desc + 32 * (size_t)i, F.mDescriptors.ptr(i), 32);
    }
    *NL = F.NL;
    for (int i = 0; i < F.NL && i < lcap; i++) {
        memcpy(&kl[i], &F.mvKeylinesUn[i], sizeof(KeyLine)); memcpy(ldesc + 32 * (size_t)i, F.mLdesc.ptr(i), 32);
        for (int k = 0; k < 3; k++) lineeq3[3 * i + k] = F.mvKeyLineFunctions[i](k);
    }
    int k = 0;
    for (int c = 0; c < FRAME_GRID_COLS; c++) for (int r = 0; r < FRAME_GRID_ROWS; r++) {
        grid_off[c * FRAME_GRID_ROWS + r] = k;
        for (size_t v : F.mGrid[c][r]) { if (k < cap) grid_idx[k] = (int32_t)v; k++; }
    }
    grid_off[FRAME_GRID_COLS * FRAME_GRID_ROWS] = k;
    bounds4[0] = Frame::mnMinX; bounds4[1] = Frame::mnMaxX; bounds4[2] = Frame::mnMinY; bounds4[3] = Frame::mnMaxY;
    return n;
}

/* Tracking::GrabImageMonocularWithPL's colour conversion (src/Tracking.cc:148-161) through the stand-in cvtColor: code per minicv.hpp */
void ref_cvt_gray(const uint8_t* src, int w, int h, int cn, int rgb, uint8_t* dst) {
    cv::Mat s(h, w, CV_MAKETYPE(CV_8U, cn), (void*)src, (size_t)w * cn), d;
    cv::cvtColor(s, d, cn == 3 ? (rgb ? CV_RGB2GRAY : CV_BGR2GRAY) : (rgb ? CV_RGBA2GRAY : CV_BGRA2GRAY));
    memcpy(dst, d.data, (size_t)w * h);
}


// ------------------------------------------------------------------------------------------------
// SURVEY.md 8(f) row 3: line projection matchers and Fuse (src/LSDmatcher.cpp, src/ORBmatcher.cc, unmodified)
// ------------------------------------------------------------------------------------------------
namespace {
void set_keylines(Frame* F, int nl, const float* kl, const int32_t* oct) {      // pt.x, pt.y, angle per line; the octave
    for (int j = 0; j < nl; j++) {
        KeyLine& k = F->mvKeylinesUn[j];
        memset(&k, 0, sizeof(k));
        k.pt.x = kl[3 * j]; k.pt.y = kl[3 * j + 1]; k.angle = kl[3 * j + 2]; k.octave = oct[j]; k.class_id = j;
    }
}
MapLine* make_ml(Scene& S, KeyFrame* kf, const double* P6, const uint8_t* desc) {
    Vector6d P; for (int k = 0; k < 6; k++) P(k) = P6 ? P6[k] : (k == 2 || k == 5 ? 1.0 : (k == 3 ? 1.0 : 0.0));
    MapLine* l = new MapLine(P, kf, &S.map); S.mls.push_back(l);
    if (desc) desc_mat(desc, 1).copyTo(l->mLDescriptor);
    return l;
}
KeyFrame* make_observer(Scene& S, const Cam& cam, int nlevels, float scaleFactor) {   // a KeyFrame with one feature and one line, to be an observation of
    orc_keypoint one; memset(&one, 0, sizeof(one)); one.x = one.y = 10.f;
    const uint8_t zero32[32] = {0};
    return make_kf(S, make_frame(S, cam, nlevels, scaleFactor, &one, 1, zero32, nullptr, nullptr, nullptr, 0, nullptr, zero32, 1));
}
}  // namespace

/* LSDmatcher::SearchByProjection(Frame& Current, const Frame& Last, th, bMono) :22-141.  state1[i]: 0 no MapLine, 1 good, 2 bad, 3 good but
   mvbLineOutlier; obs1[i]: the MapLine has an observation; oct1[i] = LastFrame.mvKeys[i].octave (the Last frame gets nl1 keypoints);
   held2[j]: 0 free, 1 a MapLine WITH observations, 2 one without.  assign2[j] = index of the Last-frame line whose MapLine sits there
   afterwards (-1 none, -2 the pre-existing one). */
int ref_line_projection_frame(int nl1, const uint8_t* state1, const uint8_t* obs1, const double* Pw6, const uint8_t* dml, const int32_t* oct1,
                              int nl2, const uint8_t* ld2, const float* kl2, const int32_t* oct2, const uint8_t* held2,
                              const float* Tcw, const float* Tlw, const float* cam8, float mb, int nlevels, float scaleFactor, float nnratio, float th, int mono,
                              int32_t* assign2) {
    Scene S;
    Cam cam; memcpy(&cam, cam8, sizeof(cam));
    std::vector<orc_keypoint> k1((size_t)std::max(nl1, 1)); memset(k1.data(), 0, k1.size() * sizeof(orc_keypoint));
    for (int i = 0; i < nl1; i++) { k1[i].x = k1[i].y = 20.f; k1[i].octave = oct1[i]; }
    std::vector<uint8_t> zero((size_t)std::max(nl1, 1) * 32, 0);
    Frame* L = make_frame(S, cam, nlevels, scaleFactor, k1.data(), nl1, zero.data(), nullptr, nullptr, nullptr, 0, Tlw, zero.data(), nl1);
    KeyFrame* KFl = make_kf(S, L);
    Frame* Cf = make_frame(S, cam, nlevels, scaleFactor, k1.data(), 0, nullptr, nullptr, nullptr, nullptr, 0, Tcw, ld2, nl2);
    Cf->mb = mb;
    set_keylines(Cf, nl2, kl2, oct2);
    std::map<MapLine*, int> index;
    for (int i = 0; i < nl1; i++) if (state1[i]) {
        MapLine* l = make_ml(S, KFl, Pw6 + 6 * (size_t)i, dml + 32 * (size_t)i);
        if (obs1[i]) l->AddObservation(KFl, i);
        if (state1[i] == 2) l->mbBad = true;
        if (state1[i] == 3) L->mvbLineOutlier[i] = true;
        L->mvpMapLines[i] = l; index[l] = i;
    }
    if (held2) for (int j = 0; j < nl2; j++) if (held2[j]) {
        MapLine* l = make_ml(S, KFl, nullptr, nullptr); if (held2[j] == 1) l->AddObservation(KFl, 0); Cf->mvpMapLines[j] = l; index[l] = -2;
    }
    LSDmatcher matcher(nnratio, true);
    const int n = matcher.SearchByProjection(*Cf, *L, th, mono != 0);
    for (int j = 0; j < nl2; j++) { MapLine* l = Cf->mvpMapLines[j]; assign2[j] = l ? index[l] : -1; }
    return n;
}

/* LSDmatcher::SearchByProjection(Frame&, const vector<MapLine*>&, th) :185-255 (Tracking::SearchLocalLines, Tracking.cc:1783) */
int ref_line_projection_mls(int nml, const uint8_t* inview, const uint8_t* bad, const uint8_t* obs, const float* proj4, const int32_t* level,
                            const float* viewcos, const uint8_t* dml, int nl2, const uint8_t* ld2, const float* kl2, const int32_t* oct2,
                            const uint8_t* held2, const float* cam8, int nlevels, float scaleFactor, float nnratio, float th, int32_t* assign2) {
    Scene S;
    Cam cam; memcpy(&cam, cam8, sizeof(cam));
    orc_keypoint none; memset(&none, 0, sizeof(none));
    Frame* F = make_frame(S, cam, nlevels, scaleFactor, &none, 0, nullptr, nullptr, nullptr, nullptr, 0, nullptr, ld2, nl2);
    set_keylines(F, nl2, kl2, oct2);
    KeyFrame* KF = make_observer(S, cam, nlevels, scaleFactor);
    std::map<MapLine*, int> index;
    std::vector<MapLine*> mls;
    for (int i = 0; i < nml; i++) {
        MapLine* l = make_ml(S, KF, nullptr, dml + 32 * (size_t)i);
        l->mbTrackInView = inview[i] != 0; l->mbBad = bad && bad[i];
        l->mTrackProjX1 = proj4[4 * i]; l->mTrackProjY1 = proj4[4 * i + 1]; l->mTrackProjX2 = proj4[4 * i + 2]; l->mTrackProjY2 = proj4[4 * i + 3];
        l->mnTrackScaleLevel = level[i]; l->mTrackViewCos = viewcos[i];
        if (obs && obs[i]) l->AddObservation(KF, 0);
        mls.push_back(l); index[l] = i;
    }
    if (held2) for (int j = 0; j < nl2; j++) if (held2[j]) {
        MapLine* l = make_ml(S, KF, nullptr, nullptr); if (held2[j] == 1) l->AddObservation(KF, 0); F->mvpMapLines[j] = l; index[l] = -2;
    }
    LSDmatcher matcher(nnratio, true);
    const int n = matcher.SearchByProjection(*F, mls, th);
    for (int j = 0; j < nl2; j++) { MapLine* l = F->mvpMapLines[j]; assign2[j] = l ? index[l] : -1; }
    return n;
}

/* ORBmatcher::Fuse(KeyFrame*, const vector<MapPoint*>&, th) :828-973.  state[i]: 0 NULL entry, 1 good, 2 bad, 3 already observed by the KeyFrame;
   nobs[i]: observations in other KeyFrames; minDist/maxDist: mfMinDistance/mfMaxDistance.  kfobs[j]: -1 the KeyFrame feature holds no MapPoint,
   >= 0 it holds one with that many OTHER observations.  fused_idx[i]: the KeyFrame feature MapPoint i ended up at or was replaced into
   (-1: not fused); Ow3, minInv, maxInv, logScale: what the reference's accessors return (inputs of the oracle's projection stage). */
int ref_fuse_points(int nmp, const uint8_t* state, const int32_t* nobs, const float* Xw, const float* normal, const float* minDist, const float* maxDist,
                    const uint8_t* dmp, int n2, const uint8_t* d2, const orc_keypoint* k2, const float* uright2, const int32_t* kfobs,
                    const float* Tcw, const float* cam8, float mbf, int nlevels, float scaleFactor, float th,
                    int32_t* fused_idx, float* Ow3, float* minInv, float* maxInv, float* logScale) {
    Scene S;
    Cam cam; memcpy(&cam, cam8, sizeof(cam));
    Frame* F = make_frame(S, cam, nlevels, scaleFactor, k2, n2, d2, nullptr, nullptr, nullptr, 0, Tcw);
    F->mbf = mbf; F->mb = mbf / cam.fx;
    if (uright2) for (int j = 0; j < n2; j++) F->mvuRight[j] = uright2[j];
    KeyFrame* KF = make_kf(S, F);
    int maxobs = 0;
    for (int i = 0; i < nmp; i++) maxobs = std::max(maxobs, nobs[i]);
    for (int j = 0; j < n2; j++) maxobs = std::max(maxobs, kfobs[j]);
    std::vector<KeyFrame*> observers;
    for (int k = 0; k < maxobs; k++) observers.push_back(make_observer(S, cam, nlevels, scaleFactor));
    for (int j = 0; j < n2; j++) if (kfobs[j] >= 0) {
        const float far[3] = {0, 0, 1000};
        MapPoint* q = make_mp(S, KF, far);
        desc_mat(d2 + 32 * (size_t)j, 1).copyTo(q->mDescriptor);
        q->AddObservation(KF, j); KF->AddMapPoint(q, j);
        for (int k = 0; k < kfobs[j]; k++) q->AddObservation(observers[k], 0);
    }
    std::vector<MapPoint*> mps(nmp, static_cast<MapPoint*>(NULL));
    for (int i = 0; i < nmp; i++) {
        if (!state[i]) continue;
        MapPoint* p = make_mp(S, observers.empty() ? KF : observers[0], Xw + 3 * (size_t)i);
        mat_from(normal + 3 * (size_t)i, 3, 1).copyTo(p->mNormalVector);
        p->mfMinDistance = minDist[i]; p->mfMaxDistance = maxDist[i];
        desc_mat(dmp + 32 * (size_t)i, 1).copyTo(p->mDescriptor);
        for (int k = 0; k < nobs[i]; k++) p->AddObservation(observers[k], 0);
        if (state[i] == 2) p->mbBad = true;
        if (state[i] == 3) p->AddObservation(KF, 0);
        mps[i] = p;
        if (minInv) { minInv[i] = p->GetMinDistanceInvariance(); maxInv[i] = p->GetMaxDistanceInvariance(); }
    }
    if (Ow3) { cv::Mat Ow = KF->GetCameraCenter(); for (int k = 0; k < 3; k++) Ow3[k] = Ow.at<float>(k); }
    if (logScale) *logScale = KF->mfLogScaleFactor;
    ORBmatcher matcher(0.6f, true);
    const int n = matcher.Fuse(KF, mps, th);
    for (int i = 0; i < nmp; i++) {
        fused_idx[i] = -1;
        MapPoint* p = mps[i];
        if (!p || state[i] != 1) continue;
        int hops = 0;
        while (p && p->isBad() && hops++ < 8) p = p->GetReplaced();
        if (p && !p->isBad() && p->IsInKeyFrame(KF)) fused_idx[i] = p->GetIndexInKeyFrame(KF);
    }
    return n;
}

/* LSDmatcher::Fuse(KeyFrame*, const vector<MapLine*>&, th) :417-548; arguments as ref_fuse_points (Pw6 doubles, normal doubles: Vector3d) */
int ref_fuse_lines(int nml, const uint8_t* state, const int32_t* nobs, const double* Pw6, const double* normal, const float* minDist, const float* maxDist,
                   const uint8_t* dml, int nl2, const uint8_t* ld2, const float* kl2, const int32_t* oct2, const int32_t* kfobs,
                   const float* Tcw, const float* cam8, int nlevels, float scaleFactor, float th,
                   int32_t* fused_idx, float* Ow3, float* minInv, float* maxInv, float* logScale) {
    Scene S;
    Cam cam; memcpy(&cam, cam8, sizeof(cam));
    orc_keypoint none; memset(&none, 0, sizeof(none));
    Frame* F = make_frame(S, cam, nlevels, scaleFactor, &none, 0, nullptr, nullptr, nullptr, nullptr, 0, Tcw, ld2, nl2);
    set_keylines(F, nl2, kl2, oct2);
    KeyFrame* KF = make_kf(S, F);
    int maxobs = 0;
    for (int i = 0; i < nml; i++) maxobs = std::max(maxobs, nobs[i]);
    for (int j = 0; j < nl2; j++) maxobs = std::max(maxobs, kfobs[j]);
    std::vector<KeyFrame*> observers;
    for (int k = 0; k < maxobs; k++) observers.push_back(make_observer(S, cam, nlevels, scaleFactor));
    for (int j = 0; j < nl2; j++) if (kfobs[j] >= 0) {
        MapLine* q = make_ml(S, KF, nullptr, ld2 + 32 * (size_t)j);
        q->AddObservation(KF, j); KF->AddMapLine(q, j);
        for (int k = 0; k < kfobs[j]; k++) q->AddObservation(observers[k], 0);
    }
    std::vector<MapLine*> mls(nml, static_cast<MapLine*>(NULL));
    for (int i = 0; i < nml; i++) {
        if (!state[i]) continue;
        MapLine* l = make_ml(S, observers.empty() ? KF : observers[0], Pw6 + 6 * (size_t)i, dml + 32 * (size_t)i);
        l->mNormalVector << normal[3 * i], normal[3 * i + 1], normal[3 * i + 2];
        l->mfMinDistance = minDist[i]; l->mfMaxDistance = maxDist[i];
        for (int k = 0; k < nobs[i]; k++) l->AddObservation(observers[k], 0);
        if (state[i] == 2) l->mbBad = true;
        mls[i] = l;
        if (minInv) { minInv[i] = l->GetMinDistanceInvariance(); maxInv[i] = l->GetMaxDistanceInvariance(); }
    }
    if (Ow3) { cv::Mat Ow = KF->GetCameraCenter(); for (int k = 0; k < 3; k++) Ow3[k] = Ow.at<float>(k); }
    if (logScale) *logScale = KF->mfLogScaleFactor;
    LSDmatcher matcher(0.6f, true);
    const int n = matcher.Fuse(KF, mls, th);
    for (int i = 0; i < nml; i++) {
        fused_idx[i] = -1;
        MapLine* l = mls[i];
        if (!l || state[i] != 1) continue;
        int hops = 0;
        while (l && l->isBad() && hops++ < 8) l = l->GetReplaced();
        if (l && !l->isBad() && l->IsInKeyFrame(KF)) fused_idx[i] = l->GetIndexInKeyFrame(KF);
    }
    return n;
}

}  // extern "C"
