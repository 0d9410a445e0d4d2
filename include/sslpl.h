/*
 * include/sslpl.h — C ABI of the H100-native point/line front-end (libsslpl_b200.so).
 *
 * This is the drop-in boundary for the three data-parallel hot paths of
 * yanyan-li/Structure-SLAM-PointLine's Tracking::TrackWithPL():
 *   (1) ORBextractor::operator()            reference: include/ORBextractor.h:45-111, src/ORBextractor.cc:1043
 *   (2) LineSegment::ExtractLineSegment     reference: include/ExtractLineSegment.h:53-76, src/ExtractLineSegment.cpp:18
 *   (3) ORBmatcher / LSDmatcher Hamming     reference: include/ORBmatcher.h:36-101, include/LSDmatcher.h:36-64
 * and, widened after those met the parity + measurement bar (SURVEY.md 8(f) "next" rows 1-3): the DBoW2 vocabulary transform of
 * Frame::ComputeBoW, ORBmatcher::SearchByProjection(Frame&, const Frame&, ...) with the Frame feature grid, and the descriptor
 * medoid of MapPoint / MapLine ::ComputeDistinctiveDescriptors.
 * The reference has no FFI; its boundary is the C++ class surface.  The adapters in
 * structure-slam-pointline_b200/host/ re-expose those class signatures on top of this ABI
 * (see INTEGRATION.md).  Plain pointers and sizes only; no torch / OpenCV types.
 *
 * Conventions: every entry point returns 0 on success or a negative sslpl_status; nothing throws;
 * the callee never allocates caller-visible memory; `*_device` variants take device pointers and
 * enqueue on the handle's stream without synchronising (call sslpl_*_sync).  Handles are not
 * thread-safe individually, but any number of handles may be used concurrently from different
 * threads (the reference calls the matchers from Tracking and LocalMapping threads at once).
 * There is NO CPU fallback: without a CUDA device every create call fails with SSLPL_ERR_CUDA.
 */
#ifndef SSLPL_H
#define SSLPL_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define SSLPL_VERSION 1
#define SSLPL_MAX_LEVELS 16

typedef enum {
    SSLPL_OK = 0,
    SSLPL_ERR_ARG = -1,        /* bad argument (null pointer, size out of the handle's capacity, ...) */
    SSLPL_ERR_CUDA = -2,       /* CUDA runtime error; see sslpl_last_error() */
    SSLPL_ERR_CAPACITY = -3,   /* an internal or caller-provided buffer was too small (no partial result) */
    SSLPL_ERR_UNSUPPORTED = -4
} sslpl_status;

const char* sslpl_last_error(void);          /* thread-local message of the last failing call */
int  sslpl_version(void);
int  sslpl_device_count(void);               /* 0 when no CUDA device / driver */
int  sslpl_default_device(void);             /* CUDA ordinal the reference-side adapters use: $SSLPL_DEVICE, else 0 */

/* pinned host memory for frames / results (so H2D/D2H run at link speed) */
int  sslpl_host_alloc(void** p, size_t bytes);
int  sslpl_host_free(void* p);

/* ---- POD mirrors of the OpenCV types that cross the reference boundary (SURVEY.md 8(a) a15) ---- */
typedef struct { float x, y, size, angle, response; int32_t octave, class_id; } sslpl_keypoint;   /* cv::KeyPoint, 28 B */
typedef struct {                                                                                  /* cv::line_descriptor::KeyLine, 68 B */
    float angle; int32_t class_id; int32_t octave; float pt_x, pt_y; float response; float size;
    float startPointX, startPointY, endPointX, endPointY;
    float sPointInOctaveX, sPointInOctaveY, ePointInOctaveX, ePointInOctaveY;
    float lineLength; int32_t numOfPixels;
} sslpl_keyline;

/* =====================================================================================
 * (1) ORB extractor — replaces ORBextractor (src/ORBextractor.cc)
 * ===================================================================================== */
typedef struct {
    int   nfeatures;      /* ORBextractor.nFeatures   (Examples/ICL.yaml:41)  */
    float scaleFactor;    /* ORBextractor.scaleFactor (ICL.yaml:44)           */
    int   nlevels;        /* ORBextractor.nLevels     (ICL.yaml:47), <= SSLPL_MAX_LEVELS */
    int   iniThFAST;      /* ICL.yaml:53 */
    int   minThFAST;      /* ICL.yaml:54 */
    int   max_width, max_height;   /* largest frame this handle will see (device workspace is sized once) */
    int   max_batch;      /* frames per call for the batched entry points (>=1) */
    int   device;         /* CUDA device ordinal */
} sslpl_orb_params;

typedef struct sslpl_orb sslpl_orb;

int  sslpl_orb_create(const sslpl_orb_params* p, sslpl_orb** out);            /* ORBextractor::ORBextractor, ORBextractor.cc:410 */
void sslpl_orb_destroy(sslpl_orb* h);
/* GetScaleFactors / GetInverseScaleFactors / GetScaleSigmaSquares / GetInverseScaleSigmaSquares
   (ORBextractor.h:63-77) + mnFeaturesPerLevel + umax; each array has nlevels (umax: 16) entries; NULL = skip */
int  sslpl_orb_tables(const sslpl_orb* h, float* scale, float* invscale, float* sigma2, float* invsigma2,
                      int* nfeat_per_level, int* umax16);
/* the same tables without a device or a handle (host arithmetic only: the adapter's constructor runs before any frame is seen) */
int  sslpl_orb_tables_host(int nfeatures, float scaleFactor, int nlevels, float* scale, float* invscale, float* sigma2, float* invsigma2,
                           int* nfeat_per_level, int* umax16);
/* Keypoint capacity per frame, a bound for every frame up to max_width: sum_l max(mnFeaturesPerLevel[l] + 16, 4 * nIni_l), with
   nIni_l = round((w_l - 32) / 30) at level l's width w_l for max_width.  DistributeOctTree splits its nIni = round(dx / dy) root
   nodes once before it looks at the level's budget, so a wide frame can keep up to 4 nIni keypoints on a level
   (ORBextractor.cc:542-669); otherwise a level keeps at most mnFeaturesPerLevel[l] + 2. */
int  sslpl_orb_max_keypoints(const sslpl_orb* h);

/* ORBextractor::operator() (ORBextractor.cc:1043) on one HOST frame (CV_8UC1, `pitch` bytes per row).
   kps[cap], desc[cap*32]; *n = number of keypoints (0 for an empty image, as the reference's silent return). */
int  sslpl_orb_extract(sslpl_orb* h, const uint8_t* img, int width, int height, int pitch,
                       sslpl_keypoint* kps, uint8_t* desc, int cap, int* n);
/* Batched frames, HOST buffers: frame f at imgs + f*frame_stride; outputs kps[f*cap + i], desc[(f*cap+i)*32], n[f]. */
int  sslpl_orb_extract_batch(sslpl_orb* h, const uint8_t* imgs, int nframes, int width, int height, int pitch,
                             size_t frame_stride, sslpl_keypoint* kps, uint8_t* desc, int cap, int* n);
/* Asynchronous form of the above: enqueues H2D + extraction + D2H on the handle's stream and returns; the host buffers
   (pinned, see sslpl_host_alloc) are valid after sslpl_orb_sync().  Needs cap >= sslpl_orb_max_keypoints(). */
int  sslpl_orb_extract_batch_begin(sslpl_orb* h, const uint8_t* imgs, int nframes, int width, int height, int pitch,
                                   size_t frame_stride, sslpl_keypoint* kps, uint8_t* desc, int cap, int* n);
/* Batched frames already resident in HBM; results stay in HBM (see sslpl_orb_device_results). Asynchronous. */
int  sslpl_orb_extract_batch_device(sslpl_orb* h, const uint8_t* d_imgs, int nframes, int width, int height, int pitch,
                                    size_t frame_stride);
/* Device result buffers of the last *_device call: d_kps[f*cap+i], d_desc[(f*cap+i)*32], d_n[f]. */
int  sslpl_orb_device_results(sslpl_orb* h, const sslpl_keypoint** d_kps, const uint8_t** d_desc, const int** d_n, int* cap);
int  sslpl_orb_sync(sslpl_orb* h);           /* wait for the handle's stream; reports deferred device-side errors */
void* sslpl_orb_stream(sslpl_orb* h);        /* cudaStream_t of the handle */
/* Run the handle on a caller-owned cudaStream_t (e.g. the framework's current stream) instead of its own. */
int  sslpl_orb_set_stream(sslpl_orb* h, void* cuda_stream);
/* mvImagePyramid[level] (ORBextractor.h:79) of frame f of the last call; bordered=1 adds the 19-px
   BORDER_REFLECT_101 frame of ComputePyramid (ORBextractor.cc:1107-1132). dst is a HOST buffer. */
int  sslpl_orb_level_size(const sslpl_orb* h, int level, int* w, int* hgt);
int  sslpl_orb_download_level(sslpl_orb* h, int frame, int level, int bordered, uint8_t* dst, int dpitch);
/* stage intermediates of the last call, for parity tests: FAST candidates (vToDistributeKeys order),
   per-level keypoints after DistributeOctTree, blurred level */
int  sslpl_orb_download_candidates(sslpl_orb* h, int frame, int level, int* xs, int* ys, int* resp, int cap, int* n);
int  sslpl_orb_download_level_keypoints(sslpl_orb* h, int frame, int level, int* xs, int* ys, int* resp, int cap, int* n);
int  sslpl_orb_download_blurred(sslpl_orb* h, int frame, int level, uint8_t* dst, int dpitch);
/* number of kernels this handle has launched since creation (bench.py's gpu_launches claim) */
long long sslpl_orb_launch_count(const sslpl_orb* h);
/* names + CUDA-event milliseconds of the kernels of the last profiled call (enable with sslpl_orb_set_profiling) */
int  sslpl_orb_set_profiling(sslpl_orb* h, int on);
int  sslpl_orb_stage_ms(sslpl_orb* h, float* ms, int cap, const char** names, int* nstages);

/* =====================================================================================
 * (3) Hamming matching — replaces ORBmatcher / LSDmatcher kernels of work
 * ===================================================================================== */
typedef struct sslpl_matcher sslpl_matcher;
typedef struct {
    int max_features;     /* largest N (points) per frame */
    int max_lines;        /* largest NL per frame */
    int max_nodes;        /* largest number of vocabulary nodes in a FeatureVector */
    int max_batch;        /* frame pairs per batched call */
    int device;
} sslpl_matcher_params;
int  sslpl_matcher_create(const sslpl_matcher_params* p, sslpl_matcher** out);
void sslpl_matcher_destroy(sslpl_matcher* m);
int  sslpl_matcher_sync(sslpl_matcher* m);
void* sslpl_matcher_stream(sslpl_matcher* m);
int  sslpl_matcher_set_stream(sslpl_matcher* m, void* cuda_stream);
long long sslpl_matcher_launch_count(const sslpl_matcher* m);

/* ORBmatcher::DescriptorDistance (ORBmatcher.cc:1650) for nq pairs a[i] vs b[i] (HOST buffers) */
int  sslpl_descriptor_distance(sslpl_matcher* m, const uint8_t* a, const uint8_t* b, int n, int32_t* dist);
/* cv::BFMatcher(NORM_HAMMING,false).knnMatch(q,t,.,2) as used by LSDmatcher.cpp:155,266,298,341,392:
   out[4*i+0..3] = trainIdx0, dist0, trainIdx1, dist1 (ties -> lower trainIdx; -1,-1 when nt < 2) */
int  sslpl_hamming_knn2(sslpl_matcher* m, const uint8_t* q, int nq, const uint8_t* t, int nt, int32_t* out);
/* Vocabulary-node assignment (synthetic one-level stand-in for DBoW2 transform, TemplatedVocabulary.h:1218-1259) */
int  sslpl_bow_assign(sslpl_matcher* m, const uint8_t* desc, int n, const uint8_t* centroids, int nc, int32_t* node);

/* DBoW2::FeatureVector flattened to CSR: nodes[nn] ascending, off[nn+1], idx[off[nn]] */
typedef struct { const int32_t* nodes; const int32_t* off; const int32_t* idx; int nn; } sslpl_featvec;

/* ORBmatcher::SearchByBoW(KeyFrame*,Frame&,vector<MapPoint*>&) (ORBmatcher.cc:159-291).
   valid1[i] != 0 <=> KF feature i has a non-bad MapPoint.  match2[j] = KF feature index matched to frame
   feature j, or -1 (the adapter maps indices back to MapPoint*).  *nmatches = return value of the reference. */
int  sslpl_search_by_bow(sslpl_matcher* m, const uint8_t* d1, int n1, const uint8_t* d2, int n2,
                         const sslpl_featvec* fv1, const sslpl_featvec* fv2,
                         const uint8_t* valid1, const float* angle1, const float* angle2,
                         float nnratio, int checkOrientation, int32_t* match2, int* nmatches);
/* ORBmatcher::SearchByBoW(KeyFrame*,KeyFrame*,vector<MapPoint*>&) (ORBmatcher.cc:525-658): match12[i] = KF2 index or -1 */
int  sslpl_search_by_bow_kf(sslpl_matcher* m, const uint8_t* d1, int n1, const uint8_t* d2, int n2,
                            const sslpl_featvec* fv1, const sslpl_featvec* fv2,
                            const uint8_t* valid1, const uint8_t* valid2, const float* angle1, const float* angle2,
                            float nnratio, int checkOrientation, int32_t* match12, int* nmatches);
/* ORBmatcher::SearchForTriangulation (ORBmatcher.cc:660-826), monocular (bOnlyStereo=false, mvuRight<0).
   kp1/kp2 = mvKeysUn; has_mp = "feature already has a MapPoint"; F12 row-major 3x3 f32; (ex,ey) epipole;
   scale = mvScaleFactors, sigma2 = mvLevelSigma2 of KF2.  pairs[2*k] = (idx1, idx2) sorted by idx1. */
int  sslpl_search_for_triangulation(sslpl_matcher* m, const uint8_t* d1, int n1, const uint8_t* d2, int n2,
                                    const sslpl_featvec* fv1, const sslpl_featvec* fv2,
                                    const uint8_t* has_mp1, const uint8_t* has_mp2,
                                    const sslpl_keypoint* kp1, const sslpl_keypoint* kp2,
                                    const float* F12, float ex, float ey, const float* scale, const float* sigma2, int nlevels,
                                    int checkOrientation, int32_t* pairs, int* nmatches);
/* LSDmatcher knnMatch-based entry points (LSDmatcher.cpp). mode 0: SearchByProjection(KF,F) :143 /
   SearchByDescriptor(KF,F) :286 -> out[tdx] = qdx table (n2 entries);  mode 1: SerachForInitialize :257 -> pairs;
   mode 2: SearchByDescriptor(KF,KF2) :329 -> out[qdx] = tdx table (n1 entries); mode 3: SearchForTriangulation :382 -> pairs.
   *nout = number of pairs written (modes 1,3); *nmatches = the reference's return value.
   Also returns Frame::lineDescriptorMAD (Frame.cc:190) in mad[0..1] when mad != NULL. */
int  sslpl_line_match(sslpl_matcher* m, int mode, const uint8_t* d1, int n1, const uint8_t* d2, int n2,
                      const uint8_t* has_ml1, const uint8_t* has_ml2, int32_t* out, int* nout, int* nmatches, double* mad);

/* Batched consecutive-frame matching, everything resident in HBM (config 5 of BASELINE.json):
   for pair p (frame p = "KeyFrame", frame p+1 = "Frame"): node assignment of both frames against the
   vocabulary, FeatureVector build, SearchByBoW (all KF features valid), rotation filter.
   d_desc/d_kps/d_n as produced by sslpl_orb_extract_batch_device (cap entries per frame, nframes frames);
   d_match[(p*cap)+j] = KF index or -1 for frame p+1's feature j; d_nmatch[p]. npairs = nframes-1. */
int  sslpl_match_bow_batch_device(sslpl_matcher* m, const uint8_t* d_desc, const sslpl_keypoint* d_kps, const int* d_n,
                                  int nframes, int cap, const uint8_t* d_centroids, int nc,
                                  float nnratio, int checkOrientation, int32_t* d_match, int32_t* d_nmatch);
/* ---- ORBmatcher::SearchByProjection(Frame &CurrentFrame, const Frame &LastFrame, th, bMono) (ORBmatcher.cc:1331-1473), the
   matcher of Tracking::TrackWithMotionModel (Tracking.cc:1227), with Frame::AssignFeaturesToGrid / GetFeaturesInArea
   (Frame.cc:133-148, 368-421) on the device.  SURVEY.md 8(f) row 2.  HOST buffers.
   Last frame (n1): valid1[i] = mvpMapPoints[i] && !mvbOutlier[i]; obs1[i] = that MapPoint's Observations() > 0; Xw[3i..] =
   GetWorldPos(); dmp[i][32] = GetDescriptor(); oct1 = mvKeys[i].octave; angle1 = mvKeysUn[i].angle.
   Current frame (n2): descriptors d2, mvKeysUn x2 / y2 / oct2 / angle2, mvuRight (NULL for monocular), claimed2[j] = the
   feature already holds a MapPoint with observations (NULL = none).  Tcw / Tlw: 3x4 row-major poses (Tlw only read when
   !bMono); cam = {fx, fy, cx, cy, mbf, mb}; bounds = {mnMinX, mnMaxX, mnMinY, mnMaxY}; scaleFactors[nlevels].
   Result: assign2[j] = index i of the last-frame MapPoint now held by current feature j; -1 = never assigned; -2 = assigned and
   then removed by the rotation check (the reference writes NULL there, ORBmatcher.cc:1461: the caller must too); *nmatches as
   returned by the reference.  The matcher handle needs max_nodes >= 3072 (grid cells) and at most 8192 features. */
int  sslpl_search_by_projection_frame(sslpl_matcher* m,
        int n1, const uint8_t* valid1, const uint8_t* obs1, const float* Xw, const uint8_t* dmp, const int32_t* oct1, const float* angle1,
        int n2, const uint8_t* d2, const float* x2, const float* y2, const int32_t* oct2, const float* angle2, const float* uright2,
        const uint8_t* claimed2, const float* Tcw, const float* Tlw, const float* cam, const float* bounds,
        const float* scaleFactors, int nlevels, float th, int bMono, int checkOrientation, int32_t* assign2, int* nmatches);
/* The same matcher over consecutive frames resident in HBM, monocular (bMono = true), asynchronous on the handle's stream like
   sslpl_match_bow_batch_device.  Pair p (npairs = nframes - 1) is what Tracking::TrackWithMotionModel (Tracking.cc:1204-1244) runs with
   frame p as LastFrame and frame p + 1 as CurrentFrame: CurrentFrame.mvpMapPoints starts all NULL (:1219), ORBmatcher::SearchByProjection
   (ORBmatcher.cc:1331-1473) runs with th, and when retry_below > 0 and it found fewer than retry_below matches (the reference: 20) it runs
   again from NULL with 2 * th (:1240-1244).
   Per frame f, `cap` entries each: d_kps = mvKeysUn (e.g. sslpl_orb_device_results, or sslpl_frame_device_keypoints_un with
   distortion), d_desc, d_n[f] (clamped to cap); d_Xw[f][cap][3] = GetWorldPos() of feature i's MapPoint; d_mpflag[f][cap]: bit0 =
   mvpMapPoints[i] && !mvbOutlier[i], bit1 = Observations() > 0; d_dmp[f][cap][32] = the MapPoints' descriptors (NULL = the frame's own
   d_desc); d_Tcw[f][12] = 3x4 row-major pose (pair p projects with frame p + 1's).  Host: cam = {fx, fy, cx, cy}, bounds = {mnMinX,
   mnMaxX, mnMinY, mnMaxY}, scaleFactors[nlevels] (nlevels <= 32).  A last-frame point whose octave is outside [0, nlevels) is skipped.
   Result: d_assign[p][cap] as assign2 above for frame p + 1's features (-1 also past d_n), d_nmatch[p] = the final count.
   Needs nframes <= max_batch + 1 and cap <= max_features + 64; the first call allocates a workspace of that size, freed with the
   handle.  Bad arguments return SSLPL_ERR_ARG and enqueue nothing. */
int  sslpl_search_by_projection_frame_batch_device(sslpl_matcher* m,
        const sslpl_keypoint* d_kps, const uint8_t* d_desc, const int* d_n, int nframes, int cap,
        const float* d_Xw, const uint8_t* d_mpflag, const uint8_t* d_dmp, const float* d_Tcw,
        const float* cam, const float* bounds, const float* scaleFactors, int nlevels, float th, int checkOrientation, int retry_below,
        int32_t* d_assign, int32_t* d_nmatch);

/* ---- ORBmatcher::SearchByProjection(Frame &F, const vector<MapPoint*> &vpMapPoints, th) (ORBmatcher.cc:45-129): the matcher of
   Tracking::SearchLocalPoints (Tracking.cc:1736), run on every frame.  Per MapPoint, in vector order, what Frame::isInFrustum left on
   it: inview = mbTrackInView, bad = isBad() (NULL = none), obs = Observations() > 0 (NULL = none), projx/projy = mTrackProjX/Y,
   projxr = mTrackProjXR (NULL for monocular), level = mnTrackScaleLevel, viewcos = mTrackViewCos, dmp = GetDescriptor().
   Frame (n2): descriptors, mvKeysUn x / y / octave, mvuRight (NULL), held2[j] = 0 nothing, 1 a MapPoint with observations (skipped),
   2 a MapPoint without (NULL = all 0).  assign2[j] = index of the MapPoint now written to F.mvpMapPoints[j] (-1: untouched). */
int  sslpl_search_by_projection_mps(sslpl_matcher* m,
        int nmp, const uint8_t* inview, const uint8_t* bad, const uint8_t* obs, const float* projx, const float* projy, const float* projxr,
        const int32_t* level, const float* viewcos, const uint8_t* dmp,
        int n2, const uint8_t* d2, const float* x2, const float* y2, const int32_t* oct2, const float* uright2, const uint8_t* held2,
        const float* bounds, const float* scaleFactors, int nlevels, float nnratio, float th, int32_t* assign2, int* nmatches);
/* ---- ORBmatcher::SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize) (ORBmatcher.cc:408-523,
   Tracking::MonocularInitialization Tracking.cc:366).  Keypoint fields are those of mvKeysUn; prev_xy[n1][2] = vbPrevMatched is
   updated like the reference does (:517-520); matches12[n1] = vnMatches12. */
int  sslpl_search_for_initialization(sslpl_matcher* m,
        int n1, const uint8_t* d1, const int32_t* oct1, const float* angle1, float* prev_xy,
        int n2, const uint8_t* d2, const float* x2, const float* y2, const int32_t* oct2, const float* angle2,
        const float* bounds, float nnratio, int checkOrientation, int windowSize, int32_t* matches12, int* nmatches);
/* ---- Tracking::MonocularInitialization's matchers (Tracking.cc:328-420) over (initial frame, frame) pairs resident in HBM, asynchronous
   on the handle's stream like the other *_batch_device calls; no caller-visible allocation.  While there is no map, every frame runs
   ORBmatcher(0.9, true).SearchForInitialization(mInitialFrame, mCurrentFrame, mvbPrevMatched, mvIniMatches, 100) (:366) and
   LSDmatcher::SerachForInitialize (:368); both frames come from the 2 x nFeatures extractor (:120, :163), so the matcher must be sized
   for it (max_features >= 2 nFeatures, or cap from that extractor).  Initializer::Initialize and the reset rules (:354-376) stay with
   the caller.
   sslpl_search_for_initialization_batch_device: ORBmatcher::SearchForInitialization (ORBmatcher.cc:408-523) for every pair d_pair[p] =
   (init row, current row) of a row set in the extractors' layout: d_kps[r][cap] = mvKeysUn (sslpl_frame_device_keypoints_un or
   sslpl_orb_device_results), d_desc[r][cap][32], d_n[r] (clamped to [0, cap]); bounds = {mnMinX, mnMaxX, mnMinY, mnMaxY} (HOST, one
   for all rows); nnratio, checkOrientation and windowSize as the reference takes them.
   Chains: a maximal run of consecutive pairs with the same init row runs strictly in order, and vbPrevMatched is carried from one pair to
   the next exactly as the reference carries it (rewritten at :516-520 and searched around by the next call).  d_prev0[npairs][cap][2]
   (f32, may be NULL; must not overlap the outputs) holds the vbPrevMatched each chain starts from and is read only at slot c0 of the
   chain that starts at pair c0; NULL means the init row's own keypoint positions (Tracking.cc:338-340).  Chains are independent, the
   inputs are never modified, and the first k pairs of a chain give exactly what a call with only those k pairs gives, so a caller cuts
   a chain where the reference resets (fewer than 100 point plus line matches) or where Initialize succeeds.  A pair with a row outside
   [0, nrows) or with current row == init row gets the count -1, writes no rows and leaves the chain's state alone.  A current row may
   appear more than once in a chain: each pair is simply the next call.
   Results per pair p:
     d_match12[p][cap]  vnMatches12 (-1 past the init row's count);
     d_prev[p][cap][2]  vbPrevMatched after this pair (rows past the init row's count are not written); a caller continuing a chain in a
                        later call passes the slot of its last good pair as that chain's d_prev0;
     d_nmatch[p]        the return value.
   Needs nrows in [2, max_batch + 1], npairs in [1, max_batch] and cap <= max_features + 64.  The grids of all rows go in the workspace of
   sslpl_search_by_projection_frame_batch_device; the first call also allocates [max_batch][max_features + 64] per-chain scratch, freed
   with the handle.  Bad arguments return SSLPL_ERR_ARG and enqueue nothing. */
int  sslpl_search_for_initialization_batch_device(sslpl_matcher* m,
        const sslpl_keypoint* d_kps, const uint8_t* d_desc, const int* d_n, int nrows, int cap, int npairs, const int32_t* d_pair,
        const float* d_prev0, const float* bounds, float nnratio, int checkOrientation, int windowSize,
        int32_t* d_match12, float* d_prev, int32_t* d_nmatch);
/* sslpl_line_search_for_initialize_batch_device: LSDmatcher::SerachForInitialize (LSDmatcher.cpp:257-284), with Frame::lineDescriptorMAD
   (Frame.cc:189-215) on the device, for every pair d_pair[p] = (init row, current row) of a line row set in the layout of
   sslpl_line_device_results: d_ldesc[r][capl][32], d_nl[r] (clamped to [0, capl]).  Pairs are independent.  Result: d_lpairs[p][capl][2] =
   (qdx, tdx) in ascending qdx, (-1, -1) after the count; d_nlmatch[p].  As in sslpl_line_search_for_triangulation_batch_device,
   d_nlmatch[p] = -1 for a row outside [0, nrows) and when the init row has lines and the current row fewer than 2 (the reference reads
   lmatches[i][1] out of bounds there; the single call returns SSLPL_ERR_ARG), and 0 when the init row has none.  Needs nrows in [1,
   max_batch + 1], npairs in [1, max_batch] and capl <= max_lines + 64; bad arguments return SSLPL_ERR_ARG and enqueue nothing. */
int  sslpl_line_search_for_initialize_batch_device(sslpl_matcher* m, const uint8_t* d_ldesc, const int* d_nl, int nrows, int capl,
        int npairs, const int32_t* d_pair, int32_t* d_lpairs, int32_t* d_nlmatch);

/* ---- Line projection matchers and Fuse (SURVEY.md 8(f) row 3).  Each reference function is a projection stage (per map element:
   gates and projected quantities, arithmetic in the reference's own cv::Mat / Eigen types - it stays in the adapter, host/matcher_b200.cc,
   which calls the reference's own accessors, e.g. MapPoint::PredictScale) followed by a search stage (the Hamming scan over the frame's
   features), which is what these entry points run on the device.  HOST buffers; results identical to the reference's loops.

   sslpl_line_search_by_projection: search stage of LSDmatcher::SearchByProjection(Frame&, const Frame&, th, bMono) (LSDmatcher.cpp:98-137)
   and of LSDmatcher::SearchByProjection(Frame&, const vector<MapLine*>&, th) (:210-251).  Per MapLine, in the reference's visiting order:
   active (passed the gates), obs (Observations() > 0), proj[4] = projected end points x1 y1 x2 y2, radius, [minLevel, maxLevel] as handed to
   Frame::GetLinesInArea (Frame.cc:423-460), its descriptor.  Frame lines: descriptors, kl2[3] = pt.x pt.y angle of mvKeylinesUn, octaves,
   held2 (1 = holds a MapLine WITH observations: never a candidate).  assign2[j] = index of the MapLine written to mvpMapLines[j] (the last
   writer; -1 none), *nmatches = the function's return value. */
int  sslpl_line_search_by_projection(sslpl_matcher* m, int nml, const uint8_t* active, const uint8_t* obs, const float* proj, const float* radius,
        const int32_t* minLevel, const int32_t* maxLevel, const uint8_t* dml,
        int nl2, const uint8_t* ld2, const float* kl2, const int32_t* oct2, const uint8_t* held2,
        float nnratio, int32_t* assign2, int* nmatches);
/* Search stage of LSDmatcher::Fuse(KeyFrame*, const vector<MapLine*>&, th) (LSDmatcher.cpp:495-523): per MapLine the projected end points and
   the level MapLine::PredictScale returned; KeyFrame lines as above (oct2 = mvKeyLines[].octave).  best_idx[i] = nearest KeyFrame line of the
   window at level in [level-1, level] (first on ties; -1 none), best_dist[i] (INT_MAX when none); the caller fuses when best_dist <= 50.
   A level outside [0, nlevels) (PredictScale is not clamped, MapLine.cpp:386-395; the reference then reads mvScaleFactors out of bounds)
   drops the line. */
int  sslpl_fuse_lines_search(sslpl_matcher* m, int nml, const uint8_t* active, const float* proj, const int32_t* level, const uint8_t* dml,
        int nl2, const uint8_t* ld2, const float* kl2, const int32_t* oct2, const float* scaleFactors, int nlevels, float th,
        int32_t* best_idx, int32_t* best_dist);
/* Search stage of ORBmatcher::Fuse(KeyFrame*, const vector<MapPoint*>&, th) (ORBmatcher.cc:889-950): per MapPoint its projection (u, v, ur =
   u - bf / z; ur may be NULL when the KeyFrame has no stereo features) and predicted level; KeyFrame features: descriptors, mvKeysUn x / y /
   octave, mvuRight (NULL = monocular), image bounds, mvScaleFactors, mvInvLevelSigma2.  Window = KeyFrame::GetFeaturesInArea(u, v,
   th * scale[level]) (KeyFrame.cc:610-649), level gate, chi-square gate (5.99 mono / 7.8 stereo), nearest descriptor (first in the grid
   traversal order on ties).  best_idx[i] (-1 none), best_dist[i] (256 none); the caller fuses when best_dist <= 50. */
int  sslpl_fuse_points_search(sslpl_matcher* m, int nmp, const uint8_t* active, const float* u, const float* v, const float* ur,
        const int32_t* level, const uint8_t* dmp,
        int n2, const uint8_t* d2, const float* x2, const float* y2, const int32_t* oct2, const float* uright2,
        const float* bounds, const float* scaleFactors, const float* invLevelSigma2, int nlevels, float th,
        int32_t* best_idx, int32_t* best_dist);

/* MapPoint::ComputeDistinctiveDescriptors (MapPoint.cc:247-312) / MapLine::ComputeDistinctiveDescriptors (MapLine.cpp:246-317),
   batched (SURVEY.md 8(f) row 3): group g owns descriptors desc[off[g] .. off[g+1]) (HOST buffers, off[0] = 0);
   best_idx[g] = index inside the group of the descriptor with the least median Hamming distance to the others (median =
   sorted[int(0.5 (N - 1))], first minimum wins; -1 for an empty group), best_median[g] = that median. */
int  sslpl_descriptor_medoid_batch(sslpl_matcher* m, const uint8_t* desc, const int32_t* off, int ngroups,
                                   int32_t* best_idx, int32_t* best_median);

/* ---- DBoW2 vocabulary: Frame::ComputeBoW / KeyFrame::ComputeBoW (Frame.cc:474-481, KeyFrame.cc:71-80), i.e.
   TemplatedVocabulary<FORB>::transform(features, BowVector&, FeatureVector&, levelsup = 4)
   (Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1127-1259).  SURVEY.md 8(f) row 1. ---- */
typedef struct sslpl_vocab sslpl_vocab;
/* The tree as arrays (what loadFromTextFile :1338-1420 builds): node 0 = root, parent[i] < i (parent[0] ignored),
   desc[i][32], weight[i], is_leaf[i] (must agree with the structure).  Word ids number the leaves in node order.  Such a vocabulary
   weights TF_IDF and scores L1_NORM, as ORBvoc.txt does (its header is "10 6 0 0"). */
int  sslpl_vocab_create(int device, int k, int L, int nnodes, const int32_t* parent, const uint8_t* desc, const double* weight,
                        const uint8_t* is_leaf, sslpl_vocab** out);
/* ORBvoc.txt text format (System.cc:70 mpVocabulary->loadFromTextFile); scoring / weighting = the header's n1 / n2, which the
   vocabulary keeps */
int  sslpl_vocab_load_text(int device, const char* path, sslpl_vocab** out, int* scoring, int* weighting);
void sslpl_vocab_destroy(sslpl_vocab* v);
int  sslpl_vocab_info(const sslpl_vocab* v, int* k, int* L, int* nnodes, int* nwords);
/* number of distinct FeatureVector node values at level L - levelsup (+1 for node 0: root / leaves above that level) */
int  sslpl_vocab_level_nodes(const sslpl_vocab* v, int levelsup, int* count);
/* Per feature (HOST buffers): word id, NodeId at level L - levelsup, leaf weight.  weight <= 0 marks a stopped word, which
   the reference leaves out of both vectors (:1162-1166).  BowVector / FeatureVector assembly from these three arrays is a
   host-side map insertion (see the Python mirror's Vocabulary.bow_vector / feature_vector_csr). */
int  sslpl_bow_transform(sslpl_matcher* m, const sslpl_vocab* v, const uint8_t* desc, int n, int levelsup,
                         int32_t* word, int32_t* node, double* weight);
/* sslpl_match_bow_batch_device with the real tree instead of the one-level synthetic vocabulary.  Optional per-feature
   outputs d_word / d_node / d_weight ([nframes][cap], may be NULL) stay in HBM for the caller's BowVector build. */
int  sslpl_match_bow_batch_device_vocab(sslpl_matcher* m, const uint8_t* d_desc, const sslpl_keypoint* d_kps, const int* d_n,
                                        int nframes, int cap, const sslpl_vocab* v, int levelsup, float nnratio, int checkOrientation,
                                        int32_t* d_match, int32_t* d_nmatch, int32_t* d_word, int32_t* d_node, double* d_weight);

/* ---- KeyFrameDatabase (src/KeyFrameDatabase.cc) over a row set resident in HBM, asynchronous on the matcher's stream like the other
   *_batch_device calls.  The row set: nrows rows, each a frame or a keyframe, in the extractors' layout d_desc[r][cap][32], d_n[r]
   (clamped to cap), and their BowVector tables d_bow_word[r][cap] int32, d_bow_val[r][cap] double, d_bow_n[r]: mBowVec as ascending
   (word, value) entries, (-1, 0.0) past the count.  Needs cap <= max_features + 64 and (P + cap) * 8 <= 200 KB with P the least power of
   two >= cap (cap <= 8256).  Bad host arguments return SSLPL_ERR_ARG and enqueue nothing.

   Frame::ComputeBoW / KeyFrame::ComputeBoW's mBowVec (Frame.cc:474-481, KeyFrame.cc:71-80) of every row, with the vocabulary tree of
   TemplatedVocabulary::transform (TemplatedVocabulary.h:1127-1197): stopped words (weight <= 0) left out, the TF_IDF weights of a word
   added in feature order (BowVector::addWeight, BowVector.cpp:34-46), then divided by the sequential sum of their absolute values in
   ascending word order (BowVector::normalize :62-84; L1 scoring normalises, so there is no division by the word count).  Only a TF_IDF /
   L1_NORM vocabulary is supported; any other returns SSLPL_ERR_UNSUPPORTED and enqueues nothing.  nrows <= 65535. */
int  sslpl_bow_vectors_batch_device(sslpl_matcher* m, const sslpl_vocab* v, const uint8_t* d_desc, const int* d_n, int nrows, int cap,
                                    int32_t* d_bow_word, double* d_bow_val, int32_t* d_bow_n);
/* TemplatedVocabulary::score(v1, v2) = L1Scoring::score (ScoringObject.cpp:23-67) of row pairs d_pair[p] = (r1, r2), r1 the first
   argument (the query): over the common words in ascending order, score += (|vi - wi| - |vi|) - |wi|; d_score[p] = -score / 2.0; NaN for
   a pair with a row outside [0, nrows).  LoopClosing::DetectLoop's minScore (LoopClosing.cc:122-142) is the float minimum of these over the
   query's non-bad covisible keyframes, starting at 1. */
int  sslpl_bow_score_batch_device(sslpl_matcher* m, const int32_t* d_bow_word, const double* d_bow_val, const int32_t* d_bow_n, int nrows,
                                  int cap, int npairs, const int32_t* d_pair, double* d_score);
/* KeyFrameDatabase::DetectLoopCandidates(pKF, minScore) (:81-202) and DetectRelocalizationCandidates(F) (:204-314, the call of
   Tracking::Relocalization, Tracking.cc:1961-1970) for nq query rows d_query[q] against the database d_db[ndb]: its rows in
   KeyFrameDatabase::add order (:45-51) with erased keyframes (:53-72) left out, which is the order of every inverted-file list.
   d_covis[nrows][10] = GetBestCovisibilityKeyFrames(10) of each row, padded with -1; an entry outside [0, nrows) or outside the database
   is a keyframe outside the database.  Loop only: d_conn_off[nq + 1] / d_conn[nconn] = the rows of the query's GetConnectedKeyFrames()
   (never listed), d_minscore[nq].  Each query starts fresh, as growing frame and keyframe ids guarantee in the reference.
   Results per query q and database position p (the reference's per-KeyFrame fields, KeyFrame.h:172-177):
     d_cand[q][ndb]  the candidate rows in the order of the returned vector, -1 after d_ncand[q];
     d_words[q][ndb] mnLoopWords / mnRelocWords, 0 when the keyframe shares no word with the query or is connected to a loop query;
     d_score[q][ndb] mLoopScore / mRelocScore written by this query (float), NaN when it did not score the keyframe.
   Reloc state: the reloc neighbour test reads mRelocScore of listed keyframes the query did not score, left by an earlier query or never
   initialised (KeyFrame.cc:45).  Query q reads the score such a keyframe got in the latest earlier query of the call that scored it, or
   else d_relocscore[row]; afterwards d_relocscore holds each keyframe's score after the last query.  So one call equals nq sequential
   reference calls on keyframes whose mRelocScore starts at d_relocscore (0 is as good as any value for a fresh keyframe).  Finding that
   earlier query walks back through the call's queries, so a call costs O(nq) per such neighbour; split sequences of thousands of frames
   into calls chained through d_relocscore.
   d_ncand[q] = -1 (no candidates, words 0, scores NaN) for a query row outside [0, nrows) or, loop only, connected offsets not within
   0 <= d_conn_off[q] <= d_conn_off[q + 1] <= nconn; and for every query when a database row is outside [0, nrows) or listed twice.
   Needs ndb in [1, 25600], nq in [1, 65535] and nconn >= 0; the first call allocates an nrows-int row -> position map (and nq ints),
   freed with the handle. */
int  sslpl_detect_loop_candidates_batch_device(sslpl_matcher* m, const int32_t* d_bow_word, const double* d_bow_val, const int32_t* d_bow_n,
        int nrows, int cap, const int32_t* d_db, int ndb, const int32_t* d_query, int nq, const int32_t* d_covis,
        const int32_t* d_conn_off, const int32_t* d_conn, int nconn, const float* d_minscore,
        int32_t* d_cand, int32_t* d_ncand, int32_t* d_words, float* d_score);
int  sslpl_detect_relocalization_candidates_batch_device(sslpl_matcher* m, const int32_t* d_bow_word, const double* d_bow_val,
        const int32_t* d_bow_n, int nrows, int cap, const int32_t* d_db, int ndb, const int32_t* d_query, int nq, const int32_t* d_covis,
        float* d_relocscore, int32_t* d_cand, int32_t* d_ncand, int32_t* d_words, float* d_score);

/* ---- Tracking::Relocalization (Tracking.cc:1961-2121) on the device ----
   sslpl_reloc_pairs_batch_device turns the candidate table of sslpl_detect_relocalization_candidates_batch_device into a pair list:
   d_pair[q * kmax + k] = (d_cand[q][k], d_query[q]) for k < min(d_ncand[q], kmax, ndb), else (-1, -1).  The slot keeps the candidate's rank,
   the order Relocalization walks; d_ncand[q] = -1 gives empty slots, and d_ncand[q] > kmax shows truncation.  Needs nq * kmax <=
   max_batch.  Asynchronous; bad arguments return SSLPL_ERR_ARG and enqueue nothing. */
int  sslpl_reloc_pairs_batch_device(sslpl_matcher* m, const int32_t* d_query, const int32_t* d_cand, const int32_t* d_ncand, int nq, int ndb,
        int kmax, int32_t* d_pair);
/* ORBmatcher::SearchByProjection(Frame &F, KeyFrame *pKF, const set<MapPoint*> &sAlreadyFound, th, ORBdist) (ORBmatcher.cc:1475-1602),
   which Relocalization runs with ORBmatcher(0.9, true) after PnP and PoseOptimization, at (10, 100) and again at (3, 64).  F.mvpMapPoints
   is read on entry and written.  One pair, host buffers.  Keyframe feature i: flag1[i] = vpMPs[i] && !isBad() && !sAlreadyFound.count(),
   Xw[i][3] = GetWorldPos(), dmp[i][32] = GetDescriptor(), dist3[i][3] = GetMinDistanceInvariance(), GetMaxDistanceInvariance(),
   mfMaxDistance, angle1[i] = mvKeysUn[i].angle.  Frame feature j: descriptor, mvKeysUn x / y / octave / angle, held2[j] =
   mvpMapPoints[j] != NULL on entry (NULL = none).  Tcw = F.mTcw 3x4 row-major, cam = {fx, fy, cx, cy}, bounds = {mnMinX, mnMaxX, mnMinY,
   mnMaxY}, the frame's mvScaleFactors[nlevels] and mfLogScaleFactor.  assign2[j] = the keyframe feature whose MapPoint was written to
   mvpMapPoints[j], -1 untouched, -2 written and then NULLed by the rotation check; *nmatches = the return value.  There is no depth test:
   a point behind the camera that projects inside the bounds is searched.  ORBdist >= 256 returns SSLPL_ERR_ARG (the reference would
   write mvpMapPoints[-1] when a window holds no free feature). */
int  sslpl_search_by_projection_kf(sslpl_matcher* m,
        int n1, const uint8_t* flag1, const float* Xw, const uint8_t* dmp, const float* dist3, const float* angle1,
        int n2, const uint8_t* d2, const float* x2, const float* y2, const int32_t* oct2, const float* angle2, const uint8_t* held2,
        const float* Tcw, const float* cam, const float* bounds, const float* scaleFactors, int nlevels, float logScaleFactor,
        float th, int ORBdist, int checkOrientation, int32_t* assign2, int* nmatches);
/* The same matcher over pairs of a row set in HBM, asynchronous on the handle's stream.  Rows (frames and keyframes alike, nrows <=
   65535) in the extractors' layout: d_kps[r][cap] = mvKeysUn, d_desc[r][cap][32], d_n[r] (clamped to [0, cap]).  Map: d_kfmp[r][cap] =
   GetMapPointMatches() as element indices (-1 or any index outside [0, nmp) = NULL), d_mpbad[m] = isBad() (NULL = none), d_mp[m][9] =
   Xw, normal, GetMinDistanceInvariance(), GetMaxDistanceInvariance(), mfMaxDistance and d_mpdesc[m][32] (the table of
   sslpl_fuse_points_batch_device).  Pair p: d_pair[p] = (keyframe row, frame row), d_Tcw[p][12] = the frame's pose for that candidate,
   d_found[p][cap] over keyframe features = sAlreadyFound.count(vpMPs[i]) (NULL = none), d_held[p][cap] over frame features =
   mvpMapPoints[j] != NULL on entry (NULL = none).  Results: d_assign[p][cap] as assign2 above (-1 past the frame's count), d_nmatch[p];
   a pair with a row outside [0, nrows) gets d_nmatch -1 and no assignment.  Needs npairs <= max_batch and cap <= max_features + 64; the
   first call of either form allocates a workspace of max_batch pairs, freed with the handle.  Bad host arguments return SSLPL_ERR_ARG and
   enqueue nothing. */
int  sslpl_search_by_projection_kf_batch_device(sslpl_matcher* m,
        const sslpl_keypoint* d_kps, const uint8_t* d_desc, const int* d_n, int nrows, int cap,
        const int32_t* d_kfmp, const uint8_t* d_mpbad, int nmp, const float* d_mp, const uint8_t* d_mpdesc,
        int npairs, const int32_t* d_pair, const float* d_Tcw, const uint8_t* d_found, const uint8_t* d_held,
        const float* cam, const float* bounds, const float* scaleFactors, int nlevels, float logScaleFactor,
        float th, int ORBdist, int checkOrientation, int32_t* d_assign, int32_t* d_nmatch);

/* ---- Keyframe-to-frame matching over (keyframe row, frame row) pairs in HBM, asynchronous on the handle's stream.  Tracking runs it in
   Relocalization (ORBmatcher(0.75, true).SearchByBoW(pKF, F) for every candidate: the pairs of sslpl_reloc_pairs_batch_device),
   TrackReferenceKeyFrame (ORBmatcher(0.9, true).SearchByBoW(mpReferenceKF, F) and LSDmatcher::SearchByProjection(mpReferenceKF, F)) and
   TrackWithMotionModel (the line matcher against the reference keyframe).
   sslpl_search_by_bow_batch_device: ORBmatcher::SearchByBoW(KeyFrame* pKF, Frame& F, vector<MapPoint*>&) (ORBmatcher.cc:159-291) for
   every pair d_pair[p] = (keyframe row, frame row).  The row set and element map are those of sslpl_search_by_projection_kf_batch_device:
   d_kps[r][cap] = mvKeysUn, d_desc[r][cap][32], d_n[r] (clamped to [0, cap]), d_kfmp[r][cap] = GetMapPointMatches() as element indices
   (-1 or any index outside [0, nmp) = NULL), d_mpbad[m] = isBad() (NULL = none bad).  A keyframe feature takes part iff its element is
   non-NULL and not bad.  Both FeatureVectors come from the vocabulary at level L - levelsup (stopped words left out), built once per row
   the pairs name.  d_match[p][cap]: the keyframe feature matched to frame feature j, or -1 (also where the rotation check dropped it, and
   past the frame's count); d_nmatch[p] = the return value.  A pair with a row outside [0, nrows), such as the (-1, -1) slots of
   sslpl_reloc_pairs_batch_device, gets d_nmatch -1 and an all -1 row.  Needs npairs <= max_batch, nrows <= 65535, cap <= max_features + 64
   and (nc + 1 + cap) * 4 <= 200 KB for the level's nc nodes; the first call allocates a workspace of 2 max_batch FeatureVectors, freed
   with the handle.  The caller keeps Relocalization's isBad() skip of a candidate and its nmatches < 15 discard. */
int  sslpl_search_by_bow_batch_device(sslpl_matcher* m,
        const sslpl_keypoint* d_kps, const uint8_t* d_desc, const int* d_n, int nrows, int cap,
        const int32_t* d_kfmp, const uint8_t* d_mpbad, int nmp,
        const sslpl_vocab* v, int levelsup,
        int npairs, const int32_t* d_pair, float nnratio, int checkOrientation,
        int32_t* d_match, int32_t* d_nmatch);
/* sslpl_match_lines_kf_batch_device: LSDmatcher::SearchByProjection(KeyFrame* pKF, Frame& F, vector<MapLine*>&) (LSDmatcher.cpp:143-183)
   for every pair d_pair[p] = (keyframe row, frame row) of a line row set in the layout of sslpl_line_device_results: d_ldesc[r][capl][32],
   d_nl[r] (clamped to [0, capl]), d_kfml[r][capl] = GetMapLineMatches() as element indices (-1 or any index outside [0, nml) = NULL; the
   reference tests no isBad() here).  d_lmatch[p][capl][tdx] = the qdx whose MapLine ends in vpMapLineMatches[tdx] (the last accepted),
   or -1; d_nlmatch[p] = the return value, which counts overwritten acceptances.  d_nlmatch[p] = -1 for a row outside [0, nrows), and
   where the keyframe has lines and the frame fewer than 2 (knnMatch leaves lmatches[i][1] undefined there).  Needs npairs <= max_batch,
   nrows <= 65535 and capl <= max_lines + 64. */
int  sslpl_match_lines_kf_batch_device(sslpl_matcher* m,
        const uint8_t* d_ldesc, const int* d_nl, int nrows, int capl,
        const int32_t* d_kfml, int nml,
        int npairs, const int32_t* d_pair, int32_t* d_lmatch, int32_t* d_nlmatch);

/* Batched line matching in HBM: knn2 + ratio rule of LSDmatcher::SearchByProjection(KF,F) (:143-183) with all
   KF lines valid: d_lmatch[p*capl + tdx] = qdx or -1; d_nlmatch[p]. */
int  sslpl_match_lines_batch_device(sslpl_matcher* m, const uint8_t* d_ldesc, const int* d_nl, int nframes, int capl,
                                    int32_t* d_lmatch, int32_t* d_nlmatch);

/* ---- LocalMapping's triangulation matchers over keyframe pairs resident in HBM (SURVEY.md 8(f) rows 2/3), asynchronous on the
   handle's stream like the other *_batch_device calls; no caller-visible allocation.  LocalMapping::CreateNewMapPoints (LocalMapping.cc:
   371-440) runs ORBmatcher::SearchForTriangulation(KF, KF2, F12, pairs, false) against each covisible neighbour, CreateNewMapLines2
   (:911-988) LSDmatcher::SearchForTriangulation(KF, KF2, pairs); here one call runs a whole list of such pairs.
   The keyframe set: nkf keyframes, `cap` (lines: `capl`) rows each, the layout of sslpl_orb_device_results / sslpl_line_device_results:
   d_kps[k][cap] = mvKeysUn, d_desc[k][cap][32], d_n[k] (clamped to cap).  The pair list: d_pair[p] = (kf1, kf2) int32, kf1 in the
   pKF1 role, kf2 in the pKF2 role.  A pair with an index outside [0, nkf) gets the count -1 and no rows.
   Needs nkf in [1, max_batch + 1] and npairs in [1, max_batch]; bad arguments return SSLPL_ERR_ARG and enqueue nothing.  Every pair's
   rows and count equal what sslpl_search_for_triangulation / sslpl_line_match(mode 3) return for it.

   ORBmatcher::SearchForTriangulation(pKF1, pKF2, F12, vMatchedPairs, bOnlyStereo = false) (ORBmatcher.cc:660-826), monocular.
   d_has_mp[k][cap] = KeyFrame::GetMapPoint(i) != NULL.  The FeatureVectors are KeyFrame::ComputeBoW's (KeyFrame.cc:71-80), computed here
   from the descriptors with the vocabulary v at levelsup.  d_geom[p][11] = F12 (3x3 row-major, LocalMapping::ComputeF12 :1286-1300) then
   the epipole ex, ey (ORBmatcher.cc:666-673), f32.  scale / sigma2 = mvScaleFactors / mvLevelSigma2 (HOST, nlevels <= SSLPL_MAX_LEVELS); a
   KF2 feature whose octave is outside [0, nlevels) is never a candidate.  Result: d_pairs[p][cap][2] = (idx1, idx2) in ascending idx1,
   (-1, -1) after the count; d_nmatch[p].  Needs cap <= max_features + 64 and the vocabulary's level nodes <= max_nodes; the first call
   allocates a [max_batch][max_features + 64] int32 table, freed with the handle. */
int  sslpl_search_for_triangulation_batch_device(sslpl_matcher* m,
        const sslpl_keypoint* d_kps, const uint8_t* d_desc, const int* d_n, int nkf, int cap,
        const uint8_t* d_has_mp, const sslpl_vocab* v, int levelsup,
        int npairs, const int32_t* d_pair, const float* d_geom,
        const float* scale, const float* sigma2, int nlevels, int checkOrientation,
        int32_t* d_pairs, int32_t* d_nmatch);
/* LSDmatcher::SearchForTriangulation(pKF1, pKF2, vMatchedPairs) (LSDmatcher.cpp:382-415), with KeyFrame::lineDescriptorMAD
   (KeyFrame.cc:820-846) on the device.  d_ldesc[k][capl][32], d_nl[k], d_has_ml[k][capl] = KeyFrame::GetMapLine(i) != NULL.
   Result: d_lpairs[p][capl][2] = (qdx, tdx) in ascending qdx, (-1, -1) after the count; d_nlmatch[p].  When KF1 has lines and KF2 fewer
   than 2 (the reference reads lmatches[i][1] out of bounds there; the single call returns SSLPL_ERR_ARG) d_nlmatch[p] = -1; when KF1 has
   none it is 0.  Needs capl <= max_lines + 64. */
int  sslpl_line_search_for_triangulation_batch_device(sslpl_matcher* m,
        const uint8_t* d_ldesc, const int* d_nl, int nkf, int capl, const uint8_t* d_has_ml,
        int npairs, const int32_t* d_pair, int32_t* d_lpairs, int32_t* d_nlmatch);

/* ---- LocalMapping::CreateNewMapPoints (LocalMapping.cc:371-637, monocular) over keyframe pairs in HBM: the matcher and the
   triangulation of every neighbour, neighbour after neighbour.  Same keyframe set, vocabulary, d_has_mp, pair list and d_geom as
   sslpl_search_for_triangulation_batch_device (checkOrientation is false, as LocalMapping's ORBmatcher(0.6, false) has it), plus
   d_kfpose[k][15] = Tcw (3x4 row-major) then Ow, f32 (the pose table of the batched Fuse calls), the HOST cam[6] = fx fy cx cy invfx invfy
   (as the KeyFrame holds them, one camera for all keyframes), scaleFactors / levelSigma2 = mvScaleFactors / mvLevelSigma2 (HOST, nlevels
   entries) and scaleFactor = mfScaleFactor.
   Chains: a maximal run of consecutive pairs with the same kf1 is one keyframe's neighbour loop, in GetBestCovisibilityKeyFrames order.
   Inside a chain the pairs run strictly in order: the KF1 features that have a MapPoint start as d_has_mp[kf1] and gain the idx1 of
   every created row (KeyFrame::AddMapPoint(pMP, idx1), :624), which the matcher of the later pairs then skips (ORBmatcher.cc:702-706).
   Chains are independent, and the inputs are never modified.  The first k pairs of a chain give what a call with only those pairs
   gives (a neighbour loop that stops at CheckNewKeyFrames, :408).  A pair with an index outside [0, nkf), with kf2 == kf1 or with a kf2
   that an earlier pair of its chain had gets the count -1, no rows, and leaves the chain's state alone.
   Results per pair p, `cap` rows each:
     d_pairs[p][cap][2]  (idx1, idx2) in ascending idx1: what SearchForTriangulation returns under the mask of that neighbour; (-1, -1)
                         after the count;
     d_nmatch[p]         the row count (-1: bad pair);
     d_status[p][cap]    per row SSLPL_CNMP_CREATED (0) or the test that rejected it, SSLPL_CNMP_*; -1 after the count;
     d_x3d[p][cap][3]    the triangulated point x3D (f32), written for every row that got past the w == 0 test (status 0 or >= 3);
                         other rows are not written;
     d_nnew[p]           the rows with status 0.
   The rows with status 0, in (pair, row) order, are the reference's MapPoint creation order.  Two created rows of one pair may share
   an idx2 (nothing marks a KF2 feature as taken): KF2's slot then ends with the later one (pKF2->AddMapPoint overwrites), so a caller
   applies them in order.  Numerics are those of the reference with cv2 4.13 and glibc >= 2.35: the 4x4 cv::SVD is OpenCV's one-sided
   Jacobi, its hypot glibc's; see DESIGN.md.  A KF1 keypoint whose octave is outside [0, nlevels) gets SSLPL_CNMP_OCTAVE1 (the
   reference indexes mvLevelSigma2 out of bounds).  Asynchronous on the matcher's stream; bad arguments return SSLPL_ERR_ARG and enqueue
   nothing. ---- */
enum {
    SSLPL_CNMP_CREATED = 0,    /* the MapPoint is created (:619-634) */
    SSLPL_CNMP_PARALLAX = 1,   /* cosParallaxRays not in (0, 0.9998) (:497, :526) */
    SSLPL_CNMP_W_ZERO = 2,     /* vt.row(3)(3) == 0 (:511) */
    SSLPL_CNMP_Z1 = 3,         /* depth in KF1 <= 0 (:533-535) */
    SSLPL_CNMP_Z2 = 4,         /* depth in KF2 <= 0 (:537-539) */
    SSLPL_CNMP_OCTAVE1 = 5,    /* KF1 keypoint octave outside [0, nlevels) (:543) */
    SSLPL_CNMP_REPROJ1 = 6,    /* reprojection chi2 in KF1 > 5.991 sigma2 (:549-559) */
    SSLPL_CNMP_REPROJ2 = 7,    /* reprojection chi2 in KF2 > 5.991 sigma2 (:578-586) */
    SSLPL_CNMP_DIST0 = 8,      /* dist1 == 0 || dist2 == 0 (:607) */
    SSLPL_CNMP_SCALE = 9       /* scale consistency (:615) */
};
int  sslpl_create_new_map_points_batch_device(sslpl_matcher* m,
        const sslpl_keypoint* d_kps, const uint8_t* d_desc, const int* d_n, int nkf, int cap,
        const uint8_t* d_has_mp, const sslpl_vocab* v, int levelsup,
        int npairs, const int32_t* d_pair, const float* d_geom, const float* d_kfpose,
        const float* cam, const float* scaleFactors, const float* levelSigma2, int nlevels, float scaleFactor,
        int32_t* d_pairs, int32_t* d_nmatch, int32_t* d_status, float* d_x3d, int32_t* d_nnew);
/* The device functions of that call on HOST tables: the 4x4 SVD of n row-major matrices A[n][16] -> W[n][4] (descending) and
   Vt[n][16] (cv::SVD::compute(A, w, u, vt, MODIFY_A | FULL_UV) on CV_32F), and glibc's hypot of nh pairs -> h[nh].  Synchronous. */
int  sslpl_matcher_debug_svd4(sslpl_matcher* m, int n, const float* A, float* W, float* Vt,
                              int nh, const double* hx, const double* hy, double* h);

/* ---- LocalMapping::CreateNewMapLines2 (LocalMapping.cc:911-1173, monocular) over keyframe pairs in HBM: the line matcher and the
   triangulation of both end points of every match, neighbour after neighbour.  The keyframe set is the layout of sslpl_line_device_results:
   d_kl[k][capl] = KeyFrame::mvKeyLines (F.mvKeylinesUn), d_ldesc[k][capl][32], d_lineeq[k][capl][3] = mvKeyLineFunctions (double),
   d_nl[k] (clamped to capl); d_has_ml[k][capl] = GetMapLine(i) != NULL.  d_kfpose[k][15] = Tcw (3x4 row-major) then Ow, f32 (the pose
   table of the points call); d_kfdepth[k] = KeyFrame::ComputeSceneMedianDepth(2) (KeyFrame.cc:711-741) as the caller computes it, f32;
   the HOST cam[6] = fx fy cx cy invfx invfy, one camera for all keyframes.
   The pair list is the caller's: it keeps the baseline gate (:955-979, ratioBaselineDepth < 0.1 drops the neighbour) and takes the
   nn = 10 best covisible keyframes.  Both differ from the points call (gate 0.01, nn = 20), so lines need their own pair list.
   Chains work as in sslpl_create_new_map_points_batch_device: a maximal run of consecutive pairs with the same kf1 is one neighbour loop,
   run in order; the KF1 mask starts as d_has_ml[kf1] and gains the qdx of every created row (AddMapLine(pML, idx1), :1159), which the
   matcher of the later pairs skips (LSDmatcher.cpp:403).  The KF2 masks are used as given (the kf2s of a chain are distinct).  Chains are
   independent, the inputs are never modified, and the first k pairs of a chain give what a call with only those pairs gives.  A pair
   with an index outside [0, nkf), with kf2 == kf1, with a kf2 repeated in its chain, or whose KF1 has lines and KF2 fewer than 2 gets
   the count -1, no rows, and leaves the chain's state alone; a KF1 without lines gives 0.
   Results per pair p, `capl` rows each:
     d_lpairs[p][capl][2]  (qdx, tdx) in ascending qdx: what LSDmatcher::SearchForTriangulation returns under the mask of that
                           neighbour; (-1, -1) after the count;
     d_nlmatch[p]          the row count (-1: bad pair);
     d_status[p][capl]     per row SSLPL_CNML_CREATED (0) or the test that rejected it, SSLPL_CNML_*; -1 after the count;
     d_line3d[p][capl][6]  s3D then e3D (f32), written for the rows with status 0 or >= 4; other rows are not written;
     d_nnew[p]             the rows with status 0.
   The rows with status 0, in (pair, row) order, are the reference's MapLine creation order.  Two created rows of one pair may share a
   tdx: KF2's slot then ends with the later one, so a caller applies them in order.  Numerics are those of the reference with cv2 4.13
   and glibc >= 2.35 (DESIGN.md).  Concurrency: in the reference CreateNewMapPoints runs in another thread at the same time and adds
   MapPoints to the same KF2s, so the depth ComputeSceneMedianDepth(2) gives at :973 and at :1098 is not deterministic there; this call
   takes one depth per keyframe as given.  Asynchronous on the matcher's stream, no caller-visible allocation (the first call allocates a
   [max_batch][max_lines + 64] int32 table, freed with the handle).  Needs nkf in [1, max_batch + 1], npairs in [1, max_batch] and capl
   in [1, max_lines + 64]; bad arguments return SSLPL_ERR_ARG and enqueue nothing. ---- */
enum {
    SSLPL_CNML_CREATED = 0,    /* the MapLine is created (:1150-1169) */
    SSLPL_CNML_PARALLAX = 1,   /* !(cos < cos + 1 && cos > 0 && cos < 0.98) (:1041-1053, :1090) */
    SSLPL_CNML_W_ZERO_S = 2,   /* vt1.row(3)(3) == 0, start point (:1066) */
    SSLPL_CNML_W_ZERO_E = 3,   /* vt2.row(3)(3) == 0, end point (:1084) */
    SSLPL_CNML_NEAR_S1 = 4,    /* |s3D - Ow1| / depth2 < 0.3 (:1099-1103) */
    SSLPL_CNML_NEAR_S2 = 5,    /* |s3D - Ow2| / depth2 < 0.3 (:1105-1109) */
    SSLPL_CNML_LONG = 6,       /* |e3D - s3D| / depth2 > 0.61 (:1112-1116) */
    SSLPL_CNML_NEAR_E1 = 7,    /* |e3D - Ow1| / depth2 < 0.3 (:1122-1126) */
    SSLPL_CNML_NEAR_E2 = 8,    /* |e3D - Ow2| / depth2 < 0.3 (:1127-1131) */
    SSLPL_CNML_ZS1 = 9,        /* start point depth in KF1 <= 0 (:1134-1136) */
    SSLPL_CNML_ZS2 = 10,       /* start point depth in KF2 <= 0 (:1138-1140) */
    SSLPL_CNML_ZE1 = 11,       /* end point depth in KF1 <= 0 (:1142-1144) */
    SSLPL_CNML_ZE2 = 12        /* end point depth in KF2 <= 0 (:1146-1148) */
};
int  sslpl_create_new_map_lines_batch_device(sslpl_matcher* m,
        const sslpl_keyline* d_kl, const uint8_t* d_ldesc, const double* d_lineeq, const int* d_nl, int nkf, int capl,
        const uint8_t* d_has_ml, int npairs, const int32_t* d_pair,
        const float* d_kfpose, const float* d_kfdepth, const float* cam,
        int32_t* d_lpairs, int32_t* d_nlmatch, int32_t* d_status, float* d_line3d, int32_t* d_nnew);

/* ---- MapPoint::PredictScale / MapLine::PredictScale (MapPoint.cc:390-405, MapLine.cpp:386-395) on the device, exact against the host's
   logf: level = (int)ceil(logf(ratio) / logScaleFactor), ratio = mfMaxDistance / dist.  The level is a monotone step function of the float
   ratio; thr[k] (k = 0 .. nlevels, nlevels + 1 floats) is the smallest positive float whose level is >= k, found by bisection over the
   float bit patterns with this process's logf (+inf when no finite ratio gets there).  Host-only, needs no device.  The device counts
   the thresholds <= ratio.  A ratio that is not finite and positive (NaN, +-inf, <= 0: dist = 0, 0 / 0) gives INT_MIN on x86-64, i.e.
   level 0 for a MapPoint (clamped to [0, nlevels - 1]) and outside the pyramid for a MapLine (not clamped: dropped).
   Needs nlevels in [1, SSLPL_MAX_LEVELS] and logScaleFactor positive and finite. ---- */
int  sslpl_predict_scale_table(float logScaleFactor, int nlevels, float* thr);
/* The device function the batched Fuse calls use, on n HOST ratios: clamp != 0 gives the MapPoint level in [0, nlevels - 1]; clamp = 0
   gives INT_MIN for a ratio that is not finite and positive, else the level when it lies in [0, nlevels), -1 for any level below 0
   and nlevels for any level >= nlevels.  Synchronous. */
int  sslpl_matcher_debug_predict_scale(sslpl_matcher* m, int n, const float* ratio, float logScaleFactor, int nlevels, int clamp,
                                       int32_t* level);

/* ---- LocalMapping::SearchInNeighbors' Fuse calls (LocalMapping.cc:1178-1279) over keyframes resident in HBM, monocular, asynchronous on
   the handle's stream; no caller-visible allocation.  ORBmatcher::Fuse(pKF, vpMapPoints, th) (ORBmatcher.cc:828-973) and
   LSDmatcher::Fuse(pKF, vpMapLines, th) (LSDmatcher.cpp:417-548) are one call per target keyframe in the reference; here one call runs a
   flat list of (keyframe, element) entries over many keyframes, projection stage included.
   The keyframe set: nkf in [1, max_batch + 1] keyframes, the layout of sslpl_orb_device_results / sslpl_line_device_results (d_kps[k][cap] =
   mvKeysUn, d_desc[k][cap][32], d_n[k]; d_kl[k][capl] = mvKeyLines, d_ldesc[k][capl][32], d_nl[k]; counts clamped to cap / capl), and
   d_kfpose[k][15] = Tcw (3x4 row-major) then Ow (GetCameraCenter), f32.  The entries: d_entry[e] = (kf, element) int32, element -1 =
   a NULL pointer in the vector; d_skip[e] (u8, NULL = none) = what the reference tests before projecting, as the caller sees it at the
   call: points isBad() || IsInKeyFrame(kf), lines isBad() (line Fuse has no IsInKeyFrame test).  cam = fx fy cx cy, bounds = mnMinX
   mnMaxX mnMinY mnMaxY, scaleFactors = mvScaleFactors, nlevels <= SSLPL_MAX_LEVELS, logScaleFactor = mfLogScaleFactor (all HOST).
   Result per entry: d_best_idx[e], d_best_dist[e] = what the projection stage followed by sslpl_fuse_points_search /
   sslpl_fuse_lines_search give for that keyframe (the caller fuses when best_dist <= 50): (-1, 256) for a point and (-1, INT_MAX) for
   a line without a candidate (skipped, NULL, failed gate, a line whose level falls outside the pyramid).  An entry whose kf is outside
   [0, nkf) or whose element is outside [-1, nel) gets (-1, -1) and reads nothing.  nentries = 0 enqueues nothing; bad arguments
   return SSLPL_ERR_ARG and enqueue nothing.
   Order dependence: the results are exact for the inputs as given.  Within one reference Fuse call a Replace recomputes the surviving
   element's descriptor (MapPoint.cc:217, MapLine.cpp:216), which later iterations read; Replace leaves position, normal and distances
   alone, so a descriptor change is the only way a result goes stale.  SearchInNeighbors is two dependent calls: phase A (the current
   keyframe's elements into every target) and phase B (the candidates, collected from the targets after phase A's bookkeeping
   :1209-1224, into the current keyframe).  The caller applies Replace / AddObservation in entry order, re-tests isBad / IsInKeyFrame
   there, and re-submits any entry whose element's descriptor a Replace recomputed since the call.

   Points: d_mp[m][9] = Xw, normal, GetMinDistanceInvariance(), GetMaxDistanceInvariance(), mfMaxDistance; d_mpdesc[m][32].
   invLevelSigma2 = mvInvLevelSigma2 (HOST).  Every keyframe's 64 x 48 grid (AssignFeaturesToGrid) is built per call in a workspace of
   max_batch + 1 grids allocated by the first call that needs it (shared with sslpl_search_by_projection_frame_batch_device) and freed
   with the handle.  A keyframe octave below 0 is never a candidate.  Stereo (mvuRight >= 0) stays with the single call. */
int  sslpl_fuse_points_batch_device(sslpl_matcher* m,
        const sslpl_keypoint* d_kps, const uint8_t* d_desc, const int* d_n, int nkf, int cap, const float* d_kfpose,
        int nmp, const float* d_mp, const uint8_t* d_mpdesc, int nentries, const int32_t* d_entry, const uint8_t* d_skip,
        const float* cam, const float* bounds, const float* scaleFactors, const float* invLevelSigma2, int nlevels, float logScaleFactor,
        float th, int32_t* d_best_idx, int32_t* d_best_dist);
/* Lines: d_ml[m][12] = SP, EP (GetWorldPos, narrowed to float), GetNormal() (narrowed to float), minInv, maxInv, mfMaxDistance;
   d_mldesc[m][32].  Needs capl <= max_lines + 64. */
int  sslpl_fuse_lines_batch_device(sslpl_matcher* m,
        const sslpl_keyline* d_kl, const uint8_t* d_ldesc, const int* d_nl, int nkf, int capl, const float* d_kfpose,
        int nml, const float* d_ml, const uint8_t* d_mldesc, int nentries, const int32_t* d_entry, const uint8_t* d_skip,
        const float* cam, const float* bounds, const float* scaleFactors, int nlevels, float logScaleFactor, float th,
        int32_t* d_best_idx, int32_t* d_best_dist);

/* ---- Optimizer::PoseOptimization(Frame*, isCorner) (Optimizer.cc:666-1022) over frames resident in HBM, monocular, asynchronous on the
   handle's stream; no caller-visible allocation.  The step after every Tracking matcher (Tracking.cc:1048, :1259, :1328, :2059-2090):
   four rounds of 10 Levenberg-Marquardt iterations on the frame's 6-DoF pose, each from the input pose, with Huber kernels in rounds
   0-2 and an inlier / outlier classification after each round.  One CTA per frame; the result of a frame depends on its own rows only.
   Frame f: d_kps[f][cap] = mvKeysUn (x, y, octave read), d_n[f] (clamped to [0, cap]); d_fmp[f][cap] = mvpMapPoints as element indices
   into d_mp[nmp][9] (the Fuse element table; Xw = columns 0..2), -1 or any index outside [0, nmp) = NULL.  Lines: d_lineeq[f][capl][3] =
   mvKeyLineFunctions (sslpl_line_device_results), d_nl[f] (clamped to [0, capl]), d_fml[f][capl] = mvpMapLines as element indices into
   d_mlpos[nml][6] (f64 mWorldPos, the table of sslpl_update_map_lines_batch_device); d_fml = NULL means no line edges,
   Optimizer::PoseOptimization(Frame*) (Optimizer.cc:1024, Relocalization), and the other line pointers are not read.  d_Tcw[f][12] = mTcw
   (3x4 row-major).  cam = {fx, fy, cx, cy} and invLevelSigma2[nlevels] = mvInvLevelSigma2 are HOST arrays, one camera for all frames.
   Results: d_Tcw_out[f][12] (may alias d_Tcw) = the pose SetPose writes (Converter::toCvMat of the final SE3Quat, narrowed to float);
   d_outlier[f][cap] / d_line_outlier[f][capl] = mvbOutlier / mvbLineOutlier, written only for features with an edge (other entries are
   left alone, so a caller passes its current rows); d_ninlier[f] = the return value, nInitialCorrespondences - nBad.  With fewer than
   3 correspondences the pose is copied, the edges' flags are written 0 and d_ninlier is 0.  A frame in which a feature with an edge has
   an octave outside [0, nlevels) gets d_ninlier = -1, its pose copied and no flags (the reference indexes mvInvLevelSigma2 out of
   bounds there).  Stereo edges (mvuRight >= 0) are not supported.  Needs nframes in [1, max_batch], cap <= max_features + 64, capl <=
   max_lines + 64 (with lines) and nlevels in [1, SSLPL_MAX_LEVELS]; bad arguments return SSLPL_ERR_ARG and enqueue nothing.
   Results are bitwise reproducible and independent of a frame's position in the batch; against g2o they agree to the tolerance DESIGN.md
   ("Pose optimisation") states, not bit for bit. */
int  sslpl_pose_optimization_batch_device(sslpl_matcher* m,
        const sslpl_keypoint* d_kps, const int* d_n, int nframes, int cap,
        const int32_t* d_fmp, int nmp, const float* d_mp,
        const double* d_lineeq, const int* d_nl, int capl, const int32_t* d_fml, int nml, const double* d_mlpos,
        const float* d_Tcw, const float* cam, const float* invLevelSigma2, int nlevels,
        float* d_Tcw_out, uint8_t* d_outlier, uint8_t* d_line_outlier, int32_t* d_ninlier);

/* =====================================================================================
 * (2) Line segments — replaces LineSegment::ExtractLineSegment (src/ExtractLineSegment.cpp:18-69)
 * ===================================================================================== */
typedef struct sslpl_line sslpl_line;
typedef struct {
    int lsdNFeatures;     /* hard-coded 40 in the reference (ExtractLineSegment.cpp:42) */
    int max_width, max_height, max_batch, device;
} sslpl_line_params;
int  sslpl_line_create(const sslpl_line_params* p, sslpl_line** out);
void sslpl_line_destroy(sslpl_line* h);
/* ExtractLineSegment(img, keylines, ldesc, keylineFunctions, scale=1, numOctaves=1): kl[cap], ldesc[cap*32], lineeq[cap*3] */
int  sslpl_line_extract(sslpl_line* h, const uint8_t* img, int width, int height, int pitch,
                        sslpl_keyline* kl, uint8_t* ldesc, double* lineeq, int cap, int* n);
int  sslpl_line_extract_batch(sslpl_line* h, const uint8_t* imgs, int nframes, int width, int height, int pitch,
                              size_t frame_stride, sslpl_keyline* kl, uint8_t* ldesc, double* lineeq, int cap, int* n);
/* asynchronous form (finish with sslpl_line_sync) */
int  sslpl_line_extract_batch_begin(sslpl_line* h, const uint8_t* imgs, int nframes, int width, int height, int pitch,
                                    size_t frame_stride, sslpl_keyline* kl, uint8_t* ldesc, double* lineeq, int cap, int* n);
int  sslpl_line_extract_batch_device(sslpl_line* h, const uint8_t* d_imgs, int nframes, int width, int height, int pitch,
                                     size_t frame_stride);
int  sslpl_line_device_results(sslpl_line* h, const sslpl_keyline** d_kl, const uint8_t** d_ldesc, const double** d_lineeq,
                               const int** d_n, int* cap);
int  sslpl_line_sync(sslpl_line* h);
void* sslpl_line_stream(sslpl_line* h);
int  sslpl_line_set_stream(sslpl_line* h, void* cuda_stream);
long long sslpl_line_launch_count(const sslpl_line* h);
/* Scheduling knob (no effect on results): the LSD region stage runs one multi-warp CTA per frame; bound how many of them one
   call keeps resident (0 = one per frame, the default).  Useful when several handles are in flight on one GPU next to wide
   kernels: resident walkers pin registers for milliseconds. */
int  sslpl_line_set_max_walkers(sslpl_line* h, int max_concurrent);
/* Statistics of the last multi-warp region-walker launch, 16 values (see csrc/line.cu): regions grown by the turn holder / as
   speculated, redo causes, cycles under the commit and claim locks, cycles per frame.  The one-warp walker leaves them 0.
   Diagnostic only. */
int  sslpl_line_walker_stats(sslpl_line* h, unsigned long long* out16);
int  sslpl_line_set_profiling(sslpl_line* h, int on);
int  sslpl_line_stage_ms(sslpl_line* h, float* ms, int cap, const char** names, int* nstages);
/* raw LSD segments (before the top-N cut) of frame f of the last call: seg[4*i] = x1,y1,x2,y2 */
int  sslpl_line_download_segments(sslpl_line* h, int frame, float* seg4, int cap, int* n);
/* debug: with SSLPL_LINE_TRACE=1 in the environment at create time, one row of 10 doubles per LSD region that reached
   region2rect: seed pixel, size before/after refine, log_nfa, x1,y1,x2,y2,width,p (detection scale) */
int  sslpl_line_debug_trace(sslpl_line* h, int frame, double* out, int cap_rows, int* n);
/* debug: the per-pixel pre-pass of frame f of the last call (waits for the handle's stream).  Input resolution w x hgt: Sobel dx, dy.
   Detection scale sw x sh: level-line angle in degrees (-1024 = NOTDEF), pix_cs[2 per pixel] = (float)cos / sin of (float)(angle in
   radians), cs0[2 per pixel] = float(cos / sin) of the angle in radians as double, gradient norm, *maxgrad = largest norm of a defined
   pixel (0 when none), seeds = defined pixel indices (y * sw + x) by descending gradient bin, raster order inside a bin (room for sw * sh
   entries), *nseeds.  Any output pointer may be NULL.  Region growing changes none of these, so they stay valid after a full call. */
int  sslpl_line_download_prep(sslpl_line* h, int frame, int* w, int* hgt, int* sw, int* sh, int16_t* dx, int16_t* dy, float* angdeg,
                              float* pix_cs, float* cs0, double* modgrad, double* maxgrad, uint32_t* seeds, int* nseeds);
/* The four debug calls below each launch one kernel on the handle's stream, counted by sslpl_line_launch_count, and wait for it. */
/* debug: the pre-pass's per-pixel ll_angle arithmetic on every 2x2 difference pair (DA = D - A, BC = B - C, each in [-255, 255]),
   entry (DA + 255) * 511 + (BC + 255): 261121 angles, cs / cs0 pairs and norms, as in sslpl_line_download_prep.  NULL = skip. */
int  sslpl_line_debug_ll_table(sslpl_line* h, float* angdeg, float* cs, float* cs0, double* modgrad);
/* debug: the LSD NFA (nfa() of lsd.cpp, as the NFA kernels evaluate it) of n triples (N[i], K[i], P[i]), with the log_nt and log-gamma
   table of a width x height frame (the handle is configured for that size as a call would).  plain = 1 evaluates the same function with
   its two shortcuts off (the pow skip and the log10 bracket of the stop test).  stop (may be NULL) receives the index i at which the
   tail loop stopped, N + 1 when it ran out, -1 for the early returns.  Requires 0 <= K <= N < sw * sh + 2 (SSLPL_ERR_ARG otherwise). */
int  sslpl_line_debug_nfa(sslpl_line* h, int width, int height, int n, const int* N, const int* K, const double* P, int plain,
                          double* out, int* stop);
/* debug: the region fit's correctly-rounded sin / cos (csrc/ddtrig.h) of n doubles on the device: full = 0 is sincos_cr (quick
   evaluation first, the form region2rect calls), full = 1 sincos_cr_full (always the long evaluation). */
int  sslpl_line_debug_sincos(sslpl_line* h, int n, const double* x, int full, double* s, double* c);
/* debug: the line path's cv::fastAtan2 (degrees) of n float pairs on the device */
int  sslpl_line_debug_atan2(sslpl_line* h, int n, const float* y, const float* x, float* out);

/* =====================================================================================
 * (4) Frame level — what Frame::Frame(imGray, ...) does with the two extractors (src/Frame.cc:69-131), the colour conversion in
 *     front of it (Tracking::GrabImageMonocularWithPL, src/Tracking.cc:148-161) and Frame::UndistortKeyPoints /
 *     ComputeImageBounds behind it (src/Frame.cc:483-543).  ONE upload of the frame; ORB and LSD+LBD on two streams.
 * ===================================================================================== */
typedef struct sslpl_frame sslpl_frame;
typedef struct { sslpl_orb_params orb; sslpl_line_params line; } sslpl_frame_params;   /* device, max_batch and max size must agree */
int  sslpl_frame_create(const sslpl_frame_params* p, sslpl_frame** out);
void sslpl_frame_destroy(sslpl_frame* h);
sslpl_orb*  sslpl_frame_orb(sslpl_frame* h);     /* the extractors it owns (device results, tables, stage times) */
sslpl_line* sslpl_frame_line(sslpl_frame* h);
long long sslpl_frame_launch_count(const sslpl_frame* h);
/* Camera.fx/fy/cx/cy and k1 k2 p1 p2 [k3] (Tracking.cc:58-86); undistortion is skipped when k1 == 0 (Frame.cc:485) */
int  sslpl_frame_set_camera(sslpl_frame* h, float fx, float fy, float cx, float cy, const float* dist, int ndist);
int  sslpl_frame_image_bounds(sslpl_frame* h, int cols, int rows, float* bounds4 /* mnMinX mnMaxX mnMinY mnMaxY */);
/* debug: k_undistort (mvKeysUn of one keypoint) on n host points xy[2 n] with the camera of the last sslpl_frame_set_camera, into
   xy_out[2 n] (may alias xy); unchanged points when k1 == 0.  Launches one kernel on the ORB stream, counted by
   sslpl_frame_launch_count, and waits for it.  sslpl_frame_image_bounds runs its four corners through this call. */
int  sslpl_frame_debug_undistort(sslpl_frame* h, int n, const float* xy, float* xy_out);
/* channels 1 (grey), 3 or 4 (interleaved 8-bit; rgb_order 1 = RGB[A], 0 = BGR[A] as Camera.RGB says).  Any output pointer but the
   counts may be NULL.  kps / kps_un / desc hold `cap` entries per frame (>= sslpl_orb_max_keypoints), the line outputs `lcap`. */
int  sslpl_frame_extract(sslpl_frame* h, const uint8_t* img, int width, int height, int pitch, int channels, int rgb_order,
                         sslpl_keypoint* kps, sslpl_keypoint* kps_un, uint8_t* desc, int cap, int* nkp,
                         sslpl_keyline* kl, uint8_t* ldesc, double* lineeq, int lcap, int* nl);
int  sslpl_frame_extract_batch(sslpl_frame* h, const uint8_t* imgs, int nframes, int width, int height, int pitch, size_t frame_stride,
                               int channels, int rgb_order,
                               sslpl_keypoint* kps, sslpl_keypoint* kps_un, uint8_t* desc, int cap, int* nkp,
                               sslpl_keyline* kl, uint8_t* ldesc, double* lineeq, int lcap, int* nl);
/* asynchronous form: enqueue only (pinned host buffers), finish with sslpl_frame_sync */
int  sslpl_frame_extract_batch_begin(sslpl_frame* h, const uint8_t* imgs, int nframes, int width, int height, int pitch, size_t frame_stride,
                                     int channels, int rgb_order,
                                     sslpl_keypoint* kps, sslpl_keypoint* kps_un, uint8_t* desc, int cap, int* nkp,
                                     sslpl_keyline* kl, uint8_t* ldesc, double* lineeq, int lcap, int* nl);
int  sslpl_frame_sync(sslpl_frame* h);
void* sslpl_frame_stream(sslpl_frame* h, int which /* 0 = ORB stream, 1 = line stream */);
int  sslpl_frame_device_gray(sslpl_frame* h, const uint8_t** d_gray, int* pitch, size_t* frame_stride);
/* mvKeysUn of the last call, in HBM ([nframes][cap], counts as in sslpl_orb_device_results): the undistorted keypoints when the camera
   has k1 != 0 (they are computed on every call then), the ORB handle's keypoints otherwise (Frame.cc:485).  Written on the ORB stream
   (sslpl_frame_stream(h, 0)): sync the frame, or order that stream before the consumer's. */
int  sslpl_frame_device_keypoints_un(sslpl_frame* h, const sslpl_keypoint** d_kps_un, int* cap);

#ifdef __cplusplus
}
#endif
#endif /* SSLPL_H */
