// match.cu — H100 (sm_90a) Hamming matchers: brute-force 2-NN (cv::BFMatcher knnMatch k=2), vocabulary-node
// assignment, SearchByBoW (KF-Frame and KF-KF), SearchForTriangulation, rotation-histogram filter, and the
// knn-based LSDmatcher entry points.  Replaces the distance work of src/ORBmatcher.cc and src/LSDmatcher.cpp.
//
// No tensor cores: 256-bit XOR + popcount per pair, reduced with warp shuffles.  Descriptors are read as
// 2 x uint4 per row.  The batched layout is "a set of frames": frame f owns desc[f*cap..], a CSR feature
// vector and optional masks; pair p matches frame p (KeyFrame role) against frame p+1 (Frame role).
#include "common.cuh"
#include "../../include/sslpl_map.h"
#include "svd4.cuh"
#include "pose.cuh"
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <vector>

namespace sslpl {

constexpr int TH_LOW = 50;          // ORBmatcher.cc:38
constexpr int MAX_DYN_SMEM = 200 * 1024;   // dynamic shared memory the two data-dependent kernels may ask for (sm_90: 227 KB per CTA, static included)
constexpr int HISTO_LENGTH = 30;    // ORBmatcher.cc:39

// A set of frames in HBM (strides in elements of the respective type)
struct FrameSet {
    const uint8_t* desc; long long desc_fs;                  // 32 B per row; frame stride in bytes
    const int* n; int n_const;                               // per-frame feature count (device array) or constant
    const int* nodes; const int* off; const int* idx; const int* nn; int nn_const;
    long long nodes_fs, off_fs, idx_fs;                      // CSR frame strides (ints)
    const uint8_t* flag; long long flag_fs;                  // valid / has-MapPoint mask (may be null)
    const float* angle; int angle_es; long long angle_fs;    // keypoint angle: element stride / frame stride in floats
    const float* x; const float* y; const int* oct;          // same strides as angle (fields of sslpl_keypoint)
    const int2* pmap; int nframes;                           // pair p = frames (pmap[p].x, pmap[p].y) of [0, nframes); NULL: (p, p + 1)
};

// the frames of pair p; false when a mapped index lies outside [0, nframes) (the pair is then left empty)
__device__ __forceinline__ bool pair_frames(const int2* pmap, int nframes, int pair, int& f1, int& f2) {
    if (!pmap) { f1 = pair; f2 = pair + 1; return true; }
    const int2 q = pmap[pair];
    f1 = q.x; f2 = q.y;
    return (unsigned)f1 < (unsigned)nframes && (unsigned)f2 < (unsigned)nframes;
}

__device__ __forceinline__ void load_desc(const uint8_t* p, uint4& a, uint4& b) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    a = __ldg(q); b = __ldg(q + 1);
}

// -------------------------------------------------------------------------------------------------
// knnMatch(k=2): one warp per query.  key = dist << 20 | trainIdx  => ascending distance, ties -> lower index
// Pair p queries frame p of q against frame p of t (t already points at the train frames), or, with a pair map, frame
// pmap[p].x of q against frame pmap[p].y of t (both arrays then start at frame 0).  kMap = false compiles the map out: the
// consecutive-pair instance keeps its registers (and occupancy) on bench.py's line path.
// -------------------------------------------------------------------------------------------------
__device__ __forceinline__ void top2_insert(unsigned& k0, unsigned& k1, unsigned k) {
    if (k < k0) { k1 = k0; k0 = k; } else if (k < k1) k1 = k;
}
// the two smallest keys of the warp, in every lane
__device__ __forceinline__ void top2_warp32(unsigned& k0, unsigned& k1) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned o0 = __shfl_xor_sync(0xffffffffu, k0, o), o1 = __shfl_xor_sync(0xffffffffu, k1, o);
        top2_insert(k0, k1, o0);
        top2_insert(k0, k1, o1);
    }
}
__device__ __forceinline__ void top2_push(unsigned long long& a1, unsigned long long& a2, unsigned long long k) {
    if (k < a1) { a2 = a1; a1 = k; } else if (k < a2) a2 = k;
}
__device__ __forceinline__ void top2_warp(unsigned long long& a1, unsigned long long& a2) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long b1 = __shfl_xor_sync(0xffffffffu, a1, o), b2 = __shfl_xor_sync(0xffffffffu, a2, o);
        const unsigned long long lo = a1 < b1 ? a1 : b1, hi = a1 < b1 ? b1 : a1, m2 = a2 < b2 ? a2 : b2;
        a1 = lo; a2 = hi < m2 ? hi : m2;
    }
}
// the smallest key of the warp, in every lane
__device__ __forceinline__ unsigned long long warp_min(unsigned long long b) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const unsigned long long t = __shfl_xor_sync(0xffffffffu, b, o); b = t < b ? t : b; }
    return b;
}

template <bool kMap>
__global__ void __launch_bounds__(256) k_knn2(const uint8_t* q, long long q_fs, const int* nq_arr, int nq_const,
                                               const uint8_t* t, long long t_fs, const int* nt_arr, int nt_const,
                                               int32_t* out, long long out_fs, int qcap, const int2* pmap, int nframes) {
    const int pair = blockIdx.y, lane = threadIdx.x & 31, qi = blockIdx.x * 8 + (threadIdx.x >> 5);
    int fq, ft;
    if (!pair_frames(kMap ? pmap : nullptr, nframes, pair, fq, ft)) return;
    const int nq = nq_arr ? min(nq_arr[fq], qcap) : nq_const, nt = nt_arr ? min(nt_arr[ft], qcap) : nt_const;
    if (qi >= nq) return;
    uint4 a0, a1;
    load_desc(q + fq * q_fs + (long long)qi * 32, a0, a1);
    const uint8_t* T = t + (kMap ? ft : pair) * t_fs;
    unsigned k0 = 0xffffffffu, k1 = 0xffffffffu;
    for (int j = lane; j < nt; j += 32) {
        uint4 b0, b1;
        load_desc(T + (long long)j * 32, b0, b1);
        top2_insert(k0, k1, ((unsigned)popc256(a0, a1, b0, b1) << 20) | (unsigned)j);
    }
    top2_warp32(k0, k1);
    if (lane == 0) {
        int4 r;
        r.x = k0 == 0xffffffffu ? -1 : (int)(k0 & 0xfffff); r.y = k0 == 0xffffffffu ? -1 : (int)(k0 >> 20);
        r.z = k1 == 0xffffffffu ? -1 : (int)(k1 & 0xfffff); r.w = k1 == 0xffffffffu ? -1 : (int)(k1 >> 20);
        reinterpret_cast<int4*>(out + pair * out_fs)[qi] = r;
    }
}

// DescriptorDistance for n pairs (ORBmatcher.cc:1650): thread per pair
__global__ void k_pair_distance(const uint8_t* a, const uint8_t* b, int n, int32_t* dist) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint4 a0, a1, b0, b1;
    load_desc(a + (long long)i * 32, a0, a1); load_desc(b + (long long)i * 32, b0, b1);
    dist[i] = popc256(a0, a1, b0, b1);
}

// -------------------------------------------------------------------------------------------------
// Vocabulary node assignment: nearest centroid, strict '<' (first wins).  Thread per descriptor,
// centroids staged in shared memory.
// -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_bow_assign(const uint8_t* desc, long long desc_fs, const int* n_arr, int n_const, int cap,
                                                     const uint8_t* centroids, int nc, int32_t* node, long long node_fs) {
    extern __shared__ uint4 s_cent[];
    const int f = blockIdx.y;
    for (int i = threadIdx.x; i < nc * 2; i += blockDim.x) s_cent[i] = __ldg(reinterpret_cast<const uint4*>(centroids) + i);
    __syncthreads();
    const int n = n_arr ? min(n_arr[f], cap) : n_const;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint4 a0, a1;
    load_desc(desc + f * desc_fs + (long long)i * 32, a0, a1);
    int best = 1 << 30, bi = 0;
    for (int c = 0; c < nc; c++) {
        const int d = popc256(a0, a1, s_cent[2 * c], s_cent[2 * c + 1]);
        if (d < best) { best = d; bi = c; }
    }
    node[f * node_fs + i] = bi;
}

// -------------------------------------------------------------------------------------------------
// DBoW2 TemplatedVocabulary<FORB>::transform (Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1218-1259): descend the
// k-ary tree by Hamming distance (strict '<': the first best child wins), one thread per descriptor.  The tree is
// stored as CSR children lists (ascending node id, as loadFromTextFile builds them) + 32-byte node descriptors; the
// upper levels stay resident in L1/L2 (ORBvoc: 1.1 M nodes x 32 B = 35 MB < 50 MB L2).
//   word  = word id of the leaf,  node = NodeId at level L - levelsup (0 if the leaf comes earlier),
//   rank  = dense index of `node` among the possible values (0 = root / early leaf, 1 + rank inside the level), or -1 for a
//           stopped word (weight <= 0), which the reference keeps out of the FeatureVector (:1162-1166).
// kMap: output row f reads its descriptors from row row_of[f] of desc (n_arr stays indexed by f); kMap = false compiles that out.
// -------------------------------------------------------------------------------------------------
struct VocabView { const int* child_off; const int* child_ids; const uint8_t* desc; const double* weight; const int* word_id; const int* level_rank; };

template <bool kMap>
__global__ void __launch_bounds__(128) k_vocab_transform(const uint8_t* desc, long long desc_fs, const int* n_arr, int n_const, int cap,
                                                          VocabView V, int nid_level, int32_t* word, int32_t* node, int32_t* rank,
                                                          double* weight, long long out_fs, const int32_t* row_of) {
    const int f = blockIdx.y;
    const int n = n_arr ? min(n_arr[f], cap) : n_const;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint4 a0, a1;
    load_desc(desc + (kMap ? row_of[f] : f) * desc_fs + (long long)i * 32, a0, a1);
    int cur = 0, nid = 0, level = 0;
    int cb = __ldg(V.child_off), ce = __ldg(V.child_off + 1);
    while (ce > cb) {
        ++level;
        int best = 1 << 30, bi = 0;
        for (int c = cb; c < ce; c++) {
            const int id = __ldg(V.child_ids + c);
            uint4 b0, b1;
            load_desc(V.desc + (long long)id * 32, b0, b1);
            const int d = popc256(a0, a1, b0, b1);
            if (d < best) { best = d; bi = id; }
        }
        cur = bi;
        if (level == nid_level) nid = cur;
        cb = __ldg(V.child_off + cur); ce = __ldg(V.child_off + cur + 1);
    }
    const double w = __ldg(V.weight + cur);
    const long long o = f * out_fs + i;
    if (word) word[o] = __ldg(V.word_id + cur);
    if (node) node[o] = nid;
    if (weight) weight[o] = w;
    if (rank) rank[o] = (w > 0) ? (nid == 0 ? 0 : 1 + __ldg(V.level_rank + nid)) : -1;
}

// FeatureVector build for a dense vocabulary (every node 0..nc-1 listed, possibly empty): CSR with
// ascending feature indices per node (FeatureVector.cpp:31-45).  One CTA per frame, thread per node.
__global__ void __launch_bounds__(128) k_build_csr(const int32_t* node, long long node_fs, const int* n_arr, int cap, int nc,
                                                    int* off, long long off_fs, int* idx, long long idx_fs) {
    __shared__ int s_warp[33];
    extern __shared__ int s_dyn[];        // nc + 1 counters, then the frame's node ids (cap ints)
    int* s_cnt = s_dyn; int* s_nd = s_dyn + nc + 1;
    const int f = blockIdx.x, tid = threadIdx.x;
    const int n = min(n_arr[f], cap);
    const int32_t* nd = node + f * node_fs;
    for (int c = tid; c <= nc; c += blockDim.x) s_cnt[c] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += blockDim.x) { const int v = nd[i]; s_nd[i] = v; if (v >= 0) atomicAdd(&s_cnt[v], 1); }   // v < 0: stopped word, not in the FeatureVector
    __syncthreads();
    block_scan_array(s_cnt, nc + 1, s_warp);                  // exclusive offsets, s_cnt[nc] = n
    for (int c = tid; c <= nc; c += blockDim.x) off[f * off_fs + c] = s_cnt[c];
    __syncthreads();
    // stable fill: thread c walks the node ids in index order (broadcast reads from shared memory)
    for (int c = tid; c < nc; c += blockDim.x) {
        int o = s_cnt[c];
        const int e = s_cnt[c + 1];
        for (int i = 0; i < n && o < e; i++) if (s_nd[i] == c) idx[f * idx_fs + o++] = i;
    }
}

// -------------------------------------------------------------------------------------------------
// SearchByBoW — one warp per (pair, node of set 1).  Nodes are independent (a feature belongs to exactly
// one node), the greedy exclusion inside a node is sequential over the KF features in list order.
//   mode 0: KF vs Frame  (ORBmatcher.cc:159-291): out = match2[F idx] = KF idx, accept best <= TH_LOW
//   mode 1: KF vs KF     (ORBmatcher.cc:525-658): out = match12[idx1] = idx2, accept best <  TH_LOW, both need MapPoints
// rot[i] holds the rotation-histogram bin of the match written at out[i] (or 255).
// -------------------------------------------------------------------------------------------------
__device__ __forceinline__ int rot_bin(float a1, float a2) {                 // ORBmatcher.cc:241-246
    float rot = __fsub_rn(a1, a2);
    if (rot < 0.0f) rot = __fadd_rn(rot, 360.0f);
    int bin = (int)roundf(__fmul_rn(rot, 1.0f / HISTO_LENGTH));
    if (bin == HISTO_LENGTH) bin = 0;
    return bin;
}

// ComputeThreeMaxima (ORBmatcher.cc:1604-1645) over a rotation histogram: the three kept bins, -1 for one it drops
__device__ __forceinline__ int3 three_maxima(const int* hist) {
    int max1 = 0, max2 = 0, max3 = 0, ind1 = -1, ind2 = -1, ind3 = -1;
    for (int i = 0; i < HISTO_LENGTH; i++) {
        const int s = hist[i];
        if (s > max1) { max3 = max2; max2 = max1; max1 = s; ind3 = ind2; ind2 = ind1; ind1 = i; }
        else if (s > max2) { max3 = max2; max2 = s; ind3 = ind2; ind2 = i; }
        else if (s > max3) { max3 = s; ind3 = i; }
    }
    if ((float)max2 < __fmul_rn(0.1f, (float)max1)) { ind2 = -1; ind3 = -1; }
    else if ((float)max3 < __fmul_rn(0.1f, (float)max1)) { ind3 = -1; }
    return make_int3(ind1, ind2, ind3);
}

__device__ __forceinline__ int find_node(const int* nodes, int nn, int id) {   // map::find on the ascending CSR node list
    int lo = 0, hi = nn;
    while (lo < hi) { int mid = (lo + hi) >> 1; if (nodes[mid] < id) lo = mid + 1; else hi = mid; }
    return (lo < nn && nodes[lo] == id) ? lo : -1;
}

// kMap (mode 0 only): pair p is the rows (S.pmap[p].x, S.pmap[p].y) of [0, S.nframes) for descriptors and angles, and the FeatureVector
// slots pslot[p] for the CSR; the keyframe row's MapPoints are kfmp[row][cap] element indices (outside [0, nmp): NULL) with isBad() flags
// mpbad[nmp] (NULL: none bad), which replace S.flag.  kMap = false compiles all of it out.
template <bool kMap>
__global__ void __launch_bounds__(128) k_bow_match(FrameSet S, int mode, float nnratio, int cap,
                                                    int32_t* out, long long out_fs, uint8_t* rot, long long rot_fs,
                                                    uint8_t* taken, long long taken_fs,
                                                    const int2* pslot, const int32_t* kfmp, const uint8_t* mpbad, int nmp) {
    const int pair = blockIdx.y, lane = threadIdx.x & 31, a = blockIdx.x * 4 + (threadIdx.x >> 5);
    int f1 = pair, f2 = pair + 1, s1 = f1, s2 = f2;                          // rows (descriptors, angles) and FeatureVector slots
    if (kMap) {
        if (!pair_frames(S.pmap, S.nframes, pair, f1, f2)) return;
        const int2 s = pslot[pair];
        s1 = s.x; s2 = s.y;
    }
    const int nn1 = S.nn ? S.nn[s1] : S.nn_const, nn2 = S.nn ? S.nn[s2] : S.nn_const;
    if (a >= nn1) return;
    const int* nodes1 = S.nodes + s1 * S.nodes_fs; const int* nodes2 = S.nodes + s2 * S.nodes_fs;
    const int b = find_node(nodes2, nn2, nodes1[a]);
    if (b < 0) return;
    const int* off1 = S.off + s1 * S.off_fs; const int* off2 = S.off + s2 * S.off_fs;
    const int* idx1 = S.idx + s1 * S.idx_fs; const int* idx2 = S.idx + s2 * S.idx_fs;
    const uint8_t* D1 = S.desc + f1 * S.desc_fs; const uint8_t* D2 = S.desc + f2 * S.desc_fs;
    const uint8_t* v1 = S.flag ? S.flag + f1 * S.flag_fs : nullptr;
    const uint8_t* v2 = S.flag ? S.flag + f2 * S.flag_fs : nullptr;
    const int32_t* mp1 = kMap ? kfmp + (long long)f1 * cap : nullptr;
    const float* A1 = S.angle + f1 * S.angle_fs; const float* A2 = S.angle + f2 * S.angle_fs;
    int32_t* O = out + pair * out_fs; uint8_t* R = rot + pair * rot_fs; uint8_t* TK = taken + pair * taken_fs;
    const int b1 = off1[a], e1 = off1[a + 1], b2 = off2[b], e2 = off2[b + 1];
    for (int i1 = b1; i1 < e1; i1++) {
        const int id1 = idx1[i1];
        if (kMap) {                                                              // :196-200
            const int e = mp1[id1];
            if ((unsigned)e >= (unsigned)nmp || (mpbad && mpbad[e])) continue;
        } else if (v1 && !v1[id1]) continue;                                     // :196-200 / :563-567
        uint4 a0, a1;
        load_desc(D1 + (long long)id1 * 32, a0, a1);
        // per-lane best / second best over this lane's candidates, in list order: key = dist << 20 | position
        unsigned k0 = 0xffffffffu, k1 = 0xffffffffu;
        for (int i2 = b2 + lane; i2 < e2; i2 += 32) {
            const int id2 = idx2[i2];
            if (TK[id2]) continue;                                               // :212 / :579 (already matched)
            if (mode == 1 && v2 && !v2[id2]) continue;                           // :579-583
            uint4 c0, c1;
            load_desc(D2 + (long long)id2 * 32, c0, c1);
            top2_insert(k0, k1, ((unsigned)popc256(a0, a1, c0, c1) << 20) | (unsigned)(i2 - b2));
        }
        top2_warp32(k0, k1);
        // bestDist1 = smallest distance (first position wins), bestDist2 = second order statistic; both start at 256
        const int best1 = k0 == 0xffffffffu ? 256 : (int)(k0 >> 20);
        const int best2 = k1 == 0xffffffffu ? 256 : (int)(k1 >> 20);
        const bool th = mode == 0 ? best1 <= TH_LOW : best1 < TH_LOW;             // :231 / :601
        if (k0 != 0xffffffffu && th && (float)best1 < __fmul_rn(nnratio, (float)best2)) {      // :233
            const int id2 = idx2[b2 + (int)(k0 & 0xfffff)];
            if (lane == 0) {
                TK[id2] = 1;
                const int bin = rot_bin(A1[(long long)id1 * S.angle_es], A2[(long long)id2 * S.angle_es]);
                if (mode == 0) { O[id2] = id1; R[id2] = (uint8_t)bin; }
                else { O[id1] = id2; R[id1] = (uint8_t)bin; }
            }
        }
        __syncwarp();
    }
}

// SearchForTriangulation (ORBmatcher.cc:660-826, monocular): warp per node of set 1; no dependency between
// idx1's (vbMatched2 is never set), so the lanes only cooperate on the scan of the node's idx2 list.
// F12 and the epipole of pair p are geom[11 p ..] (F row-major, ex, ey) when geom != NULL, else T's.  A KF2 feature whose octave is
// outside [0, nlevels) is never a candidate (mvScaleFactors / mvLevelSigma2 have no entry for it).  kMap = false (the single-pair
// call) compiles S.pmap and geom out.
struct TriArgs { float F[9]; float ex, ey; int nlevels; float scale[SSLPL_MAX_LEVELS]; float sigma2[SSLPL_MAX_LEVELS]; };

template <bool kMap>
__global__ void __launch_bounds__(128) k_tri_match(FrameSet S, TriArgs T, const float* geom, int32_t* out, long long out_fs, uint8_t* rot, long long rot_fs) {
    const int pair = blockIdx.y, lane = threadIdx.x & 31, a = blockIdx.x * 4 + (threadIdx.x >> 5);
    int f1, f2;
    if (!pair_frames(kMap ? S.pmap : nullptr, S.nframes, pair, f1, f2)) return;
    const int nn1 = S.nn ? S.nn[f1] : S.nn_const, nn2 = S.nn ? S.nn[f2] : S.nn_const;
    if (a >= nn1) return;
    const float* G = kMap ? geom : nullptr;
    float F[9], ex, ey;
#pragma unroll
    for (int k = 0; k < 9; k++) F[k] = G ? G[11LL * pair + k] : T.F[k];
    ex = G ? G[11LL * pair + 9] : T.ex; ey = G ? G[11LL * pair + 10] : T.ey;
    const int* nodes1 = S.nodes + f1 * S.nodes_fs; const int* nodes2 = S.nodes + f2 * S.nodes_fs;
    const int b = find_node(nodes2, nn2, nodes1[a]);
    if (b < 0) return;
    const int* off1 = S.off + f1 * S.off_fs; const int* off2 = S.off + f2 * S.off_fs;
    const int* idx1 = S.idx + f1 * S.idx_fs; const int* idx2 = S.idx + f2 * S.idx_fs;
    const uint8_t* D1 = S.desc + f1 * S.desc_fs; const uint8_t* D2 = S.desc + f2 * S.desc_fs;
    const uint8_t* m1 = S.flag + f1 * S.flag_fs; const uint8_t* m2 = S.flag + f2 * S.flag_fs;
    const long long es = S.angle_es;
    const float* A1 = S.angle + f1 * S.angle_fs; const float* A2 = S.angle + f2 * S.angle_fs;
    const float* X1 = S.x + f1 * S.angle_fs; const float* Y1 = S.y + f1 * S.angle_fs;
    const float* X2 = S.x + f2 * S.angle_fs; const float* Y2 = S.y + f2 * S.angle_fs;
    const int* OC2 = S.oct + f2 * S.angle_fs;
    const int b1 = off1[a], e1 = off1[a + 1], b2 = off2[b], e2 = off2[b + 1];
    for (int i1 = b1; i1 < e1; i1++) {
        const int id1 = idx1[i1];
        if (m1[id1]) continue;                                                    // :702-706
        uint4 a0, a1;
        load_desc(D1 + (long long)id1 * 32, a0, a1);
        const float x1 = X1[id1 * es], y1 = Y1[id1 * es];
        // epipolar line l = x1' F12 (CheckDistEpipolarLine :143-145), f32 without contraction
        const float la = __fadd_rn(__fadd_rn(__fmul_rn(x1, F[0]), __fmul_rn(y1, F[3])), F[6]);
        const float lb = __fadd_rn(__fadd_rn(__fmul_rn(x1, F[1]), __fmul_rn(y1, F[4])), F[7]);
        const float lc = __fadd_rn(__fadd_rn(__fmul_rn(x1, F[2]), __fmul_rn(y1, F[5])), F[8]);
        const float den = __fadd_rn(__fmul_rn(la, la), __fmul_rn(lb, lb));
        unsigned best = 0xffffffffu;              // min over (dist << 20 | (0xfffff - position)): min distance, LAST wins (:741)
        for (int i2 = b2 + lane; i2 < e2; i2 += 32) {
            const int id2 = idx2[i2];
            if (m2[id2]) continue;                                                // :725-729
            uint4 c0, c1;
            load_desc(D2 + (long long)id2 * 32, c0, c1);
            const int dist = popc256(a0, a1, c0, c1);
            if (dist > TH_LOW) continue;
            const float x2 = X2[id2 * es], y2 = Y2[id2 * es];
            const int oc = OC2[id2 * es];
            if ((unsigned)oc >= (unsigned)T.nlevels) continue;
            const float dex = __fsub_rn(ex, x2), dey = __fsub_rn(ey, y2);
            if (__fadd_rn(__fmul_rn(dex, dex), __fmul_rn(dey, dey)) < __fmul_rn(100.f, T.scale[oc])) continue;    // :749-751
            const float num = __fadd_rn(__fadd_rn(__fmul_rn(la, x2), __fmul_rn(lb, y2)), lc);
            if (den == 0.f) continue;
            const float dsqr = __fdiv_rn(__fmul_rn(num, num), den);
            if (!((double)dsqr < 3.84 * (double)T.sigma2[oc])) continue;          // :156 (double compare)
            const unsigned key = ((unsigned)dist << 20) | (0xfffffu - (unsigned)(i2 - b2));
            best = min(best, key);
        }
        best = __reduce_min_sync(0xffffffffu, best);
        if (best != 0xffffffffu && lane == 0) {
            const int id2 = idx2[b2 + (int)(0xfffffu - (best & 0xfffffu))];
            out[pair * out_fs + id1] = id2;
            rot[pair * rot_fs + id1] = (uint8_t)rot_bin(A1[id1 * es], A2[id2 * es]);
        }
    }
}

// -------------------------------------------------------------------------------------------------
// SURVEY.md 8(f) row 2: Frame::AssignFeaturesToGrid (Frame.cc:133-148, PosInGrid :462-472) as a CSR over the 64 x 48 cells
// (cell id = ix * 48 + iy: the traversal order of GetFeaturesInArea, Frame.cc:368-421) and
// ORBmatcher::SearchByProjection(Frame &CurrentFrame, const Frame &LastFrame, th, bMono) (ORBmatcher.cc:1331-1473).
// The matcher is a greedy scan over the last frame's MapPoints in index order (a feature of the current frame that has
// received a MapPoint with observations is skipped by later points), so ONE WARP walks a frame pair sequentially; the lanes
// share the grid cells of each search window.  First-wins ties are kept by reducing (distance, traversal position) keys.
// The batched form walks many consecutive pairs at once, one warp (CTA) per pair, with the same kernel.
// -------------------------------------------------------------------------------------------------
constexpr int GRID_COLS = 64, GRID_ROWS = 48;        // Frame.h:45-46
constexpr int TH_HIGH = 100;                         // ORBmatcher.cc:37

// The image bounds (mnMinX, mnMaxX, mnMinY, mnMaxY), the inverse grid cell size and mvScaleFactors of a frame
struct GridGeom { float minX, maxX, minY, maxY, invW, invH; float scale[32]; };

// G from bounds = (minX, maxX, minY, maxY) and scaleFactors[nlevels] (NULL with nlevels = 0: no scale table; the caller bounds nlevels
// by 32).  Degenerate bounds would give an infinite or negative cell size: SSLPL_ERR_ARG.
static int grid_geom(GridGeom& G, const float* bounds, const float* scaleFactors, int nlevels) {
    SSLPL_REQUIRE(bounds[1] > bounds[0] && bounds[3] > bounds[2], SSLPL_ERR_ARG, "degenerate image bounds");
    G = GridGeom{};
    G.minX = bounds[0]; G.maxX = bounds[1]; G.minY = bounds[2]; G.maxY = bounds[3];
    G.invW = (float)GRID_COLS / (bounds[1] - bounds[0]); G.invH = (float)GRID_ROWS / (bounds[3] - bounds[2]);   // Frame.cc:115-116
    for (int k = 0; k < nlevels; k++) G.scale[k] = scaleFactors[k];
    return SSLPL_OK;
}

struct ProjArgs {
    float T[12];                                     // Tcw, 3x4 row-major (when ProjPair::Tcw is NULL)
    float fx, fy, cx, cy, mbf;
    GridGeom G;
    float th;
    int forward, backward, checkOri, use_right;
    int nlevels;                                     // a last-frame point whose octave is outside [0, nlevels) is skipped
    int retry_below;                                 // a pair with fewer matches reruns with 2 * th (Tracking.cc:1240-1244); <= 0: never
};

// Where the walker of pair p reads and writes: the last frame at the *1 pointers + p * (their frame stride), the current frame at
// the *2 pointers + p * (theirs), the per-pair tables at + p * ws_fs.  Keypoint fields are read with an element stride (1: separate
// arrays, 7: fields of sslpl_keypoint).  The single-pair entry point runs pair 0 only.
struct ProjPair {
    const int* n; int n1, n2, cap;                   // n != NULL: counts n[p] (last) and n[p + 1] (current), clamped to cap; else n1, n2
    const float* Tcw;                                // pose of pair p at Tcw + 12 p; NULL = ProjArgs::T
    const uint8_t* flag1;                            // bit0 = MapPoint && !outlier, bit1 = Observations() > 0
    const float* Xw; const uint8_t* dmp; const float* angle1; const int* oct1;
    long long flag1_fs, xw_fs, dmp_fs, kp1_fs; int es1;
    const uint8_t* d2; const float* x2; const float* y2; const float* angle2; const int* oct2; const float* uright2;
    long long d2_fs, kp2_fs; int es2;
    const uint8_t* claimed0;                         // current features holding a MapPoint with observations on entry (NULL = none)
    const int* goff; const int* gidx; long long goff_fs, gidx_fs;     // 64 x 48 grid CSR of the current frame
    uint8_t* claimed; int32_t* assign2; int32_t* sel; uint8_t* rbin; long long ws_fs;
    int32_t* nmatch;                                 // nmatch[p]
};

// Frame::AssignFeaturesToGrid's cell of every feature (PosInGrid, Frame.cc:462-472): frame f = blockIdx.y, fields at element stride es
__global__ void __launch_bounds__(128) k_grid_cells(const float* x, const float* y, int es, long long fs, const int* n_arr, int n_const, int cap,
                                                    const __grid_constant__ GridGeom G, int32_t* cell, long long cell_fs) {
    const int f = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = n_arr ? min(n_arr[f], cap) : n_const;
    if (i >= n) return;
    const long long e = f * fs + (long long)i * es;
    const int px = (int)roundf(__fmul_rn(__fsub_rn(x[e], G.minX), G.invW)), py = (int)roundf(__fmul_rn(__fsub_rn(y[e], G.minY), G.invH));
    cell[f * cell_fs + i] = (px < 0 || px >= GRID_COLS || py < 0 || py >= GRID_ROWS) ? -1 : px * GRID_ROWS + py;
}

// The cells of Frame::GetFeaturesInArea(x, y, r) (Frame.cc:375-393) on the grid of k_grid_cells, in its traversal order: cell rank
// c = 0 .. ncell - 1 is cell (cx0 + c / ny, cy0 + c % ny).
struct GridWin { int cx0, cy0, ny, ncell; };

// false when the window misses the grid
__device__ __forceinline__ bool grid_window(const GridGeom& G, float x, float y, float r, GridWin& w) {
    const int cx0 = max(0, (int)floorf(__fmul_rn(__fsub_rn(__fsub_rn(x, G.minX), r), G.invW)));
    if (cx0 >= GRID_COLS) return false;
    const int cx1 = min(GRID_COLS - 1, (int)ceilf(__fmul_rn(__fadd_rn(__fsub_rn(x, G.minX), r), G.invW)));
    if (cx1 < 0) return false;
    const int cy0 = max(0, (int)floorf(__fmul_rn(__fsub_rn(__fsub_rn(y, G.minY), r), G.invH)));
    if (cy0 >= GRID_ROWS) return false;
    const int cy1 = min(GRID_ROWS - 1, (int)ceilf(__fmul_rn(__fadd_rn(__fsub_rn(y, G.minY), r), G.invH)));
    if (cy1 < 0) return false;
    w.cx0 = cx0; w.cy0 = cy0; w.ny = cy1 - cy0 + 1; w.ncell = (cx1 - cx0 + 1) * w.ny;
    return true;
}

// The candidates of window w, lane by lane: lane l walks the cells of rank l, l + 32, ... and passes each feature j of the grid CSR
// to cand(j, dist), which applies the caller's filters and returns false to skip j, or sets dist to the descriptor distance and returns
// true.  take() gets the key (dist << 40) | (cell rank << 20) | position in the cell: ascending keys are ascending distances in
// GetFeaturesInArea's order, so the smallest key is the reference's first strict minimum and the two smallest are its best /
// second-best pair.  (A bool rather than a sentinel distance: each filter then branches straight to the next feature; with a
// sentinel, k_point_fuse_search<true> needs 3 more registers.)
template <class Cand, class Take>
__device__ __forceinline__ void grid_scan(const int* goff, const int* gidx, const GridWin& w, int lane, Cand cand, Take take) {
    for (int c = lane; c < w.ncell; c += 32) {
        const int cell = (w.cx0 + c / w.ny) * GRID_ROWS + w.cy0 + c % w.ny;
        const int b = goff[cell], e = goff[cell + 1];
        for (int q = b; q < e; q++) {
            int d;
            if (cand(gidx[q], d)) take(((unsigned long long)d << 40) | ((unsigned long long)c << 20) | (unsigned)(q - b));
        }
    }
}
// the smallest key of the window, in every lane (~0 when no candidate)
template <class Cand>
__device__ __forceinline__ unsigned long long grid_min(const int* goff, const int* gidx, const GridWin& w, int lane, Cand cand) {
    unsigned long long best = ~0ull;
    grid_scan(goff, gidx, w, lane, cand, [&](unsigned long long k) { if (k < best) best = k; });
    return warp_min(best);
}
// the two smallest keys of the window, in every lane (~0 for a missing one)
template <class Cand>
__device__ __forceinline__ void grid_top2(const int* goff, const int* gidx, const GridWin& w, int lane, Cand cand,
                                          unsigned long long& b1, unsigned long long& b2) {
    b1 = ~0ull; b2 = ~0ull;
    grid_scan(goff, gidx, w, lane, cand, [&](unsigned long long k) { top2_push(b1, b2, k); });
    top2_warp(b1, b2);
}
// the feature of a window key
__device__ __forceinline__ int grid_key_feature(const int* goff, const int* gidx, const GridWin& w, unsigned long long key) {
    const int c = (int)((key >> 20) & 0xfffff), pos = (int)(key & 0xfffff);
    return gidx[goff[(w.cx0 + c / w.ny) * GRID_ROWS + w.cy0 + c % w.ny] + pos];
}

// The rotation check of the one-warp walkers (ComputeThreeMaxima, ORBmatcher.cc:1604-1645, over the histogram s_hist) on matches
// [0, n): bin(i) is the rotation bin of match i, or -1 when i has none; drop(i) removes a match outside the three kept bins.  Returns
// the number removed, in every lane.
template <class Bin, class Drop>
__device__ __forceinline__ int warp_rot_check(const int* s_hist, int n, int lane, Bin bin, Drop drop) {
    __shared__ int s_keep[3];
    if (lane == 0) { const int3 k = three_maxima(s_hist); s_keep[0] = k.x; s_keep[1] = k.y; s_keep[2] = k.z; }
    __syncwarp();
    const int k0 = s_keep[0], k1 = s_keep[1], k2 = s_keep[2];
    int ndrop = 0;
    for (int i0 = 0; i0 < n; i0 += 32) {
        const int i = i0 + lane;
        const int b = i < n ? bin(i) : -1;
        const bool d = b >= 0 && b != k0 && b != k1 && b != k2;
        if (d) drop(i);
        ndrop += __popc(__ballot_sync(0xffffffffu, d));
    }
    return ndrop;
}

// Rcw * x + tcw of a pose (Tcw 3x4 row-major): cv::gemm runs a plain 3x3 * 3x1 (+ 3x1) CV_32F product in FLOAT, products summed left
// to right, the addend last (probed on cv2 4.13, tools/probe_cv_gemm.py; the reference compiled over that model agrees with the oracle
// in tests/test_ref_parity_cpu.py).  Explicit _rn intrinsics: no FMA contraction.
__device__ __forceinline__ float rt_row(const float* T, float x0, float x1, float x2) {
    return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[0], x0), __fmul_rn(T[1], x1)), __fmul_rn(T[2], x2)), T[3]);
}

// One warp per frame pair (blockIdx.x); see ProjPair for the layout.
__global__ void __launch_bounds__(32) k_proj_match(const __grid_constant__ ProjArgs A, const __grid_constant__ ProjPair P) {
    __shared__ int s_hist[HISTO_LENGTH];
    __shared__ float s_T[12];
    const int lane = threadIdx.x, p = blockIdx.x;
    const int n1 = P.n ? min(P.n[p], P.cap) : P.n1, n2 = P.n ? min(P.n[p + 1], P.cap) : P.n2;
    const uint8_t* flag1 = P.flag1 + p * P.flag1_fs;
    const float* Xw = P.Xw + p * P.xw_fs; const uint8_t* dmp = P.dmp + p * P.dmp_fs;
    const float* angle1 = P.angle1 + p * P.kp1_fs; const int* oct1 = P.oct1 + p * P.kp1_fs;
    const long long es1 = P.es1, es2 = P.es2;
    const uint8_t* d2 = P.d2 + p * P.d2_fs;
    const float* x2 = P.x2 + p * P.kp2_fs; const float* y2 = P.y2 + p * P.kp2_fs; const float* angle2 = P.angle2 + p * P.kp2_fs;
    const int* oct2 = P.oct2 + p * P.kp2_fs; const float* uright2 = P.uright2;      // stereo: single pair only
    const int* goff = P.goff + p * P.goff_fs; const int* gidx = P.gidx + p * P.gidx_fs;
    uint8_t* claimed = P.claimed + p * P.ws_fs; int32_t* assign2 = P.assign2 + p * P.ws_fs;
    int32_t* sel = P.sel + p * P.ws_fs; uint8_t* rbin = P.rbin + p * P.ws_fs;
    if (lane < 12) s_T[lane] = P.Tcw ? P.Tcw[12LL * p + lane] : A.T[lane];
    const int nout = P.n ? P.cap : n2;                           // the batched table is written whole
    int nmatches = 0;
    for (int pass = 0;; pass++) {
        // TrackWithMotionModel NULLs mvpMapPoints before each SearchByProjection (Tracking.cc:1219, 1242): assignments and claims restart
        const float th = pass == 0 ? A.th : __fmul_rn(2.0f, A.th);
        for (int j = lane; j < nout; j += 32) assign2[j] = -1;
        for (int j = lane; j < n2; j += 32) claimed[j] = P.claimed0 ? P.claimed0[j] : 0;
        if (lane < HISTO_LENGTH) s_hist[lane] = 0;
        __syncwarp();
        nmatches = 0;
        for (int i = 0; i < n1; i++) {
            if (lane == 0) sel[i] = -1;
            const int fl = flag1[i];
            if (!(fl & 1)) continue;
            const float X0 = Xw[3 * i], X1 = Xw[3 * i + 1], X2 = Xw[3 * i + 2];
            const float xc = rt_row(s_T, X0, X1, X2), yc = rt_row(s_T + 4, X0, X1, X2), zc = rt_row(s_T + 8, X0, X1, X2);   // :1364
            const float invzc = (float)(1.0 / (double)zc);
            if (invzc < 0) continue;
            const float u = __fadd_rn(__fmul_rn(__fmul_rn(A.fx, xc), invzc), A.cx), v = __fadd_rn(__fmul_rn(__fmul_rn(A.fy, yc), invzc), A.cy);
            if (u < A.G.minX || u > A.G.maxX || v < A.G.minY || v > A.G.maxY) continue;
            const int lo = oct1[i * es1];
            if ((unsigned)lo >= (unsigned)A.nlevels) continue;        // outside mvScaleFactors: never read scale[] out of range
            const float r = __fmul_rn(th, A.G.scale[lo]);
            const int minLevel = A.forward ? lo : (A.backward ? 0 : lo - 1), maxLevel = A.forward ? -1 : (A.backward ? lo : lo + 1);
            GridWin w;                                               // GetFeaturesInArea (Frame.cc:368-421)
            if (!grid_window(A.G, u, v, r, w)) continue;
            const bool checkLevels = (minLevel > 0) || (maxLevel >= 0);
            uint4 a0, a1;
            load_desc(dmp + (long long)i * 32, a0, a1);
            const float ur = __fsub_rn(u, __fmul_rn(A.mbf, invzc));
            // captured by value: by reference, ptxas spills at this kernel's 64 registers
            const unsigned long long best = grid_min(goff, gidx, w, lane, [=](int j, int& d) {
                if (checkLevels) {
                    const int o = oct2[j * es2];
                    if (o < minLevel) return false;
                    if (maxLevel >= 0 && o > maxLevel) return false;
                }
                if (!(fabsf(__fsub_rn(x2[j * es2], u)) < r && fabsf(__fsub_rn(y2[j * es2], v)) < r)) return false;
                if (claimed[j]) return false;                           // :1400-1402
                if (A.use_right && uright2[j * es2] > 0) { if (fabsf(__fsub_rn(ur, uright2[j * es2])) > r) return false; }
                uint4 b0, b1;
                load_desc(d2 + (long long)j * 32, b0, b1);
                d = popc256(a0, a1, b0, b1);
                return true;
            });
            const int bestDist = best == ~0ull ? 256 : (int)(best >> 40);
            if (bestDist <= TH_HIGH) {
                const int j = grid_key_feature(goff, gidx, w, best);
                if (lane == 0) {
                    assign2[j] = i; claimed[j] = (fl >> 1) & 1;
                    sel[i] = j;
                    const int bin = rot_bin(angle1[i * es1], angle2[j * es2]);
                    rbin[i] = (uint8_t)bin;
                    if (A.checkOri) s_hist[bin]++;
                }
                nmatches++;
            }
            __syncwarp();
        }
        __syncwarp();
        if (A.checkOri)                                              // assigned, then removed: the reference NULLs it explicitly (:1461)
            nmatches -= warp_rot_check(s_hist, n1, lane, [&](int i) { return sel[i] >= 0 ? (int)rbin[i] : -1; },
                                       [&](int i) { assign2[sel[i]] = -2; });
        if (pass > 0 || nmatches >= A.retry_below) break;
        __syncwarp();                                                // the rotation check's writes land before the next pass resets
    }
    if (lane == 0) P.nmatch[p] = nmatches;
}

// -------------------------------------------------------------------------------------------------
// ORBmatcher::SearchByProjection(Frame &F, const vector<MapPoint*> &vpMapPoints, th) — ORBmatcher.cc:45-129 (Tracking::SearchLocalPoints,
// every frame) and ORBmatcher::SearchForInitialization — ORBmatcher.cc:408-523.  Both are greedy scans whose later iterations see
// what earlier ones wrote (a feature that received a MapPoint with observations is skipped; a feature matched at distance d only
// yields to a strictly smaller distance), so, like k_proj_match, ONE WARP walks the list in order and its lanes share the grid
// cells of each search window.  The reference's sequential best / second-best update keeps the two smallest candidates in
// (distance, traversal position) order: that is what the two-key reduction below computes.
// -------------------------------------------------------------------------------------------------
constexpr int TH_LOW_I = 50;                        // ORBmatcher.cc:38
struct WinArgs { GridGeom G; float th, nnratio; int bFactor, use_right, checkOri, window; };

__global__ void __launch_bounds__(32) k_proj_match_mps(const __grid_constant__ WinArgs A, int nmp, const uint8_t* flag /* bit0 in view && !bad, bit1 obs>0 */,
                                                        const float* px, const float* py, const float* pxr, const int* level, const float* viewcos, const uint8_t* dmp,
                                                        int n2, const uint8_t* d2, const float* x2, const float* y2, const int* oct2, const float* uright2,
                                                        uint8_t* claimed, const int* goff, const int* gidx, int32_t* assign2, int32_t* nmatch) {
    const int lane = threadIdx.x;
    for (int j = lane; j < n2; j += 32) assign2[j] = -1;
    __syncwarp();
    int nmatches = 0;
    for (int i = 0; i < nmp; i++) {
        const int fl = flag[i];
        if (!(fl & 1)) continue;                                  // !mbTrackInView || isBad() (:54-58)
        const int lvl = level[i];
        float r = (double)viewcos[i] > 0.998 ? 2.5f : 4.0f;       // RadiusByViewingCos (:131-137)
        if (A.bFactor) r = __fmul_rn(r, A.th);
        const float rad = __fmul_rn(r, A.G.scale[lvl]);
        const float u = px[i], v = py[i];
        GridWin w;
        if (!grid_window(A.G, u, v, rad, w)) continue;
        const int minLevel = lvl - 1, maxLevel = lvl;            // GetFeaturesInArea(..., nPredictedLevel-1, nPredictedLevel)
        const bool checkLevels = (minLevel > 0) || (maxLevel >= 0);
        uint4 a0, a1;
        load_desc(dmp + (long long)i * 32, a0, a1);
        unsigned long long b1, b2;
        grid_top2(goff, gidx, w, lane, [&](int j, int& d) {
            if (checkLevels) { const int o = oct2[j]; if (o < minLevel) return false; if (maxLevel >= 0 && o > maxLevel) return false; }
            if (!(fabsf(__fsub_rn(x2[j], u)) < rad && fabsf(__fsub_rn(y2[j], v)) < rad)) return false;
            if (claimed[j]) return false;                            // holds a MapPoint with observations (:86-88)
            if (A.use_right && uright2[j] > 0) { if (fabsf(__fsub_rn(pxr[i], uright2[j])) > rad) return false; }
            uint4 c0, c1;
            load_desc(d2 + (long long)j * 32, c0, c1);
            d = popc256(a0, a1, c0, c1);
            return d < 256;                                       // never below the initial bestDist = bestDist2 = 256
        }, b1, b2);
        if (b1 == ~0ull) continue;
        const int bestDist = (int)(b1 >> 40);
        if (bestDist <= TH_HIGH) {
            const int j = grid_key_feature(goff, gidx, w, b1);
            int bestDist2 = 256, bestLevel2 = -1;
            if (b2 != ~0ull) { bestDist2 = (int)(b2 >> 40); bestLevel2 = oct2[grid_key_feature(goff, gidx, w, b2)]; }
            if (oct2[j] == bestLevel2 && (float)bestDist > __fmul_rn(A.nnratio, (float)bestDist2)) continue;   // :117
            if (lane == 0) { assign2[j] = i; claimed[j] = (fl >> 1) & 1; }
            nmatches++;
        }
        __syncwarp();
    }
    if (lane == 0) *nmatch = nmatches;
}

// ---------------- SURVEY.md 8(f) row 3: line projection search, Fuse search ----------------
// Frame::GetLinesInArea (Frame.cc:423-460) = KeyFrame::GetLinesInArea (KeyFrame.cc:651-684) for one frame line: the mid-point test is
// evaluated in double and narrowed (as the mixed float/double expression of the reference is), without FMA contraction.
struct LineWin { double mx, my; float r2, r, slope; double rs; int minLevel, maxLevel; bool checkLevels; };
__device__ __forceinline__ LineWin line_win(float x1, float y1, float x2, float y2, float r, int minLevel, int maxLevel) {
    LineWin w;
    w.mx = __dmul_rn(0.5, (double)__fadd_rn(x1, x2)); w.my = __dmul_rn(0.5, (double)__fadd_rn(y1, y2));
    w.r = r; w.r2 = __fmul_rn(r, r);
    w.slope = __fdiv_rn(__fsub_rn(y1, y2), __fsub_rn(x1, x2));
    w.rs = __dmul_rn((double)r, 0.01);
    w.minLevel = minLevel; w.maxLevel = maxLevel; w.checkLevels = (minLevel > 0) || (maxLevel > 0);
    return w;
}
__device__ __forceinline__ bool line_in_area(const LineWin& w, float ptx, float pty, float angle, int octave) {
    const double dx = __dsub_rn(w.mx, (double)ptx), dy = __dsub_rn(w.my, (double)pty);
    const float distance = __double2float_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
    if (distance > w.r2) return false;
    const float slope = __fsub_rn(w.slope, angle);
    if ((double)slope > w.rs) return false;
    if (w.checkLevels) {
        if (octave < w.minLevel) return false;
        if (w.maxLevel >= 0 && octave > w.maxLevel) return false;
    }
    return true;
}

// Search stage of both LSDmatcher::SearchByProjection overloads (LSDmatcher.cpp:98-137 = :210-251).  The MapLines are visited in
// vector order by ONE warp, because a frame line taken by a MapLine with observations is skipped by the later ones (:104-106);
// the lanes share the scan over the frame's lines.  keys: (distance << 32) | line index = the scan order of the reference.
__global__ void __launch_bounds__(32) k_line_window_search(int nml, const uint8_t* flag /* bit0 active, bit1 obs>0 */, const float4* proj, const float* radius,
                                                            const int* minLevel, const int* maxLevel, const uint8_t* dml,
                                                            int nl2, const uint8_t* ld2, const float* kl2, const int* oct2, uint8_t* claimed,
                                                            float nnratio, int32_t* assign2, int32_t* nmatch) {
    const int lane = threadIdx.x;
    for (int j = lane; j < nl2; j += 32) assign2[j] = -1;
    __syncwarp();
    int nmatches = 0;
    for (int i = 0; i < nml; i++) {
        const int fl = flag[i];
        if (!(fl & 1)) continue;
        const float4 p = proj[i];
        const LineWin w = line_win(p.x, p.y, p.z, p.w, radius[i], minLevel[i], maxLevel[i]);
        uint4 a0, a1;
        load_desc(dml + (long long)i * 32, a0, a1);
        unsigned long long b1 = ~0ull, b2 = ~0ull;
        for (int j = lane; j < nl2; j += 32) {
            if (!line_in_area(w, kl2[3 * j], kl2[3 * j + 1], kl2[3 * j + 2], oct2[j])) continue;
            if (claimed[j]) continue;
            uint4 c0, c1;
            load_desc(ld2 + (long long)j * 32, c0, c1);
            const int dist = popc256(a0, a1, c0, c1);
            if (dist >= 256) continue;                            // never below the initial bestDist = bestDist2 = 256
            top2_push(b1, b2, ((unsigned long long)dist << 32) | (unsigned)j);
        }
        top2_warp(b1, b2);
        if (b1 == ~0ull) continue;
        const int bestDist = (int)(b1 >> 32);
        if (bestDist <= TH_HIGH) {
            const int j = (int)(b1 & 0xffffffffu);
            int bestDist2 = 256, bestLevel2 = -1;
            if (b2 != ~0ull) { bestDist2 = (int)(b2 >> 32); bestLevel2 = oct2[(int)(b2 & 0xffffffffu)]; }
            if (oct2[j] == bestLevel2 && (float)bestDist > __fmul_rn(nnratio, (float)bestDist2)) continue;
            if (lane == 0) { assign2[j] = i; claimed[j] = (fl >> 1) & 1; }
            nmatches++;
        }
        __syncwarp();
    }
    if (lane == 0) *nmatch = nmatches;
}

// -------------------------------------------------------------------------------------------------
// MapPoint::PredictScale / MapLine::PredictScale (MapPoint.cc:390-405, MapLine.cpp:386-395): (int)ceil(logf(ratio) / logScaleFactor).
// The level is a monotone step function of the float ratio, so the host finds, with its own logf, the smallest positive float t_k
// whose level is >= k for k = 0 .. nlevels (sslpl_predict_scale_table) and the device counts the thresholds <= ratio: the same levels
// as the host's libm by construction.  A ratio that is not finite and positive (NaN, +-inf, <= 0) has logf = NaN or -inf, which
// x86-64 converts to INT_MIN: clamped to level 0 (points), outside the pyramid (lines).
// clamp: [0, nlevels - 1];  !clamp: INT_MIN as above, else -1 for any level below 0, nlevels for any level >= nlevels.
// -------------------------------------------------------------------------------------------------
struct PredictTable { float thr[SSLPL_MAX_LEVELS + 1]; int nlevels; };

__device__ __forceinline__ int predict_scale(float ratio, const float* thr, int nlevels, bool clamp) {
    int c = 0;
    for (int k = 0; k <= nlevels; k++) c += thr[k] <= ratio;
    if (!(ratio > 0.f && ratio < INFINITY)) return clamp ? 0 : INT_MIN;
    return clamp ? min(max(c - 1, 0), nlevels - 1) : c - 1;
}

__global__ void k_predict_scale(int n, const float* ratio, const __grid_constant__ PredictTable T, int clamp, int32_t* level) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) level[i] = predict_scale(ratio[i], T.thr, T.nlevels, clamp != 0);
}

// Mat::dot of two float rows of 3 (double products and sum; the reference's sum starts from 0.0, which changes only the sign of an
// exact zero, and no caller reads that sign), cv::norm (double accumulation, the double it returns) and (float)cv::norm(d), and the
// double dot product with the normal of the viewing-angle gate
__device__ __forceinline__ double dot3d(float a0, float a1, float a2, float b0, float b1, float b2) {
    return __dadd_rn(__dadd_rn(__dmul_rn((double)a0, (double)b0), __dmul_rn((double)a1, (double)b1)), __dmul_rn((double)a2, (double)b2));
}
__device__ __forceinline__ double norm3d_d(float d0, float d1, float d2) { return __dsqrt_rn(dot3d(d0, d1, d2, d0, d1, d2)); }
__device__ __forceinline__ float norm3d(float d0, float d1, float d2) { return __double2float_rn(norm3d_d(d0, d1, d2)); }
__device__ __forceinline__ bool view_ok(float d0, float d1, float d2, float n0, float n1, float n2, float dist) {
    return !(dot3d(d0, d1, d2, n0, n1, n2) < __dmul_rn(0.5, (double)dist));
}

// Where the batched Fuse calls read: entry e = (keyframe, element) pair, the keyframe set (strides in elements of its arrays), the
// element table and the keyframe poses pose[k][15] = Tcw (3x4 row-major), Ow.  Unused (zero) in the single-call instances.
struct FuseMap {
    const int2* entry; const uint8_t* skip; int nkf, nel;
    const float* kp; long long kp_fs; const uint8_t* desc; long long desc_fs; const int* n; int cap;
    const float* pose; const float* el; const uint8_t* eldesc;
    const int* goff; const int* gidx; long long goff_fs, gidx_fs;      // points: the 64 x 48 grid CSR of every keyframe
    float fx, fy, cx, cy;
    GridGeom G;
    PredictTable T;
    float invSigma2[SSLPL_MAX_LEVELS];
};

// entry e of a batched call: false (and (-1, -1) written) when its keyframe or element index is out of range
__device__ __forceinline__ bool fuse_entry(const FuseMap& M, int e, int lane, int& k, int& p, int32_t* best_idx, int32_t* best_dist) {
    const int2 q = M.entry[e];
    k = q.x; p = q.y;
    if ((unsigned)k < (unsigned)M.nkf && p >= -1 && p < M.nel) return true;
    if (lane == 0) { best_idx[e] = -1; best_dist[e] = -1; }
    return false;
}

// Projection stage of ORBmatcher::Fuse (ORBmatcher.cc:828-894) for MapPoint p in keyframe k, with the reference's operation order.
// el[p][9] = Xw, normal, minInv, maxInv, maxRaw.
__device__ __forceinline__ bool fuse_project_point(const FuseMap& M, int k, int p, float& u, float& v, int& lvl) {
    const float* T = M.pose + 15LL * k;
    const float* P = M.el + 9LL * p;
    const float X0 = P[0], X1 = P[1], X2 = P[2];
    const float zc = rt_row(T + 8, X0, X1, X2);
    if (zc < 0.0f) return false;
    const float invz = __fdiv_rn(1.0f, zc);
    u = __fadd_rn(__fmul_rn(M.fx, __fmul_rn(rt_row(T, X0, X1, X2), invz)), M.cx);
    v = __fadd_rn(__fmul_rn(M.fy, __fmul_rn(rt_row(T + 4, X0, X1, X2), invz)), M.cy);
    if (!(u >= M.G.minX && u < M.G.maxX && v >= M.G.minY && v < M.G.maxY)) return false;     // KeyFrame::IsInImage KeyFrame.cc:686-689
    const float d0 = __fsub_rn(X0, T[12]), d1 = __fsub_rn(X1, T[13]), d2 = __fsub_rn(X2, T[14]);
    const float dist = norm3d(d0, d1, d2);
    if (dist < P[6] || dist > P[7]) return false;
    if (!view_ok(d0, d1, d2, P[3], P[4], P[5], dist)) return false;
    lvl = predict_scale(__fdiv_rn(P[8], dist), M.T.thr, M.T.nlevels, true);
    return true;
}

// Projection stage of LSDmatcher::Fuse (LSDmatcher.cpp:417-497) for MapLine p in keyframe k, with the reference's operation order.
// el[p][12] = SP, EP, normal, minInv, maxInv, maxRaw.  A level outside the pyramid drops the line.
__device__ __forceinline__ bool fuse_project_line(const FuseMap& M, int k, int p, float4& q, int& lvl) {
    const float* T = M.pose + 15LL * k;
    const float* L = M.el + 12LL * p;
    const float s0 = L[0], s1 = L[1], s2 = L[2], e0 = L[3], e1 = L[4], e2 = L[5];
    const float sz = rt_row(T + 8, s0, s1, s2), ez = rt_row(T + 8, e0, e1, e2);
    if (sz < 0.0f || ez < 0.0f) return false;
    const float iz1 = __fdiv_rn(1.0f, sz), iz2 = __fdiv_rn(1.0f, ez);
    q.x = __fadd_rn(__fmul_rn(__fmul_rn(M.fx, rt_row(T, s0, s1, s2)), iz1), M.cx);
    q.y = __fadd_rn(__fmul_rn(__fmul_rn(M.fy, rt_row(T + 4, s0, s1, s2)), iz1), M.cy);
    if (q.x < M.G.minX || q.x > M.G.maxX || q.y < M.G.minY || q.y > M.G.maxY) return false;
    q.z = __fadd_rn(__fmul_rn(__fmul_rn(M.fx, rt_row(T, e0, e1, e2)), iz2), M.cx);
    q.w = __fadd_rn(__fmul_rn(__fmul_rn(M.fy, rt_row(T + 4, e0, e1, e2)), iz2), M.cy);
    if (q.z < M.G.minX || q.z > M.G.maxX || q.w < M.G.minY || q.w > M.G.maxY) return false;
    const float d0 = __fsub_rn(__fmul_rn(0.5f, __fadd_rn(s0, e0)), T[12]), d1 = __fsub_rn(__fmul_rn(0.5f, __fadd_rn(s1, e1)), T[13]),
                d2 = __fsub_rn(__fmul_rn(0.5f, __fadd_rn(s2, e2)), T[14]);
    const float dist = norm3d(d0, d1, d2);
    if (dist < L[9] || dist > L[10]) return false;
    if (!view_ok(d0, d1, d2, L[6], L[7], L[8], dist)) return false;
    lvl = predict_scale(__fdiv_rn(L[11], dist), M.T.thr, M.T.nlevels, false);
    return lvl >= 0 && lvl < M.T.nlevels;
}

// Search stage of LSDmatcher::Fuse (LSDmatcher.cpp:499-523): independent per MapLine, one warp each.  kMap: warp i runs entry i of a
// batched call (fuse_project_line, then the same search over keyframe k's sslpl_keyline rows); false compiles the map out.
template <bool kMap>
__global__ void __launch_bounds__(128) k_line_fuse_search(int nml, const uint8_t* active, const float4* proj, const int* level, const uint8_t* dml,
                                                           int nl2, const uint8_t* ld2, const float* kl2, const int* oct2, const float* scale, float th,
                                                           int32_t* best_idx, int32_t* best_dist, const __grid_constant__ FuseMap M) {
    const int i = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (i >= nml) return;
    // keyline fields: (pt.x, pt.y, angle) rows and a separate octave array, or sslpl_keyline (angle, class_id, octave, pt_x, pt_y, ...)
    constexpr int es = kMap ? 17 : 3, ox = kMap ? 3 : 0, oy = kMap ? 4 : 1, oa = kMap ? 0 : 2, oes = kMap ? 17 : 1;
    unsigned long long b = ~0ull;
    bool act;
    int lvl;
    float4 p;
    if (kMap) {
        int k, e;
        if (!fuse_entry(M, i, lane, k, e, best_idx, best_dist)) return;
        act = e >= 0 && !(M.skip && M.skip[i]) && fuse_project_line(M, k, e, p, lvl);
        nl2 = min(M.n[k], M.cap); ld2 = M.desc + k * M.desc_fs; kl2 = M.kp + k * M.kp_fs;
        oct2 = reinterpret_cast<const int*>(kl2 + 2); scale = M.G.scale; dml = M.eldesc + (long long)e * 32;
    } else {
        act = active[i];
        dml += (long long)i * 32;
    }
    if (act) {
        if (!kMap) { lvl = level[i]; p = proj[i]; }
        const LineWin w = line_win(p.x, p.y, p.z, p.w, __fmul_rn(th, scale[lvl]), -1, -1);
        uint4 a0, a1;
        load_desc(dml, a0, a1);
        for (int j = lane; j < nl2; j += 32) {
            const int o = oct2[oes * j];
            if (!line_in_area(w, kl2[es * j + ox], kl2[es * j + oy], kl2[es * j + oa], o)) continue;
            if (o < lvl - 1 || o > lvl) continue;
            uint4 c0, c1;
            load_desc(ld2 + (long long)j * 32, c0, c1);
            const unsigned long long k = ((unsigned long long)popc256(a0, a1, c0, c1) << 32) | (unsigned)j;
            b = k < b ? k : b;
        }
        b = warp_min(b);
    }
    if (lane == 0) { best_idx[i] = b == ~0ull ? -1 : (int)(b & 0xffffffffu); best_dist[i] = b == ~0ull ? 0x7fffffff : (int)(b >> 32); }
}

// Search stage of ORBmatcher::Fuse (ORBmatcher.cc:896-950): independent per MapPoint, one warp each over the grid cells of the window.
// kMap: warp i runs entry i of a batched call (fuse_project_point, then the same search over keyframe k's sslpl_keypoint rows and grid;
// monocular, a keyframe octave below 0 is never a candidate); false compiles the map out.
template <bool kMap>
__global__ void __launch_bounds__(128) k_point_fuse_search(const __grid_constant__ WinArgs A, int nmp, const uint8_t* active, const float* pu, const float* pv, const float* pur,
                                                            const int* level, const uint8_t* dmp, const uint8_t* d2, const float* x2, const float* y2, const int* oct2,
                                                            const float* uright2, const float* invSigma2, const int* goff, const int* gidx,
                                                            int32_t* best_idx, int32_t* best_dist, const __grid_constant__ FuseMap M) {
    const int i = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (i >= nmp) return;
    constexpr int es = kMap ? 7 : 1;                     // keypoint fields: separate arrays or sslpl_keypoint rows
    unsigned long long b = ~0ull;
    GridWin w;
    bool act;
    int lvl;
    float u, v, ur;
    if (kMap) {
        int k, e;
        if (!fuse_entry(M, i, lane, k, e, best_idx, best_dist)) return;
        act = e >= 0 && !(M.skip && M.skip[i]) && fuse_project_point(M, k, e, u, v, lvl);
        ur = 0.f;
        d2 = M.desc + k * M.desc_fs; x2 = M.kp + k * M.kp_fs; y2 = x2 + 1; oct2 = reinterpret_cast<const int*>(x2 + 5);
        goff = M.goff + k * M.goff_fs; gidx = M.gidx + k * M.gidx_fs; invSigma2 = M.invSigma2; dmp = M.eldesc + (long long)e * 32;
    } else {
        act = active[i];
        dmp += (long long)i * 32;
    }
    if (act) {
        if (!kMap) { lvl = level[i]; u = pu[i]; v = pv[i]; ur = pur[i]; }
        const float rad = __fmul_rn(A.th, A.G.scale[lvl]);
        if (grid_window(A.G, u, v, rad, w)) {
            uint4 a0, a1;
            load_desc(dmp, a0, a1);
            b = grid_min(goff, gidx, w, lane, [&](int j, int& d) {
                const float kx = x2[es * j], ky = y2[es * j];
                if (!(fabsf(__fsub_rn(kx, u)) < rad && fabsf(__fsub_rn(ky, v)) < rad)) return false;        // KeyFrame::GetFeaturesInArea KeyFrame.cc:642
                const int o = oct2[es * j];
                if (o < lvl - 1 || o > lvl) return false;                                                    // :905
                if (kMap && o < 0) return false;
                const float ex = __fsub_rn(u, kx), ey = __fsub_rn(v, ky);
                float e2 = __fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey));
                const float kr = A.use_right ? uright2[j] : -1.f;
                if (kr >= 0) {                                                                            // stereo chi-square, 3 dof (:908-921)
                    const float er = __fsub_rn(ur, kr);
                    e2 = __fadd_rn(e2, __fmul_rn(er, er));
                    if ((double)__fmul_rn(e2, invSigma2[o]) > 7.8) return false;
                } else if ((double)__fmul_rn(e2, invSigma2[o]) > 5.99) return false;                         // :923-932
                uint4 c0, c1;
                load_desc(d2 + (long long)j * 32, c0, c1);
                d = popc256(a0, a1, c0, c1);
                return d < 256;                                                                           // bestDist starts at 256, strict <
            });
        }
    }
    if (lane == 0) {
        int bi = -1, bd = 256;
        if (b != ~0ull) { bi = grid_key_feature(goff, gidx, w, b); bd = (int)(b >> 40); }
        best_idx[i] = bi; best_dist[i] = bd;
    }
}

// ORBmatcher::SearchForInitialization (ORBmatcher.cc:408-523) of one pair, run by one warp (the block's only one): F1's n1 features
// (descriptors d1, octave / angle at element stride es) are searched around prev[i] = vbPrevMatched[i] (x, y interleaved) among F2's n2
// features (fields at stride es) on F2's grid CSR goff / gidx.  matchedDist / matches21 [n2] and rbin [n1] are scratch; writes
// matches12[n1] and prev (:517-520) and returns the count in every lane.
template <int es>
__device__ __forceinline__ int init_match(const WinArgs& A, int n1, const uint8_t* d1, const int* oct1, const float* angle1, float* prev,
                                          int n2, const uint8_t* d2, const float* x2, const float* y2, const int* oct2, const float* angle2,
                                          const int* goff, const int* gidx, int* matchedDist, int* matches21, int32_t* matches12, uint8_t* rbin) {
    __shared__ int s_hist[HISTO_LENGTH];
    const int lane = threadIdx.x;
    for (int j = lane; j < n2; j += 32) { matchedDist[j] = 0x7fffffff; matches21[j] = -1; }
    for (int i = lane; i < n1; i += 32) { matches12[i] = -1; rbin[i] = 255; }
    if (lane < HISTO_LENGTH) s_hist[lane] = 0;
    __syncwarp();
    int nmatches = 0;
    const float rad = (float)A.window;
    for (int i1 = 0; i1 < n1; i1++) {
        const int level1 = oct1[es * i1];
        if (level1 > 0) continue;                                 // :426
        const float u = prev[2 * i1], v = prev[2 * i1 + 1];
        GridWin w;
        if (!grid_window(A.G, u, v, rad, w)) continue;
        uint4 a0, a1;
        load_desc(d1 + (long long)i1 * 32, a0, a1);
        unsigned long long b1, b2;
        grid_top2(goff, gidx, w, lane, [&](int j, int& d) {
            { const int o = oct2[es * j]; if (o < level1 || o > level1) return false; }   // GetFeaturesInArea(..., level1, level1): levels are checked (maxLevel >= 0)
            if (!(fabsf(__fsub_rn(x2[es * j], u)) < rad && fabsf(__fsub_rn(y2[es * j], v)) < rad)) return false;
            uint4 c0, c1;
            load_desc(d2 + (long long)j * 32, c0, c1);
            d = popc256(a0, a1, c0, c1);
            return matchedDist[j] > d;                            // :448
        }, b1, b2);
        if (b1 == ~0ull) continue;
        const int bestDist = (int)(b1 >> 40);
        const float bestDist2 = b2 == ~0ull ? (float)0x7fffffff : (float)(int)(b2 >> 40);
        if (bestDist <= TH_LOW_I && (float)bestDist < __fmul_rn(bestDist2, A.nnratio)) {       // :462-464
            const int j = grid_key_feature(goff, gidx, w, b1);
            const int old = matches21[j];
            if (old >= 0) nmatches--;
            if (lane == 0) {
                if (old >= 0) matches12[old] = -1;
                matches12[i1] = j; matches21[j] = i1; matchedDist[j] = bestDist;
                if (A.checkOri) { const int bin = rot_bin(angle1[es * i1], angle2[es * j]); rbin[i1] = (uint8_t)bin; s_hist[bin]++; }
            }
            nmatches++;
        }
        __syncwarp();
    }
    __syncwarp();
    if (A.checkOri)                                               // rbin[i] stays set when a later feature takes match i's j
        nmatches -= warp_rot_check(s_hist, n1, lane, [&](int i) { return rbin[i] != 255 && matches12[i] >= 0 ? (int)rbin[i] : -1; },
                                   [&](int i) { matches12[i] = -1; });
    __syncwarp();
    for (int i = lane; i < n1; i += 32) {                         // :517-520
        const int j = matches12[i];
        if (j >= 0) { prev[2 * i] = x2[es * j]; prev[2 * i + 1] = y2[es * j]; }
    }
    __syncwarp();
    return nmatches;
}

// The single pair: fields in separate arrays
__global__ void __launch_bounds__(32) k_init_match(const __grid_constant__ WinArgs A, int n1, const uint8_t* d1, const int* oct1, const float* angle1,
                                                    float* prev, int n2, const uint8_t* d2, const float* x2, const float* y2, const int* oct2,
                                                    const float* angle2, const int* goff, const int* gidx, int* matchedDist, int* matches21,
                                                    int32_t* matches12, uint8_t* rbin, int32_t* nmatch) {
    const int n = init_match<1>(A, n1, d1, oct1, angle1, prev, n2, d2, x2, y2, oct2, angle2, goff, gidx, matchedDist, matches21, matches12, rbin);
    if (threadIdx.x == 0) *nmatch = n;
}

// -------------------------------------------------------------------------------------------------
// MapPoint / MapLine ::ComputeDistinctiveDescriptors (MapPoint.cc:247-312, MapLine.cpp:246-317), batched over groups of
// observed descriptors (CSR): the descriptor with the least median Hamming distance to the others, first minimum wins.
// One CTA per group, one thread per row; the median of a row (rank r = int(0.5 (N-1)) of N distances in 0..256) is found by
// bisection on the value with count(d <= v) (8 passes over the row, descriptors stay in L1) — no sort, no per-thread arrays.
// -------------------------------------------------------------------------------------------------
// The median of row i: the smallest v with count(d <= v) >= r + 1 over the rows j in [0, n) with use(j) (the self-distance 0 counted),
// returned as the key (median, i) whose minimum is the first least median.  row(j) is the address of row j's descriptor.
template <class Row, class Use>
__device__ __forceinline__ unsigned medoid_key(Row row, Use use, int n, int r, int i) {
    uint4 a0, a1;
    load_desc(row(i), a0, a1);
    int lo = 0, hi = 256;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        int cnt = 0;
        for (int j = 0; j < n; j++) {
            if (!use(j)) continue;
            uint4 b0, b1;
            load_desc(row(j), b0, b1);
            cnt += (j == i ? 0 : popc256(a0, a1, b0, b1)) <= mid;
        }
        if (cnt >= r + 1) hi = mid; else lo = mid + 1;
    }
    return ((unsigned)lo << 20) | (unsigned)i;
}

__global__ void __launch_bounds__(128) k_medoid(const uint8_t* desc, const int32_t* off, int32_t* best_idx, int32_t* best_median) {
    __shared__ unsigned s_best;
    const int gI = blockIdx.x, b = off[gI], N = off[gI + 1] - b;
    if (threadIdx.x == 0) s_best = 0xffffffffu;
    __syncthreads();
    if (N > 0) {
        const int r = (int)(0.5 * (double)(N - 1));
        unsigned mine = 0xffffffffu;
        const auto row = [&](int j) { return desc + (long long)(b + j) * 32; };
        for (int i = threadIdx.x; i < N; i += blockDim.x)
            mine = min(mine, medoid_key(row, [](int) { return true; }, N, r, i));
        atomicMin(&s_best, mine);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        best_idx[gI] = N > 0 ? (int)(s_best & 0xfffffu) : -1;
        best_median[gI] = N > 0 ? (int)(s_best >> 20) : -1;
    }
}

// Rotation-histogram filter (ComputeThreeMaxima, ORBmatcher.cc:1604-1645; application :270-288) and match
// count, one CTA per pair.  compact != 0 additionally writes the (i, out[i]) pairs in ascending i (:818-823).
__global__ void __launch_bounds__(256) k_rot_filter(int32_t* out, long long out_fs, const uint8_t* rot, long long rot_fs,
                                                     const int* n_arr, int n_frame_off, int n_const, int cap, int checkOri,
                                                     int32_t* nmatch, int32_t* pairs, long long pairs_fs) {
    __shared__ int s_hist[HISTO_LENGTH];
    __shared__ int s_keep[3];
    __shared__ int s_warp[33];
    const int pair = blockIdx.x, tid = threadIdx.x;
    const int n = n_arr ? min(n_arr[pair + n_frame_off], cap) : n_const;
    int32_t* O = out + pair * out_fs; const uint8_t* R = rot + pair * rot_fs;
    if (tid < HISTO_LENGTH) s_hist[tid] = 0;
    __syncthreads();
    if (checkOri) {
        for (int i = tid; i < n; i += 256) if (O[i] >= 0) atomicAdd(&s_hist[R[i]], 1);
        __syncthreads();
        if (tid == 0) { const int3 k = three_maxima(s_hist); s_keep[0] = k.x; s_keep[1] = k.y; s_keep[2] = k.z; }
        __syncthreads();
        const int k0 = s_keep[0], k1 = s_keep[1], k2 = s_keep[2];
        for (int i = tid; i < n; i += 256)
            if (O[i] >= 0) { const int b = R[i]; if (b != k0 && b != k1 && b != k2) O[i] = -1; }
        __syncthreads();
    }
    // count (and optionally compact in ascending index order)
    const int chunk = (n + 255) / 256, pb = min(n, tid * chunk), pe = min(n, pb + chunk);
    int c = 0;
    for (int i = pb; i < pe; i++) c += O[i] >= 0;
    int total;
    int o = block_exclusive_scan(c, s_warp, &total);
    if (pairs) for (int i = pb; i < pe; i++) if (O[i] >= 0) { pairs[pair * pairs_fs + 2 * o] = i; pairs[pair * pairs_fs + 2 * o + 1] = O[i]; o++; }
    if (tid == 0) nmatch[pair] = total;
}

__global__ void k_fill_i32(int32_t* p, long long n, int v) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// LSDmatcher::SearchByProjection(KF,F) ratio rule on a knn2 table (LSDmatcher.cpp:161-180): out[tdx] = qdx, the
// LAST accepted query wins (atomicMax over ascending qdx), nmatch counts every acceptance like the reference.
// kMap: pair p is the rows (pmap[p].x, pmap[p].y) of [0, nrows) (keyframe, frame), the keyframe's MapLines are kfml[row][cap] element
// indices (outside [0, nml): NULL) and n_arr is indexed by row; the pair's count (zeroed by the caller) becomes -1 when a row is outside
// the set or when the keyframe has lines and the frame fewer than 2.  kMap = false compiles all of it out.
template <bool kMap>
__global__ void __launch_bounds__(128) k_line_ratio(const int32_t* knn, long long knn_fs, const int* n_arr, int n_const, int cap,
                                                     const uint8_t* has_ml1, long long ml_fs,
                                                     int32_t* out, long long out_fs, int32_t* nmatch,
                                                     const int2* pmap, int nrows, const int32_t* kfml, int nml) {
    const int pair = blockIdx.y, q = blockIdx.x * blockDim.x + threadIdx.x;
    int nq, fk = pair, ff;
    if (kMap) {
        const bool ok = pair_frames(pmap, nrows, pair, fk, ff);
        nq = ok ? max(0, min(n_arr[fk], cap)) : 0;
        if (!ok || (nq > 0 && min(n_arr[ff], cap) < 2)) {                       // knnMatch would leave lmatches[i][1] undefined (:167)
            if (q == 0) nmatch[pair] = -1;
            return;
        }
    } else nq = n_arr ? min(n_arr[pair], cap) : n_const;
    if (q >= nq) return;
    const int4 r = reinterpret_cast<const int4*>(knn + pair * knn_fs)[q];
    if (r.x < 0 || r.z < 0) return;
    const float ratio = __fdiv_rn((float)r.y, (float)r.w);                         // :167
    if ((double)ratio < (double)(1.0f / 1.5f)) {                                    // :169
        if (kMap) { if ((unsigned)kfml[(long long)fk * cap + q] >= (unsigned)nml) return; }   // :173-174
        else if (has_ml1 && !has_ml1[pair * ml_fs + q]) return;
        atomicMax(&out[pair * out_fs + r.x], q);
        atomicAdd(&nmatch[pair], 1);
    }
}

// A pair of the batched triangulation matcher whose keyframe indices lie outside [0, nframes) gets the count -1 (its rows stay empty)
__global__ void k_bad_pairs(const int2* pmap, int npairs, int nframes, int32_t* nmatch) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    int f1, f2;
    if (p < npairs && !pair_frames(pmap, nframes, p, f1, f2)) nmatch[p] = -1;
}

// SearchByBoW(KeyFrame, Frame) over (keyframe row, frame row) pairs builds the FeatureVector of each row the pairs name once, in a slot:
// side k of pair p (0 keyframe, 1 frame) is slot 2p + k, and a row's FeatureVector lives in the smallest slot that names it.
// k_kfbow_claim leaves that slot in slot_of_row[row] (filled with INT_MAX before); k_kfbow_slots then gives each slot its row (-1 for a
// slot whose row an earlier slot holds) and clamped count (0 there), and each pair its two slots and its frame's clamped count.
__global__ void k_kfbow_claim(const int2* pmap, int npairs, int nrows, int32_t* slot_of_row) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x, p = t >> 1;
    int kr, fr;
    if (p >= npairs || !pair_frames(pmap, nrows, p, kr, fr)) return;
    atomicMin(slot_of_row + ((t & 1) ? fr : kr), t);
}
__global__ void k_kfbow_slots(const int2* pmap, int npairs, int nrows, const int* n, int cap, const int32_t* slot_of_row,
                              int32_t* slot_row, int* slot_n, int2* pslot, int* frame_n) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x, p = t >> 1;
    if (p >= npairs) return;
    int kr, fr;
    const bool ok = pair_frames(pmap, nrows, p, kr, fr);
    const int r = (t & 1) ? fr : kr;
    const bool own = ok && slot_of_row[r] == t;
    slot_row[t] = own ? r : -1;
    slot_n[t] = own ? min(max(n[r], 0), cap) : 0;
    if (t & 1) return;
    pslot[p] = ok ? make_int2(slot_of_row[kr], slot_of_row[fr]) : make_int2(0, 0);
    frame_n[p] = ok ? min(max(n[fr], 0), cap) : 0;
}

// LSDmatcher::SearchForTriangulation (LSDmatcher.cpp:382-415), one CTA per keyframe pair, on the knn2 table of (KF1 lines, KF2 lines):
//   KeyFrame::lineDescriptorMAD's nn12_mad (KeyFrame.cc:820-846; the host form is line_mad() below) over all n1 query rows.  The
//   distances are integers in [0, 256], so both medians are exact selections over a 257-bin histogram: med12 = element nq / 2 of the
//   d1 - d0 sorted in DESCENDING order (conpare_descriptor_by_NN12_dist), then element nq / 2 of |d1 - d0 - med12| in ascending order;
//   then the filter of :398-410 (skip rows whose KF1 or KF2 line has a MapLine, accept d1 - d0 > fac nn12_mad, fac = 0.1) and an ordered
//   compaction: lpairs[p][k] = (qdx, tdx) in ascending qdx, (-1, -1) past the count.
// nlmatch[p] = -1 when an index is outside [0, nframes) or when KF1 has lines and KF2 fewer than 2 (the reference would read
// lmatches[i][1] out of bounds, :402); 0 when KF1 has none.
// With has_ml NULL and fac = 0.5 it is LSDmatcher::SerachForInitialize (LSDmatcher.cpp:257-284; Frame::lineDescriptorMAD, Frame.cc:189-215,
// computes the same nn12_mad), which tests no MapLines.
// nn12_mad * fac of the n1 >= 1 rows of knn table K (fac: 0.1 for SearchForTriangulation :406, 0.5 for SerachForInitialize :270), computed
// by the whole CTA (every thread gets it); s_hist[257] and s_sel are the caller's shared memory
__device__ __forceinline__ double line_mad_thr(const int4* K, int n1, int tid, int* s_hist, int* s_sel, double fac) {
    const int k = n1 / 2;
    for (int i = tid; i < 257; i += 256) s_hist[i] = 0;
    __syncthreads();
    for (int i = tid; i < n1; i += 256) { const int4 r = K[i]; atomicAdd(&s_hist[r.w - r.y], 1); }
    __syncthreads();
    if (tid == 0) {                                            // descending order: count down from 256
        int c = 0, v = 256;
        for (; v > 0; v--) { c += s_hist[v]; if (c > k) break; }
        *s_sel = v;
    }
    __syncthreads();
    const int med12 = *s_sel;
    for (int i = tid; i < 257; i += 256) s_hist[i] = 0;
    __syncthreads();
    for (int i = tid; i < n1; i += 256) { const int4 r = K[i]; atomicAdd(&s_hist[abs(r.w - r.y - med12)], 1); }
    __syncthreads();
    if (tid == 0) {                                            // ascending order
        int c = 0, v = 0;
        for (; v < 256; v++) { c += s_hist[v]; if (c > k) break; }
        *s_sel = v;
    }
    __syncthreads();
    return __dmul_rn(__dmul_rn(1.4826, (double)*s_sel), fac);
}
// the KF2 and distance tests of :403-408 for knn row r (the KF1 test is the caller's)
__device__ __forceinline__ bool line_row_ok(int4 r, const uint8_t* h2, double thr) {
    return !h2[r.x] && (double)(r.w - r.y) > thr;
}

__global__ void __launch_bounds__(256) k_line_tri(const int32_t* knn, long long knn_fs, const int* nl, int capl, const int2* pmap, int nframes,
                                                   const uint8_t* has_ml, double fac, int32_t* lpairs, int32_t* nlmatch) {
    __shared__ int s_hist[257];
    __shared__ int s_warp[33];
    __shared__ int s_sel;
    const int p = blockIdx.x, tid = threadIdx.x;
    int f1, f2, n1 = 0, total = 0;
    bool ok = pair_frames(pmap, nframes, p, f1, f2);
    if (ok) {
        n1 = max(0, min(nl[f1], capl));
        ok = n1 == 0 || min(nl[f2], capl) >= 2;
    }
    const int4* K = reinterpret_cast<const int4*>(knn + p * knn_fs);
    int32_t* O = lpairs + 2LL * capl * p;
    if (ok && n1 > 0) {                                        // CTA-uniform
        const double thr = line_mad_thr(K, n1, tid, s_hist, &s_sel, fac);
        const uint8_t* h1 = has_ml ? has_ml + (long long)f1 * capl : nullptr; const uint8_t* h2 = has_ml ? has_ml + (long long)f2 * capl : nullptr;
        const auto keep = [&](int i, int4 r) { return (!has_ml || (!h1[i] && !h2[r.x])) && (double)(r.w - r.y) > thr; };
        const int chunk = (n1 + 255) / 256, pb = min(n1, tid * chunk), pe = min(n1, pb + chunk);
        int c = 0;
        for (int i = pb; i < pe; i++) c += keep(i, K[i]);
        int o = block_exclusive_scan(c, s_warp, &total);
        for (int i = pb; i < pe; i++) {
            const int4 r = K[i];
            if (keep(i, r)) { O[2 * o] = i; O[2 * o + 1] = r.x; o++; }
        }
    }
    for (int i = total + tid; i < capl; i += 256) { O[2 * i] = -1; O[2 * i + 1] = -1; }
    if (tid == 0) nlmatch[p] = ok ? total : -1;
}

// The table k_create_lines_chain starts from: for pair p, tw[p][qdx] = tdx when row qdx of LSDmatcher::SearchForTriangulation passes the
// KF2 and distance tests (the KF1 mask left out), else -1, for qdx < n1.  Pairs that k_line_tri gives no rows or -1 are left unwritten.
__global__ void __launch_bounds__(256) k_line_tri_table(const int32_t* knn, long long knn_fs, const int* nl, int capl, const int2* pmap,
                                                         int nframes, const uint8_t* has_ml, int32_t* tw) {
    __shared__ int s_hist[257];
    __shared__ int s_sel;
    const int p = blockIdx.x, tid = threadIdx.x;
    int f1, f2;
    if (!pair_frames(pmap, nframes, p, f1, f2)) return;
    const int n1 = max(0, min(nl[f1], capl));
    if (n1 == 0 || min(nl[f2], capl) < 2) return;              // CTA-uniform
    const int4* K = reinterpret_cast<const int4*>(knn + p * knn_fs);
    const double thr = line_mad_thr(K, n1, tid, s_hist, &s_sel, 0.1);
    const uint8_t* h2 = has_ml + (long long)f2 * capl;
    int32_t* T = tw + (long long)capl * p;
    for (int i = tid; i < n1; i += 256) { const int4 r = K[i]; T[i] = line_row_ok(r, h2, thr) ? r.x : -1; }
}

// ---------------- LocalMapping::CreateNewMapPoints' neighbour loop (LocalMapping.cc:371-637, monocular) ----------------
// Status codes of include/sslpl.h (SSLPL_CNMP_*), one per `continue` of the per-match body in reference order.
enum { CNMP_CREATED = 0, CNMP_PARALLAX, CNMP_W_ZERO, CNMP_Z1, CNMP_Z2, CNMP_OCTAVE1, CNMP_REPROJ1, CNMP_REPROJ2, CNMP_DIST0, CNMP_SCALE };

struct CreateArgs {
    float fx, fy, cx, cy, invfx, invfy;   // KeyFrame::fx .. invfy (one camera for both keyframes)
    float ratioFactor;                    // 1.5f * mfScaleFactor (:400)
    int nlevels;
    float scale[SSLPL_MAX_LEVELS], sigma2[SSLPL_MAX_LEVELS];
};

// cv::addWeighted(a, alpha, b, -1, 0) of CV_32F, as tools/probe_cv_matexpr.py measured it: in double, rounded once
__device__ __forceinline__ float add_weighted_m1(float a, float alpha, float b) {
    return __double2float_rn(__dadd_rn(__dadd_rn(__dmul_rn((double)a, (double)alpha), -(double)b), 0.0));
}
// float(Rcw.row(r).dot(x3Dt) + tcw.at<float>(r)) for row r = T[0..3] of a pose (:533, :545)
__device__ __forceinline__ float cam_row(const float* T, const float* X) {
    return __double2float_rn(__dadd_rn(dot3d(T[0], T[1], T[2], X[0], X[1], X[2]), (double)T[3]));
}
// Rwc * xn (cv::gemm's float path) with Rwc = Rcw.t(): column i of Rcw
__device__ __forceinline__ void ray(const float* T, const float* xn, float* r) {
#pragma unroll
    for (int i = 0; i < 3; i++)
        r[i] = __fadd_rn(__fadd_rn(__fmul_rn(T[i], xn[0]), __fmul_rn(T[4 + i], xn[1])), __fmul_rn(T[8 + i], xn[2]));
}
// the monocular reprojection chi-square test (:549-558 / :578-585): true = rejected
__device__ __forceinline__ bool reproj_bad(const CreateArgs& C, const float* T, const float* X, float z, float kx, float ky, float sigma2) {
    const float x = cam_row(T, X), y = cam_row(T + 4, X);
    const float invz = __double2float_rn(__ddiv_rn(1.0, (double)z));                                   // const float invz = 1.0 / z
    const float u = __fadd_rn(__fmul_rn(__fmul_rn(C.fx, x), invz), C.cx), v = __fadd_rn(__fmul_rn(__fmul_rn(C.fy, y), invz), C.cy);
    const float ex = __fsub_rn(u, kx), ey = __fsub_rn(v, ky);
    return (double)__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)) > __dmul_rn(5.991, (double)sigma2);
}

// The per-match body of CreateNewMapPoints (:459-634) for KF1 keypoint (x1, y1, o1) and KF2 keypoint (x2, y2, o2) with poses T1 / T2
// (pose[15] = Tcw 3x4 row-major, Ow) -> status; X is set when the row gets past the w == 0 test (*written = true).
__device__ __forceinline__ int create_point(const CreateArgs& C, const float* T1, const float* T2, float x1, float y1, int o1,
                                            float x2, float y2, int o2, float* X, bool* written) {
    *written = false;
    const float xn1[3] = {__fmul_rn(__fsub_rn(x1, C.cx), C.invfx), __fmul_rn(__fsub_rn(y1, C.cy), C.invfy), 1.f};   // :475-476
    const float xn2[3] = {__fmul_rn(__fsub_rn(x2, C.cx), C.invfx), __fmul_rn(__fsub_rn(y2, C.cy), C.invfy), 1.f};
    float r1[3], r2[3];
    ray(T1, xn1, r1); ray(T2, xn2, r2);                                                                          // :479-480
    const float cosp = __double2float_rn(__ddiv_rn(dot3d(r1[0], r1[1], r1[2], r2[0], r2[1], r2[2]),
                                                   __dmul_rn(norm3d_d(r1[0], r1[1], r1[2]), norm3d_d(r2[0], r2[1], r2[2]))));   // :482
    if (!(cosp < __fadd_rn(cosp, 1.f) && cosp > 0.f && (double)cosp < 0.9998)) return CNMP_PARALLAX;             // :484-497, :526
    float A[16], W[4], Vt[16];
#pragma unroll
    for (int k = 0; k < 4; k++) {                                                                                // :500-504
        A[k] = add_weighted_m1(T1[8 + k], xn1[0], T1[k]);
        A[4 + k] = add_weighted_m1(T1[8 + k], xn1[1], T1[4 + k]);
        A[8 + k] = add_weighted_m1(T2[8 + k], xn2[0], T2[k]);
        A[12 + k] = add_weighted_m1(T2[8 + k], xn2[1], T2[4 + k]);
    }
    svd4_jacobi(A, W, Vt);                                                                                       // :506-509
    if (Vt[15] == 0.f) return CNMP_W_ZERO;                                                                       // :511
    const float inv = __double2float_rn(__ddiv_rn(1.0, (double)Vt[15]));                                         // :515, convertTo
#pragma unroll
    for (int k = 0; k < 3; k++) X[k] = __fadd_rn(__fmul_rn(Vt[12 + k], inv), 0.f);
    *written = true;
    const float z1 = cam_row(T1 + 8, X);                                                                         // :533-539
    if (z1 <= 0.f) return CNMP_Z1;
    const float z2 = cam_row(T2 + 8, X);
    if (z2 <= 0.f) return CNMP_Z2;
    if ((unsigned)o1 >= (unsigned)C.nlevels) return CNMP_OCTAVE1;                                                // mvLevelSigma2[kp1.octave]
    if (reproj_bad(C, T1, X, z1, x1, y1, C.sigma2[o1])) return CNMP_REPROJ1;
    if (reproj_bad(C, T2, X, z2, x2, y2, C.sigma2[o2])) return CNMP_REPROJ2;
    const float dist1 = norm3d(__fsub_rn(X[0], T1[12]), __fsub_rn(X[1], T1[13]), __fsub_rn(X[2], T1[14]));       // :601-605
    const float dist2 = norm3d(__fsub_rn(X[0], T2[12]), __fsub_rn(X[1], T2[13]), __fsub_rn(X[2], T2[14]));
    if (dist1 == 0.f || dist2 == 0.f) return CNMP_DIST0;
    const float ratioDist = __fdiv_rn(dist2, dist1), ratioOctave = __fdiv_rn(C.scale[o1], C.scale[o2]);           // :610-616
    if (__fmul_rn(ratioDist, C.ratioFactor) < ratioOctave || ratioDist > __fmul_rn(ratioOctave, C.ratioFactor)) return CNMP_SCALE;
    return CNMP_CREATED;
}

// The steps the chain kernels below share.  A chain is a maximal run [c0, c1) of consecutive pairs with the same kf1; false when pair c0
// does not start one.
__device__ __forceinline__ bool chain_range(const int2* pmap, int npairs, int c0, int& kf1, int& c1) {
    kf1 = pmap[c0].x;
    if (c0 > 0 && pmap[c0 - 1].x == kf1) return false;
    c1 = c0 + 1;
    while (c1 < npairs && pmap[c1].x == kf1) c1++;
    return true;
}

// SearchForInitialization over the chains of a pair list (pmap[p] = (init row, current row) of a row set of sslpl_keypoint rows kp,
// descriptors desc and counts n, cap rows each): block c0 runs the chain that starts at pair c0 (chain_range; other blocks return at
// once), pair after pair, because each pair reads the vbPrevMatched the one before it left and the greedy scan inside a pair is itself
// sequential.  The chain's state starts as prev0[c0] (NULL: the init row's keypoint positions); a good pair p copies it to prev[p],
// updates it there and makes prev[p] the state of the next pair.  A pair with a row outside [0, nrows) or the init row as its current row
// gets nmatch -1, writes no rows and leaves the state alone.  Row r2's grid CSR is goff + r2 goff_fs, gidx + r2 gidx_fs; the chain's
// scratch is ws_* + c0 ws_fs.
__global__ void __launch_bounds__(32) k_init_chain(const __grid_constant__ WinArgs A, const int2* pmap, int npairs, int nrows, const float* kp,
                                                    const uint8_t* desc, const int* n_arr, int cap, const float* prev0,
                                                    const int* goff, const int* gidx, long long goff_fs, long long gidx_fs,
                                                    int* ws_dist, int* ws_m21, uint8_t* ws_rbin, long long ws_fs,
                                                    int32_t* match12, float* prev, int32_t* nmatch) {
    const int c0 = blockIdx.x, lane = threadIdx.x;
    int r1, c1;
    if (!chain_range(pmap, npairs, c0, r1, c1)) return;
    const bool ok1 = (unsigned)r1 < (unsigned)nrows;
    const int n1 = ok1 ? max(0, min(n_arr[r1], cap)) : 0;
    const float* K1 = kp + 7LL * cap * (ok1 ? r1 : 0);
    const float* src = prev0 ? prev0 + 2LL * cap * c0 : nullptr;
    for (int p = c0; p < c1; p++) {
        const int r2 = pmap[p].y;
        if (!ok1 || (unsigned)r2 >= (unsigned)nrows || r2 == r1) {
            if (lane == 0) nmatch[p] = -1;
            continue;
        }
        float* P = prev + 2LL * cap * p;
        for (int i = lane; i < n1; i += 32) {                     // Tracking.cc:338-340 without prev0
            P[2 * i] = src ? src[2 * i] : K1[7 * i];
            P[2 * i + 1] = src ? src[2 * i + 1] : K1[7 * i + 1];
        }
        __syncwarp();
        const int n2 = max(0, min(n_arr[r2], cap));
        const float* K2 = kp + 7LL * cap * r2;
        int32_t* M = match12 + (long long)cap * p;
        const int n = init_match<7>(A, n1, desc + 32LL * cap * r1, reinterpret_cast<const int*>(K1 + 5), K1 + 3, P, n2, desc + 32LL * cap * r2,
                                    K2, K2 + 1, reinterpret_cast<const int*>(K2 + 5), K2 + 3, goff + goff_fs * r2, gidx + gidx_fs * r2,
                                    ws_dist + ws_fs * c0, ws_m21 + ws_fs * c0, M, ws_rbin + ws_fs * c0);
        for (int i = n1 + lane; i < cap; i += 32) M[i] = -1;
        if (lane == 0) nmatch[p] = n;
        src = P;
    }
}

// s_bits = row kf1 of the mask as a bitmap of cap bits (all clear when !ok1), visible to the whole CTA on return
__device__ __forceinline__ void chain_load_bits(unsigned* s_bits, const uint8_t* mask, int kf1, bool ok1, int cap, int tid) {
    const int words = (cap + 31) / 32;
    for (int w = tid; w < words; w += 256) {
        unsigned b = 0;
        for (int k = 0; k < 32 && ok1 && 32 * w + k < cap; k++) b |= (mask[(long long)kf1 * cap + 32 * w + k] != 0) << k;
        s_bits[w] = b;
    }
    __syncthreads();
}
// pair p of the chain from c0 gets -1 (and leaves the bitmap alone) for kf1 or kf2 outside [0, nkf), kf2 == kf1 or a kf2 repeated in the chain
__device__ __forceinline__ bool chain_pair_bad(const int2* pmap, int c0, int p, int kf1, bool ok1, int nkf, int& kf2) {
    kf2 = pmap[p].y;
    bool bad = !ok1 || (unsigned)kf2 >= (unsigned)nkf || kf2 == kf1;
    for (int q = c0; q < p && !bad; q++) bad = pmap[q].y == kf2;
    return bad;
}
// rows R[k] = (i, T[i]) of the i < n1 with T[i] >= 0 and bit i clear, in ascending i (block scan); returns the count
__device__ __forceinline__ int chain_compact(const int32_t* T, int n1, const unsigned* s_bits, int* s_warp, int32_t* R, int tid) {
    const int chunk = (n1 + 255) / 256, pb = min(n1, tid * chunk), pe = min(n1, pb + chunk);
    int c = 0, total;
    for (int i = pb; i < pe; i++) c += T[i] >= 0 && !((s_bits[i >> 5] >> (i & 31)) & 1u);
    int o = block_exclusive_scan(c, s_warp, &total);
    for (int i = pb; i < pe; i++)
        if (T[i] >= 0 && !((s_bits[i >> 5] >> (i & 31)) & 1u)) { R[2 * o] = i; R[2 * o + 1] = T[i]; o++; }
    return total;
}
// rows and statuses past the count cleared to -1, the pair's counts written; the bitmap bits set for pair p are visible on return
__device__ __forceinline__ void chain_pair_end(int32_t* R, int32_t* S, int total, int cap, bool bad, int created, int p, int32_t* nmatch,
                                               int32_t* nnew, int tid) {
    for (int i = total + tid; i < cap; i += 256) { R[2 * i] = -1; R[2 * i + 1] = -1; S[i] = -1; }
    if (tid == 0) { nmatch[p] = bad ? -1 : total; nnew[p] = created; }
    __syncthreads();
}

// One CTA per chain (a maximal run of consecutive pairs with the same kf1: one keyframe's neighbour loop); CTAs that do not start a chain
// return at once.  The KF1 features that have a MapPoint are a bitmap in shared memory, loaded from has_mp; for each pair in order the
// CTA drops the unfiltered SearchForTriangulation rows (tw[p][idx1] = idx2 or -1) whose idx1 is set, compacts the rest in ascending idx1
// (block scan), triangulates one row per thread and sets the bits of the created rows (AddMapPoint(pMP, idx1), :624) before the next pair.
// A pair with an index outside [0, nkf), kf2 == kf1 or a kf2 repeated in its chain gets count -1 and leaves the bitmap alone.
__global__ void __launch_bounds__(256, 1) k_create_points_chain(const int2* pmap, int npairs, int nkf, const int32_t* tw, int cap,
        const float* kp, const int* n_arr, const uint8_t* has_mp, const float* pose, const __grid_constant__ CreateArgs C,
        int32_t* rows, int32_t* nmatch, int32_t* status, float* x3d, int32_t* nnew) {
    extern __shared__ unsigned s_bits[];
    __shared__ int s_warp[33];
    const int c0 = blockIdx.x, tid = threadIdx.x;
    int kf1, c1;
    if (!chain_range(pmap, npairs, c0, kf1, c1)) return;
    const bool ok1 = (unsigned)kf1 < (unsigned)nkf;
    const int n1 = ok1 ? max(0, min(n_arr[kf1], cap)) : 0;
    chain_load_bits(s_bits, has_mp, kf1, ok1, cap, tid);
    const float* K1 = kp + 7LL * cap * (ok1 ? kf1 : 0);
    for (int p = c0; p < c1; p++) {
        int kf2;
        const bool bad = chain_pair_bad(pmap, c0, p, kf1, ok1, nkf, kf2);
        int32_t* R = rows + 2LL * cap * p; int32_t* S = status + (long long)cap * p; float* X3 = x3d + 3LL * cap * p;
        int total = 0, created = 0;
        if (!bad) {                                                              // CTA-uniform
            total = chain_compact(tw + (long long)cap * p, n1, s_bits, s_warp, R, tid);
            __syncthreads();                                                     // the rows (global) and every bitmap read are done
            const float* K2 = kp + 7LL * cap * kf2;
            const float* T1 = pose + 15LL * kf1; const float* T2 = pose + 15LL * kf2;
            float t1[15], t2[15];
#pragma unroll
            for (int k = 0; k < 15; k++) { t1[k] = T1[k]; t2[k] = T2[k]; }
            for (int r = tid; r < total; r += 256) {
                const int i1 = R[2 * r], i2 = R[2 * r + 1];
                float X[3]; bool written;
                const int st = create_point(C, t1, t2, K1[7 * i1], K1[7 * i1 + 1], __float_as_int(K1[7 * i1 + 5]),
                                            K2[7 * i2], K2[7 * i2 + 1], __float_as_int(K2[7 * i2 + 5]), X, &written);
                S[r] = st;
                if (written) { X3[3 * r] = X[0]; X3[3 * r + 1] = X[1]; X3[3 * r + 2] = X[2]; }
                if (st == CNMP_CREATED) { atomicOr(&s_bits[i1 >> 5], 1u << (i1 & 31)); created++; }
            }
            int all;
            block_exclusive_scan(created, s_warp, &all);
            created = all;
        }
        chain_pair_end(R, S, total, cap, bad, created, p, nmatch, nnew, tid);
    }
}

// ---------------- LocalMapping::CreateNewMapLines2's neighbour loop (LocalMapping.cc:911-1173, monocular) ----------------
// Status codes of include/sslpl.h (SSLPL_CNML_*), one per `continue` of the per-match body in reference order.
enum { CNML_CREATED = 0, CNML_PARALLAX, CNML_W_ZERO_S, CNML_W_ZERO_E, CNML_NEAR_S1, CNML_NEAR_S2, CNML_LONG, CNML_NEAR_E1, CNML_NEAR_E2,
       CNML_ZS1, CNML_ZS2, CNML_ZE1, CNML_ZE2 };

struct LineCam { float fx, fy, cx, cy, invfx, invfy; };   // KeyFrame::fx .. invfy (one camera for both keyframes)

// (a + b) / 2 of CV_32F: MatExpr's addWeighted(a, 0.5, b, 0.5, 0), in double, rounded once
__device__ __forceinline__ float mid_aw(float a, float b) {
    return __double2float_rn(__dadd_rn(__dadd_rn(__dmul_rn((double)a, 0.5), __dmul_rn((double)b, 0.5)), 0.0));
}
// M = K * Tcw (:1047-1048), 3x3 by 3x4: cv::gemm's float path (inner length 3 = output height), K's zeros in the sum order
__device__ __forceinline__ void proj_mat(const LineCam& C, const float* T, float* M) {
    const float K[9] = {C.fx, 0.f, C.cx, 0.f, C.fy, C.cy, 0.f, 0.f, 1.f};
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 4; j++)
            M[4 * i + j] = __fadd_rn(__fadd_rn(__fmul_rn(K[3 * i], T[j]), __fmul_rn(K[3 * i + 1], T[4 + j])), __fmul_rn(K[3 * i + 2], T[8 + j]));
}
// row j of klF.t() * M (:1057-1058): cv::gemm 1x3 by 3x4, accumulated in double from 0 and rounded once
__device__ __forceinline__ float plane_row(const float* l, const float* M, int j) {
    return __double2float_rn(__dadd_rn(__dadd_rn(__dadd_rn(0.0, __dmul_rn((double)l[0], (double)M[j])), __dmul_rn((double)l[1], (double)M[4 + j])),
                                       __dmul_rn((double)l[2], (double)M[8 + j])));
}
// One end point (:1056-1070 / :1073-1088): A = [P1; P2; x T1.row(2) - T1.row(0); y T1.row(2) - T1.row(1)], its SVD and the
// dehomogenised null vector X; false when vt(3, 3) == 0
__device__ __forceinline__ bool tri_end(const float* P1, const float* P2, const float* T1, float x, float y, float* X) {
    float A[16], W[4], Vt[16];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        A[k] = P1[k]; A[4 + k] = P2[k];
        A[8 + k] = add_weighted_m1(T1[8 + k], x, T1[k]);
        A[12 + k] = add_weighted_m1(T1[8 + k], y, T1[4 + k]);
    }
    svd4_jacobi(A, W, Vt);
    if (Vt[15] == 0.f) return false;
    const float inv = __double2float_rn(__ddiv_rn(1.0, (double)Vt[15]));                                         // rowRange(0, 3) / w
#pragma unroll
    for (int k = 0; k < 3; k++) X[k] = __fadd_rn(__fmul_rn(Vt[12 + k], inv), 0.f);
    return true;
}
// (float)cv::norm(a - b) / depth (:1099-1131)
__device__ __forceinline__ float dist_ratio(const float* a, const float* b, float depth) {
    return __fdiv_rn(norm3d(__fsub_rn(a[0], b[0]), __fsub_rn(a[1], b[1]), __fsub_rn(a[2], b[2])), depth);
}

// The per-match body of CreateNewMapLines2 (:1007-1169) for KF1 segment (s1, e1) with line function l1 and KF2 segment (s2, e2) with l2,
// poses T1 / T2 (pose[15] = Tcw 3x4 row-major, Ow), projection matrices M1 / M2 and KF2's median depth -> status; X = s3D, e3D is set
// when both SVDs gave a w != 0 (*written = true).
__device__ __forceinline__ int create_line(const LineCam& C, const float* T1, const float* T2, const float* M1, const float* M2, float depth2,
                                           const float* s1, const float* e1, const double* l1, const float* s2, const float* e2,
                                           const double* l2, float* X, bool* written) {
    *written = false;
    const float S1[2] = {__fmul_rn(__fsub_rn(s1[0], C.cx), C.invfx), __fmul_rn(__fsub_rn(s1[1], C.cy), C.invfy)};   // :1025-1036
    const float E1[2] = {__fmul_rn(__fsub_rn(e1[0], C.cx), C.invfx), __fmul_rn(__fsub_rn(e1[1], C.cy), C.invfy)};
    const float S2[2] = {__fmul_rn(__fsub_rn(s2[0], C.cx), C.invfx), __fmul_rn(__fsub_rn(s2[1], C.cy), C.invfy)};
    const float E2[2] = {__fmul_rn(__fsub_rn(e2[0], C.cx), C.invfx), __fmul_rn(__fsub_rn(e2[1], C.cy), C.invfy)};
    const float m1[3] = {mid_aw(S1[0], E1[0]), mid_aw(S1[1], E1[1]), mid_aw(1.f, 1.f)};
    const float m2[3] = {mid_aw(S2[0], E2[0]), mid_aw(S2[1], E2[1]), mid_aw(1.f, 1.f)};
    float r1[3], r2[3];
    ray(T1, m1, r1); ray(T2, m2, r2);                                                                           // :1038-1039
    const float cosp = __double2float_rn(__ddiv_rn(dot3d(r1[0], r1[1], r1[2], r2[0], r2[1], r2[2]),
                                                   __dmul_rn(norm3d_d(r1[0], r1[1], r1[2]), norm3d_d(r2[0], r2[1], r2[2]))));   // :1041
    if (!(cosp < __fadd_rn(cosp, 1.f) && cosp > 0.f && (double)cosp < 0.98)) return CNML_PARALLAX;             // :1043, :1053, :1090
    const float f1[3] = {__double2float_rn(l1[0]), __double2float_rn(l1[1]), __double2float_rn(l1[2])};          // klF1, klF2 (:1016-1021)
    const float f2[3] = {__double2float_rn(l2[0]), __double2float_rn(l2[1]), __double2float_rn(l2[2])};
    float P1[4], P2[4];
#pragma unroll
    for (int j = 0; j < 4; j++) { P1[j] = plane_row(f1, M1, j); P2[j] = plane_row(f2, M2, j); }
    if (!tri_end(P1, P2, T1, S1[0], S1[1], X)) return CNML_W_ZERO_S;
    if (!tri_end(P1, P2, T1, E1[0], E1[1], X + 3)) return CNML_W_ZERO_E;
    *written = true;
    const float* s3 = X; const float* e3 = X + 3;
    if ((double)dist_ratio(s3, T1 + 12, depth2) < 0.3) return CNML_NEAR_S1;                                     // :1098-1109
    if ((double)dist_ratio(s3, T2 + 12, depth2) < 0.3) return CNML_NEAR_S2;
    if ((double)dist_ratio(e3, s3, depth2) > 0.61) return CNML_LONG;                                            // :1112-1116
    if ((double)dist_ratio(e3, T1 + 12, depth2) < 0.3) return CNML_NEAR_E1;                                     // :1122-1131
    if ((double)dist_ratio(e3, T2 + 12, depth2) < 0.3) return CNML_NEAR_E2;
    if (cam_row(T1 + 8, s3) <= 0.f) return CNML_ZS1;                                                            // :1134-1148
    if (cam_row(T2 + 8, s3) <= 0.f) return CNML_ZS2;
    if (cam_row(T1 + 8, e3) <= 0.f) return CNML_ZE1;
    if (cam_row(T2 + 8, e3) <= 0.f) return CNML_ZE2;
    return CNML_CREATED;
}

// One CTA per chain, as k_create_points_chain: the KF1 lines that have a MapLine are a bitmap in shared memory, loaded from has_ml; for
// each pair in order the CTA drops the k_line_tri_table rows whose qdx is set, compacts the rest in ascending qdx (block scan),
// triangulates both end points of one row per thread and sets the bits of the created rows (AddMapLine(pML, idx1), :1159) before the
// next pair.  A pair with an index outside [0, nkf), kf2 == kf1, a kf2 repeated in its chain, or KF1 with lines and KF2 with fewer than
// 2 gets count -1 and leaves the bitmap alone; KF1 without lines gives 0.  kl = sslpl_keyline rows (17 floats), lineeq 3 doubles per row.
__global__ void __launch_bounds__(256, 1) k_create_lines_chain(const int2* pmap, int npairs, int nkf, const int32_t* tw, int capl,
        const float* kl, const double* lineeq, const int* nl, const uint8_t* has_ml, const float* pose, const float* depth,
        const __grid_constant__ LineCam C, int32_t* rows, int32_t* nmatch, int32_t* status, float* line3d, int32_t* nnew) {
    extern __shared__ unsigned s_bits[];
    __shared__ int s_warp[33];
    __shared__ float s_T[2][15], s_M[2][12];
    const int c0 = blockIdx.x, tid = threadIdx.x;
    int kf1, c1;
    if (!chain_range(pmap, npairs, c0, kf1, c1)) return;
    const bool ok1 = (unsigned)kf1 < (unsigned)nkf;
    const int n1 = ok1 ? max(0, min(nl[kf1], capl)) : 0;
    chain_load_bits(s_bits, has_ml, kf1, ok1, capl, tid);
    const long long o1 = (long long)capl * (ok1 ? kf1 : 0);
    for (int p = c0; p < c1; p++) {
        int kf2;
        bool bad = chain_pair_bad(pmap, c0, p, kf1, ok1, nkf, kf2);
        if (!bad) bad = n1 > 0 && min(nl[kf2], capl) < 2;
        int32_t* R = rows + 2LL * capl * p; int32_t* S = status + (long long)capl * p; float* L3 = line3d + 6LL * capl * p;
        int total = 0, created = 0;
        if (!bad && n1 > 0) {                                                    // CTA-uniform
            total = chain_compact(tw + (long long)capl * p, n1, s_bits, s_warp, R, tid);
            if (tid < 30) s_T[tid / 15][tid % 15] = pose[15LL * (tid < 15 ? kf1 : kf2) + tid % 15];
            __syncthreads();                                                     // the rows (global), the poses and every bitmap read are done
            if (tid < 2) proj_mat(C, s_T[tid], s_M[tid]);
            __syncthreads();
            const long long o2 = (long long)capl * kf2;
            const float d2 = depth[kf2];
            for (int r = tid; r < total; r += 256) {
                const int i1 = R[2 * r], i2 = R[2 * r + 1];
                const float* k1 = kl + 17 * (o1 + i1); const float* k2 = kl + 17 * (o2 + i2);
                float X[6]; bool written;
                const int st = create_line(C, s_T[0], s_T[1], s_M[0], s_M[1], d2, k1 + 7, k1 + 9, lineeq + 3 * (o1 + i1), k2 + 7, k2 + 9,
                                           lineeq + 3 * (o2 + i2), X, &written);
                S[r] = st;
                if (written) {
#pragma unroll
                    for (int k = 0; k < 6; k++) L3[6 * r + k] = X[k];
                }
                if (st == CNML_CREATED) { atomicOr(&s_bits[i1 >> 5], 1u << (i1 & 31)); created++; }
            }
            int all;
            block_exclusive_scan(created, s_warp, &all);
            created = all;
        }
        chain_pair_end(R, S, total, capl, bad, created, p, nmatch, nnew, tid);
    }
}

// sslpl_matcher_debug_svd4: svd4_jacobi on n row-major 4x4 matrices (W, Vt), glibc_hypot on nh pairs
__global__ void k_debug_svd4(int n, const float* A, float* W, float* Vt, int nh, const double* hx, const double* hy, double* h) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        float a[16], w[4], v[16];
#pragma unroll
        for (int k = 0; k < 16; k++) a[k] = A[16LL * i + k];
        svd4_jacobi(a, w, v);
#pragma unroll
        for (int k = 0; k < 4; k++) W[4LL * i + k] = w[k];
#pragma unroll
        for (int k = 0; k < 16; k++) Vt[16LL * i + k] = v[k];
    }
    if (i < nh) h[i] = glibc_hypot(hx[i], hy[i]);
}

// ---------------- MapPoint / MapLine ComputeDistinctiveDescriptors and UpdateNormalAndDepth / UpdateAverageDir (include/sslpl_map.h) ----------------
struct MapUpd {
    const float* kp; long long kp_fs; const uint8_t* desc; long long desc_fs; const int* n; int cap, nkf;   // the keyframe set
    const float* pose; const uint8_t* kfbad;
    int nel; float* el; uint8_t* eldesc; const double* pos; double* nrm64;    // element rows (lines: pos = mWorldPos in double)
    int nupd; const int32_t* elem; const int32_t* refkf; const int32_t* off; const int2* obs; const int32_t* first;
    int what, nlevels; float scale[SSLPL_MAX_LEVELS];
    int32_t* status;
};

// first[e] = the first entry of this call that names element e
__global__ void k_first_entry(const int32_t* elem, int nupd, int nel, int32_t* first) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nupd) return;
    const int e = elem[i];
    if ((unsigned)e < (unsigned)nel) atomicMin(first + e, i);
}

// One warp per entry.  The medoid is k_medoid's selection over the rows of the good keyframes, a lane per row.  The normal: the lanes
// compute each observation's ray and its scale in parallel, then every lane runs the sum in observation order (each step rounds on the
// previous one), reading the terms by shuffle.  Points: el[m][9] = Xw, normal, minInv, maxInv, maxRaw; lines: el[m][12] = SP, EP,
// normal, minInv, maxInv, maxRaw with the position read from pos[m][6].
template <bool kLine>
__global__ void __launch_bounds__(128) k_map_update(const __grid_constant__ MapUpd U) {
    constexpr int es = kLine ? 17 : 7, oct_at = kLine ? 2 : 5, ew = kLine ? 12 : 9;   // sslpl_keyline / sslpl_keypoint words, octave field
    constexpr unsigned full = 0xffffffffu;
    const int u = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (u >= U.nupd) return;
    const bool geom = U.what & SSLPL_MAPUPD_GEOM, dsc = U.what & SSLPL_MAPUPD_DESC;
    const int e = U.elem[u], o0 = U.off[u], N = U.off[u + 1] - o0, rk = geom ? U.refkf[u] : 0;
    bool bad = (unsigned)e >= (unsigned)U.nel || U.first[e] != u || o0 < 0 || N < 0 || N > U.nkf || (unsigned)rk >= (unsigned)U.nkf;
    if (!bad && N == 0) {
        if (lane == 0) U.status[u] = SSLPL_MAPUPD_NO_OBS;
        return;
    }
    const int2* obs = U.obs + o0;
    int refpos = INT_MAX;                                                  // first position of the reference keyframe in the list
    if (!bad) {
        bool b = false;
        for (int i = lane; i < N; i += 32) {
            const int2 q = obs[i];
            b |= (unsigned)q.x >= (unsigned)U.nkf || q.y < 0 || q.y >= min(U.n[min(max(q.x, 0), U.nkf - 1)], U.cap);
            for (int j = 0; j < i && !b; j++) b |= obs[j].x == q.x;
            if (q.x == rk) refpos = min(refpos, i);
        }
        bad = __any_sync(full, b);
        refpos = __reduce_min_sync(full, refpos);
    }
    int oct = 0;
    if (!bad && geom) {
        const int ridx = refpos < N ? obs[refpos].y : 0;                  // observations[pRefKF] default-inserts 0
        if (ridx >= min(U.n[rk], U.cap)) bad = true;
        else oct = __float_as_int(U.kp[U.kp_fs * rk + (long long)es * ridx + oct_at]);
    }
    if (bad) {
        if (lane == 0) U.status[u] = SSLPL_MAPUPD_BAD;
        return;
    }
    int st = SSLPL_MAPUPD_OK;
    if (dsc) {
        const auto good = [&](int j) { return U.kfbad == nullptr || !U.kfbad[obs[j].x]; };
        const auto row = [&](int j) { const int2 q = obs[j]; return U.desc + U.desc_fs * q.x + 32LL * q.y; };
        int ng = 0;
        for (int i = lane; i < N; i += 32) ng += good(i);
        ng = __reduce_add_sync(full, ng);
        if (ng == 0) {
            st = SSLPL_MAPUPD_NO_GOOD_KF;
        } else {
            const int r = (int)(0.5 * (double)(ng - 1));
            unsigned key = 0xffffffffu;
            for (int i = lane; i < N; i += 32)
                if (good(i)) key = min(key, medoid_key(row, good, N, r, i));
            key = __reduce_min_sync(full, key);
            if (lane < 8) reinterpret_cast<uint32_t*>(U.eldesc + 32LL * e)[lane] = reinterpret_cast<const uint32_t*>(row((int)(key & 0xfffffu)))[lane];
        }
    }
    if (!geom) {
        if (lane == 0) U.status[u] = st;
        return;
    }
    float* P = U.el + (long long)ew * e;
    const float* Oref = U.pose + 15LL * rk + 12;
    float nf[3], X[3];                                                     // the normal as stored; the point whose distance is taken
    if (!kLine) {
        // normal = normal + normali / cv::norm(normali): scaleAdd(normali, 1.0 / norm, normal), fma with the scale narrowed to float;
        // normal / n: convertTo with the scale 1.0 / n narrowed to float
        X[0] = P[0]; X[1] = P[1]; X[2] = P[2];
        float s0 = 0.f, s1 = 0.f, s2 = 0.f;
        for (int b = 0; b < N; b += 32) {
            float q0 = 0.f, q1 = 0.f, q2 = 0.f, a = 0.f;
            if (b + lane < N) {
                const float* Ow = U.pose + 15LL * obs[b + lane].x + 12;
                q0 = __fsub_rn(X[0], Ow[0]); q1 = __fsub_rn(X[1], Ow[1]); q2 = __fsub_rn(X[2], Ow[2]);
                a = __double2float_rn(__ddiv_rn(1.0, norm3d_d(q0, q1, q2)));
            }
            for (int j = 0; j < min(32, N - b); j++) {
                const float aj = __shfl_sync(full, a, j);
                s0 = __fmaf_rn(__shfl_sync(full, q0, j), aj, s0);
                s1 = __fmaf_rn(__shfl_sync(full, q1, j), aj, s1);
                s2 = __fmaf_rn(__shfl_sync(full, q2, j), aj, s2);
            }
        }
        const float inv = __double2float_rn(__ddiv_rn(1.0, (double)N));
        nf[0] = __fadd_rn(__fmul_rn(s0, inv), 0.f); nf[1] = __fadd_rn(__fmul_rn(s1, inv), 0.f); nf[2] = __fadd_rn(__fmul_rn(s2, inv), 0.f);
    } else {
        // Eigen in double: middlePos = 0.5 * (head + tail), normali = middlePos - OWi, normal += normali / normali.norm(), normal / n;
        // the distance from MP = 0.5 * (SP + EP) of the float narrowing (addWeighted)
        const double* W = U.pos + 6LL * e;
        const double m0 = __dmul_rn(0.5, __dadd_rn(W[0], W[3])), m1 = __dmul_rn(0.5, __dadd_rn(W[1], W[4])), m2 = __dmul_rn(0.5, __dadd_rn(W[2], W[5]));
        double s0 = 0.0, s1 = 0.0, s2 = 0.0;
        for (int b = 0; b < N; b += 32) {
            double q0 = 0.0, q1 = 0.0, q2 = 0.0;
            if (b + lane < N) {
                const float* Ow = U.pose + 15LL * obs[b + lane].x + 12;
                q0 = __dsub_rn(m0, (double)Ow[0]); q1 = __dsub_rn(m1, (double)Ow[1]); q2 = __dsub_rn(m2, (double)Ow[2]);
                const double nr = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(q0, q0), __dmul_rn(q1, q1)), __dmul_rn(q2, q2)));
                q0 = __ddiv_rn(q0, nr); q1 = __ddiv_rn(q1, nr); q2 = __ddiv_rn(q2, nr);
            }
            for (int j = 0; j < min(32, N - b); j++) {
                s0 = __dadd_rn(s0, __shfl_sync(full, q0, j));
                s1 = __dadd_rn(s1, __shfl_sync(full, q1, j));
                s2 = __dadd_rn(s2, __shfl_sync(full, q2, j));
            }
        }
        const double dn = (double)N;
        s0 = __ddiv_rn(s0, dn); s1 = __ddiv_rn(s1, dn); s2 = __ddiv_rn(s2, dn);
        if (U.nrm64 && lane == 0) { U.nrm64[3LL * e] = s0; U.nrm64[3LL * e + 1] = s1; U.nrm64[3LL * e + 2] = s2; }
        nf[0] = __double2float_rn(s0); nf[1] = __double2float_rn(s1); nf[2] = __double2float_rn(s2);
#pragma unroll
        for (int c = 0; c < 3; c++) X[c] = mid_aw(__double2float_rn(W[c]), __double2float_rn(W[c + 3]));
    }
    if (lane != 0) return;
    P[ew - 6] = nf[0]; P[ew - 5] = nf[1]; P[ew - 4] = nf[2];
    if (oct < 0 || oct >= U.nlevels) {
        st = SSLPL_MAPUPD_REF_OCTAVE;
    } else {
        const float dist = norm3d(__fsub_rn(X[0], Oref[0]), __fsub_rn(X[1], Oref[1]), __fsub_rn(X[2], Oref[2]));
        const float mx = __fmul_rn(dist, U.scale[oct]), mn = __fdiv_rn(mx, U.scale[U.nlevels - 1]);
        P[ew - 3] = __fmul_rn(0.8f, mn); P[ew - 2] = __fmul_rn(1.2f, mx); P[ew - 1] = mx;
    }
    U.status[u] = st;
}

// -------------------------------------------------------------------------------------------------
// Keyframe database (src/KeyFrameDatabase.cc) over a row set in HBM.  Every double sum below is sequential in ascending word order,
// as the reference's std::map walks run; the parallelism is across rows, pairs, queries and database positions only.
// -------------------------------------------------------------------------------------------------
struct BowRows { int32_t* word; double* val; int32_t* n; int cap; };

// BowVector of one row (TemplatedVocabulary::transform :1145-1195 with TF_IDF weighting and L1 scoring): k_vocab_transform left the
// row's word ids and leaf weights in word / val [r][cap].  One CTA per row: the (word, feature) keys of the weighted features are sorted
// in shared memory (P = a power of two >= cap), each run adds its weights in feature order (BowVector::addWeight :34-46), one thread
// takes the L1 norm in word order and every value is divided by it (normalize :62-84).  Entries past the count become (-1, 0.0).
__global__ void __launch_bounds__(512) k_bow_vector(BowRows B, const int* d_n, int P) {
    extern __shared__ unsigned long long s_key[];      // P keys, then cap weights (doubles)
    __shared__ int s_warp[33];
    __shared__ double s_norm;
    double* s_w = reinterpret_cast<double*>(s_key + P);
    const int r = blockIdx.x, tid = threadIdx.x, cap = B.cap;
    const int n = min(max(d_n[r], 0), cap);
    int32_t* W = B.word + (long long)r * cap; double* V = B.val + (long long)r * cap;
    for (int i = tid; i < P; i += blockDim.x) {
        unsigned long long k = ~0ull;
        if (i < n) {
            const double w = V[i];
            s_w[i] = w;
            if (w > 0) k = ((unsigned long long)(unsigned)W[i] << 32) | (unsigned)i;
        }
        s_key[i] = k;
    }
    __syncthreads();
    for (int k = 2; k <= P; k <<= 1)                   // bitonic sort, ascending
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < P; i += blockDim.x) {
                const int l = i ^ j;
                if (l > i) {
                    const unsigned long long a = s_key[i], b = s_key[l];
                    if ((a > b) == ((i & k) == 0)) { s_key[i] = b; s_key[l] = a; }
                }
            }
            __syncthreads();
        }
    // runs of equal words: run starts are numbered in order by a block scan over chunks of blockDim keys
    int nruns = 0;
    for (int base = 0; base < n; base += blockDim.x) {
        const int i = base + tid;
        const unsigned long long k = i < n ? s_key[i] : ~0ull;
        const bool start = k != ~0ull && (i == 0 || (s_key[i - 1] >> 32) != (k >> 32));
        int total;
        const int o = nruns + block_exclusive_scan(start ? 1 : 0, s_warp, &total);
        double sum = 0.0;
        if (start) {
            for (int j = i; j < n && (s_key[j] >> 32) == (k >> 32); j++) sum = __dadd_rn(sum, s_w[(unsigned)s_key[j]]);
        }
        if (start) { W[o] = (int32_t)(k >> 32); V[o] = sum; }
        nruns += total;
    }
    __syncthreads();
    if (tid == 0) {
        double norm = 0.0;
        for (int o = 0; o < nruns; o++) norm = __dadd_rn(norm, fabs(V[o]));
        s_norm = norm;
        B.n[r] = nruns;
    }
    __syncthreads();
    const double norm = s_norm;
    for (int o = tid; o < cap; o += blockDim.x) {
        if (o < nruns) { if (norm > 0.0) V[o] = __ddiv_rn(V[o], norm); }
        else { W[o] = -1; V[o] = 0.0; }
    }
}

// L1Scoring::score (ScoringObject.cpp:23-67) of a sorted BowVector (qw, qv, nq) against row r: the common words in ascending order, each
// term ((|v - w| - |v|) - |w|) added to the sum in that order; the caller negates and halves.  The merge visits the same common words
// as the reference's lower_bound jumps.
__device__ __forceinline__ double l1_sum(const int32_t* qw, const double* qv, int nq, const int32_t* dw, const double* dv, int nd) {
    double s = 0.0;
    int i = 0, j = 0;
    while (i < nq && j < nd) {
        const int a = qw[i], b = dw[j];
        if (a == b) {
            const double vi = qv[i], wi = dv[j];
            s = __dadd_rn(s, __dsub_rn(__dsub_rn(fabs(__dsub_rn(vi, wi)), fabs(vi)), fabs(wi)));
            i++; j++;
        } else if (a < b) i++;
        else j++;
    }
    return s;
}

__device__ __forceinline__ int bow_count(const BowRows& B, int r) { return min(max(B.n[r], 0), B.cap); }

// TemplatedVocabulary::score(v1, v2) for row pairs; NaN for a pair with a row outside [0, nrows).  Thread per pair.
__global__ void __launch_bounds__(128) k_bow_score(BowRows B, int nrows, int npairs, const int2* pair, double* score) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= npairs) return;
    const int2 q = pair[p];
    if ((unsigned)q.x >= (unsigned)nrows || (unsigned)q.y >= (unsigned)nrows) { score[p] = __longlong_as_double(0x7ff8000000000000LL); return; }
    const long long o1 = (long long)q.x * B.cap, o2 = (long long)q.y * B.cap;
    const double s = l1_sum(B.word + o1, B.val + o1, bow_count(B, q.x), B.word + o2, B.val + o2, bow_count(B, q.y));
    score[p] = __ddiv_rn(-s, 2.0);
}

// The database of one call: its rows in add order, the row -> position map (-1: not in the database), the error word (non-zero: a
// database row outside [0, nrows) or listed twice, which fails every query) and maxw[q], the largest word count of query q.
struct KfdbArgs {
    BowRows B; int nrows;
    const int32_t* db; int ndb; int32_t* pos_of_row; int32_t* err; int32_t* maxw;
    const int32_t* query; int nq;
    const int32_t* covis;                        // [nrows][10], -1 padded
    const int32_t* conn_off; const int32_t* conn; int nconn; const float* minscore;    // loop only
    float* relocscore;                           // reloc only
    int32_t* cand; int32_t* ncand; int32_t* words; float* score;
};
constexpr int KFDB_POS_BITS = 15;               // sort key of a listed keyframe: (index of its first common word in the query) << 15 | position
constexpr int KFDB_CHUNK = 128;                 // database positions per CTA of k_kfdb_count / k_kfdb_score, one per thread

__global__ void k_kfdb_posmap(KfdbArgs A) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= A.ndb) return;
    const int r = A.db[p];
    if ((unsigned)r >= (unsigned)A.nrows || atomicCAS(A.pos_of_row + r, -1, p) != -1) atomicOr(A.err, 1);
}

// a query row outside [0, nrows), or (loop) a connected-keyframe range outside [0, nconn), fails the query; a bad database fails all
template <bool kLoop>
__device__ __forceinline__ bool kfdb_query_ok(const KfdbArgs& A, int q) {
    if (*A.err != 0 || (unsigned)A.query[q] >= (unsigned)A.nrows) return false;
    if (!kLoop) return true;
    const int c0 = A.conn_off[q], c1 = A.conn_off[q + 1];
    return 0 <= c0 && c0 <= c1 && c1 <= A.nconn;
}

__device__ __forceinline__ int block_max(int v, int* s_red) {
    for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    int m = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) m = max(m, s_red[w]);
    return m;
}

// minCommonWords = maxCommonWords * 0.8f, a float product truncated to int (KeyFrameDatabase.cc:132, 243)
__device__ __forceinline__ int min_common_words(int maxw) { return (int)__fmul_rn((float)maxw, 0.8f); }

// the query's BowVector into shared memory: cap values, then cap word ids; returns its length
__device__ __forceinline__ int stage_query(const KfdbArgs& A, int qr, double* s_qv) {
    const int cap = A.B.cap, nqw = bow_count(A.B, qr);
    int32_t* s_qw = reinterpret_cast<int32_t*>(s_qv + cap);
    for (int i = threadIdx.x; i < nqw; i += blockDim.x) { s_qv[i] = A.B.val[(long long)qr * cap + i]; s_qw[i] = A.B.word[(long long)qr * cap + i]; }
    __syncthreads();
    return nqw;
}

// Word counts and first common words of query blockIdx.y against KFDB_CHUNK database positions (a thread per position, a merge of the
// query's BowVector, staged in shared memory, against the position's).  words[q][p] = mnLoopWords / mnRelocWords (0: not listed,
// connected keyframes of a loop query included), cand[q][p] = the listed position's sort key (-1: not listed) for k_kfdb_accumulate,
// score[q][p] = NaN until k_kfdb_score; the chunk's largest count goes to maxw[q].  A failed query leaves 0 / NaN / -1.
template <bool kLoop>
__global__ void __launch_bounds__(KFDB_CHUNK) k_kfdb_count(KfdbArgs A) {
    extern __shared__ double s_qv[];
    __shared__ int s_red[32];
    __shared__ unsigned char s_conn[KFDB_CHUNK];
    const int q = blockIdx.y, tid = threadIdx.x, p0 = blockIdx.x * KFDB_CHUNK, p = p0 + tid;
    const long long qo = (long long)q * A.ndb;
    const bool in = p < A.ndb;
    if (in) { A.words[qo + p] = 0; A.score[qo + p] = __int_as_float(0x7fc00000); A.cand[qo + p] = -1; }
    if (!kfdb_query_ok<kLoop>(A, q)) return;
    s_conn[tid] = 0;
    const int nqw = stage_query(A, A.query[q], s_qv);
    if (kLoop) {                                  // GetConnectedKeyFrames() of the query: never listed (:98-108)
        for (int c = A.conn_off[q] + tid; c < A.conn_off[q + 1]; c += blockDim.x) {
            const int r = A.conn[c];
            const int cp = (unsigned)r < (unsigned)A.nrows ? A.pos_of_row[r] : -1;
            if (cp >= p0 && cp < p0 + KFDB_CHUNK) s_conn[cp - p0] = 1;
        }
        __syncthreads();
    }
    int cnt = 0;
    if (in && !s_conn[tid]) {
        const int32_t* s_qw = reinterpret_cast<const int32_t*>(s_qv + A.B.cap);
        const int r = A.db[p];
        const int32_t* dw = A.B.word + (long long)r * A.B.cap;
        const int nd = bow_count(A.B, r);
        int first = -1, i = 0, j = 0;
        while (i < nqw && j < nd) {
            const int a = s_qw[i], b = dw[j];
            if (a == b) { if (cnt == 0) first = i; cnt++; i++; j++; }
            else if (a < b) i++;
            else j++;
        }
        A.words[qo + p] = cnt;
        if (cnt) A.cand[qo + p] = (first << KFDB_POS_BITS) | p;
    }
    const int m = block_max(cnt, s_red);
    if (tid == 0 && m > 0) atomicMax(A.maxw + q, m);
}

// mLoopScore / mRelocScore, si = (float)score(query, kf), of the positions of the chunk with more than minCommonWords common words
template <bool kLoop>
__global__ void __launch_bounds__(KFDB_CHUNK) k_kfdb_score(KfdbArgs A) {
    extern __shared__ double s_qv[];
    const int q = blockIdx.y, p = blockIdx.x * KFDB_CHUNK + threadIdx.x;
    const long long qo = (long long)q * A.ndb;
    if (!kfdb_query_ok<kLoop>(A, q)) return;
    const bool need = p < A.ndb && A.words[qo + p] > min_common_words(A.maxw[q]);
    if (!__syncthreads_or(need)) return;
    const int nqw = stage_query(A, A.query[q], s_qv);
    if (!need) return;
    const long long o = (long long)A.db[p] * A.B.cap;
    const double s = l1_sum(reinterpret_cast<const int32_t*>(s_qv + A.B.cap), s_qv, nqw, A.B.word + o, A.B.val + o, bow_count(A.B, A.db[p]));
    A.score[qo + p] = __double2float_rn(__ddiv_rn(-s, 2.0));
}

// The covisibility accumulation, retention and deduplication of one query (CTA) (:146-201 loop, :259-313 reloc).  lScoreAndMatch is
// the scored positions (loop: si >= minScore) in the order of their sort keys, sorted here in shared memory; accScore / pBestKF of an
// entry depend on no other entry, so they are computed in parallel, and the first occurrence of each pBestKF in that order is found with
// an atomicMin on the entry index in cand[q][pBestKF's position] before cand[q] receives the result.  Reloc: a listed neighbour this
// query did not score reads the score of the latest earlier query of the call that scored it, else relocscore[row].
template <bool kLoop>
__global__ void __launch_bounds__(512) k_kfdb_accumulate(KfdbArgs A) {
    extern __shared__ int s_ent[];                // per entry: sort key, then pBestKF's position; then accScore (floats)
    __shared__ int s_red[33];
    __shared__ int s_cnt;
    const int q = blockIdx.x, tid = threadIdx.x, ndb = A.ndb;
    const long long qo = (long long)q * ndb;
    float* s_acc = reinterpret_cast<float*>(s_ent + ndb);
    if (!kfdb_query_ok<kLoop>(A, q)) { if (tid == 0) A.ncand[q] = -1; return; }
    const int minw = min_common_words(A.maxw[q]);
    const float minScore = kLoop ? A.minscore[q] : 0.f;
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    for (int p = tid; p < ndb; p += blockDim.x)
        if (A.words[qo + p] > minw && (!kLoop || A.score[qo + p] >= minScore)) s_ent[atomicAdd(&s_cnt, 1)] = A.cand[qo + p];
    __syncthreads();
    const int ne = s_cnt;
    int P = 1;
    while (P < ne) P <<= 1;
    for (int k = 2; k <= P; k <<= 1)              // bitonic sort of ne keys; the missing tail of the power of two counts as +inf
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < ne; i += blockDim.x) {
                const int l = (j == (k >> 1)) ? (i ^ (k - 1)) : (i ^ j);
                if (l > i && l < ne) {
                    const int a = s_ent[i], b = s_ent[l];
                    if (a > b) { s_ent[i] = b; s_ent[l] = a; }
                }
            }
            __syncthreads();
        }
    float best_acc = minScore;
    for (int e = tid; e < ne; e += blockDim.x) {
        const int p = s_ent[e] & ((1 << KFDB_POS_BITS) - 1);
        const float si = A.score[qo + p];
        float acc = si, bestScore = si;
        int bestp = p;
        const int32_t* nb = A.covis + (long long)A.db[p] * 10;
        for (int c = 0; c < 10; c++) {
            const int r2 = nb[c];
            const int p2 = (unsigned)r2 < (unsigned)A.nrows ? A.pos_of_row[r2] : -1;
            if (p2 < 0) continue;
            const int w2 = A.words[qo + p2];
            if (w2 <= (kLoop ? minw : 0)) continue;
            float s2 = A.score[qo + p2];
            if (!kLoop && w2 <= minw) {
                int q2 = q - 1;
                while (q2 >= 0 && isnan(A.score[(long long)q2 * ndb + p2])) q2--;
                s2 = q2 >= 0 ? A.score[(long long)q2 * ndb + p2] : A.relocscore[r2];
            }
            acc = __fadd_rn(acc, s2);
            if (s2 > bestScore) { bestp = p2; bestScore = s2; }
        }
        s_acc[e] = acc;
        best_acc = fmaxf(best_acc, acc);
        s_ent[e] = bestp;
    }
    for (int o = 16; o > 0; o >>= 1) best_acc = fmaxf(best_acc, __shfl_xor_sync(0xffffffffu, best_acc, o));
    __syncthreads();
    if ((tid & 31) == 0) s_red[tid >> 5] = __float_as_int(best_acc);
    for (int p = tid; p < ndb; p += blockDim.x) A.cand[qo + p] = INT_MAX;
    __syncthreads();
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) best_acc = fmaxf(best_acc, __int_as_float(s_red[w]));
    const float keep = __fmul_rn(0.75f, best_acc);
    for (int e = tid; e < ne; e += blockDim.x)
        if (s_acc[e] > keep) atomicMin(A.cand + qo + s_ent[e], e);
    __syncthreads();
    for (int e = tid; e < ne; e += blockDim.x)     // s_acc[e] becomes the entry's output flag
        s_acc[e] = (s_acc[e] > keep && A.cand[qo + s_ent[e]] == e) ? 1.f : 0.f;
    __syncthreads();
    int nout = 0;
    for (int base = 0; base < ne; base += blockDim.x) {
        const int e = base + tid;
        const bool out = e < ne && s_acc[e] != 0.f;
        int total;
        const int o = nout + block_exclusive_scan(out ? 1 : 0, s_red, &total);
        if (out) A.cand[qo + o] = A.db[s_ent[e]];
        nout += total;
    }
    __syncthreads();
    for (int p = nout + tid; p < ndb; p += blockDim.x) A.cand[qo + p] = -1;
    if (tid == 0) A.ncand[q] = nout;
}

// After a reloc call: each database keyframe keeps the score of the last query that scored it (mRelocScore, :241).
__global__ void k_kfdb_reloc_state(KfdbArgs A) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= A.ndb || *A.err) return;
    for (int q = A.nq - 1; q >= 0; q--) {
        const float s = A.score[(long long)q * A.ndb + p];
        if (!isnan(s)) { A.relocscore[A.db[p]] = s; return; }
    }
}

// -------------------------------------------------------------------------------------------------
// Tracking::Relocalization (Tracking.cc:1961-2121) on the device.  k_reloc_pairs turns DetectRelocalizationCandidates' table into
// (candidate keyframe row, query row) pairs, slot q * kmax + k for the candidate of rank k; (-1, -1) past min(ncand[q], kmax, ndb).
// -------------------------------------------------------------------------------------------------
__global__ void k_reloc_pairs(int nq, const int32_t* query, const int32_t* cand, const int32_t* ncand, int ndb, int kmax, int2* pair) {
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= (long long)nq * kmax) return;
    const int q = (int)(s / kmax), k = (int)(s % kmax);
    pair[s] = k < min(ncand[q], min(kmax, ndb)) ? make_int2(cand[(long long)q * ndb + k], query[q]) : make_int2(-1, -1);
}

// ORBmatcher::SearchByProjection(Frame &F, KeyFrame *pKF, sAlreadyFound, th, ORBdist) — ORBmatcher.cc:1475-1602, run after PnP and
// PoseOptimization on each candidate.  Pair p = (keyframe row, frame row) of a row set (sslpl_keypoint rows, descriptors, counts, all of
// stride cap); the keyframe's MapPoints are element indices kfmp[row][i] into el[m][9] = Xw, normal, GetMinDistanceInvariance(),
// GetMaxDistanceInvariance(), mfMaxDistance and eldesc[m][32] (the Fuse / map-refresh element table).
struct RelocArgs {
    float fx, fy, cx, cy, th;
    int ORBdist, checkOri;
    GridGeom G;                                      // the frame's bounds, grid and mvScaleFactors
    PredictTable T;                                  // MapPoint::PredictScale(dist, Frame*) (MapPoint.cc:407-422) with the frame's mfLogScaleFactor
};
struct RelocSet {
    const int2* pair; int npairs, nrows, cap;
    const float* kp; const uint8_t* desc; const int* n;               // row r at kp + 7 cap r, desc + 32 cap r; n[r] clamped to [0, cap]
    const int32_t* kfmp; const uint8_t* mpbad; const float* el; const uint8_t* eldesc; int nel;
    const float* Tcw;                                // pair p's pose at Tcw + 12 p
    const uint8_t* found; const uint8_t* held;       // [p][cap]: sAlreadyFound.count(vpMPs[i]), F.mvpMapPoints[j] != NULL (NULL = none)
    float* xy; int* wn; const int* goff; const int* gidx; long long goff_fs;   // per pair: the frame's (x, y) rows and count, its grid CSR
    uint8_t* claimed; int32_t* sel; uint8_t* rbin; long long ws_fs;            // per pair walker tables
    int32_t* assign; int32_t* nmatch;                // [p][cap], [p]
};

__device__ __forceinline__ bool reloc_pair(const RelocSet& R, int p, int& kr, int& fr) {
    const int2 q = R.pair[p];
    kr = q.x; fr = q.y;
    return (unsigned)kr < (unsigned)R.nrows && (unsigned)fr < (unsigned)R.nrows;
}
__device__ __forceinline__ int reloc_count(const RelocSet& R, int r) { return min(max(R.n[r], 0), R.cap); }

// The (x, y) of pair p's frame rows into the pair's slot, for k_grid_cells / k_build_csr (an invalid pair gets no features)
__global__ void __launch_bounds__(128) k_reloc_gather_xy(const __grid_constant__ RelocSet R) {
    const int p = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    int kr, fr;
    const bool ok = reloc_pair(R, p, kr, fr);
    const int n = ok ? reloc_count(R, fr) : 0;
    if (i == 0) R.wn[p] = n;
    if (i >= n) return;
    const float* k = R.kp + 7LL * R.cap * fr + 7LL * i;
    R.xy[(long long)p * 2 * R.ws_fs + 2 * i] = k[0];
    R.xy[(long long)p * 2 * R.ws_fs + 2 * i + 1] = k[1];
}

// One warp per pair.  The keyframe's MapPoints are walked in index order (an assignment makes the frame feature unavailable to later
// points); the lanes share each search window.
__global__ void __launch_bounds__(32) k_proj_match_kf(const __grid_constant__ RelocArgs A, const __grid_constant__ RelocSet R) {
    __shared__ int s_hist[HISTO_LENGTH];
    __shared__ float s_T[12], s_Ow[3];
    const int lane = threadIdx.x, p = blockIdx.x;
    int32_t* assign = R.assign + (long long)p * R.cap;
    for (int j = lane; j < R.cap; j += 32) assign[j] = -1;
    int kr, fr;
    if (!reloc_pair(R, p, kr, fr)) { if (lane == 0) R.nmatch[p] = -1; return; }
    const int n1 = reloc_count(R, kr), n2 = reloc_count(R, fr);
    const float* kp1 = R.kp + 7LL * R.cap * kr; const float* kp2 = R.kp + 7LL * R.cap * fr;
    const uint8_t* d2 = R.desc + 32LL * R.cap * fr;
    const int32_t* kfmp = R.kfmp + (long long)R.cap * kr;
    const uint8_t* found = R.found ? R.found + (long long)p * R.cap : nullptr;
    const uint8_t* held = R.held ? R.held + (long long)p * R.cap : nullptr;
    const int* goff = R.goff + p * R.goff_fs; const int* gidx = R.gidx + p * R.ws_fs;
    uint8_t* claimed = R.claimed + p * R.ws_fs; int32_t* sel = R.sel + p * R.ws_fs; uint8_t* rbin = R.rbin + p * R.ws_fs;
    if (lane < 12) s_T[lane] = R.Tcw[12LL * p + lane];
    if (lane < HISTO_LENGTH) s_hist[lane] = 0;
    for (int j = lane; j < n2; j += 32) claimed[j] = held && held[j] ? 1 : 0;         // a frame feature holding any MapPoint is skipped (:1543)
    __syncwarp();
    // Ow = -Rcw.t()*tcw (:1480): a transposed operand takes cv::gemm's general path, double accumulation (as twc in k_proj_match)
    if (lane < 3) s_Ow[lane] = __double2float_rn(-__dadd_rn(__dadd_rn(__dmul_rn((double)s_T[lane], (double)s_T[3]),
                                                                     __dmul_rn((double)s_T[4 + lane], (double)s_T[7])),
                                                           __dmul_rn((double)s_T[8 + lane], (double)s_T[11])));
    __syncwarp();
    const float* T = s_T;
    int nmatches = 0;
    for (int i = 0; i < n1; i++) {
        if (lane == 0) sel[i] = -1;
        const int e = kfmp[i];
        if ((unsigned)e >= (unsigned)R.nel) continue;                                  // NULL (:1497)
        if ((R.mpbad && R.mpbad[e]) || (found && found[i])) continue;                  // :1499
        const float* P = R.el + 9LL * e;
        const float X0 = P[0], X1 = P[1], X2 = P[2];
        // no depth test: a point behind the camera is searched when it projects inside the bounds; z = 0 gives inf / NaN, which either
        // fails the bounds or finds no feature in the window (every comparison with NaN is false)
        const float xc = rt_row(T, X0, X1, X2), yc = rt_row(T + 4, X0, X1, X2), zc = rt_row(T + 8, X0, X1, X2);
        const float invzc = (float)(1.0 / (double)zc);
        const float u = __fadd_rn(__fmul_rn(__fmul_rn(A.fx, xc), invzc), A.cx), v = __fadd_rn(__fmul_rn(__fmul_rn(A.fy, yc), invzc), A.cy);
        if (u < A.G.minX || u > A.G.maxX || v < A.G.minY || v > A.G.maxY) continue;
        const float dist3D = norm3d(__fsub_rn(X0, s_Ow[0]), __fsub_rn(X1, s_Ow[1]), __fsub_rn(X2, s_Ow[2]));
        if (dist3D < P[6] || dist3D > P[7]) continue;                                 // :1523-1524
        const int lvl = predict_scale(__fdiv_rn(P[8], dist3D), A.T.thr, A.T.nlevels, true);
        const float r = __fmul_rn(A.th, A.G.scale[lvl]);
        GridWin w;                                                                     // GetFeaturesInArea(u, v, r, lvl - 1, lvl + 1)
        if (!grid_window(A.G, u, v, r, w)) continue;
        uint4 a0, a1;
        load_desc(R.eldesc + 32LL * e, a0, a1);
        const unsigned long long best = grid_min(goff, gidx, w, lane, [&](int j, int& d) {
            const int o = __float_as_int(kp2[7LL * j + 5]);
            if (o < lvl - 1 || o > lvl + 1) return false;
            if (!(fabsf(__fsub_rn(kp2[7LL * j], u)) < r && fabsf(__fsub_rn(kp2[7LL * j + 1], v)) < r)) return false;
            if (claimed[j]) return false;
            uint4 b0, b1;
            load_desc(d2 + 32LL * j, b0, b1);
            d = popc256(a0, a1, b0, b1);
            return true;
        });
        if (best != ~0ull && (int)(best >> 40) <= A.ORBdist) {                        // :1561 (ORBdist < 256: no candidate never passes)
            const int j = grid_key_feature(goff, gidx, w, best);
            if (lane == 0) {
                assign[j] = i; claimed[j] = 1; sel[i] = j;
                const int bin = rot_bin(kp1[7LL * i + 3], kp2[7LL * j + 3]);             // pKF->mvKeysUn[i].angle - F.mvKeysUn[j].angle (:1568)
                rbin[i] = (uint8_t)bin;
                if (A.checkOri) s_hist[bin]++;
            }
            nmatches++;
        }
        __syncwarp();
    }
    __syncwarp();
    if (A.checkOri)                                                                    // assigned, then NULLed by the rotation check (:1595)
        nmatches -= warp_rot_check(s_hist, n1, lane, [&](int i) { return sel[i] >= 0 ? (int)rbin[i] : -1; },
                                   [&](int i) { assign[sel[i]] = -2; });
    if (lane == 0) R.nmatch[p] = nmatches;
}

}  // namespace sslpl

// =================================================================================================
using namespace sslpl;

struct sslpl_vocab {
    int device = 0, k = 0, L = 0, nnodes = 0, nwords = 0;
    int scoring = 0, weighting = 0;      // DBoW2 ScoringType / WeightingType: L1_NORM / TF_IDF unless a text file's header says otherwise
    uint8_t* arena = nullptr;
    sslpl::VocabView view{};
    std::vector<int> depth;              // per node
    std::vector<int> level_count;        // nodes per depth
};

struct sslpl_matcher : sslpl::StreamHandle {
    sslpl_matcher_params p;
    int cap = 0;                     // rows per frame slot of the single-call staging (max(features, lines))
    // single-call staging: 2 frame slots
    uint8_t* desc; int* nodes; int* off; int* idx; uint8_t* flag; float* kpf; int* nn2; int* ncnt;
    int32_t* out; uint8_t* rot; uint8_t* taken; int32_t* pairs; int32_t* nmatch; int32_t* knn; uint8_t* cent; int32_t* node;
    int32_t* word; double* wgt;      // per-feature outputs of the vocabulary transform (single-call staging)
    // batch workspace
    int32_t* b_node; int* b_off; int* b_idx; uint8_t* b_rot; uint8_t* b_taken; int32_t* b_knn; int* iota;
    // workspace of sslpl_search_by_projection_frame_batch_device, allocated by its first call: per frame the grid cell of every
    // feature and the grid CSR, per pair the walker's claimed / sel / rbin tables ([max_batch + 1][max_features + 64] each)
    uint8_t* pw = nullptr;
    int32_t* pw_cell = nullptr; int* pw_off = nullptr; int* pw_idx = nullptr; int32_t* pw_sel = nullptr; uint8_t* pw_claimed = nullptr; uint8_t* pw_rbin = nullptr;
    // per-pair match table of sslpl_search_for_triangulation_batch_device ([max_batch][max_features + 64]), allocated by its first call
    int32_t* tw = nullptr;
    // per-pair row table of sslpl_create_new_map_lines_batch_device ([max_batch][max_lines + 64]), allocated by its first call
    int32_t* ltw = nullptr;
    // workspace of the SearchByProjection(Frame, KeyFrame) calls, allocated by the first one: per pair ([max_batch][cap]) the frame's
    // (x, y) rows, grid cells and CSR and the walker's tables; the single call's element table, pair and pose
    uint8_t* rw = nullptr;
    float* rw_xy = nullptr; int* rw_n = nullptr; int32_t* rw_cell = nullptr; int* rw_off = nullptr; int* rw_idx = nullptr;
    int32_t* rw_sel = nullptr; uint8_t* rw_claimed = nullptr; uint8_t* rw_rbin = nullptr;
    float* rw_el = nullptr; uint8_t* rw_eldesc = nullptr; int32_t* rw_kfmp = nullptr; int32_t* rw_pair = nullptr; float* rw_T = nullptr;
    int32_t* rw_nmatch = nullptr;
    // workspace of sslpl_search_by_bow_batch_device, allocated by its first call: per slot ([2 max_batch]) its row, count, node indices
    // and FeatureVector CSR; per pair its two slots and its frame's count
    uint8_t* kb = nullptr;
    int32_t* kb_row = nullptr; int* kb_n = nullptr; int32_t* kb_node = nullptr; int* kb_off = nullptr; int* kb_idx = nullptr;
    int2* kb_pslot = nullptr; int* kb_fn = nullptr;
    // per-chain scratch of sslpl_search_for_initialization_batch_device ([max_batch][max_features + 64]), allocated by its first call
    uint8_t* iw = nullptr;
    int* iw_dist = nullptr; int* iw_m21 = nullptr; uint8_t* iw_rbin = nullptr;
};

namespace {

int carve(sslpl_matcher* m, Arena& A) {
    const int cap = m->cap, NN = m->p.max_nodes + 1, B = m->p.max_batch + 1;
    m->desc = A.take<uint8_t>((size_t)2 * cap * 32);
    m->nodes = A.take<int>((size_t)2 * NN); m->off = A.take<int>((size_t)2 * (NN + 1)); m->idx = A.take<int>((size_t)2 * cap);
    m->flag = A.take<uint8_t>((size_t)2 * cap);
    m->kpf = A.take<float>((size_t)2 * cap * 7);
    m->nn2 = A.take<int>(2); m->ncnt = A.take<int>(2);
    m->out = A.take<int32_t>(cap); m->rot = A.take<uint8_t>(cap); m->taken = A.take<uint8_t>(cap);
    m->pairs = A.take<int32_t>((size_t)2 * cap); m->nmatch = A.take<int32_t>(B);
    m->knn = A.take<int32_t>((size_t)4 * cap);
    m->cent = A.take<uint8_t>((size_t)NN * 32); m->node = A.take<int32_t>(cap);
    m->word = A.take<int32_t>(cap); m->wgt = A.take<double>(cap);
    const int fc = m->p.max_features + 64, lc = m->p.max_lines + 64;
    m->b_node = A.take<int32_t>((size_t)B * fc); m->b_off = A.take<int>((size_t)B * (NN + 1)); m->b_idx = A.take<int>((size_t)B * fc);
    m->b_rot = A.take<uint8_t>((size_t)B * fc); m->b_taken = A.take<uint8_t>((size_t)B * fc);
    m->b_knn = A.take<int32_t>((size_t)B * lc * 4);
    m->iota = A.take<int>(NN);
    return 0;
}

int featvec_ok(const sslpl_matcher* m, const sslpl_featvec* fv, int n) {
    SSLPL_REQUIRE(fv && fv->nn >= 0 && fv->nn <= m->p.max_nodes, SSLPL_ERR_ARG, "feature vector has more nodes than max_nodes");
    if (fv->nn == 0) return SSLPL_OK;
    SSLPL_REQUIRE(fv->nodes && fv->off && fv->idx, SSLPL_ERR_ARG, "null feature vector arrays");
    SSLPL_REQUIRE(fv->off[fv->nn] <= n, SSLPL_ERR_ARG, "feature vector indexes more features than given");
    return SSLPL_OK;
}

// a feature vector that featvec_ok accepted
int upload_featvec(sslpl_matcher* m, int slot, const sslpl_featvec* fv) {
    const int NN = m->p.max_nodes + 1;
    if (fv->nn == 0) return SSLPL_OK;
    SSLPL_CUDA(cudaMemcpyAsync(m->nodes + slot * NN, fv->nodes, sizeof(int) * fv->nn, cudaMemcpyHostToDevice, m->stream));
    SSLPL_CUDA(cudaMemcpyAsync(m->off + slot * (NN + 1), fv->off, sizeof(int) * (fv->nn + 1), cudaMemcpyHostToDevice, m->stream));
    SSLPL_CUDA(cudaMemcpyAsync(m->idx + slot * m->cap, fv->idx, sizeof(int) * fv->off[fv->nn], cudaMemcpyHostToDevice, m->stream));
    return SSLPL_OK;
}

FrameSet staging_set(sslpl_matcher* m) {
    const int NN = m->p.max_nodes + 1;
    FrameSet S; memset(&S, 0, sizeof(S));
    S.desc = m->desc; S.desc_fs = (long long)m->cap * 32;
    S.nodes = m->nodes; S.off = m->off; S.idx = m->idx; S.nodes_fs = NN; S.off_fs = NN + 1; S.idx_fs = m->cap;
    S.nn = m->nn2;
    S.flag = m->flag; S.flag_fs = m->cap;
    S.angle = m->kpf + 3; S.x = m->kpf; S.y = m->kpf + 1; S.oct = reinterpret_cast<const int*>(m->kpf + 5);
    S.angle_es = 7; S.angle_fs = (long long)m->cap * 7;
    return S;
}

// A frame set in HBM ([..][cap] descriptors and sslpl_keypoint rows) whose FeatureVectors k_build_csr wrote into b_off / b_idx for a
// dense vocabulary level: every frame lists the nodes 0..nc-1, so all share the iota array
FrameSet dense_set(sslpl_matcher* m, const uint8_t* d_desc, const sslpl_keypoint* d_kps, int cap, int nc, const uint8_t* flag) {
    FrameSet S; memset(&S, 0, sizeof(S));
    S.desc = d_desc; S.desc_fs = (long long)cap * 32;
    S.nodes = m->iota; S.nodes_fs = 0; S.nn = nullptr; S.nn_const = nc;
    S.off = m->b_off; S.idx = m->b_idx; S.off_fs = m->p.max_nodes + 2; S.idx_fs = m->p.max_features + 64;
    S.flag = flag; S.flag_fs = cap;
    const float* kf = reinterpret_cast<const float*>(d_kps);
    S.angle = kf + 3; S.x = kf; S.y = kf + 1; S.oct = reinterpret_cast<const int*>(kf + 5); S.angle_es = 7; S.angle_fs = (long long)cap * 7;
    return S;
}

int fill(sslpl_matcher* m, int32_t* p, long long n, int v) {
    if (n <= 0) return SSLPL_OK;
    launch(m, k_fill_i32, (unsigned)((n + 255) / 256), 256, 0, p, n, v);
    return SSLPL_OK;
}

// k_build_csr keeps nc + 1 counters and a frame's cap node ids in shared memory
int csr_fits(int nc, int cap) {
    SSLPL_REQUIRE((size_t)((nc + 1 + cap) * sizeof(int)) <= (size_t)MAX_DYN_SMEM, SSLPL_ERR_CAPACITY,
                  "nodes + features exceed the shared memory of one CTA ((nc + 1 + cap) * 4 <= 200 KB)");
    return SSLPL_OK;
}

// The single-pair grid matchers build the 64 x 48 grid CSR of the current frame in staging slot 1 of the node lists (max_nodes >= 3072)
// with one k_build_csr CTA; at most 8192 features keep that CTA within MAX_DYN_SMEM.
constexpr int GRID_MAX_FEATURES = 8192;
static_assert((GRID_COLS * GRID_ROWS + 1 + GRID_MAX_FEATURES + 64) * sizeof(int) <= MAX_DYN_SMEM, "grid CSR of one frame exceeds MAX_DYN_SMEM");
int grid_staging_ok(const sslpl_matcher* m) {
    SSLPL_REQUIRE(m->cap <= GRID_MAX_FEATURES + 64, SSLPL_ERR_ARG, "the matcher capacity exceeds 8192 features");
    SSLPL_REQUIRE(m->p.max_nodes >= GRID_COLS * GRID_ROWS, SSLPL_ERR_ARG, "the matcher needs max_nodes >= 3072 (64 x 48 grid cells)");
    return SSLPL_OK;
}
// Frame::AssignFeaturesToGrid of the n2 features at (x[i], y[i]) into goff / gidx.  h_small is written here: the caller has synchronised
// the stream since h_small's last asynchronous copy, and does not write it again before its next synchronisation.
int grid_staging_build(sslpl_matcher* m, const float* x, const float* y, int n2, const GridGeom& G, int*& goff, int*& gidx) {
    const int nc = GRID_COLS * GRID_ROWS;
    goff = m->off + (m->p.max_nodes + 2); gidx = m->idx + m->cap;
    m->h_small[0] = n2;
    SSLPL_CUDA(cudaMemcpyAsync(m->ncnt, m->h_small, sizeof(int), cudaMemcpyHostToDevice, m->stream));
    launch(m, k_grid_cells, (n2 + 127) / 128, 128, 0, x, y, 1, 0, nullptr, n2, n2, G, m->node, 0);
    launch(m, k_build_csr, 1, 128, (nc + 1 + m->cap) * sizeof(int), m->node, 0, m->ncnt, m->cap, nc, goff, 0, gidx, 0);
    return SSLPL_OK;
}

// The per-frame grid workspace of the batched projection matchers ([max_batch + 1] frames): per frame the grid cell of every feature
// and the grid CSR, and the motion-model walker's claimed / sel / rbin tables.
int ensure_grid_ws(sslpl_matcher* m) {
    const int B = m->p.max_batch + 1, fc = m->p.max_features + 64, nc = GRID_COLS * GRID_ROWS;
    Arena W;
    for (int k = 0; k < 2; k++) {
        m->pw_cell = W.take<int32_t>((size_t)B * fc); m->pw_off = W.take<int>((size_t)B * (nc + 1)); m->pw_idx = W.take<int>((size_t)B * fc);
        m->pw_sel = W.take<int32_t>((size_t)B * fc); m->pw_claimed = W.take<uint8_t>((size_t)B * fc); m->pw_rbin = W.take<uint8_t>((size_t)B * fc);
        if (k == 0) {
            if (int rc = first_use(m->pw, W.used)) return rc;
            W.base = m->pw; W.size = W.used; W.used = 0;
        }
    }
    return SSLPL_OK;
}
// Frame::AssignFeaturesToGrid of nframes frames in HBM (sslpl_keypoint rows from kp, frame stride 7 cap floats, counts n[f]): the grid CSR
// of frame f at pw_off + f (nc + 1), pw_idx + f fc; the caller has checked csr_fits(3072, cap)
int grid_batch_build(sslpl_matcher* m, const float* kp, const int* n, int nframes, int cap, const GridGeom& G) {
    if (int rc = ensure_grid_ws(m)) return rc;
    const int fc = m->p.max_features + 64, nc = GRID_COLS * GRID_ROWS;
    launch(m, k_grid_cells, dim3((cap + 127) / 128, nframes), 128, 0, kp, kp + 1, 7, 7LL * cap, n, 0, cap, G, m->pw_cell, fc);
    launch(m, k_build_csr, nframes, 128, (nc + 1 + cap) * sizeof(int), m->pw_cell, fc, n, cap, nc, m->pw_off, nc + 1, m->pw_idx, fc);
    return SSLPL_OK;
}

int ensure_reloc_ws(sslpl_matcher* m) {
    const int B = m->p.max_batch, W = m->cap, nc = GRID_COLS * GRID_ROWS;
    Arena A;
    for (int k = 0; k < 2; k++) {
        m->rw_xy = A.take<float>((size_t)B * W * 2); m->rw_n = A.take<int>(B); m->rw_cell = A.take<int32_t>((size_t)B * W);
        m->rw_off = A.take<int>((size_t)B * (nc + 1)); m->rw_idx = A.take<int>((size_t)B * W);
        m->rw_sel = A.take<int32_t>((size_t)B * W); m->rw_claimed = A.take<uint8_t>((size_t)B * W); m->rw_rbin = A.take<uint8_t>((size_t)B * W);
        m->rw_el = A.take<float>((size_t)W * 9); m->rw_eldesc = A.take<uint8_t>((size_t)W * 32); m->rw_kfmp = A.take<int32_t>((size_t)2 * W);
        m->rw_pair = A.take<int32_t>(2); m->rw_T = A.take<float>(12); m->rw_nmatch = A.take<int32_t>(1);
        if (k == 0) {
            if (int rc = first_use(m->rw, A.used)) return rc;
            A.base = m->rw; A.size = A.used; A.used = 0;
        }
    }
    return SSLPL_OK;
}

int ensure_kfbow_ws(sslpl_matcher* m) {
    const int S = 2 * m->p.max_batch, B = m->p.max_batch, fc = m->p.max_features + 64, NN = m->p.max_nodes + 1;
    Arena A;
    for (int k = 0; k < 2; k++) {
        m->kb_row = A.take<int32_t>(S); m->kb_n = A.take<int>(S);
        m->kb_node = A.take<int32_t>((size_t)S * fc); m->kb_off = A.take<int>((size_t)S * (NN + 1)); m->kb_idx = A.take<int>((size_t)S * fc);
        m->kb_pslot = A.take<int2>(B); m->kb_fn = A.take<int>(B);
        if (k == 0) {
            if (int rc = first_use(m->kb, A.used)) return rc;
            A.base = m->kb; A.size = A.used; A.used = 0;
        }
    }
    return SSLPL_OK;
}

int ensure_init_ws(sslpl_matcher* m) {
    const int B = m->p.max_batch, fc = m->p.max_features + 64;
    Arena A;
    for (int k = 0; k < 2; k++) {
        m->iw_dist = A.take<int>((size_t)B * fc); m->iw_m21 = A.take<int>((size_t)B * fc); m->iw_rbin = A.take<uint8_t>((size_t)B * fc);
        if (k == 0) {
            if (int rc = first_use(m->iw, A.used)) return rc;
            A.base = m->iw; A.size = A.used; A.used = 0;
        }
    }
    return SSLPL_OK;
}

// the sizes of a batched call over a keyframe set: nkf keyframes of cap rows (cap <= rows + 64: max_features or max_lines)
int kf_set_ok(const sslpl_matcher* m, int nkf, int cap, int rows) {
    SSLPL_REQUIRE(nkf >= 1 && nkf <= m->p.max_batch + 1, SSLPL_ERR_ARG, "nkf outside [1, max_batch + 1]");
    SSLPL_REQUIRE(cap >= 1 && cap <= rows + 64, SSLPL_ERR_ARG, "cap outside [1, max_features + 64] (lines: [1, max_lines + 64])");
    return SSLPL_OK;
}
// ... and npairs keyframe pairs
int kf_pairs_ok(const sslpl_matcher* m, int nkf, int cap, int rows, int npairs) {
    if (int rc = kf_set_ok(m, nkf, cap, rows)) return rc;
    SSLPL_REQUIRE(npairs >= 1 && npairs <= m->p.max_batch, SSLPL_ERR_ARG, "npairs outside [1, max_batch]");
    return SSLPL_OK;
}

// upload angles (or full keypoints) into the 7-float-per-row staging of a slot
int upload_angles(sslpl_matcher* m, int slot, const float* angle, int n) {
    if (n == 0) return SSLPL_OK;
    SSLPL_CUDA(cudaMemcpy2DAsync(m->kpf + (size_t)slot * m->cap * 7 + 3, 7 * sizeof(float), angle, sizeof(float), sizeof(float), n,
                                 cudaMemcpyHostToDevice, m->stream));
    return SSLPL_OK;
}

int common_bow(sslpl_matcher* m, int mode, const uint8_t* d1, int n1, const uint8_t* d2, int n2,
               const sslpl_featvec* fv1, const sslpl_featvec* fv2, const uint8_t* valid1, const uint8_t* valid2,
               const float* angle1, const float* angle2, float nnratio, int checkOri, int32_t* match, int* nmatches) {
    SSLPL_REQUIRE(m && match && nmatches && fv1 && fv2, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(n1 >= 0 && n2 >= 0 && n1 <= m->p.max_features && n2 <= m->p.max_features, SSLPL_ERR_ARG, "feature count exceeds max_features");
    SSLPL_REQUIRE((n1 == 0 || (d1 && angle1 && valid1)) && (n2 == 0 || (d2 && angle2)), SSLPL_ERR_ARG, "null descriptor/angle/valid array");
    SSLPL_REQUIRE(mode == 0 || n2 == 0 || valid2, SSLPL_ERR_ARG, "valid2 required for the KF-KF variant");
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    const int nout = mode == 0 ? n2 : n1;
    if (nout == 0) { *nmatches = 0; return SSLPL_OK; }
    int rc;
    if ((rc = featvec_ok(m, fv1, n1)) || (rc = featvec_ok(m, fv2, n2))) return rc;
    cudaStream_t st = m->stream;
    const int cap = m->cap;
    if (n1) SSLPL_CUDA(cudaMemcpyAsync(m->desc, d1, (size_t)n1 * 32, cudaMemcpyHostToDevice, st));
    if (n2) SSLPL_CUDA(cudaMemcpyAsync(m->desc + (size_t)cap * 32, d2, (size_t)n2 * 32, cudaMemcpyHostToDevice, st));
    if ((rc = upload_featvec(m, 0, fv1)) || (rc = upload_featvec(m, 1, fv2))) return rc;
    if ((rc = upload_angles(m, 0, angle1, n1)) || (rc = upload_angles(m, 1, angle2, n2))) return rc;
    if (n1) SSLPL_CUDA(cudaMemcpyAsync(m->flag, valid1, n1, cudaMemcpyHostToDevice, st));
    if (n2 && valid2) SSLPL_CUDA(cudaMemcpyAsync(m->flag + cap, valid2, n2, cudaMemcpyHostToDevice, st));
    else if (n2) SSLPL_CUDA(cudaMemsetAsync(m->flag + cap, 1, n2, st));
    m->h_small[0] = fv1->nn; m->h_small[1] = fv2->nn;
    SSLPL_CUDA(cudaMemcpyAsync(m->nn2, m->h_small, 2 * sizeof(int), cudaMemcpyHostToDevice, st));
    fill(m, m->out, nout, -1);
    SSLPL_CUDA(cudaMemsetAsync(m->rot, 255, nout, st));
    SSLPL_CUDA(cudaMemsetAsync(m->taken, 0, std::max(n2, 1), st));
    if (fv1->nn > 0 && fv2->nn > 0)
        launch(m, k_bow_match<false>, dim3((fv1->nn + 3) / 4, 1), 128, 0, staging_set(m), mode, nnratio, cap, m->out, 0, m->rot, 0, m->taken, 0,
               nullptr, nullptr, nullptr, 0);
    launch(m, k_rot_filter, 1, 256, 0, m->out, 0, m->rot, 0, nullptr, 0, nout, cap, checkOri, m->nmatch, nullptr, 0);
    SSLPL_CUDA(cudaGetLastError());
    SSLPL_CUDA(cudaMemcpyAsync(match, m->out, sizeof(int32_t) * nout, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->h_small + 8, m->nmatch, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaStreamSynchronize(st));
    *nmatches = m->h_small[8];
    return SSLPL_OK;
}

int run_knn2(sslpl_matcher* m, const uint8_t* q, int nq, const uint8_t* t, int nt, int32_t* out_host) {
    SSLPL_REQUIRE(nq >= 0 && nt >= 0 && nq <= m->cap && nt <= m->cap, SSLPL_ERR_ARG, "row count exceeds the matcher capacity");
    SSLPL_REQUIRE(nt < (1 << 20), SSLPL_ERR_ARG, "too many train rows");
    if (nq == 0) return SSLPL_OK;
    cudaStream_t st = m->stream;
    SSLPL_CUDA(cudaMemcpyAsync(m->desc, q, (size_t)nq * 32, cudaMemcpyHostToDevice, st));
    if (nt) SSLPL_CUDA(cudaMemcpyAsync(m->desc + (size_t)m->cap * 32, t, (size_t)nt * 32, cudaMemcpyHostToDevice, st));
    launch(m, k_knn2<false>, dim3((nq + 7) / 8, 1), 256, 0, m->desc, 0, nullptr, nq, m->desc + (size_t)m->cap * 32, 0, nullptr, nt, m->knn, 0, nq,
           nullptr, 0);
    SSLPL_CUDA(cudaGetLastError());
    if (out_host) {
        SSLPL_CUDA(cudaMemcpyAsync(out_host, m->knn, sizeof(int32_t) * 4 * nq, cudaMemcpyDeviceToHost, st));
        SSLPL_CUDA(cudaStreamSynchronize(st));
    }
    return SSLPL_OK;
}

// Frame::lineDescriptorMAD, Frame.cc:190-215 (host: two medians over <= NL values)
void line_mad(const int32_t* knn, int nq, double* nn_mad, double* nn12_mad) {
    if (nq <= 0) { *nn_mad = 0; *nn12_mad = 0; return; }
    std::vector<float> a(nq), g(nq);
    for (int i = 0; i < nq; i++) a[i] = (float)knn[4 * i + 1];
    std::sort(a.begin(), a.end());
    const double med = a[nq / 2];
    for (int i = 0; i < nq; i++) a[i] = fabsf((float)((float)knn[4 * i + 1] - med));
    std::sort(a.begin(), a.end());
    *nn_mad = 1.4826 * a[nq / 2];
    for (int i = 0; i < nq; i++) g[i] = (float)knn[4 * i + 3] - (float)knn[4 * i + 1];
    std::sort(g.begin(), g.end(), [](float x, float y) { return x > y; });
    const double med12 = g[nq / 2];
    for (int i = 0; i < nq; i++) a[i] = fabsf((float)((float)knn[4 * i + 3] - (float)knn[4 * i + 1] - med12));
    std::sort(a.begin(), a.end());
    *nn12_mad = 1.4826 * a[nq / 2];
}

int matcher_init(sslpl_matcher* m) {
    if (int rc = m->open(m->p.device)) return rc;
    Arena A; carve(m, A);
    if (int rc = m->alloc_arena(A.used + (1 << 16))) return rc;
    Arena B; B.base = m->arena; B.size = m->arena_size; carve(m, B);
    std::vector<int> iota(m->p.max_nodes + 1);
    for (int i = 0; i <= m->p.max_nodes; i++) iota[i] = i;
    SSLPL_CUDA(cudaMemcpy(m->iota, iota.data(), sizeof(int) * iota.size(), cudaMemcpyHostToDevice));
    // the two kernels with data-dependent dynamic shared memory may use the whole 227 KB of an sm_90 CTA
    SSLPL_CUDA(cudaFuncSetAttribute(k_bow_assign, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_DYN_SMEM));
    SSLPL_CUDA(cudaFuncSetAttribute(k_build_csr, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_DYN_SMEM));
    SSLPL_CUDA(cudaFuncSetAttribute(k_bow_vector, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_DYN_SMEM));
    SSLPL_CUDA(cudaFuncSetAttribute(k_kfdb_count<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_DYN_SMEM));
    SSLPL_CUDA(cudaFuncSetAttribute(k_kfdb_count<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_DYN_SMEM));
    SSLPL_CUDA(cudaFuncSetAttribute(k_kfdb_score<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_DYN_SMEM));
    SSLPL_CUDA(cudaFuncSetAttribute(k_kfdb_score<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_DYN_SMEM));
    SSLPL_CUDA(cudaFuncSetAttribute(k_kfdb_accumulate<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_DYN_SMEM));
    SSLPL_CUDA(cudaFuncSetAttribute(k_kfdb_accumulate<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_DYN_SMEM));
    return SSLPL_OK;
}

}  // namespace

extern "C" {

void sslpl_matcher_destroy(sslpl_matcher* m);

int sslpl_matcher_create(const sslpl_matcher_params* p, sslpl_matcher** out) {
    SSLPL_REQUIRE(p && out, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(p->max_features >= 1 && p->max_lines >= 0 && p->max_nodes >= 1 && p->max_batch >= 1, SSLPL_ERR_ARG, "bad matcher capacity");
    SSLPL_REQUIRE(p->max_features < (1 << 20) && p->max_lines < (1 << 20), SSLPL_ERR_ARG, "capacity too large");
    sslpl_matcher* m = new sslpl_matcher();
    m->p = *p;
    m->cap = std::max(p->max_features, p->max_lines) + 64;
    const int rc = matcher_init(m);
    if (rc != SSLPL_OK) { sslpl_matcher_destroy(m); return rc; }
    *out = m;
    return SSLPL_OK;
}

void sslpl_matcher_destroy(sslpl_matcher* m) {
    if (!m) return;
    m->close();
    if (m->pw) cudaFree(m->pw);
    if (m->tw) cudaFree(m->tw);
    if (m->ltw) cudaFree(m->ltw);
    if (m->rw) cudaFree(m->rw);
    if (m->kb) cudaFree(m->kb);
    if (m->iw) cudaFree(m->iw);
    delete m;
}

int sslpl_matcher_sync(sslpl_matcher* m) { SSLPL_REQUIRE(m, SSLPL_ERR_ARG, "null handle"); return m->sync(nullptr, nullptr); }
void* sslpl_matcher_stream(sslpl_matcher* m) { return m ? (void*)m->stream : nullptr; }
int sslpl_matcher_set_stream(sslpl_matcher* m, void* cuda_stream) { SSLPL_REQUIRE(m, SSLPL_ERR_ARG, "null handle"); return m->set_stream(cuda_stream); }
long long sslpl_matcher_launch_count(const sslpl_matcher* m) { return m ? m->launches : 0; }

int sslpl_descriptor_distance(sslpl_matcher* m, const uint8_t* a, const uint8_t* b, int n, int32_t* dist) {
    SSLPL_REQUIRE(m && (n == 0 || (a && b && dist)), SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(n >= 0 && n <= m->cap, SSLPL_ERR_ARG, "n exceeds the matcher capacity");
    if (n == 0) return SSLPL_OK;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    cudaStream_t st = m->stream;
    SSLPL_CUDA(cudaMemcpyAsync(m->desc, a, (size_t)n * 32, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->desc + (size_t)m->cap * 32, b, (size_t)n * 32, cudaMemcpyHostToDevice, st));
    launch(m, k_pair_distance, (n + 127) / 128, 128, 0, m->desc, m->desc + (size_t)m->cap * 32, n, m->out);
    SSLPL_CUDA(cudaGetLastError());
    SSLPL_CUDA(cudaMemcpyAsync(dist, m->out, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaStreamSynchronize(st));
    return SSLPL_OK;
}

int sslpl_hamming_knn2(sslpl_matcher* m, const uint8_t* q, int nq, const uint8_t* t, int nt, int32_t* out) {
    SSLPL_REQUIRE(m && (nq == 0 || (q && out)) && (nt == 0 || t), SSLPL_ERR_ARG, "null argument");
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    return run_knn2(m, q, nq, t, nt, out);
}

int sslpl_bow_assign(sslpl_matcher* m, const uint8_t* desc, int n, const uint8_t* centroids, int nc, int32_t* node) {
    SSLPL_REQUIRE(m && (n == 0 || (desc && node)) && centroids, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(n >= 0 && n <= m->cap && nc >= 1 && nc <= m->p.max_nodes, SSLPL_ERR_ARG, "n or nc exceeds the matcher capacity");
    if (n == 0) return SSLPL_OK;
    SSLPL_REQUIRE((size_t)(nc * 32) <= (size_t)MAX_DYN_SMEM, SSLPL_ERR_CAPACITY, "too many centroids for one shared-memory tile (nc <= 6400)");
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    cudaStream_t st = m->stream;
    SSLPL_CUDA(cudaMemcpyAsync(m->desc, desc, (size_t)n * 32, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->cent, centroids, (size_t)nc * 32, cudaMemcpyHostToDevice, st));
    launch(m, k_bow_assign, dim3((n + 127) / 128, 1), 128, nc * 32, m->desc, 0, nullptr, n, n, m->cent, nc, m->node, 0);
    SSLPL_CUDA(cudaGetLastError());
    SSLPL_CUDA(cudaMemcpyAsync(node, m->node, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaStreamSynchronize(st));
    return SSLPL_OK;
}

int sslpl_search_by_bow(sslpl_matcher* m, const uint8_t* d1, int n1, const uint8_t* d2, int n2,
                        const sslpl_featvec* fv1, const sslpl_featvec* fv2, const uint8_t* valid1, const float* angle1, const float* angle2,
                        float nnratio, int checkOri, int32_t* match2, int* nmatches) {
    return common_bow(m, 0, d1, n1, d2, n2, fv1, fv2, valid1, nullptr, angle1, angle2, nnratio, checkOri, match2, nmatches);
}

int sslpl_search_by_bow_kf(sslpl_matcher* m, const uint8_t* d1, int n1, const uint8_t* d2, int n2,
                           const sslpl_featvec* fv1, const sslpl_featvec* fv2, const uint8_t* valid1, const uint8_t* valid2,
                           const float* angle1, const float* angle2, float nnratio, int checkOri, int32_t* match12, int* nmatches) {
    return common_bow(m, 1, d1, n1, d2, n2, fv1, fv2, valid1, valid2, angle1, angle2, nnratio, checkOri, match12, nmatches);
}

int sslpl_search_for_triangulation(sslpl_matcher* m, const uint8_t* d1, int n1, const uint8_t* d2, int n2,
                                   const sslpl_featvec* fv1, const sslpl_featvec* fv2, const uint8_t* has_mp1, const uint8_t* has_mp2,
                                   const sslpl_keypoint* kp1, const sslpl_keypoint* kp2, const float* F12, float ex, float ey,
                                   const float* scale, const float* sigma2, int nlevels, int checkOri, int32_t* pairs, int* nmatches) {
    SSLPL_REQUIRE(m && pairs && nmatches && fv1 && fv2 && F12 && scale && sigma2, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(n1 >= 0 && n2 >= 0 && n1 <= m->p.max_features && n2 <= m->p.max_features, SSLPL_ERR_ARG, "feature count exceeds max_features");
    SSLPL_REQUIRE(nlevels >= 1 && nlevels <= SSLPL_MAX_LEVELS, SSLPL_ERR_ARG, "nlevels out of range");
    SSLPL_REQUIRE((n1 == 0 || (d1 && kp1 && has_mp1)) && (n2 == 0 || (d2 && kp2 && has_mp2)), SSLPL_ERR_ARG, "null array");
    *nmatches = 0;
    if (n1 == 0 || n2 == 0) return SSLPL_OK;
    for (int i = 0; i < n2; i++) SSLPL_REQUIRE(kp2[i].octave >= 0 && kp2[i].octave < nlevels, SSLPL_ERR_ARG, "keypoint octave out of range");
    int rc;
    if ((rc = featvec_ok(m, fv1, n1)) || (rc = featvec_ok(m, fv2, n2))) return rc;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    cudaStream_t st = m->stream;
    const int cap = m->cap;
    SSLPL_CUDA(cudaMemcpyAsync(m->desc, d1, (size_t)n1 * 32, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->desc + (size_t)cap * 32, d2, (size_t)n2 * 32, cudaMemcpyHostToDevice, st));
    if ((rc = upload_featvec(m, 0, fv1)) || (rc = upload_featvec(m, 1, fv2))) return rc;
    SSLPL_CUDA(cudaMemcpyAsync(m->kpf, kp1, (size_t)n1 * 28, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->kpf + (size_t)cap * 7, kp2, (size_t)n2 * 28, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->flag, has_mp1, n1, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->flag + cap, has_mp2, n2, cudaMemcpyHostToDevice, st));
    m->h_small[0] = fv1->nn; m->h_small[1] = fv2->nn;
    SSLPL_CUDA(cudaMemcpyAsync(m->nn2, m->h_small, 2 * sizeof(int), cudaMemcpyHostToDevice, st));
    fill(m, m->out, n1, -1);
    SSLPL_CUDA(cudaMemsetAsync(m->rot, 255, n1, st));
    TriArgs T;
    for (int i = 0; i < 9; i++) T.F[i] = F12[i];
    T.ex = ex; T.ey = ey; T.nlevels = nlevels;
    for (int i = 0; i < SSLPL_MAX_LEVELS; i++) { T.scale[i] = i < nlevels ? scale[i] : 0.f; T.sigma2[i] = i < nlevels ? sigma2[i] : 0.f; }
    if (fv1->nn > 0 && fv2->nn > 0) launch(m, k_tri_match<false>, dim3((fv1->nn + 3) / 4, 1), 128, 0, staging_set(m), T, nullptr, m->out, 0, m->rot, 0);
    launch(m, k_rot_filter, 1, 256, 0, m->out, 0, m->rot, 0, nullptr, 0, n1, cap, checkOri, m->nmatch, m->pairs, 0);
    SSLPL_CUDA(cudaGetLastError());
    SSLPL_CUDA(cudaMemcpyAsync(m->h_small + 8, m->nmatch, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaStreamSynchronize(st));
    *nmatches = m->h_small[8];
    if (*nmatches > 0) {
        SSLPL_CUDA(cudaMemcpyAsync(pairs, m->pairs, sizeof(int32_t) * 2 * (*nmatches), cudaMemcpyDeviceToHost, st));
        SSLPL_CUDA(cudaStreamSynchronize(st));
    }
    return SSLPL_OK;
}

int sslpl_line_match(sslpl_matcher* m, int mode, const uint8_t* d1, int n1, const uint8_t* d2, int n2,
                     const uint8_t* has_ml1, const uint8_t* has_ml2, int32_t* out, int* nout, int* nmatches, double* mad) {
    SSLPL_REQUIRE(m && out && nmatches && mode >= 0 && mode <= 3, SSLPL_ERR_ARG, "bad argument");
    SSLPL_REQUIRE(n1 >= 0 && n2 >= 0 && n1 <= m->p.max_lines && n2 <= m->p.max_lines, SSLPL_ERR_ARG, "line count exceeds max_lines");
    // the reference indexes lmatches[i][1] unconditionally (LSDmatcher.cpp:167): it requires >= 2 train rows
    SSLPL_REQUIRE(n1 == 0 || n2 >= 2, SSLPL_ERR_ARG, "knnMatch(k=2) needs at least 2 train descriptors (reference reads out of bounds otherwise)");
    SSLPL_REQUIRE((mode != 0 && mode != 3) || n1 == 0 || has_ml1, SSLPL_ERR_ARG, "has_ml1 required");
    SSLPL_REQUIRE((mode != 2 && mode != 3) || n2 == 0 || has_ml2, SSLPL_ERR_ARG, "has_ml2 required");
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    std::vector<int32_t> knn(4 * (size_t)std::max(n1, 1));
    int rc = run_knn2(m, d1, n1, d2, n2, knn.data());
    if (rc) return rc;
    double nn_mad = 0, nn12_mad = 0;
    line_mad(knn.data(), n1, &nn_mad, &nn12_mad);
    if (mad) { mad[0] = nn_mad; mad[1] = nn12_mad; }
    int nm = 0, k = 0;
    if (mode == 0) for (int j = 0; j < n2; j++) out[j] = -1;
    if (mode == 2) for (int i = 0; i < n1; i++) out[i] = -1;
    const float minRatio = 1.0f / 1.5f;
    for (int i = 0; i < n1; i++) {                      // knn rows are already in queryIdx order (:161)
        const int tdx = knn[4 * i];
        const float dist0 = (float)knn[4 * i + 1], dist1 = (float)knn[4 * i + 3];
        if (mode == 0) {
            const double dist_12 = dist0 / dist1;
            if (dist_12 < minRatio && has_ml1[i]) { out[tdx] = i; nm++; }
        } else if (mode == 1) {
            if ((double)(dist1 - dist0) > nn12_mad * 0.5) { out[2 * k] = i; out[2 * k + 1] = tdx; k++; nm++; }
        } else if (mode == 2) {
            if ((double)(dist1 - dist0) > nn12_mad * 0.5 && has_ml2[tdx]) { out[i] = tdx; nm++; }
        } else {
            if (has_ml1[i] || has_ml2[tdx]) continue;
            if ((double)(dist1 - dist0) > nn12_mad * 0.1) { out[2 * k] = i; out[2 * k + 1] = tdx; k++; nm++; }
        }
    }
    if (nout) *nout = k;
    *nmatches = nm;
    return SSLPL_OK;
}

// common tail of the batched consecutive-frame SearchByBoW: b_node holds the dense node index (or -1) of every feature; the caller has
// checked csr_fits(nc, cap)
static int bow_batch_tail(sslpl_matcher* m, const uint8_t* d_desc, const sslpl_keypoint* d_kps, const int* d_n, int nframes, int cap, int nc,
                          float nnratio, int checkOri, int32_t* d_match, int32_t* d_nmatch) {
    cudaStream_t st = m->stream;
    const int npairs = nframes - 1, fc = m->p.max_features + 64, NN = m->p.max_nodes + 1;
    launch(m, k_build_csr, nframes, 128, (nc + 1 + cap) * sizeof(int), m->b_node, fc, d_n, cap, nc, m->b_off, NN + 1, m->b_idx, fc);
    fill(m, d_match, (long long)npairs * cap, -1);
    SSLPL_CUDA(cudaMemsetAsync(m->b_rot, 255, (size_t)npairs * fc, st));
    SSLPL_CUDA(cudaMemsetAsync(m->b_taken, 0, (size_t)npairs * fc, st));
    launch(m, k_bow_match<false>, dim3((nc + 3) / 4, npairs), 128, 0, dense_set(m, d_desc, d_kps, cap, nc, nullptr), 0, nnratio, cap, d_match, cap,
           m->b_rot, fc, m->b_taken, fc, nullptr, nullptr, nullptr, 0);
    launch(m, k_rot_filter, npairs, 256, 0, d_match, cap, m->b_rot, fc, d_n, 1, 0, cap, checkOri, d_nmatch, nullptr, 0);
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}

int sslpl_match_bow_batch_device(sslpl_matcher* m, const uint8_t* d_desc, const sslpl_keypoint* d_kps, const int* d_n,
                                 int nframes, int cap, const uint8_t* d_centroids, int nc, float nnratio, int checkOri,
                                 int32_t* d_match, int32_t* d_nmatch) {
    SSLPL_REQUIRE(m && d_desc && d_kps && d_n && d_centroids && d_match && d_nmatch, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(nframes >= 2 && nframes <= m->p.max_batch + 1, SSLPL_ERR_ARG, "nframes exceeds max_batch+1");
    SSLPL_REQUIRE(cap >= 1 && cap <= m->p.max_features + 64 && nc >= 1 && nc <= m->p.max_nodes, SSLPL_ERR_ARG, "cap or nc exceeds the matcher capacity");
    SSLPL_REQUIRE((size_t)(nc * 32) <= (size_t)MAX_DYN_SMEM, SSLPL_ERR_CAPACITY, "too many centroids for one shared-memory tile (nc <= 6400)");
    if (int rc = csr_fits(nc, cap)) return rc;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    const int fc = m->p.max_features + 64;
    launch(m, k_bow_assign, dim3((cap + 127) / 128, nframes), 128, nc * 32, d_desc, (long long)cap * 32, d_n, 0, cap, d_centroids, nc, m->b_node, fc);
    return bow_batch_tail(m, d_desc, d_kps, d_n, nframes, cap, nc, nnratio, checkOri, d_match, d_nmatch);
}

// ---------------- projection-gated matcher (SURVEY.md 8(f) row 2) ----------------
int sslpl_search_by_projection_frame(sslpl_matcher* m,
        int n1, const uint8_t* valid1, const uint8_t* obs1, const float* Xw, const uint8_t* dmp, const int32_t* oct1, const float* angle1,
        int n2, const uint8_t* d2, const float* x2, const float* y2, const int32_t* oct2, const float* angle2, const float* uright2,
        const uint8_t* claimed2, const float* Tcw, const float* Tlw, const float* cam, const float* bounds,
        const float* scaleFactors, int nlevels, float th, int bMono, int checkOri, int32_t* assign2, int* nmatches) {
    SSLPL_REQUIRE(m && assign2 && nmatches && Tcw && cam && bounds && scaleFactors, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(n1 >= 0 && n2 >= 0 && n1 <= m->cap && n2 <= m->cap, SSLPL_ERR_ARG, "n1 / n2 exceed the matcher capacity");
    if (int rc = grid_staging_ok(m)) return rc;
    SSLPL_REQUIRE(nlevels >= 1 && nlevels <= 32, SSLPL_ERR_ARG, "nlevels out of range");
    SSLPL_REQUIRE(n1 == 0 || (valid1 && obs1 && Xw && dmp && oct1 && angle1), SSLPL_ERR_ARG, "null last-frame array");
    SSLPL_REQUIRE(n2 == 0 || (d2 && x2 && y2 && oct2 && angle2), SSLPL_ERR_ARG, "null current-frame array");
    SSLPL_REQUIRE(bMono || Tlw, SSLPL_ERR_ARG, "the stereo direction test needs the last frame's pose");
    ProjArgs A; memset(&A, 0, sizeof(A));
    if (int rc = grid_geom(A.G, bounds, scaleFactors, nlevels)) return rc;
    for (int j = 0; j < n2; j++) assign2[j] = -1;
    *nmatches = 0;
    if (n1 == 0 || n2 == 0) return SSLPL_OK;
    for (int i = 0; i < n1; i++) SSLPL_REQUIRE(oct1[i] >= 0 && oct1[i] < nlevels, SSLPL_ERR_ARG, "last-frame octave outside the scale-factor table");
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    cudaStream_t st = m->stream;
    const int cap = m->cap;
    for (int k = 0; k < 12; k++) A.T[k] = Tcw[k];
    A.fx = cam[0]; A.fy = cam[1]; A.cx = cam[2]; A.cy = cam[3]; A.mbf = cam[4];
    A.th = th; A.checkOri = checkOri ? 1 : 0; A.use_right = uright2 ? 1 : 0; A.nlevels = nlevels;
    if (!bMono) {                                                        // tlc = Rlw * (-Rcw^T tcw) + tlw against the baseline (:1352-1353)
        float twc[3];
        for (int r = 0; r < 3; r++) twc[r] = (float)(-((double)Tcw[r] * Tcw[3] + (double)Tcw[4 + r] * Tcw[7] + (double)Tcw[8 + r] * Tcw[11]));
        // twc = -Rcw.t()*tcw carries a transpose flag => cv::gemm's general path (double accumulation, above); tlc = Rlw*twc+tlw
        // is a plain product => float path.  Host code: volatile keeps the compiler from contracting the float chain.
        volatile float s = Tlw[8] * twc[0]; s = s + Tlw[9] * twc[1]; s = s + Tlw[10] * twc[2];
        const float tlcz = s + Tlw[11];
        A.forward = tlcz > cam[5]; A.backward = -tlcz > cam[5];
    }
    // staging (pinned scratch would avoid the pageable copies; this entry point is per frame pair, not the batched path)
    std::vector<uint8_t> fl(n1);
    for (int i = 0; i < n1; i++) fl[i] = (uint8_t)((valid1[i] ? 1 : 0) | (obs1[i] ? 2 : 0));
    float* k0 = m->kpf; float* k1 = m->kpf + (size_t)cap * 7;
    SSLPL_CUDA(cudaMemcpyAsync(m->desc, dmp, (size_t)n1 * 32, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->desc + (size_t)cap * 32, d2, (size_t)n2 * 32, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k0, Xw, sizeof(float) * 3 * n1, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k0 + 3 * (size_t)cap, angle1, sizeof(float) * n1, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k0 + 4 * (size_t)cap, oct1, sizeof(int) * n1, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k1, x2, sizeof(float) * n2, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k1 + (size_t)cap, y2, sizeof(float) * n2, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k1 + 2 * (size_t)cap, angle2, sizeof(float) * n2, cudaMemcpyHostToDevice, st));
    if (uright2) SSLPL_CUDA(cudaMemcpyAsync(k1 + 3 * (size_t)cap, uright2, sizeof(float) * n2, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k1 + 4 * (size_t)cap, oct2, sizeof(int) * n2, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->flag, fl.data(), n1, cudaMemcpyHostToDevice, st));
    if (claimed2) SSLPL_CUDA(cudaMemcpyAsync(m->flag + cap, claimed2, n2, cudaMemcpyHostToDevice, st));
    else SSLPL_CUDA(cudaMemsetAsync(m->flag + cap, 0, n2, st));
    SSLPL_CUDA(cudaStreamSynchronize(st));                               // fl (pageable) is reused by the caller
    int *goff, *gidx;
    if (int rc = grid_staging_build(m, k1, k1 + cap, n2, A.G, goff, gidx)) return rc;
    ProjPair P; memset(&P, 0, sizeof(P));
    P.n1 = n1; P.n2 = n2; P.cap = cap;
    P.flag1 = m->flag; P.Xw = k0; P.dmp = m->desc; P.angle1 = k0 + 3 * (size_t)cap; P.oct1 = reinterpret_cast<const int*>(k0 + 4 * (size_t)cap); P.es1 = 1;
    P.d2 = m->desc + (size_t)cap * 32; P.x2 = k1; P.y2 = k1 + cap; P.angle2 = k1 + 2 * (size_t)cap; P.oct2 = reinterpret_cast<const int*>(k1 + 4 * (size_t)cap);
    P.uright2 = k1 + 3 * (size_t)cap; P.es2 = 1;
    P.claimed0 = m->flag + cap; P.goff = goff; P.gidx = gidx;
    P.claimed = m->taken; P.assign2 = m->out; P.sel = m->pairs; P.rbin = m->rot; P.nmatch = m->nmatch;
    launch(m, k_proj_match, 1, 32, 0, A, P);
    SSLPL_CUDA(cudaGetLastError());
    SSLPL_CUDA(cudaMemcpyAsync(assign2, m->out, sizeof(int32_t) * n2, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->h_small, m->nmatch, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaStreamSynchronize(st));
    *nmatches = m->h_small[0];
    return SSLPL_OK;
}

// The same matcher over consecutive frames in HBM (monocular: bMono = true, as Tracking passes it for a monocular sensor): pair p
// projects frame p's MapPoints with frame p + 1's pose.  Grid cells of every current frame (frame on grid.y), one k_build_csr
// launch for all of them, then one walker warp per pair, which also runs TrackWithMotionModel's 2 * th retry (Tracking.cc:1240-1244).
int sslpl_search_by_projection_frame_batch_device(sslpl_matcher* m, const sslpl_keypoint* d_kps, const uint8_t* d_desc, const int* d_n,
        int nframes, int cap, const float* d_Xw, const uint8_t* d_mpflag, const uint8_t* d_dmp, const float* d_Tcw,
        const float* cam, const float* bounds, const float* scaleFactors, int nlevels, float th, int checkOri, int retry_below,
        int32_t* d_assign, int32_t* d_nmatch) {
    SSLPL_REQUIRE(m && d_kps && d_desc && d_n && d_Xw && d_mpflag && d_Tcw && cam && bounds && scaleFactors && d_assign && d_nmatch,
                  SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(nframes >= 2 && nframes <= m->p.max_batch + 1, SSLPL_ERR_ARG, "nframes outside [2, max_batch + 1]");
    SSLPL_REQUIRE(cap >= 1 && cap <= m->p.max_features + 64, SSLPL_ERR_ARG, "cap outside [1, max_features + 64]");
    SSLPL_REQUIRE(nlevels >= 1 && nlevels <= 32, SSLPL_ERR_ARG, "nlevels out of range");
    SSLPL_REQUIRE(th > 0.f, SSLPL_ERR_ARG, "th must be positive");
    ProjArgs A; memset(&A, 0, sizeof(A));
    if (int rc = grid_geom(A.G, bounds, scaleFactors, nlevels)) return rc;
    const int nc = GRID_COLS * GRID_ROWS, npairs = nframes - 1;
    if (int rc = csr_fits(nc, cap)) return rc;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    const int fc = m->p.max_features + 64;
    A.fx = cam[0]; A.fy = cam[1]; A.cx = cam[2]; A.cy = cam[3];
    A.th = th; A.checkOri = checkOri ? 1 : 0; A.nlevels = nlevels; A.retry_below = retry_below;
    const float* kf = reinterpret_cast<const float*>(d_kps);            // sslpl_keypoint = 7 x 4 B: x y size angle response octave class_id
    const long long kfs = 7LL * cap;
    if (int rc = grid_batch_build(m, kf + kfs, d_n + 1, npairs, cap, A.G)) return rc;
    ProjPair P; memset(&P, 0, sizeof(P));
    P.n = d_n; P.cap = cap; P.Tcw = d_Tcw + 12;
    P.flag1 = d_mpflag; P.Xw = d_Xw; P.dmp = d_dmp ? d_dmp : d_desc; P.angle1 = kf + 3; P.oct1 = reinterpret_cast<const int*>(kf + 5);
    P.flag1_fs = cap; P.xw_fs = 3LL * cap; P.dmp_fs = 32LL * cap; P.kp1_fs = kfs; P.es1 = 7;
    P.d2 = d_desc + 32LL * cap; P.x2 = kf + kfs; P.y2 = kf + kfs + 1; P.angle2 = kf + kfs + 3; P.oct2 = reinterpret_cast<const int*>(kf + kfs + 5);
    P.d2_fs = 32LL * cap; P.kp2_fs = kfs; P.es2 = 7;
    P.goff = m->pw_off; P.gidx = m->pw_idx; P.goff_fs = nc + 1; P.gidx_fs = fc;
    P.claimed = m->pw_claimed; P.assign2 = d_assign; P.sel = m->pw_sel; P.rbin = m->pw_rbin; P.ws_fs = cap;
    P.nmatch = d_nmatch;
    launch(m, k_proj_match, npairs, 32, 0, A, P);
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}

int sslpl_search_by_projection_mps(sslpl_matcher* m,
        int nmp, const uint8_t* inview, const uint8_t* bad, const uint8_t* obs, const float* projx, const float* projy, const float* projxr,
        const int32_t* level, const float* viewcos, const uint8_t* dmp,
        int n2, const uint8_t* d2, const float* x2, const float* y2, const int32_t* oct2, const float* uright2, const uint8_t* held2,
        const float* bounds, const float* scaleFactors, int nlevels, float nnratio, float th, int32_t* assign2, int* nmatches) {
    SSLPL_REQUIRE(m && assign2 && nmatches && bounds && scaleFactors, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(nmp >= 0 && n2 >= 0 && nmp <= m->cap && n2 <= m->cap, SSLPL_ERR_ARG, "nmp / n2 exceed the matcher capacity");
    if (int rc = grid_staging_ok(m)) return rc;
    SSLPL_REQUIRE(nlevels >= 1 && nlevels <= 32, SSLPL_ERR_ARG, "nlevels out of range");
    SSLPL_REQUIRE(nmp == 0 || (inview && projx && projy && level && viewcos && dmp), SSLPL_ERR_ARG, "null MapPoint array");
    SSLPL_REQUIRE(n2 == 0 || (d2 && x2 && y2 && oct2), SSLPL_ERR_ARG, "null frame array");
    SSLPL_REQUIRE(!uright2 || projxr, SSLPL_ERR_ARG, "stereo frame features need mTrackProjXR");
    WinArgs A; memset(&A, 0, sizeof(A));
    if (int rc = grid_geom(A.G, bounds, scaleFactors, nlevels)) return rc;
    for (int j = 0; j < n2; j++) assign2[j] = -1;
    *nmatches = 0;
    if (nmp == 0 || n2 == 0) return SSLPL_OK;
    for (int i = 0; i < nmp; i++) SSLPL_REQUIRE(level[i] >= 0 && level[i] < nlevels, SSLPL_ERR_ARG, "predicted level outside the scale-factor table");
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    cudaStream_t st = m->stream;
    const int cap = m->cap;
    A.th = th; A.nnratio = nnratio; A.bFactor = th != 1.0f; A.use_right = uright2 ? 1 : 0;
    std::vector<uint8_t> fl(nmp), cl(n2, 0);
    for (int i = 0; i < nmp; i++) fl[i] = (uint8_t)(((inview[i] && !(bad && bad[i])) ? 1 : 0) | ((obs && obs[i]) ? 2 : 0));
    if (held2) for (int j = 0; j < n2; j++) cl[j] = held2[j] == 1;
    float* k0 = m->kpf; float* k1 = m->kpf + (size_t)cap * 7;
    SSLPL_CUDA(cudaMemcpyAsync(m->desc, dmp, (size_t)nmp * 32, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->desc + (size_t)cap * 32, d2, (size_t)n2 * 32, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k0, projx, sizeof(float) * nmp, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k0 + (size_t)cap, projy, sizeof(float) * nmp, cudaMemcpyHostToDevice, st));
    if (projxr) SSLPL_CUDA(cudaMemcpyAsync(k0 + 2 * (size_t)cap, projxr, sizeof(float) * nmp, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k0 + 3 * (size_t)cap, viewcos, sizeof(float) * nmp, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k0 + 4 * (size_t)cap, level, sizeof(int) * nmp, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k1, x2, sizeof(float) * n2, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k1 + (size_t)cap, y2, sizeof(float) * n2, cudaMemcpyHostToDevice, st));
    if (uright2) SSLPL_CUDA(cudaMemcpyAsync(k1 + 3 * (size_t)cap, uright2, sizeof(float) * n2, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k1 + 4 * (size_t)cap, oct2, sizeof(int) * n2, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->flag, fl.data(), nmp, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->flag + cap, cl.data(), n2, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaStreamSynchronize(st));                               // pageable staging vectors go out of scope
    int *goff, *gidx;
    if (int rc = grid_staging_build(m, k1, k1 + cap, n2, A.G, goff, gidx)) return rc;
    launch(m, k_proj_match_mps, 1, 32, 0, A, nmp, m->flag, k0, k0 + cap, k0 + 2 * (size_t)cap, reinterpret_cast<const int*>(k0 + 4 * (size_t)cap), k0 + 3 * (size_t)cap, m->desc,
                                       n2, m->desc + (size_t)cap * 32, k1, k1 + cap, reinterpret_cast<const int*>(k1 + 4 * (size_t)cap), k1 + 3 * (size_t)cap,
                                       m->flag + cap, goff, gidx, m->out, m->nmatch);
    SSLPL_CUDA(cudaGetLastError());
    SSLPL_CUDA(cudaMemcpyAsync(assign2, m->out, sizeof(int32_t) * n2, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->h_small, m->nmatch, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaStreamSynchronize(st));
    *nmatches = m->h_small[0];
    return SSLPL_OK;
}

int sslpl_search_for_initialization(sslpl_matcher* m,
        int n1, const uint8_t* d1, const int32_t* oct1, const float* angle1, float* prev_xy /* [n1][2], in/out */,
        int n2, const uint8_t* d2, const float* x2, const float* y2, const int32_t* oct2, const float* angle2,
        const float* bounds, float nnratio, int checkOri, int windowSize, int32_t* matches12, int* nmatches) {
    SSLPL_REQUIRE(m && matches12 && nmatches && bounds, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(n1 >= 0 && n2 >= 0 && n1 <= m->cap && n2 <= m->cap, SSLPL_ERR_ARG, "n1 / n2 exceed the matcher capacity");
    if (int rc = grid_staging_ok(m)) return rc;
    SSLPL_REQUIRE(n1 == 0 || (d1 && oct1 && angle1 && prev_xy), SSLPL_ERR_ARG, "null first-frame array");
    SSLPL_REQUIRE(n2 == 0 || (d2 && x2 && y2 && oct2 && angle2), SSLPL_ERR_ARG, "null second-frame array");
    WinArgs A; memset(&A, 0, sizeof(A));
    if (int rc = grid_geom(A.G, bounds, nullptr, 0)) return rc;
    for (int i = 0; i < n1; i++) matches12[i] = -1;
    *nmatches = 0;
    if (n1 == 0 || n2 == 0) return SSLPL_OK;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    cudaStream_t st = m->stream;
    const int cap = m->cap;
    A.nnratio = nnratio; A.checkOri = checkOri ? 1 : 0; A.window = windowSize;
    float* k0 = m->kpf; float* k1 = m->kpf + (size_t)cap * 7;          // k0: prev [n1][2] in the first 2 cap floats, angle1, oct1
    SSLPL_CUDA(cudaMemcpyAsync(m->desc, d1, (size_t)n1 * 32, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->desc + (size_t)cap * 32, d2, (size_t)n2 * 32, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k0, prev_xy, sizeof(float) * 2 * n1, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k0 + 3 * (size_t)cap, angle1, sizeof(float) * n1, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k0 + 4 * (size_t)cap, oct1, sizeof(int) * n1, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k1, x2, sizeof(float) * n2, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k1 + (size_t)cap, y2, sizeof(float) * n2, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k1 + 2 * (size_t)cap, angle2, sizeof(float) * n2, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(k1 + 4 * (size_t)cap, oct2, sizeof(int) * n2, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaStreamSynchronize(st));
    int *goff, *gidx;
    if (int rc = grid_staging_build(m, k1, k1 + cap, n2, A.G, goff, gidx)) return rc;
    launch(m, k_init_match, 1, 32, 0, A, n1, m->desc, reinterpret_cast<const int*>(k0 + 4 * (size_t)cap), k0 + 3 * (size_t)cap, k0,
                                   n2, m->desc + (size_t)cap * 32, k1, k1 + cap, reinterpret_cast<const int*>(k1 + 4 * (size_t)cap), k1 + 2 * (size_t)cap,
                                   goff, gidx, m->knn, m->knn + cap, m->out, m->rot, m->nmatch);
    SSLPL_CUDA(cudaGetLastError());
    SSLPL_CUDA(cudaMemcpyAsync(matches12, m->out, sizeof(int32_t) * n1, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaMemcpyAsync(prev_xy, k0, sizeof(float) * 2 * n1, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->h_small, m->nmatch, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaStreamSynchronize(st));
    *nmatches = m->h_small[0];
    return SSLPL_OK;
}

// The same matcher over the chains of a pair list of a row set in HBM: the grid of every row (one grid_batch_build), then k_init_chain, one
// warp per chain.
int sslpl_search_for_initialization_batch_device(sslpl_matcher* m,
        const sslpl_keypoint* d_kps, const uint8_t* d_desc, const int* d_n, int nrows, int cap, int npairs, const int32_t* d_pair,
        const float* d_prev0, const float* bounds, float nnratio, int checkOri, int windowSize,
        int32_t* d_match12, float* d_prev, int32_t* d_nmatch) {
    SSLPL_REQUIRE(m && d_kps && d_desc && d_n && d_pair && bounds && d_match12 && d_prev && d_nmatch, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(nrows >= 2 && nrows <= m->p.max_batch + 1, SSLPL_ERR_ARG, "nrows outside [2, max_batch + 1]");
    SSLPL_REQUIRE(npairs >= 1 && npairs <= m->p.max_batch, SSLPL_ERR_ARG, "npairs outside [1, max_batch]");
    SSLPL_REQUIRE(cap >= 1 && cap <= m->p.max_features + 64, SSLPL_ERR_ARG, "cap outside [1, max_features + 64]");
    WinArgs A; memset(&A, 0, sizeof(A));
    if (int rc = grid_geom(A.G, bounds, nullptr, 0)) return rc;
    const int nc = GRID_COLS * GRID_ROWS;
    if (int rc = csr_fits(nc, cap)) return rc;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    A.nnratio = nnratio; A.checkOri = checkOri ? 1 : 0; A.window = windowSize;
    if (int rc = ensure_init_ws(m)) return rc;
    const float* kf = reinterpret_cast<const float*>(d_kps);
    if (int rc = grid_batch_build(m, kf, d_n, nrows, cap, A.G)) return rc;
    const int fc = m->p.max_features + 64;
    launch(m, k_init_chain, npairs, 32, 0, A, reinterpret_cast<const int2*>(d_pair), npairs, nrows, kf, d_desc, d_n, cap, d_prev0,
           m->pw_off, m->pw_idx, (long long)(nc + 1), (long long)fc, m->iw_dist, m->iw_m21, m->iw_rbin, (long long)fc, d_match12, d_prev, d_nmatch);
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}

// Frame::GetFeaturesInArea on its own (Frame.cc:368-421) is host logic over the same CSR; the matcher above is its only
// device consumer.  (The per-frame grid build is k_grid_cells + k_build_csr.)

// ---------------- line projection search and Fuse search (SURVEY.md 8(f) row 3) ----------------

int sslpl_line_search_by_projection(sslpl_matcher* m, int nml, const uint8_t* active, const uint8_t* obs, const float* proj, const float* radius,
                                    const int32_t* minLevel, const int32_t* maxLevel, const uint8_t* dml,
                                    int nl2, const uint8_t* ld2, const float* kl2, const int32_t* oct2, const uint8_t* held2,
                                    float nnratio, int32_t* assign2, int* nmatches) {
    SSLPL_REQUIRE(m && nmatches && nml >= 0 && nl2 >= 0, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(nml == 0 || (active && proj && radius && minLevel && maxLevel && dml), SSLPL_ERR_ARG, "null MapLine array");
    SSLPL_REQUIRE(nl2 == 0 || (ld2 && kl2 && oct2 && assign2), SSLPL_ERR_ARG, "null frame-line array");
    for (int j = 0; j < nl2; j++) assign2[j] = -1;
    *nmatches = 0;
    if (nml == 0 || nl2 == 0) return SSLPL_OK;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    cudaStream_t st = m->stream;
    const size_t need = (size_t)nml * (1 + 16 + 4 + 4 + 4 + 32) + (size_t)nl2 * (32 + 12 + 4 + 1 + 4) + 16 * 256 + 4096;
    if (int rc = ensure_scratch(m, need)) return rc;
    std::vector<uint8_t> fl(nml), cl(nl2, 0);
    for (int i = 0; i < nml; i++) fl[i] = (uint8_t)((active[i] ? 1 : 0) | ((obs && obs[i]) ? 2 : 0));
    if (held2) for (int j = 0; j < nl2; j++) cl[j] = held2[j] == 1;
    Arena A; A.base = m->scratch; A.used = 0;
    cudaError_t e = cudaSuccess;
    uint8_t* d_fl = stage(A, fl.data(), nml, st, e); float* d_proj = stage(A, proj, (size_t)4 * nml, st, e); float* d_rad = stage(A, radius, nml, st, e);
    int32_t* d_min = stage(A, minLevel, nml, st, e); int32_t* d_max = stage(A, maxLevel, nml, st, e); uint8_t* d_dml = stage(A, dml, (size_t)32 * nml, st, e);
    uint8_t* d_ld2 = stage(A, ld2, (size_t)32 * nl2, st, e); float* d_kl2 = stage(A, kl2, (size_t)3 * nl2, st, e); int32_t* d_oct = stage(A, oct2, nl2, st, e);
    uint8_t* d_cl = stage(A, cl.data(), nl2, st, e); int32_t* d_out = A.take<int32_t>(nl2 + 8);
    SSLPL_CUDA(e);
    SSLPL_CUDA(cudaStreamSynchronize(st));                               // the pageable staging vectors go out of scope
    launch(m, k_line_window_search, 1, 32, 0, nml, d_fl, reinterpret_cast<const float4*>(d_proj), d_rad, d_min, d_max, d_dml, nl2, d_ld2, d_kl2, d_oct, d_cl,
                                           nnratio, d_out, m->nmatch);
    SSLPL_CUDA(cudaGetLastError());
    SSLPL_CUDA(cudaMemcpyAsync(assign2, d_out, sizeof(int32_t) * nl2, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->h_small, m->nmatch, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaStreamSynchronize(st));
    *nmatches = m->h_small[0];
    return SSLPL_OK;
}

int sslpl_fuse_lines_search(sslpl_matcher* m, int nml, const uint8_t* active, const float* proj, const int32_t* level, const uint8_t* dml,
                            int nl2, const uint8_t* ld2, const float* kl2, const int32_t* oct2, const float* scaleFactors, int nlevels, float th,
                            int32_t* best_idx, int32_t* best_dist) {
    SSLPL_REQUIRE(m && nml >= 0 && nl2 >= 0 && scaleFactors && nlevels >= 1 && nlevels <= 32, SSLPL_ERR_ARG, "bad argument");
    SSLPL_REQUIRE(nml == 0 || (active && proj && level && dml && best_idx && best_dist), SSLPL_ERR_ARG, "null MapLine array");
    SSLPL_REQUIRE(nl2 == 0 || (ld2 && kl2 && oct2), SSLPL_ERR_ARG, "null KeyFrame-line array");
    for (int i = 0; i < nml; i++) { best_idx[i] = -1; best_dist[i] = 0x7fffffff; }
    if (nml == 0 || nl2 == 0) return SSLPL_OK;
    std::vector<uint8_t> act(nml);
    for (int i = 0; i < nml; i++) act[i] = active[i] && level[i] >= 0 && level[i] < nlevels;      // MapLine::PredictScale is not clamped: out-of-pyramid levels are dropped
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    cudaStream_t st = m->stream;
    const size_t need = (size_t)nml * (1 + 16 + 4 + 32 + 8) + (size_t)nl2 * (32 + 12 + 4) + 16 * 256 + 4096;
    if (int rc = ensure_scratch(m, need)) return rc;
    Arena A; A.base = m->scratch; A.used = 0;
    cudaError_t e = cudaSuccess;
    uint8_t* d_act = stage(A, act.data(), nml, st, e); float* d_proj = stage(A, proj, (size_t)4 * nml, st, e); int32_t* d_lvl = stage(A, level, nml, st, e);
    uint8_t* d_dml = stage(A, dml, (size_t)32 * nml, st, e); uint8_t* d_ld2 = stage(A, ld2, (size_t)32 * nl2, st, e);
    float* d_kl2 = stage(A, kl2, (size_t)3 * nl2, st, e); int32_t* d_oct = stage(A, oct2, nl2, st, e); float* d_sc = stage(A, scaleFactors, nlevels, st, e);
    int32_t* d_bi = A.take<int32_t>(nml + 8); int32_t* d_bd = A.take<int32_t>(nml + 8);
    SSLPL_CUDA(e);
    SSLPL_CUDA(cudaStreamSynchronize(st));
    FuseMap Z; memset(&Z, 0, sizeof(Z));
    launch(m, k_line_fuse_search<false>, (nml + 3) / 4, 128, 0, nml, d_act, reinterpret_cast<const float4*>(d_proj), d_lvl, d_dml, nl2, d_ld2, d_kl2,
           d_oct, d_sc, th, d_bi, d_bd, Z);
    SSLPL_CUDA(cudaGetLastError());
    SSLPL_CUDA(cudaMemcpyAsync(best_idx, d_bi, sizeof(int32_t) * nml, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaMemcpyAsync(best_dist, d_bd, sizeof(int32_t) * nml, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaStreamSynchronize(st));
    return SSLPL_OK;
}

int sslpl_fuse_points_search(sslpl_matcher* m, int nmp, const uint8_t* active, const float* u, const float* v, const float* ur, const int32_t* level, const uint8_t* dmp,
                             int n2, const uint8_t* d2, const float* x2, const float* y2, const int32_t* oct2, const float* uright2,
                             const float* bounds, const float* scaleFactors, const float* invLevelSigma2, int nlevels, float th,
                             int32_t* best_idx, int32_t* best_dist) {
    SSLPL_REQUIRE(m && nmp >= 0 && n2 >= 0 && bounds && scaleFactors && invLevelSigma2 && nlevels >= 1 && nlevels <= 32, SSLPL_ERR_ARG, "bad argument");
    SSLPL_REQUIRE(n2 <= m->cap, SSLPL_ERR_ARG, "n2 exceeds the matcher capacity");
    if (int rc = grid_staging_ok(m)) return rc;
    SSLPL_REQUIRE(nmp == 0 || (active && u && v && level && dmp && best_idx && best_dist), SSLPL_ERR_ARG, "null MapPoint array");
    SSLPL_REQUIRE(n2 == 0 || (d2 && x2 && y2 && oct2), SSLPL_ERR_ARG, "null KeyFrame array");
    WinArgs A; memset(&A, 0, sizeof(A));
    if (int rc = grid_geom(A.G, bounds, scaleFactors, nlevels)) return rc;
    for (int i = 0; i < nmp; i++) { best_idx[i] = -1; best_dist[i] = 256; }
    if (nmp == 0 || n2 == 0) return SSLPL_OK;
    for (int i = 0; i < nmp; i++) SSLPL_REQUIRE(!active[i] || (level[i] >= 0 && level[i] < nlevels), SSLPL_ERR_ARG, "predicted level outside the pyramid");
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    cudaStream_t st = m->stream;
    A.th = th; A.use_right = uright2 ? 1 : 0;
    const size_t need = (size_t)nmp * (1 + 12 + 4 + 32 + 8) + (size_t)n2 * (32 + 16) + 32 * 4 + 16 * 256 + 4096;
    if (int rc = ensure_scratch(m, need)) return rc;
    Arena S; S.base = m->scratch; S.used = 0;
    cudaError_t e = cudaSuccess;
    std::vector<float> urz;
    if (!ur) { urz.assign(nmp, 0.f); ur = urz.data(); }
    uint8_t* d_act = stage(S, active, nmp, st, e); float* d_u = stage(S, u, nmp, st, e); float* d_v = stage(S, v, nmp, st, e); float* d_ur = stage(S, ur, nmp, st, e);
    int32_t* d_lvl = stage(S, level, nmp, st, e); uint8_t* d_dmp = stage(S, dmp, (size_t)32 * nmp, st, e);
    uint8_t* d_d2 = stage(S, d2, (size_t)32 * n2, st, e); float* d_x2 = stage(S, x2, n2, st, e); float* d_y2 = stage(S, y2, n2, st, e);
    int32_t* d_oct = stage(S, oct2, n2, st, e); float* d_ur2 = stage(S, uright2, uright2 ? n2 : 0, st, e); float* d_is2 = stage(S, invLevelSigma2, nlevels, st, e);
    int32_t* d_bi = S.take<int32_t>(nmp + 8); int32_t* d_bd = S.take<int32_t>(nmp + 8);
    SSLPL_CUDA(e);
    SSLPL_CUDA(cudaStreamSynchronize(st));
    int *goff, *gidx;
    if (int rc = grid_staging_build(m, d_x2, d_y2, n2, A.G, goff, gidx)) return rc;
    FuseMap Z; memset(&Z, 0, sizeof(Z));
    launch(m, k_point_fuse_search<false>, (nmp + 3) / 4, 128, 0, A, nmp, d_act, d_u, d_v, d_ur, d_lvl, d_dmp, d_d2, d_x2, d_y2, d_oct, d_ur2, d_is2,
           goff, gidx, d_bi, d_bd, Z);
    SSLPL_CUDA(cudaGetLastError());
    SSLPL_CUDA(cudaMemcpyAsync(best_idx, d_bi, sizeof(int32_t) * nmp, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaMemcpyAsync(best_dist, d_bd, sizeof(int32_t) * nmp, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaStreamSynchronize(st));
    return SSLPL_OK;
}

// ---------------- descriptor medoids (SURVEY.md 8(f) row 3) ----------------
int sslpl_descriptor_medoid_batch(sslpl_matcher* m, const uint8_t* desc, const int32_t* off, int ngroups, int32_t* best_idx, int32_t* best_median) {
    SSLPL_REQUIRE(m && off && ngroups >= 0 && (ngroups == 0 || (best_idx && best_median)), SSLPL_ERR_ARG, "null argument");
    if (ngroups == 0) return SSLPL_OK;
    const int total = off[ngroups];
    SSLPL_REQUIRE(off[0] == 0 && total >= 0 && (total == 0 || desc), SSLPL_ERR_ARG, "bad group offsets");
    for (int g = 0; g < ngroups; g++) SSLPL_REQUIRE(off[g + 1] >= off[g] && off[g + 1] - off[g] < (1 << 20), SSLPL_ERR_ARG, "group offsets must be non-decreasing (groups < 2^20 rows)");
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    cudaStream_t st = m->stream;
    const size_t need = align_up((size_t)total * 32 + 256, 256) + align_up(sizeof(int32_t) * (size_t)(ngroups + 1), 256) + 2 * align_up(sizeof(int32_t) * (size_t)ngroups, 256);
    if (int rc = ensure_scratch(m, need)) return rc;
    Arena A; A.base = m->scratch; A.used = 0;
    uint8_t* d_desc = A.take<uint8_t>((size_t)total * 32 + 32); int32_t* d_off = A.take<int32_t>(ngroups + 1);
    int32_t* d_bi = A.take<int32_t>(ngroups); int32_t* d_bm = A.take<int32_t>(ngroups);
    if (total) SSLPL_CUDA(cudaMemcpyAsync(d_desc, desc, (size_t)total * 32, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(d_off, off, sizeof(int32_t) * (ngroups + 1), cudaMemcpyHostToDevice, st));
    launch(m, k_medoid, ngroups, 128, 0, d_desc, d_off, d_bi, d_bm);
    SSLPL_CUDA(cudaGetLastError());
    SSLPL_CUDA(cudaMemcpyAsync(best_idx, d_bi, sizeof(int32_t) * ngroups, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaMemcpyAsync(best_median, d_bm, sizeof(int32_t) * ngroups, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaStreamSynchronize(st));
    return SSLPL_OK;
}

// ---------------- DBoW2 vocabulary (SURVEY.md 8(f) row 1) ----------------
static int vocab_level_nodes(const sslpl_vocab* v, int levelsup) {
    const int lvl = v->L - levelsup;
    return 1 + ((lvl >= 1 && lvl < (int)v->level_count.size()) ? v->level_count[lvl] : 0);
}

int sslpl_vocab_create(int device, int k, int L, int nnodes, const int32_t* parent, const uint8_t* desc, const double* weight,
                       const uint8_t* is_leaf, sslpl_vocab** out) {
    SSLPL_REQUIRE(out && parent && desc && weight && is_leaf, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(k >= 1 && L >= 1 && nnodes >= 1, SSLPL_ERR_ARG, "bad vocabulary shape");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { set_error("no CUDA device available: libsslpl_b200 has no CPU fallback"); return SSLPL_ERR_CUDA; }
    SSLPL_CUDA(cudaSetDevice(device));
    std::vector<int> cnt(nnodes + 1, 0), depth(nnodes, 0), word(nnodes, -1), rank(nnodes, 0);
    for (int i = 1; i < nnodes; i++) {
        SSLPL_REQUIRE(parent[i] >= 0 && parent[i] < i, SSLPL_ERR_ARG, "vocabulary: parent[i] must be an earlier node");
        cnt[parent[i] + 1]++; depth[i] = depth[parent[i]] + 1;
    }
    for (int i = 0; i < nnodes; i++) cnt[i + 1] += cnt[i];                    // CSR offsets
    std::vector<int> ids(std::max(nnodes - 1, 1)), fillp(cnt.begin(), cnt.end() - 1);
    for (int i = 1; i < nnodes; i++) ids[fillp[parent[i]]++] = i;             // ascending ids inside every list
    int nwords = 0, maxd = 0;
    for (int i = 1; i < nnodes; i++) {
        const bool leaf = cnt[i + 1] == cnt[i];
        SSLPL_REQUIRE(leaf == (is_leaf[i] != 0), SSLPL_ERR_ARG, "vocabulary: is_leaf disagrees with the tree structure");
        if (leaf) word[i] = nwords++;
        maxd = std::max(maxd, depth[i]);
    }
    sslpl_vocab* v = new sslpl_vocab();
    v->device = device; v->k = k; v->L = L; v->nnodes = nnodes; v->nwords = nwords; v->depth = depth;
    v->level_count.assign(maxd + 1, 0);
    for (int i = 0; i < nnodes; i++) rank[i] = v->level_count[depth[i]]++;    // rank among the nodes of the same depth, ascending id
    Arena A;
    A.base = nullptr; A.used = 0;
    auto carve_all = [&](Arena& a, sslpl::VocabView& w) {
        w.child_off = a.take<int>(nnodes + 1); w.child_ids = a.take<int>(ids.size()); w.desc = a.take<uint8_t>((size_t)nnodes * 32);
        w.weight = a.take<double>(nnodes); w.word_id = a.take<int>(nnodes); w.level_rank = a.take<int>(nnodes);
    };
    sslpl::VocabView dry{}; carve_all(A, dry);
    const size_t bytes = A.used + 256;
    cudaError_t e = cudaMalloc(&v->arena, bytes);
    if (e != cudaSuccess) { set_error("cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e)); delete v; return SSLPL_ERR_CUDA; }
    Arena B2; B2.base = v->arena; B2.used = 0;
    carve_all(B2, v->view);
    SSLPL_CUDA(cudaMemcpy(const_cast<int*>(v->view.child_off), cnt.data(), sizeof(int) * (nnodes + 1), cudaMemcpyHostToDevice));
    SSLPL_CUDA(cudaMemcpy(const_cast<int*>(v->view.child_ids), ids.data(), sizeof(int) * ids.size(), cudaMemcpyHostToDevice));
    SSLPL_CUDA(cudaMemcpy(const_cast<uint8_t*>(v->view.desc), desc, (size_t)nnodes * 32, cudaMemcpyHostToDevice));
    SSLPL_CUDA(cudaMemcpy(const_cast<double*>(v->view.weight), weight, sizeof(double) * nnodes, cudaMemcpyHostToDevice));
    SSLPL_CUDA(cudaMemcpy(const_cast<int*>(v->view.word_id), word.data(), sizeof(int) * nnodes, cudaMemcpyHostToDevice));
    SSLPL_CUDA(cudaMemcpy(const_cast<int*>(v->view.level_rank), rank.data(), sizeof(int) * nnodes, cudaMemcpyHostToDevice));
    *out = v;
    return SSLPL_OK;
}

// ORBvoc.txt text format of TemplatedVocabulary::loadFromTextFile (TemplatedVocabulary.h:1338-1420):
// "k L scoring weighting" then one line per node: "parent is_leaf b0 .. b31 weight".  Blank lines are skipped (the reference's
// `while(!f.eof())` loop turns the trailing newline into one bogus node with an uninitialised parent).
int sslpl_vocab_load_text(int device, const char* path, sslpl_vocab** out, int* scoring, int* weighting) {
    SSLPL_REQUIRE(path && out, SSLPL_ERR_ARG, "null argument");
    FILE* f = fopen(path, "r");
    if (!f) { set_error("cannot open vocabulary file %s", path); return SSLPL_ERR_ARG; }
    int k = 0, L = 0, n1 = 0, n2 = 0;
    if (fscanf(f, "%d %d %d %d", &k, &L, &n1, &n2) != 4 || k < 0 || k > 20 || L < 1 || L > 10 || n1 < 0 || n1 > 5 || n2 < 0 || n2 > 3) {
        fclose(f); set_error("%s is not a DBoW2 text vocabulary", path); return SSLPL_ERR_ARG;
    }
    std::vector<int32_t> parent(1, -1); std::vector<uint8_t> desc(32, 0), leaf(1, 0); std::vector<double> weight(1, 0.0);
    for (;;) {
        int pid, isleaf;
        if (fscanf(f, "%d %d", &pid, &isleaf) != 2) break;
        uint8_t d[32];
        bool ok = true;
        for (int i = 0; i < 32 && ok; i++) { int b; ok = fscanf(f, "%d", &b) == 1; d[i] = (uint8_t)b; }
        double w = 0;
        ok = ok && fscanf(f, "%lf", &w) == 1;
        if (!ok) { fclose(f); set_error("%s: truncated node line", path); return SSLPL_ERR_ARG; }
        parent.push_back(pid); leaf.push_back(isleaf > 0 ? 1 : 0); weight.push_back(w); desc.insert(desc.end(), d, d + 32);
    }
    fclose(f);
    if (scoring) *scoring = n1;
    if (weighting) *weighting = n2;
    if (int rc = sslpl_vocab_create(device, k, L, (int)parent.size(), parent.data(), desc.data(), weight.data(), leaf.data(), out)) return rc;
    (*out)->scoring = n1; (*out)->weighting = n2;
    return SSLPL_OK;
}

void sslpl_vocab_destroy(sslpl_vocab* v) {
    if (!v) return;
    cudaSetDevice(v->device);
    if (v->arena) cudaFree(v->arena);
    delete v;
}

int sslpl_vocab_info(const sslpl_vocab* v, int* k, int* L, int* nnodes, int* nwords) {
    SSLPL_REQUIRE(v, SSLPL_ERR_ARG, "null vocabulary");
    if (k) *k = v->k;
    if (L) *L = v->L;
    if (nnodes) *nnodes = v->nnodes;
    if (nwords) *nwords = v->nwords;
    return SSLPL_OK;
}

int sslpl_vocab_level_nodes(const sslpl_vocab* v, int levelsup, int* count) {
    SSLPL_REQUIRE(v && count, SSLPL_ERR_ARG, "null argument");
    *count = vocab_level_nodes(v, levelsup);
    return SSLPL_OK;
}

int sslpl_bow_transform(sslpl_matcher* m, const sslpl_vocab* v, const uint8_t* desc, int n, int levelsup,
                        int32_t* word, int32_t* node, double* weight) {
    SSLPL_REQUIRE(m && v && (n == 0 || (desc && word && node && weight)), SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(n >= 0 && n <= m->cap, SSLPL_ERR_ARG, "n exceeds the matcher capacity");
    SSLPL_REQUIRE(v->device == m->p.device, SSLPL_ERR_ARG, "vocabulary and matcher live on different devices");
    if (n == 0) return SSLPL_OK;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    cudaStream_t st = m->stream;
    SSLPL_CUDA(cudaMemcpyAsync(m->desc, desc, (size_t)n * 32, cudaMemcpyHostToDevice, st));
    launch(m, k_vocab_transform<false>, dim3((n + 127) / 128, 1), 128, 0, m->desc, 0, nullptr, n, n, v->view, v->L - levelsup, m->word, m->node,
           nullptr, m->wgt, 0, nullptr);
    SSLPL_CUDA(cudaGetLastError());
    SSLPL_CUDA(cudaMemcpyAsync(word, m->word, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaMemcpyAsync(node, m->node, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaMemcpyAsync(weight, m->wgt, sizeof(double) * n, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaStreamSynchronize(st));
    return SSLPL_OK;
}

int sslpl_match_bow_batch_device_vocab(sslpl_matcher* m, const uint8_t* d_desc, const sslpl_keypoint* d_kps, const int* d_n,
                                       int nframes, int cap, const sslpl_vocab* v, int levelsup, float nnratio, int checkOri,
                                       int32_t* d_match, int32_t* d_nmatch, int32_t* d_word, int32_t* d_node, double* d_weight) {
    SSLPL_REQUIRE(m && v && d_desc && d_kps && d_n && d_match && d_nmatch, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(nframes >= 2 && nframes <= m->p.max_batch + 1, SSLPL_ERR_ARG, "nframes exceeds max_batch+1");
    const int nc = vocab_level_nodes(v, levelsup);
    SSLPL_REQUIRE(cap >= 1 && cap <= m->p.max_features + 64 && nc <= m->p.max_nodes, SSLPL_ERR_ARG, "cap or the vocabulary level exceeds the matcher capacity (max_nodes)");
    SSLPL_REQUIRE(v->device == m->p.device, SSLPL_ERR_ARG, "vocabulary and matcher live on different devices");
    if (int rc = csr_fits(nc, cap)) return rc;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    const int fc = m->p.max_features + 64;
    const dim3 grid((cap + 127) / 128, nframes);
    // optional per-feature outputs use the caller's [nframes][cap] layout; the dense node index goes to the workspace ([..][fc])
    if (d_word || d_node || d_weight)
        launch(m, k_vocab_transform<false>, grid, 128, 0, d_desc, (long long)cap * 32, d_n, 0, cap, v->view, v->L - levelsup, d_word, d_node, nullptr,
               d_weight, cap, nullptr);
    launch(m, k_vocab_transform<false>, grid, 128, 0, d_desc, (long long)cap * 32, d_n, 0, cap, v->view, v->L - levelsup, nullptr, nullptr, m->b_node,
           nullptr, fc, nullptr);
    return bow_batch_tail(m, d_desc, d_kps, d_n, nframes, cap, nc, nnratio, checkOri, d_match, d_nmatch);
}

// ---------------- Keyframe database over a row set in HBM (KeyFrameDatabase.cc) ----------------
// k_bow_vector keeps a power of two >= cap keys and cap weights (bow_rows_ok bounds them), k_kfdb_count / k_kfdb_score the query's
// cap (word, value) pairs (12 cap bytes, less than the former), k_kfdb_accumulate 8 bytes per database position: each in one CTA's
// shared memory.
constexpr int KFDB_MAX_DB = MAX_DYN_SMEM / 8;
static_assert(KFDB_MAX_DB <= (1 << KFDB_POS_BITS), "database positions must fit the sort key");
static int bow_pow2(int cap) { int P = 1; while (P < cap) P <<= 1; return P; }

static int bow_rows_ok(const sslpl_matcher* m, const int32_t* w, const double* v, const int32_t* n, int nrows, int cap) {
    SSLPL_REQUIRE(m && w && v && n, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(nrows >= 1, SSLPL_ERR_ARG, "nrows must be >= 1");
    SSLPL_REQUIRE(cap >= 1 && cap <= m->p.max_features + 64, SSLPL_ERR_ARG, "cap outside [1, max_features + 64]");
    SSLPL_REQUIRE((size_t)(bow_pow2(cap) + cap) * 8 <= (size_t)MAX_DYN_SMEM && cap < (1 << (31 - KFDB_POS_BITS)), SSLPL_ERR_ARG,
                  "cap exceeds what one CTA's shared memory holds (a power of two >= cap, plus cap, times 8 bytes <= 200 KB)");
    return SSLPL_OK;
}

int sslpl_bow_vectors_batch_device(sslpl_matcher* m, const sslpl_vocab* v, const uint8_t* d_desc, const int* d_n, int nrows, int cap,
                                   int32_t* d_bow_word, double* d_bow_val, int32_t* d_bow_n) {
    if (int rc = bow_rows_ok(m, d_bow_word, d_bow_val, d_bow_n, nrows, cap)) return rc;
    SSLPL_REQUIRE(v && d_desc && d_n, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(nrows <= 65535, SSLPL_ERR_ARG, "nrows exceeds 65535");
    SSLPL_REQUIRE(v->device == m->p.device, SSLPL_ERR_ARG, "vocabulary and matcher live on different devices");
    SSLPL_REQUIRE(v->scoring == 0 && v->weighting == 0, SSLPL_ERR_UNSUPPORTED, "BowVectors are built for TF_IDF weighting and L1 scoring only");
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    launch(m, k_vocab_transform<false>, dim3((cap + 127) / 128, nrows), 128, 0, d_desc, (long long)cap * 32, d_n, 0, cap, v->view, 0,
           d_bow_word, nullptr, nullptr, d_bow_val, cap, nullptr);
    const int P = bow_pow2(cap);
    launch(m, k_bow_vector, nrows, 512, (size_t)(P + cap) * 8, BowRows{d_bow_word, d_bow_val, d_bow_n, cap}, d_n, P);
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}

int sslpl_bow_score_batch_device(sslpl_matcher* m, const int32_t* d_bow_word, const double* d_bow_val, const int32_t* d_bow_n, int nrows,
                                 int cap, int npairs, const int32_t* d_pair, double* d_score) {
    if (int rc = bow_rows_ok(m, d_bow_word, d_bow_val, d_bow_n, nrows, cap)) return rc;
    SSLPL_REQUIRE(d_pair && d_score, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(npairs >= 1, SSLPL_ERR_ARG, "npairs must be >= 1");
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    launch(m, k_bow_score, (npairs + 127) / 128, 128, 0, BowRows{const_cast<int32_t*>(d_bow_word), const_cast<double*>(d_bow_val),
           const_cast<int32_t*>(d_bow_n), cap}, nrows, npairs, reinterpret_cast<const int2*>(d_pair), d_score);
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}

// DetectLoopCandidates (kLoop) / DetectRelocalizationCandidates for nq queries: the row -> position map of the database, then the scores
// of every query, then the accumulation of every query; reloc then leaves the keyframes' final scores in relocscore.
extern "C++" {
template <bool kLoop>
int kfdb_detect(sslpl_matcher* m, KfdbArgs A) {
    if (int rc = bow_rows_ok(m, A.B.word, A.B.val, A.B.n, A.nrows, A.B.cap)) return rc;
    SSLPL_REQUIRE(A.db && A.query && A.covis && A.cand && A.ncand && A.words && A.score, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(kLoop ? (A.conn_off && A.conn && A.minscore) : A.relocscore != nullptr, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(A.ndb >= 1 && A.ndb <= KFDB_MAX_DB, SSLPL_ERR_ARG, "ndb outside [1, 25600]");
    SSLPL_REQUIRE(A.nq >= 1 && A.nq <= 65535, SSLPL_ERR_ARG, "nq outside [1, 65535]");
    SSLPL_REQUIRE(!kLoop || A.nconn >= 0, SSLPL_ERR_ARG, "nconn must be >= 0");
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    // scratch: the row -> position map, the error word, maxw[nq]
    const size_t map_bytes = align_up((size_t)A.nrows * 4, 256);
    if (int rc = ensure_scratch(m, map_bytes + 256 + (size_t)A.nq * 4)) return rc;
    A.pos_of_row = reinterpret_cast<int32_t*>(m->scratch);
    A.err = reinterpret_cast<int32_t*>(m->scratch + map_bytes);
    A.maxw = reinterpret_cast<int32_t*>(m->scratch + map_bytes + 256);
    fill(m, A.pos_of_row, A.nrows, -1);
    SSLPL_CUDA(cudaMemsetAsync(A.err, 0, 256 + (size_t)A.nq * 4, m->stream));
    launch(m, k_kfdb_posmap, (A.ndb + 255) / 256, 256, 0, A);
    const dim3 chunks((A.ndb + KFDB_CHUNK - 1) / KFDB_CHUNK, A.nq);
    launch(m, k_kfdb_count<kLoop>, chunks, KFDB_CHUNK, (size_t)A.B.cap * 12, A);
    launch(m, k_kfdb_score<kLoop>, chunks, KFDB_CHUNK, (size_t)A.B.cap * 12, A);
    launch(m, k_kfdb_accumulate<kLoop>, A.nq, 512, (size_t)A.ndb * 8, A);
    if (!kLoop) launch(m, k_kfdb_reloc_state, (A.ndb + 255) / 256, 256, 0, A);
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}
}  // extern "C++"

int sslpl_detect_loop_candidates_batch_device(sslpl_matcher* m, const int32_t* d_bow_word, const double* d_bow_val, const int32_t* d_bow_n,
        int nrows, int cap, const int32_t* d_db, int ndb, const int32_t* d_query, int nq, const int32_t* d_covis,
        const int32_t* d_conn_off, const int32_t* d_conn, int nconn, const float* d_minscore,
        int32_t* d_cand, int32_t* d_ncand, int32_t* d_words, float* d_score) {
    KfdbArgs A; memset(&A, 0, sizeof(A));
    A.B = BowRows{const_cast<int32_t*>(d_bow_word), const_cast<double*>(d_bow_val), const_cast<int32_t*>(d_bow_n), cap};
    A.nrows = nrows; A.db = d_db; A.ndb = ndb; A.query = d_query; A.nq = nq; A.covis = d_covis;
    A.conn_off = d_conn_off; A.conn = d_conn; A.nconn = nconn; A.minscore = d_minscore;
    A.cand = d_cand; A.ncand = d_ncand; A.words = d_words; A.score = d_score;
    return kfdb_detect<true>(m, A);
}

int sslpl_detect_relocalization_candidates_batch_device(sslpl_matcher* m, const int32_t* d_bow_word, const double* d_bow_val,
        const int32_t* d_bow_n, int nrows, int cap, const int32_t* d_db, int ndb, const int32_t* d_query, int nq, const int32_t* d_covis,
        float* d_relocscore, int32_t* d_cand, int32_t* d_ncand, int32_t* d_words, float* d_score) {
    KfdbArgs A; memset(&A, 0, sizeof(A));
    A.B = BowRows{const_cast<int32_t*>(d_bow_word), const_cast<double*>(d_bow_val), const_cast<int32_t*>(d_bow_n), cap};
    A.nrows = nrows; A.db = d_db; A.ndb = ndb; A.query = d_query; A.nq = nq; A.covis = d_covis; A.relocscore = d_relocscore;
    A.cand = d_cand; A.ncand = d_ncand; A.words = d_words; A.score = d_score;
    return kfdb_detect<false>(m, A);
}

int sslpl_match_lines_batch_device(sslpl_matcher* m, const uint8_t* d_ldesc, const int* d_nl, int nframes, int capl,
                                   int32_t* d_lmatch, int32_t* d_nlmatch) {
    SSLPL_REQUIRE(m && d_ldesc && d_nl && d_lmatch && d_nlmatch, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(nframes >= 2 && nframes <= m->p.max_batch + 1 && capl >= 1 && capl <= m->p.max_lines + 64, SSLPL_ERR_ARG, "batch or capacity exceeds the matcher capacity");
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    cudaStream_t st = m->stream;
    const int npairs = nframes - 1, lc = m->p.max_lines + 64;
    launch(m, k_knn2<false>, dim3((capl + 7) / 8, npairs), 256, 0, d_ldesc, (long long)capl * 32, d_nl, 0, d_ldesc + (size_t)capl * 32, (long long)capl * 32,
           d_nl, 0, m->b_knn, (long long)lc * 4, capl, nullptr, 0);
    fill(m, d_lmatch, (long long)npairs * capl, -1);
    SSLPL_CUDA(cudaMemsetAsync(d_nlmatch, 0, sizeof(int32_t) * npairs, st));
    launch(m, k_line_ratio<false>, dim3((capl + 127) / 128, npairs), 128, 0, m->b_knn, (long long)lc * 4, d_nl, 0, capl, nullptr, 0, d_lmatch, capl,
           d_nlmatch, nullptr, 0, nullptr, 0);
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}

// ---------------- LocalMapping's matchers over keyframe pairs in HBM (SURVEY.md 8(f) rows 2/3) ----------------
// SearchForTriangulation for a list of (KF1, KF2) pairs of one keyframe set: the FeatureVector of every keyframe (KeyFrame::ComputeBoW's,
// from the descriptors), then k_tri_match over the pair map with per-pair F12 / epipole, the rotation filter and the ordered compaction.
static int tri_match_stage(sslpl_matcher* m,
        const sslpl_keypoint* d_kps, const uint8_t* d_desc, const int* d_n, int nkf, int cap, const uint8_t* d_has_mp,
        const sslpl_vocab* v, int levelsup, int npairs, const int32_t* d_pair, const float* d_geom,
        const float* scale, const float* sigma2, int nlevels) {
    SSLPL_REQUIRE(d_kps && d_desc && d_n && d_has_mp && v && d_pair && d_geom && scale && sigma2, SSLPL_ERR_ARG, "null argument");
    if (int rc = kf_pairs_ok(m, nkf, cap, m->p.max_features, npairs)) return rc;
    SSLPL_REQUIRE(nlevels >= 1 && nlevels <= SSLPL_MAX_LEVELS, SSLPL_ERR_ARG, "nlevels out of range");
    const int nc = vocab_level_nodes(v, levelsup);
    SSLPL_REQUIRE(nc <= m->p.max_nodes, SSLPL_ERR_ARG, "the vocabulary level exceeds the matcher capacity (max_nodes)");
    SSLPL_REQUIRE(v->device == m->p.device, SSLPL_ERR_ARG, "vocabulary and matcher live on different devices");
    if (int rc = csr_fits(nc, cap)) return rc;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    const int fc = m->p.max_features + 64, NN = m->p.max_nodes + 1;
    if (int rc = first_use(m->tw, sizeof(int32_t) * (size_t)m->p.max_batch * fc)) return rc;
    launch(m, k_vocab_transform<false>, dim3((cap + 127) / 128, nkf), 128, 0, d_desc, (long long)cap * 32, d_n, 0, cap, v->view, v->L - levelsup,
           nullptr, nullptr, m->b_node, nullptr, fc, nullptr);
    launch(m, k_build_csr, nkf, 128, (nc + 1 + cap) * sizeof(int), m->b_node, fc, d_n, cap, nc, m->b_off, NN + 1, m->b_idx, fc);
    fill(m, m->tw, (long long)npairs * cap, -1);
    FrameSet S = dense_set(m, d_desc, d_kps, cap, nc, d_has_mp);
    S.pmap = reinterpret_cast<const int2*>(d_pair); S.nframes = nkf;
    TriArgs T; memset(&T, 0, sizeof(T));
    T.nlevels = nlevels;
    for (int i = 0; i < nlevels; i++) { T.scale[i] = scale[i]; T.sigma2[i] = sigma2[i]; }
    // b_rot is only read where the table holds a match, and k_tri_match writes both together
    launch(m, k_tri_match<true>, dim3((nc + 3) / 4, npairs), 128, 0, S, T, d_geom, m->tw, cap, m->b_rot, fc);
    return SSLPL_OK;
}

int sslpl_search_for_triangulation_batch_device(sslpl_matcher* m,
        const sslpl_keypoint* d_kps, const uint8_t* d_desc, const int* d_n, int nkf, int cap, const uint8_t* d_has_mp,
        const sslpl_vocab* v, int levelsup, int npairs, const int32_t* d_pair, const float* d_geom,
        const float* scale, const float* sigma2, int nlevels, int checkOrientation, int32_t* d_pairs, int32_t* d_nmatch) {
    SSLPL_REQUIRE(m && d_pairs && d_nmatch, SSLPL_ERR_ARG, "null argument");
    if (int rc = tri_match_stage(m, d_kps, d_desc, d_n, nkf, cap, d_has_mp, v, levelsup, npairs, d_pair, d_geom, scale, sigma2, nlevels)) return rc;
    const int fc = m->p.max_features + 64;
    fill(m, d_pairs, 2LL * npairs * cap, -1);
    launch(m, k_rot_filter, npairs, 256, 0, m->tw, cap, m->b_rot, fc, nullptr, 0, cap, cap, checkOrientation, d_nmatch, d_pairs, 2LL * cap);
    launch(m, k_bad_pairs, (npairs + 127) / 128, 128, 0, reinterpret_cast<const int2*>(d_pair), npairs, nkf, d_nmatch);
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}

// LSDmatcher::SearchForTriangulation for a list of (KF1, KF2) pairs: k_knn2 over the pair map (query = KF1's lines, train = KF2's), then
// k_line_tri (lineDescriptorMAD, the filter and the compaction) per pair.
int sslpl_line_search_for_triangulation_batch_device(sslpl_matcher* m, const uint8_t* d_ldesc, const int* d_nl, int nkf, int capl,
        const uint8_t* d_has_ml, int npairs, const int32_t* d_pair, int32_t* d_lpairs, int32_t* d_nlmatch) {
    SSLPL_REQUIRE(m && d_ldesc && d_nl && d_has_ml && d_pair && d_lpairs && d_nlmatch, SSLPL_ERR_ARG, "null argument");
    if (int rc = kf_pairs_ok(m, nkf, capl, m->p.max_lines, npairs)) return rc;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    const int lc = m->p.max_lines + 64;
    const int2* pmap = reinterpret_cast<const int2*>(d_pair);
    launch(m, k_knn2<true>, dim3((capl + 7) / 8, npairs), 256, 0, d_ldesc, (long long)capl * 32, d_nl, 0, d_ldesc, (long long)capl * 32, d_nl, 0,
           m->b_knn, (long long)lc * 4, capl, pmap, nkf);
    launch(m, k_line_tri, npairs, 256, 0, m->b_knn, (long long)lc * 4, d_nl, capl, pmap, nkf, d_has_ml, 0.1, d_lpairs, d_nlmatch);
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}

// LSDmatcher::SerachForInitialize for a list of (initial frame, frame) pairs: k_knn2 over the pair map, then k_line_tri without masks at
// 0.5 nn12_mad per pair.
int sslpl_line_search_for_initialize_batch_device(sslpl_matcher* m, const uint8_t* d_ldesc, const int* d_nl, int nrows, int capl,
        int npairs, const int32_t* d_pair, int32_t* d_lpairs, int32_t* d_nlmatch) {
    SSLPL_REQUIRE(m && d_ldesc && d_nl && d_pair && d_lpairs && d_nlmatch, SSLPL_ERR_ARG, "null argument");
    if (int rc = kf_pairs_ok(m, nrows, capl, m->p.max_lines, npairs)) return rc;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    const int lc = m->p.max_lines + 64;
    const int2* pmap = reinterpret_cast<const int2*>(d_pair);
    launch(m, k_knn2<true>, dim3((capl + 7) / 8, npairs), 256, 0, d_ldesc, (long long)capl * 32, d_nl, 0, d_ldesc, (long long)capl * 32, d_nl, 0,
           m->b_knn, (long long)lc * 4, capl, pmap, nrows);
    launch(m, k_line_tri, npairs, 256, 0, m->b_knn, (long long)lc * 4, d_nl, capl, pmap, nrows, nullptr, 0.5, d_lpairs, d_nlmatch);
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}

// LocalMapping::CreateNewMapPoints' neighbour loop over the chains of a pair list: the unfiltered SearchForTriangulation rows of every pair
// (tri_match_stage, checkOrientation false), then k_create_points_chain, one CTA per chain.
int sslpl_create_new_map_points_batch_device(sslpl_matcher* m,
        const sslpl_keypoint* d_kps, const uint8_t* d_desc, const int* d_n, int nkf, int cap, const uint8_t* d_has_mp,
        const sslpl_vocab* v, int levelsup, int npairs, const int32_t* d_pair, const float* d_geom, const float* d_kfpose,
        const float* cam, const float* scaleFactors, const float* levelSigma2, int nlevels, float scaleFactor,
        int32_t* d_pairs, int32_t* d_nmatch, int32_t* d_status, float* d_x3d, int32_t* d_nnew) {
    SSLPL_REQUIRE(m && d_kfpose && cam && d_pairs && d_nmatch && d_status && d_x3d && d_nnew, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(scaleFactor > 0.f && scaleFactor < INFINITY, SSLPL_ERR_ARG, "scaleFactor must be positive and finite");
    CreateArgs C; memset(&C, 0, sizeof(C));
    C.fx = cam[0]; C.fy = cam[1]; C.cx = cam[2]; C.cy = cam[3]; C.invfx = cam[4]; C.invfy = cam[5];
    C.ratioFactor = 1.5f * scaleFactor;
    if (int rc = tri_match_stage(m, d_kps, d_desc, d_n, nkf, cap, d_has_mp, v, levelsup, npairs, d_pair, d_geom, scaleFactors, levelSigma2, nlevels)) return rc;
    C.nlevels = nlevels;
    for (int i = 0; i < nlevels; i++) { C.scale[i] = scaleFactors[i]; C.sigma2[i] = levelSigma2[i]; }
    const size_t smem = sizeof(unsigned) * (size_t)((cap + 31) / 32);
    launch(m, k_create_points_chain, npairs, 256, smem, reinterpret_cast<const int2*>(d_pair), npairs, nkf, m->tw, cap,
           reinterpret_cast<const float*>(d_kps), d_n, d_has_mp, d_kfpose, C, d_pairs, d_nmatch, d_status, d_x3d, d_nnew);
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}

// LocalMapping::CreateNewMapLines2's neighbour loop over the chains of a pair list: k_knn2 over the pair map, the KF1-unmasked rows of
// every pair (k_line_tri_table), then k_create_lines_chain, one CTA per chain.
int sslpl_create_new_map_lines_batch_device(sslpl_matcher* m,
        const sslpl_keyline* d_kl, const uint8_t* d_ldesc, const double* d_lineeq, const int* d_nl, int nkf, int capl,
        const uint8_t* d_has_ml, int npairs, const int32_t* d_pair, const float* d_kfpose, const float* d_kfdepth, const float* cam,
        int32_t* d_lpairs, int32_t* d_nlmatch, int32_t* d_status, float* d_line3d, int32_t* d_nnew) {
    SSLPL_REQUIRE(m && d_kl && d_ldesc && d_lineeq && d_nl && d_has_ml && d_pair && d_kfpose && d_kfdepth && cam && d_lpairs && d_nlmatch &&
                  d_status && d_line3d && d_nnew, SSLPL_ERR_ARG, "null argument");
    if (int rc = kf_pairs_ok(m, nkf, capl, m->p.max_lines, npairs)) return rc;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    const int lc = m->p.max_lines + 64;
    if (int rc = first_use(m->ltw, sizeof(int32_t) * (size_t)m->p.max_batch * lc)) return rc;
    LineCam C;
    C.fx = cam[0]; C.fy = cam[1]; C.cx = cam[2]; C.cy = cam[3]; C.invfx = cam[4]; C.invfy = cam[5];
    const int2* pmap = reinterpret_cast<const int2*>(d_pair);
    launch(m, k_knn2<true>, dim3((capl + 7) / 8, npairs), 256, 0, d_ldesc, (long long)capl * 32, d_nl, 0, d_ldesc, (long long)capl * 32, d_nl, 0,
           m->b_knn, (long long)lc * 4, capl, pmap, nkf);
    launch(m, k_line_tri_table, npairs, 256, 0, m->b_knn, (long long)lc * 4, d_nl, capl, pmap, nkf, d_has_ml, m->ltw);
    const size_t smem = sizeof(unsigned) * (size_t)((capl + 31) / 32);
    launch(m, k_create_lines_chain, npairs, 256, smem, pmap, npairs, nkf, m->ltw, capl, reinterpret_cast<const float*>(d_kl), d_lineeq, d_nl,
           d_has_ml, d_kfpose, d_kfdepth, C, d_lpairs, d_nlmatch, d_status, d_line3d, d_nnew);
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}

int sslpl_matcher_debug_svd4(sslpl_matcher* m, int n, const float* A, float* W, float* Vt, int nh, const double* hx, const double* hy, double* h) {
    SSLPL_REQUIRE(m && n >= 0 && nh >= 0 && (n == 0 || (A && W && Vt)) && (nh == 0 || (hx && hy && h)), SSLPL_ERR_ARG, "null argument");
    const int nt = std::max(n, nh);
    if (nt == 0) return SSLPL_OK;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    cudaStream_t st = m->stream;
    if (int rc = ensure_scratch(m, (size_t)n * 36 * sizeof(float) + (size_t)nh * 3 * sizeof(double) + 4096)) return rc;
    Arena Ar; Ar.base = m->scratch; Ar.used = 0;
    cudaError_t e = cudaSuccess;
    const float* d_A = stage(Ar, A, (size_t)16 * n, st, e); float* d_W = Ar.take<float>((size_t)4 * n + 8); float* d_V = Ar.take<float>((size_t)16 * n + 8);
    const double* d_hx = stage(Ar, hx, nh, st, e); const double* d_hy = stage(Ar, hy, nh, st, e); double* d_h = Ar.take<double>((size_t)nh + 8);
    SSLPL_CUDA(e);
    launch(m, k_debug_svd4, (nt + 127) / 128, 128, 0, n, d_A, d_W, d_V, nh, d_hx, d_hy, d_h);
    SSLPL_CUDA(cudaGetLastError());
    if (n) {
        SSLPL_CUDA(cudaMemcpyAsync(W, d_W, sizeof(float) * 4 * (size_t)n, cudaMemcpyDeviceToHost, st));
        SSLPL_CUDA(cudaMemcpyAsync(Vt, d_V, sizeof(float) * 16 * (size_t)n, cudaMemcpyDeviceToHost, st));
    }
    if (nh) SSLPL_CUDA(cudaMemcpyAsync(h, d_h, sizeof(double) * (size_t)nh, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaStreamSynchronize(st));
    return SSLPL_OK;
}

// ---------------- PredictScale thresholds and LocalMapping::SearchInNeighbors' Fuse over keyframes in HBM (SURVEY.md 8(f) rows 2/3) ----------------
// t_k = the smallest positive float r with (int)ceil(logf(r) / logScaleFactor) >= k, by bisection over the bit patterns of the positive
// floats with this process's logf (+inf when no finite r gets there).  The level is compared in float: for any logScaleFactor of a float
// scale factor > 1 (>= 1.19e-7) |ceil(logf(r) / s)| < 2^31, where the float compare and the int conversion agree.
int sslpl_predict_scale_table(float logScaleFactor, int nlevels, float* thr) {
    SSLPL_REQUIRE(thr, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(nlevels >= 1 && nlevels <= SSLPL_MAX_LEVELS, SSLPL_ERR_ARG, "nlevels outside [1, SSLPL_MAX_LEVELS]");
    SSLPL_REQUIRE(logScaleFactor > 0.f && logScaleFactor < INFINITY, SSLPL_ERR_ARG, "logScaleFactor must be positive and finite");
    for (int k = 0; k <= nlevels; k++) {
        uint32_t lo = 1, hi = 0x7f800000u;                                // hi = +inf: never evaluated
        while (lo < hi) {
            const uint32_t mid = lo + (hi - lo) / 2;
            float r; memcpy(&r, &mid, 4);
            if (std::ceil(logf(r) / logScaleFactor) >= (float)k) hi = mid; else lo = mid + 1;
        }
        memcpy(&thr[k], &lo, 4);
    }
    return SSLPL_OK;
}

static int predict_table(PredictTable& T, float logScaleFactor, int nlevels) {
    memset(&T, 0, sizeof(T));
    T.nlevels = nlevels;
    return sslpl_predict_scale_table(logScaleFactor, nlevels, T.thr);
}

int sslpl_matcher_debug_predict_scale(sslpl_matcher* m, int n, const float* ratio, float logScaleFactor, int nlevels, int clamp, int32_t* level) {
    SSLPL_REQUIRE(m && n >= 0 && (n == 0 || (ratio && level)), SSLPL_ERR_ARG, "null argument");
    PredictTable T;
    if (int rc = predict_table(T, logScaleFactor, nlevels)) return rc;
    if (n == 0) return SSLPL_OK;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    cudaStream_t st = m->stream;
    if (int rc = ensure_scratch(m, (size_t)n * 8 + 1024)) return rc;
    Arena A; A.base = m->scratch; A.used = 0;
    cudaError_t e = cudaSuccess;
    float* d_r = stage(A, ratio, n, st, e); int32_t* d_l = A.take<int32_t>(n + 8);
    SSLPL_CUDA(e);
    launch(m, k_predict_scale, (n + 255) / 256, 256, 0, n, d_r, T, clamp, d_l);
    SSLPL_CUDA(cudaGetLastError());
    SSLPL_CUDA(cudaMemcpyAsync(level, d_l, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaStreamSynchronize(st));
    return SSLPL_OK;
}

static int fuse_map_common(FuseMap& M, sslpl_matcher* m, int nkf, int cap, int rows, int nel, int nentries, const int32_t* d_entry,
                           const uint8_t* d_skip, const float* d_kfpose, const float* d_el, const uint8_t* d_eldesc, const float* cam,
                           const float* bounds, const float* scaleFactors, int nlevels, float logScaleFactor) {
    SSLPL_REQUIRE(d_entry && d_kfpose && d_el && d_eldesc && cam && bounds && scaleFactors, SSLPL_ERR_ARG, "null argument");
    if (int rc = kf_set_ok(m, nkf, cap, rows)) return rc;
    SSLPL_REQUIRE(nel >= 0 && nentries >= 0, SSLPL_ERR_ARG, "negative count");
    SSLPL_REQUIRE(nlevels >= 1 && nlevels <= SSLPL_MAX_LEVELS, SSLPL_ERR_ARG, "nlevels outside [1, SSLPL_MAX_LEVELS]");
    memset(&M, 0, sizeof(M));
    if (int rc = grid_geom(M.G, bounds, scaleFactors, nlevels)) return rc;
    if (int rc = predict_table(M.T, logScaleFactor, nlevels)) return rc;
    M.entry = reinterpret_cast<const int2*>(d_entry); M.skip = d_skip; M.nkf = nkf; M.nel = nel;
    M.pose = d_kfpose; M.el = d_el; M.eldesc = d_eldesc;
    M.fx = cam[0]; M.fy = cam[1]; M.cx = cam[2]; M.cy = cam[3];
    return SSLPL_OK;
}

// ORBmatcher::Fuse(pKF, vpMapPoints, th) for a flat list of (keyframe, MapPoint) entries: the 64 x 48 grid of every keyframe (frame on
// grid.y, one k_build_csr CTA per keyframe), then one warp per entry: projection stage and search (k_point_fuse_search<true>).
int sslpl_fuse_points_batch_device(sslpl_matcher* m,
        const sslpl_keypoint* d_kps, const uint8_t* d_desc, const int* d_n, int nkf, int cap, const float* d_kfpose,
        int nmp, const float* d_mp, const uint8_t* d_mpdesc, int nentries, const int32_t* d_entry, const uint8_t* d_skip,
        const float* cam, const float* bounds, const float* scaleFactors, const float* invLevelSigma2, int nlevels, float logScaleFactor, float th,
        int32_t* d_best_idx, int32_t* d_best_dist) {
    SSLPL_REQUIRE(m && d_kps && d_desc && d_n && invLevelSigma2 && d_best_idx && d_best_dist, SSLPL_ERR_ARG, "null argument");
    FuseMap M;
    if (int rc = fuse_map_common(M, m, nkf, cap, m->p.max_features, nmp, nentries, d_entry, d_skip, d_kfpose, d_mp, d_mpdesc, cam, bounds,
                                 scaleFactors, nlevels, logScaleFactor)) return rc;
    const int nc = GRID_COLS * GRID_ROWS;
    if (int rc = csr_fits(nc, cap)) return rc;
    if (nentries == 0) return SSLPL_OK;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    const int fc = m->p.max_features + 64;
    for (int k = 0; k < nlevels; k++) M.invSigma2[k] = invLevelSigma2[k];
    const float* kf = reinterpret_cast<const float*>(d_kps);              // sslpl_keypoint = 7 x 4 B: x y size angle response octave class_id
    M.kp = kf; M.kp_fs = 7LL * cap; M.desc = d_desc; M.desc_fs = 32LL * cap; M.n = d_n; M.cap = cap;
    WinArgs A; memset(&A, 0, sizeof(A));
    A.G = M.G; A.th = th;
    if (int rc = grid_batch_build(m, kf, d_n, nkf, cap, A.G)) return rc;
    M.goff = m->pw_off; M.gidx = m->pw_idx; M.goff_fs = nc + 1; M.gidx_fs = fc;
    launch(m, k_point_fuse_search<true>, (nentries + 3) / 4, 128, 0, A, nentries, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
           nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, d_best_idx, d_best_dist, M);
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}

// LSDmatcher::Fuse(pKF, vpMapLines, th) for a flat list of (keyframe, MapLine) entries: one warp per entry, projection stage and search
// over the keyframe's sslpl_keyline rows (k_line_fuse_search<true>).
int sslpl_fuse_lines_batch_device(sslpl_matcher* m,
        const sslpl_keyline* d_kl, const uint8_t* d_ldesc, const int* d_nl, int nkf, int capl, const float* d_kfpose,
        int nml, const float* d_ml, const uint8_t* d_mldesc, int nentries, const int32_t* d_entry, const uint8_t* d_skip,
        const float* cam, const float* bounds, const float* scaleFactors, int nlevels, float logScaleFactor, float th,
        int32_t* d_best_idx, int32_t* d_best_dist) {
    SSLPL_REQUIRE(m && d_kl && d_ldesc && d_nl && d_best_idx && d_best_dist, SSLPL_ERR_ARG, "null argument");
    FuseMap M;
    if (int rc = fuse_map_common(M, m, nkf, capl, m->p.max_lines, nml, nentries, d_entry, d_skip, d_kfpose, d_ml, d_mldesc, cam, bounds,
                                 scaleFactors, nlevels, logScaleFactor)) return rc;
    if (nentries == 0) return SSLPL_OK;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    M.kp = reinterpret_cast<const float*>(d_kl); M.kp_fs = 17LL * capl; M.desc = d_ldesc; M.desc_fs = 32LL * capl; M.n = d_nl; M.cap = capl;
    launch(m, k_line_fuse_search<true>, (nentries + 3) / 4, 128, 0, nentries, nullptr, nullptr, nullptr, nullptr, 0, nullptr, nullptr, nullptr,
           nullptr, th, d_best_idx, d_best_dist, M);
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}

// The map-element refresh of include/sslpl_map.h: the first entry of every element (k_first_entry over a table in the scratch), then
// one warp per entry (k_map_update<kLine>, passed as `kernel`).
static int map_update(sslpl_matcher* m, void (*kernel)(MapUpd), MapUpd& U, int rows, int nel, bool el_ok, const float* scaleFactors, int nlevels,
                      const int32_t* d_elem, const int32_t* d_refkf, const int32_t* d_obs_off, const int32_t* d_obs, int nupd) {
    SSLPL_REQUIRE(U.kp && U.desc && U.n, SSLPL_ERR_ARG, "null argument");
    if (int rc = kf_set_ok(m, U.nkf, U.cap, rows)) return rc;
    SSLPL_REQUIRE(U.what >= 1 && U.what <= 3, SSLPL_ERR_ARG, "what outside {1, 2, 3}");
    SSLPL_REQUIRE(nel >= 0 && nupd >= 0, SSLPL_ERR_ARG, "negative count");
    SSLPL_REQUIRE(nlevels >= 1 && nlevels <= SSLPL_MAX_LEVELS, SSLPL_ERR_ARG, "nlevels outside [1, SSLPL_MAX_LEVELS]");
    const bool geom = U.what & SSLPL_MAPUPD_GEOM, dsc = U.what & SSLPL_MAPUPD_DESC;
    SSLPL_REQUIRE((!dsc || U.eldesc) && (!geom || (el_ok && U.pose && scaleFactors)), SSLPL_ERR_ARG, "null argument");
    if (nupd == 0) return SSLPL_OK;
    SSLPL_REQUIRE(d_elem && d_obs_off && d_obs && U.status && (!geom || d_refkf), SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(reinterpret_cast<uintptr_t>(d_obs) % 8 == 0, SSLPL_ERR_ARG, "d_obs must be 8-byte aligned (read as int2 pairs)");
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    if (geom) for (int k = 0; k < nlevels; k++) U.scale[k] = scaleFactors[k];
    U.nlevels = nlevels; U.nel = nel; U.nupd = nupd;
    U.elem = d_elem; U.refkf = d_refkf; U.off = d_obs_off; U.obs = reinterpret_cast<const int2*>(d_obs);
    if (int rc = ensure_scratch(m, sizeof(int32_t) * ((size_t)nel + 1))) return rc;
    int32_t* first = reinterpret_cast<int32_t*>(m->scratch);
    U.first = first;
    if (nel > 0) {
        if (int rc = fill(m, first, nel, INT_MAX)) return rc;
        launch(m, k_first_entry, (nupd + 255) / 256, 256, 0, d_elem, nupd, nel, first);
    }
    launch(m, kernel, (nupd + 3) / 4, 128, 0, U);
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}

int sslpl_update_map_points_batch_device(sslpl_matcher* m,
        const sslpl_keypoint* d_kps, const uint8_t* d_desc, const int* d_n, int nkf, int cap,
        const float* d_kfpose, const uint8_t* d_kfbad,
        int nmp, float* d_mp, uint8_t* d_mpdesc,
        int nupd, const int32_t* d_elem, const int32_t* d_refkf, const int32_t* d_obs_off, const int32_t* d_obs,
        const float* scaleFactors, int nlevels, int what, int32_t* d_status) {
    SSLPL_REQUIRE(m, SSLPL_ERR_ARG, "null handle");
    MapUpd U;
    memset(&U, 0, sizeof(U));
    U.kp = reinterpret_cast<const float*>(d_kps); U.kp_fs = 7LL * cap; U.desc = d_desc; U.desc_fs = 32LL * cap; U.n = d_n; U.cap = cap;
    U.nkf = nkf; U.pose = d_kfpose; U.kfbad = d_kfbad; U.el = d_mp; U.eldesc = d_mpdesc; U.what = what; U.status = d_status;
    return map_update(m, k_map_update<false>, U, m->p.max_features, nmp, d_mp != nullptr, scaleFactors, nlevels, d_elem, d_refkf, d_obs_off, d_obs, nupd);
}

int sslpl_update_map_lines_batch_device(sslpl_matcher* m,
        const sslpl_keyline* d_kl, const uint8_t* d_ldesc, const int* d_nl, int nkf, int capl,
        const float* d_kfpose, const uint8_t* d_kfbad,
        int nml, const double* d_mlpos, float* d_ml, uint8_t* d_mldesc, double* d_mlnormal,
        int nupd, const int32_t* d_elem, const int32_t* d_refkf, const int32_t* d_obs_off, const int32_t* d_obs,
        const float* scaleFactors, int nlevels, int what, int32_t* d_status) {
    SSLPL_REQUIRE(m, SSLPL_ERR_ARG, "null handle");
    MapUpd U;
    memset(&U, 0, sizeof(U));
    U.kp = reinterpret_cast<const float*>(d_kl); U.kp_fs = 17LL * capl; U.desc = d_ldesc; U.desc_fs = 32LL * capl; U.n = d_nl; U.cap = capl;
    U.nkf = nkf; U.pose = d_kfpose; U.kfbad = d_kfbad; U.el = d_ml; U.eldesc = d_mldesc; U.pos = d_mlpos; U.nrm64 = d_mlnormal;
    U.what = what; U.status = d_status;
    return map_update(m, k_map_update<true>, U, m->p.max_lines, nml, d_ml && d_mlpos, scaleFactors, nlevels, d_elem, d_refkf, d_obs_off, d_obs, nupd);
}

// The arguments of SearchByProjection(Frame, KeyFrame) common to the single and the batched call
static int reloc_args(RelocArgs& A, const float* cam, const float* bounds, const float* scaleFactors, int nlevels, float logScaleFactor, float th,
               int ORBdist, int checkOri) {
    SSLPL_REQUIRE(cam && bounds && scaleFactors, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(nlevels >= 1 && nlevels <= SSLPL_MAX_LEVELS, SSLPL_ERR_ARG, "nlevels outside [1, SSLPL_MAX_LEVELS]");
    memset(&A, 0, sizeof(A));
    if (int rc = grid_geom(A.G, bounds, scaleFactors, nlevels)) return rc;
    SSLPL_REQUIRE(th > 0.f, SSLPL_ERR_ARG, "th must be positive");
    // with no candidate in the window bestDist stays 256 and bestIdx2 -1: ORBdist >= 256 would make the reference write mvpMapPoints[-1]
    SSLPL_REQUIRE(ORBdist < 256, SSLPL_ERR_ARG, "ORBdist must be below 256");
    if (int rc = predict_table(A.T, logScaleFactor, nlevels)) return rc;
    A.fx = cam[0]; A.fy = cam[1]; A.cx = cam[2]; A.cy = cam[3];
    A.th = th; A.ORBdist = ORBdist; A.checkOri = checkOri ? 1 : 0;
    return SSLPL_OK;
}

// The grid of every pair's frame (AssignFeaturesToGrid over the pair's gathered rows), then one walker warp per pair.  R's row set, map,
// pairs and outputs are set; the workspace is ensure_reloc_ws's.
static int reloc_run(sslpl_matcher* m, const RelocArgs& A, RelocSet& R) {
    const int nc = GRID_COLS * GRID_ROWS, W = m->cap;
    R.xy = m->rw_xy; R.wn = m->rw_n; R.goff = m->rw_off; R.gidx = m->rw_idx; R.goff_fs = nc + 1;
    R.claimed = m->rw_claimed; R.sel = m->rw_sel; R.rbin = m->rw_rbin; R.ws_fs = W;
    launch(m, k_reloc_gather_xy, dim3((R.cap + 127) / 128, R.npairs), 128, 0, R);
    launch(m, k_grid_cells, dim3((R.cap + 127) / 128, R.npairs), 128, 0, m->rw_xy, m->rw_xy + 1, 2, 2LL * W, m->rw_n, 0, R.cap,
           A.G, m->rw_cell, (long long)W);
    launch(m, k_build_csr, R.npairs, 128, (nc + 1 + R.cap) * sizeof(int), m->rw_cell, (long long)W, m->rw_n, R.cap, nc, m->rw_off,
           (long long)(nc + 1), m->rw_idx, (long long)W);
    launch(m, k_proj_match_kf, R.npairs, 32, 0, A, R);
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}


int sslpl_search_by_projection_kf(sslpl_matcher* m,
        int n1, const uint8_t* flag1, const float* Xw, const uint8_t* dmp, const float* dist3, const float* angle1,
        int n2, const uint8_t* d2, const float* x2, const float* y2, const int32_t* oct2, const float* angle2, const uint8_t* held2,
        const float* Tcw, const float* cam, const float* bounds, const float* scaleFactors, int nlevels, float logScaleFactor,
        float th, int ORBdist, int checkOrientation, int32_t* assign2, int* nmatches) {
    SSLPL_REQUIRE(m && Tcw && assign2 && nmatches, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(n1 >= 0 && n2 >= 0 && n1 <= m->p.max_features && n2 <= m->p.max_features, SSLPL_ERR_ARG, "feature count exceeds max_features");
    SSLPL_REQUIRE(n1 == 0 || (flag1 && Xw && dmp && dist3 && angle1), SSLPL_ERR_ARG, "null keyframe array");
    SSLPL_REQUIRE(n2 == 0 || (d2 && x2 && y2 && oct2 && angle2), SSLPL_ERR_ARG, "null frame array");
    RelocArgs A;
    if (int rc = reloc_args(A, cam, bounds, scaleFactors, nlevels, logScaleFactor, th, ORBdist, checkOrientation)) return rc;
    const int W = m->cap, nc = GRID_COLS * GRID_ROWS;
    if (int rc = csr_fits(nc, W)) return rc;
    for (int j = 0; j < n2; j++) assign2[j] = -1;
    *nmatches = 0;
    if (n1 == 0 || n2 == 0) return SSLPL_OK;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    if (int rc = ensure_reloc_ws(m)) return rc;
    cudaStream_t st = m->stream;
    // row 0 = the keyframe (mvKeysUn angles), row 1 = the frame; MapPoint i of the keyframe is element i
    std::vector<sslpl_keypoint> kp((size_t)W + n2);
    memset(kp.data(), 0, kp.size() * sizeof(sslpl_keypoint));
    for (int i = 0; i < n1; i++) kp[i].angle = angle1[i];
    for (int j = 0; j < n2; j++) { sslpl_keypoint& k = kp[(size_t)W + j]; k.x = x2[j]; k.y = y2[j]; k.octave = oct2[j]; k.angle = angle2[j]; }
    std::vector<float> el((size_t)n1 * 9, 0.f);
    std::vector<int32_t> kfmp(n1), misc = {n1, n2, 0, 1};
    for (int i = 0; i < n1; i++) {
        kfmp[i] = flag1[i] ? i : -1;
        for (int c = 0; c < 3; c++) { el[9 * (size_t)i + c] = Xw[3 * (size_t)i + c]; el[9 * (size_t)i + 6 + c] = dist3[3 * (size_t)i + c]; }
    }
    SSLPL_CUDA(cudaMemcpyAsync(m->kpf, kp.data(), kp.size() * sizeof(sslpl_keypoint), cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->desc + 32LL * W, d2, (size_t)n2 * 32, cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->ncnt, misc.data(), 2 * sizeof(int), cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->rw_pair, misc.data() + 2, 2 * sizeof(int), cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->rw_T, Tcw, 12 * sizeof(float), cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->rw_kfmp, kfmp.data(), (size_t)n1 * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->rw_el, el.data(), el.size() * sizeof(float), cudaMemcpyHostToDevice, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->rw_eldesc, dmp, (size_t)n1 * 32, cudaMemcpyHostToDevice, st));
    if (held2) SSLPL_CUDA(cudaMemcpyAsync(m->flag, held2, n2, cudaMemcpyHostToDevice, st));
    RelocSet R; memset(&R, 0, sizeof(R));
    R.pair = reinterpret_cast<const int2*>(m->rw_pair); R.npairs = 1; R.nrows = 2; R.cap = W;
    R.kp = m->kpf; R.desc = m->desc; R.n = m->ncnt;
    R.kfmp = m->rw_kfmp; R.el = m->rw_el; R.eldesc = m->rw_eldesc; R.nel = n1;
    R.Tcw = m->rw_T; R.held = held2 ? m->flag : nullptr;
    R.assign = m->out; R.nmatch = m->rw_nmatch;
    if (int rc = reloc_run(m, A, R)) return rc;
    SSLPL_CUDA(cudaMemcpyAsync(assign2, m->out, sizeof(int32_t) * n2, cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaMemcpyAsync(m->h_small, m->rw_nmatch, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    SSLPL_CUDA(cudaStreamSynchronize(st));
    *nmatches = m->h_small[0];
    return SSLPL_OK;
}

int sslpl_search_by_projection_kf_batch_device(sslpl_matcher* m,
        const sslpl_keypoint* d_kps, const uint8_t* d_desc, const int* d_n, int nrows, int cap,
        const int32_t* d_kfmp, const uint8_t* d_mpbad, int nmp, const float* d_mp, const uint8_t* d_mpdesc,
        int npairs, const int32_t* d_pair, const float* d_Tcw, const uint8_t* d_found, const uint8_t* d_held,
        const float* cam, const float* bounds, const float* scaleFactors, int nlevels, float logScaleFactor,
        float th, int ORBdist, int checkOrientation, int32_t* d_assign, int32_t* d_nmatch) {
    SSLPL_REQUIRE(m && d_kps && d_desc && d_n && d_kfmp && d_pair && d_Tcw && d_assign && d_nmatch, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(nmp >= 0 && (nmp == 0 || (d_mp && d_mpdesc)), SSLPL_ERR_ARG, "null element table");
    SSLPL_REQUIRE(nrows >= 1 && nrows <= 65535, SSLPL_ERR_ARG, "nrows outside [1, 65535]");
    SSLPL_REQUIRE(cap >= 1 && cap <= m->p.max_features + 64, SSLPL_ERR_ARG, "cap outside [1, max_features + 64]");
    SSLPL_REQUIRE(npairs >= 1 && npairs <= m->p.max_batch, SSLPL_ERR_ARG, "npairs outside [1, max_batch]");
    RelocArgs A;
    if (int rc = reloc_args(A, cam, bounds, scaleFactors, nlevels, logScaleFactor, th, ORBdist, checkOrientation)) return rc;
    if (int rc = csr_fits(GRID_COLS * GRID_ROWS, cap)) return rc;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    if (int rc = ensure_reloc_ws(m)) return rc;
    RelocSet R; memset(&R, 0, sizeof(R));
    R.pair = reinterpret_cast<const int2*>(d_pair); R.npairs = npairs; R.nrows = nrows; R.cap = cap;
    R.kp = reinterpret_cast<const float*>(d_kps); R.desc = d_desc; R.n = d_n;
    R.kfmp = d_kfmp; R.mpbad = d_mpbad; R.el = d_mp; R.eldesc = d_mpdesc; R.nel = nmp;
    R.Tcw = d_Tcw; R.found = d_found; R.held = d_held;
    R.assign = d_assign; R.nmatch = d_nmatch;
    return reloc_run(m, A, R);
}

int sslpl_reloc_pairs_batch_device(sslpl_matcher* m, const int32_t* d_query, const int32_t* d_cand, const int32_t* d_ncand, int nq, int ndb,
                                   int kmax, int32_t* d_pair) {
    SSLPL_REQUIRE(m && d_query && d_cand && d_ncand && d_pair, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(nq >= 1 && ndb >= 1 && kmax >= 1, SSLPL_ERR_ARG, "nq, ndb and kmax must be positive");
    SSLPL_REQUIRE((long long)nq * kmax <= m->p.max_batch, SSLPL_ERR_ARG, "nq * kmax exceeds max_batch");
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    const int ns = nq * kmax;
    launch(m, k_reloc_pairs, (ns + 127) / 128, 128, 0, nq, d_query, d_cand, d_ncand, ndb, kmax, reinterpret_cast<int2*>(d_pair));
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}

// ORBmatcher::SearchByBoW(KeyFrame*, Frame&) over (keyframe row, frame row) pairs: the row -> slot map (k_kfbow_claim / k_kfbow_slots),
// the FeatureVector of every named row once (k_vocab_transform<true>, k_build_csr), k_bow_match<true>, the rotation filter and count,
// then -1 for the pairs outside the rows.
int sslpl_search_by_bow_batch_device(sslpl_matcher* m,
        const sslpl_keypoint* d_kps, const uint8_t* d_desc, const int* d_n, int nrows, int cap,
        const int32_t* d_kfmp, const uint8_t* d_mpbad, int nmp,
        const sslpl_vocab* v, int levelsup,
        int npairs, const int32_t* d_pair, float nnratio, int checkOrientation,
        int32_t* d_match, int32_t* d_nmatch) {
    SSLPL_REQUIRE(m && d_kps && d_desc && d_n && d_kfmp && v && d_pair && d_match && d_nmatch, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(nmp >= 0, SSLPL_ERR_ARG, "nmp must be >= 0");
    SSLPL_REQUIRE(nrows >= 1 && nrows <= 65535, SSLPL_ERR_ARG, "nrows outside [1, 65535]");
    SSLPL_REQUIRE(cap >= 1 && cap <= m->p.max_features + 64, SSLPL_ERR_ARG, "cap outside [1, max_features + 64]");
    SSLPL_REQUIRE(npairs >= 1 && npairs <= m->p.max_batch, SSLPL_ERR_ARG, "npairs outside [1, max_batch]");
    SSLPL_REQUIRE(npairs <= 32767, SSLPL_ERR_ARG, "npairs exceeds 32767 (two FeatureVector slots per pair on one grid axis)");
    const int nc = vocab_level_nodes(v, levelsup);
    SSLPL_REQUIRE(nc <= m->p.max_nodes, SSLPL_ERR_ARG, "the vocabulary level exceeds the matcher capacity (max_nodes)");
    SSLPL_REQUIRE(v->device == m->p.device, SSLPL_ERR_ARG, "vocabulary and matcher live on different devices");
    if (int rc = csr_fits(nc, cap)) return rc;
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    if (int rc = ensure_kfbow_ws(m)) return rc;
    if (int rc = ensure_scratch(m, (size_t)nrows * 4)) return rc;
    cudaStream_t st = m->stream;
    const int fc = m->p.max_features + 64, NN = m->p.max_nodes + 1, ns = 2 * npairs;
    const int2* pmap = reinterpret_cast<const int2*>(d_pair);
    int32_t* slot_of_row = reinterpret_cast<int32_t*>(m->scratch);
    fill(m, slot_of_row, nrows, INT_MAX);
    launch(m, k_kfbow_claim, (ns + 127) / 128, 128, 0, pmap, npairs, nrows, slot_of_row);
    launch(m, k_kfbow_slots, (ns + 127) / 128, 128, 0, pmap, npairs, nrows, d_n, cap, (const int32_t*)slot_of_row, m->kb_row, m->kb_n,
           m->kb_pslot, m->kb_fn);
    launch(m, k_vocab_transform<true>, dim3((cap + 127) / 128, ns), 128, 0, d_desc, (long long)cap * 32, (const int*)m->kb_n, 0, cap, v->view,
           v->L - levelsup, nullptr, nullptr, m->kb_node, nullptr, fc, (const int32_t*)m->kb_row);
    launch(m, k_build_csr, ns, 128, (nc + 1 + cap) * sizeof(int), m->kb_node, fc, m->kb_n, cap, nc, m->kb_off, NN + 1, m->kb_idx, fc);
    fill(m, d_match, (long long)npairs * cap, -1);
    SSLPL_CUDA(cudaMemsetAsync(m->b_taken, 0, (size_t)npairs * fc, st));
    FrameSet S = dense_set(m, d_desc, d_kps, cap, nc, nullptr);
    S.off = m->kb_off; S.idx = m->kb_idx; S.pmap = pmap; S.nframes = nrows;
    // b_rot is only read where the table holds a match, and k_bow_match writes both together
    launch(m, k_bow_match<true>, dim3((nc + 3) / 4, npairs), 128, 0, S, 0, nnratio, cap, d_match, cap, m->b_rot, fc, m->b_taken, fc,
           (const int2*)m->kb_pslot, d_kfmp, d_mpbad, nmp);
    launch(m, k_rot_filter, npairs, 256, 0, d_match, cap, m->b_rot, fc, (const int*)m->kb_fn, 0, 0, cap, checkOrientation ? 1 : 0, d_nmatch,
           nullptr, 0);
    launch(m, k_bad_pairs, (npairs + 127) / 128, 128, 0, pmap, npairs, nrows, d_nmatch);
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}

// LSDmatcher::SearchByProjection(KeyFrame*, Frame&) over (keyframe row, frame row) pairs: k_knn2 over the pair map (query = the keyframe's
// lines, train = the frame's), then the ratio rule with the keyframe's MapLines.
int sslpl_match_lines_kf_batch_device(sslpl_matcher* m,
        const uint8_t* d_ldesc, const int* d_nl, int nrows, int capl,
        const int32_t* d_kfml, int nml,
        int npairs, const int32_t* d_pair, int32_t* d_lmatch, int32_t* d_nlmatch) {
    SSLPL_REQUIRE(m && d_ldesc && d_nl && d_kfml && d_pair && d_lmatch && d_nlmatch, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(nml >= 0, SSLPL_ERR_ARG, "nml must be >= 0");
    SSLPL_REQUIRE(nrows >= 1 && nrows <= 65535, SSLPL_ERR_ARG, "nrows outside [1, 65535]");
    SSLPL_REQUIRE(capl >= 1 && capl <= m->p.max_lines + 64, SSLPL_ERR_ARG, "capl outside [1, max_lines + 64]");
    SSLPL_REQUIRE(npairs >= 1 && npairs <= m->p.max_batch, SSLPL_ERR_ARG, "npairs outside [1, max_batch]");
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    const int lc = m->p.max_lines + 64;
    const int2* pmap = reinterpret_cast<const int2*>(d_pair);
    launch(m, k_knn2<true>, dim3((capl + 7) / 8, npairs), 256, 0, d_ldesc, (long long)capl * 32, d_nl, 0, d_ldesc, (long long)capl * 32, d_nl, 0,
           m->b_knn, (long long)lc * 4, capl, pmap, nrows);
    fill(m, d_lmatch, (long long)npairs * capl, -1);
    SSLPL_CUDA(cudaMemsetAsync(d_nlmatch, 0, sizeof(int32_t) * npairs, m->stream));
    launch(m, k_line_ratio<true>, dim3((capl + 127) / 128, npairs), 128, 0, m->b_knn, (long long)lc * 4, d_nl, 0, capl, nullptr, 0, d_lmatch,
           capl, d_nlmatch, pmap, nrows, d_kfml, nml);
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}

// Optimizer::PoseOptimization over frames in HBM: k_pose_opt (pose.cuh), one CTA per frame.
int sslpl_pose_optimization_batch_device(sslpl_matcher* m,
        const sslpl_keypoint* d_kps, const int* d_n, int nframes, int cap,
        const int32_t* d_fmp, int nmp, const float* d_mp,
        const double* d_lineeq, const int* d_nl, int capl, const int32_t* d_fml, int nml, const double* d_mlpos,
        const float* d_Tcw, const float* cam, const float* invLevelSigma2, int nlevels,
        float* d_Tcw_out, uint8_t* d_outlier, uint8_t* d_line_outlier, int32_t* d_ninlier) {
    SSLPL_REQUIRE(m && d_kps && d_n && d_fmp && d_Tcw && cam && invLevelSigma2 && d_Tcw_out && d_outlier && d_ninlier,
                  SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(nframes >= 1 && nframes <= m->p.max_batch, SSLPL_ERR_ARG, "nframes outside [1, max_batch]");
    SSLPL_REQUIRE(cap >= 1 && cap <= m->p.max_features + 64, SSLPL_ERR_ARG, "cap outside [1, max_features + 64]");
    SSLPL_REQUIRE(nmp >= 0 && (nmp == 0 || d_mp), SSLPL_ERR_ARG, "nmp must be >= 0, with an element table when > 0");
    SSLPL_REQUIRE(nlevels >= 1 && nlevels <= SSLPL_MAX_LEVELS, SSLPL_ERR_ARG, "nlevels outside [1, SSLPL_MAX_LEVELS]");
    if (d_fml) {
        SSLPL_REQUIRE(d_lineeq && d_nl && d_line_outlier, SSLPL_ERR_ARG, "null line argument");
        SSLPL_REQUIRE(capl >= 1 && capl <= m->p.max_lines + 64, SSLPL_ERR_ARG, "capl outside [1, max_lines + 64]");
        SSLPL_REQUIRE(nml >= 0 && (nml == 0 || d_mlpos), SSLPL_ERR_ARG, "nml must be >= 0, with a position table when > 0");
    }
    SSLPL_CUDA(cudaSetDevice(m->p.device));
    PoseArgs A; memset(&A, 0, sizeof(A));
    A.kps = reinterpret_cast<const float*>(d_kps); A.n = d_n; A.cap = cap;
    A.fmp = d_fmp; A.nmp = nmp; A.mp = d_mp;
    if (d_fml) { A.lineeq = d_lineeq; A.nl = d_nl; A.capl = capl; A.fml = d_fml; A.nml = nml; A.mlpos = d_mlpos; A.line_outlier = d_line_outlier; }
    A.Tcw = d_Tcw; A.Tcw_out = d_Tcw_out; A.outlier = d_outlier; A.ninlier = d_ninlier;
    A.fx = cam[0]; A.fy = cam[1]; A.cx = cam[2]; A.cy = cam[3];
    A.nlevels = nlevels;
    for (int l = 0; l < nlevels; l++) A.invs2[l] = invLevelSigma2[l];
    launch(m, k_pose_opt, nframes, POSE_THREADS, 0, A);
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}

}  // extern "C"
