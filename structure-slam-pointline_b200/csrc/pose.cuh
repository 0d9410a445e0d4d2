// pose.cuh — Optimizer::PoseOptimization (Optimizer.cc:666-1022) on the device: the SE3Quat pose of the reference's g2o
// (Thirdparty/g2o/g2o/types/se3quat.h), EdgeSE3ProjectXYZOnlyPose and EdgeLineProjectXYZOnlyPose (lineEdge.h:155-240), the Huber
// kernel, a dense 6 x 6 LDLT and OptimizationAlgorithmLevenberg::solve (optimization_algorithm_levenberg.cpp:61-161), one CTA per frame.
// Included by match.cu, whose sslpl_pose_optimization_batch_device launches k_pose_opt.  All arithmetic is FP64 as in g2o; the
// reductions run in a fixed order so a frame's result does not depend on the batch around it.  See DESIGN.md, "Pose optimisation".
#pragma once
#include "common.cuh"
#include <cfloat>

namespace sslpl {

constexpr int POSE_THREADS = 256;
constexpr int POSE_ROUNDS = 4, POSE_ITERS = 10, POSE_TRIALS = 10;   // its[4] = {10, ...}; maxTrialsAfterFailure = 10
constexpr float POSE_CHI2_MONO = 5.991f;                            // chi2Mono[it]; a line compares each endpoint with 2 * chi2Mono[it]

// g2o::SE3Quat: unit quaternion (w, x, y, z) with w >= 0 after normalizeRotation, and a translation
struct SE3 { double q[4]; double t[3]; };

struct PoseArgs {
    const float* kps; const int* n; int cap;                 // mvKeysUn rows (sslpl_keypoint: x y size angle response octave class_id)
    const int32_t* fmp; int nmp; const float* mp;             // mvpMapPoints as element indices; element table [nmp][9], Xw = 0..2
    const double* lineeq; const int* nl; int capl;            // mvKeyLineFunctions [capl][3]
    const int32_t* fml; int nml; const double* mlpos;         // mvpMapLines as element indices (NULL = no line edges); mWorldPos [nml][6]
    const float* Tcw; float* Tcw_out; uint8_t* outlier; uint8_t* line_outlier; int32_t* ninlier;
    double fx, fy, cx, cy;
    int nlevels; double invs2[SSLPL_MAX_LEVELS];              // mvInvLevelSigma2, widened as setInformation widens it
};

__device__ __forceinline__ void quat_normalize_pos(double* q) {         // SE3Quat::normalizeRotation
    if (q[0] < 0) { q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3]; }
    const double s = 1.0 / sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    q[0] *= s; q[1] *= s; q[2] *= s; q[3] *= s;
}

// Eigen's Quaternion(const Matrix3&) (Shepperd's branches, Quaternion.h quaternionbase_assign_impl), then normalizeRotation
__device__ __forceinline__ void quat_from_matrix(const double R[3][3], double* q) {
    double t = R[0][0] + R[1][1] + R[2][2];
    if (t > 0) {
        t = sqrt(t + 1.0);
        q[0] = 0.5 * t; t = 0.5 / t;
        q[1] = (R[2][1] - R[1][2]) * t; q[2] = (R[0][2] - R[2][0]) * t; q[3] = (R[1][0] - R[0][1]) * t;
    } else {
        int i = 0;
        if (R[1][1] > R[0][0]) i = 1;
        if (R[2][2] > R[i][i]) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        t = sqrt(R[i][i] - R[j][j] - R[k][k] + 1.0);
        double v[3];
        v[i] = 0.5 * t; t = 0.5 / t;
        q[0] = (R[k][j] - R[j][k]) * t;
        v[j] = (R[j][i] + R[i][j]) * t; v[k] = (R[k][i] + R[i][k]) * t;
        q[1] = v[0]; q[2] = v[1]; q[3] = v[2];
    }
    quat_normalize_pos(q);
}

__device__ __forceinline__ void quat_to_matrix(const double* q, double R[3][3]) {   // QuaternionBase::toRotationMatrix
    const double w = q[0], x = q[1], y = q[2], z = q[3];
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0][0] = 1 - (tyy + tzz); R[0][1] = txy - twz; R[0][2] = txz + twy;
    R[1][0] = txy + twz; R[1][1] = 1 - (txx + tzz); R[1][2] = tyz - twx;
    R[2][0] = txz - twy; R[2][1] = tyz + twx; R[2][2] = 1 - (txx + tyy);
}

// SE3Quat::map: q * X + t, with Eigen's quaternion-vector product (v + 2w (u x v) + u x (2 u x v))
__device__ __forceinline__ void se3_map(const SE3& P, const double* X, double* Y) {
    const double* u = P.q + 1; const double w = P.q[0];
    double uv[3] = {u[1] * X[2] - u[2] * X[1], u[2] * X[0] - u[0] * X[2], u[0] * X[1] - u[1] * X[0]};
    uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
    Y[0] = X[0] + w * uv[0] + (u[1] * uv[2] - u[2] * uv[1]) + P.t[0];
    Y[1] = X[1] + w * uv[1] + (u[2] * uv[0] - u[0] * uv[2]) + P.t[1];
    Y[2] = X[2] + w * uv[2] + (u[0] * uv[1] - u[1] * uv[0]) + P.t[2];
}

// Converter::toSE3Quat of a 3x4 row-major f32 pose
__device__ __forceinline__ void se3_from_f32(const float* T, SE3& P) {
    double R[3][3];
    for (int r = 0; r < 3; r++) { for (int c = 0; c < 3; c++) R[r][c] = T[4 * r + c]; P.t[r] = T[4 * r + 3]; }
    quat_from_matrix(R, P.q);
}

// SE3Quat::exp(d) * P with d = (omega, upsilon)
__device__ __noinline__ void se3_exp_mul(const double* d, const SE3& P, SE3& out) {
    const double w0 = d[0], w1 = d[1], w2 = d[2];
    const double theta = sqrt(w0 * w0 + w1 * w1 + w2 * w2);
    const double O[3][3] = {{0, -w2, w1}, {w2, 0, -w0}, {-w1, w0, 0}};
    double O2[3][3];
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) O2[r][c] = O[r][0] * O[0][c] + O[r][1] * O[1][c] + O[r][2] * O[2][c];
    double R[3][3], V[3][3];
    if (theta < 0.00001) {
        for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) { R[r][c] = (r == c) + O[r][c] + O2[r][c]; V[r][c] = R[r][c]; }
    } else {
        const double s = sin(theta), co = cos(theta), a = s / theta, b = (1 - co) / (theta * theta), c3 = (theta - s) / (theta * theta * theta);
        for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) {
            R[r][c] = (r == c) + a * O[r][c] + b * O2[r][c];
            V[r][c] = (r == c) + b * O[r][c] + c3 * O2[r][c];
        }
    }
    SE3 E;
    quat_from_matrix(R, E.q);
    for (int r = 0; r < 3; r++) E.t[r] = V[r][0] * d[3] + V[r][1] * d[4] + V[r][2] * d[5];
    se3_map(E, P.t, out.t);                                                 // t = E.t + E.q * P.t
    const double* a = E.q; const double* b = P.q;                          // Eigen quaternion product a * b
    out.q[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
    out.q[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
    out.q[2] = a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3];
    out.q[3] = a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1];
    quat_normalize_pos(out.q);
}

// EdgeSE3ProjectXYZOnlyPose: e = obs - pi(P X); J = d e / d(omega, upsilon) (types_six_dof_expmap.cpp:266-288) when J != nullptr
__device__ __forceinline__ void mono_edge(const SE3& P, const double* X, double ox, double oy, const PoseArgs& A,
                                          double& e0, double& e1, double (*J)[6]) {
    double Y[3]; se3_map(P, X, Y);
    e0 = ox - (Y[0] / Y[2] * A.fx + A.cx);
    e1 = oy - (Y[1] / Y[2] * A.fy + A.cy);
    if (!J) return;
    const double x = Y[0], y = Y[1], invz = 1.0 / Y[2], invz2 = invz * invz;
    J[0][0] = x * y * invz2 * A.fx; J[0][1] = -(1 + (x * x * invz2)) * A.fx; J[0][2] = y * invz * A.fx;
    J[0][3] = -invz * A.fx; J[0][4] = 0; J[0][5] = x * invz2 * A.fx;
    J[1][0] = (1 + y * y * invz2) * A.fy; J[1][1] = -x * y * invz2 * A.fy; J[1][2] = -x * invz * A.fy;
    J[1][3] = 0; J[1][4] = -invz * A.fy; J[1][5] = y * invz2 * A.fy;
}

// EdgeLineProjectXYZOnlyPose: e = l0 u + l1 v + l2 (error(1) = error(2) = 0); J its only non-zero row (lineEdge.h:174-205)
__device__ __forceinline__ double line_edge(const SE3& P, const double* X, const double* l, const PoseArgs& A, double* J) {
    double Y[3]; se3_map(P, X, Y);
    const double u = Y[0] / Y[2] * A.fx + A.cx, v = Y[1] / Y[2] * A.fy + A.cy;
    const double e = l[0] * u + l[1] * v + l[2];
    if (J) {
        const double x = Y[0], y = Y[1], invz = 1.0 / Y[2], invz2 = invz * invz, lx = l[0], ly = l[1], fx = A.fx, fy = A.fy;
        J[0] = -fy * ly - fx * lx * x * y * invz2 - fy * ly * y * y * invz2;
        J[1] = fx * lx + fx * lx * x * x * invz2 + fy * ly * x * y * invz2;
        J[2] = -fx * lx * y * invz + fy * ly * x * invz;
        J[3] = fx * lx * invz;
        J[4] = fy * ly * invz;
        J[5] = -(fx * lx * x + fy * ly * y) * invz2;
    }
    return e;
}

// RobustKernelHuber::robustify: rho(chi2) and rho'(chi2)
__device__ __forceinline__ void huber(double e, double delta, double& r0, double& r1) {
    const double dsqr = delta * delta;
    if (e <= dsqr) { r0 = e; r1 = 1.0; }
    else { const double s = sqrt(e); r0 = 2 * s * delta - dsqr; r1 = delta / s; }
}

// A += w * outer(j, j) on the 21 upper-triangle terms (row-major), b -= w * j * e
__device__ __forceinline__ void accum(double* acc, const double* j, double w, double we) {
    int k = 0;
#pragma unroll
    for (int r = 0; r < 6; r++)
#pragma unroll
        for (int c = r; c < 6; c++) acc[k++] += w * j[r] * j[c];
#pragma unroll
    for (int r = 0; r < 6; r++) acc[21 + r] -= we * j[r];
}

// Sum of NV doubles per thread over the block, in a fixed order (warp tree, then the warps in index order); the result is in
// s_out[0..NV) for every thread after the call.  s_red holds (POSE_THREADS / 32) * NV doubles.
template <int NV>
__device__ __forceinline__ void block_sum(double* v, double* s_red, double* s_out) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < NV; i++) {
        double x = v[i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
        if (lane == 0) s_red[wid * NV + i] = x;
    }
    __syncthreads();
    if (threadIdx.x < NV) {
        double s = 0;
        for (int w = 0; w < POSE_THREADS / 32; w++) s += s_red[w * NV + threadIdx.x];
        s_out[threadIdx.x] = s;
    }
    __syncthreads();
}

// The frame's active edges at pose P: robust chi2 (robust = the Huber kernels are still attached) and, with kSystem, H and b
// (acc[0..21) = H's upper triangle, acc[21..27) = b, acc[27] = chi2).  Level-0 edges only: outlier flag 0.
template <bool kSystem>
__device__ void pose_pass(const PoseArgs& A, int f, int n, int nl, const SE3& P, bool robust, double* s_red, double* s_out) {
    constexpr int NV = kSystem ? 28 : 1;
    const double dMono = (double)(float)sqrt(5.991), dLine = (double)(float)sqrt(7.815);
    double acc[NV];
#pragma unroll
    for (int i = 0; i < NV; i++) acc[i] = 0;
    const float* kp = A.kps + (size_t)f * A.cap * 7;
    for (int i = threadIdx.x; i < n; i += POSE_THREADS) {
        const int m = A.fmp[(size_t)f * A.cap + i];
        if (m < 0 || m >= A.nmp || A.outlier[(size_t)f * A.cap + i]) continue;
        const double X[3] = {A.mp[(size_t)m * 9], A.mp[(size_t)m * 9 + 1], A.mp[(size_t)m * 9 + 2]};
        const double inv = A.invs2[__float_as_int(kp[7 * i + 5])];
        double e0, e1, J[2][6];
        mono_edge(P, X, kp[7 * i], kp[7 * i + 1], A, e0, e1, kSystem ? J : nullptr);
        const double chi2 = e0 * (inv * e0) + e1 * (inv * e1);
        double r0 = chi2, r1 = 1.0;
        if (robust) huber(chi2, dMono, r0, r1);
        acc[NV - 1] += r0;
        if constexpr (kSystem) {
            const double w = r1 * inv;
            accum(acc, J[0], w, w * e0);
            accum(acc, J[1], w, w * e1);
        }
    }
    if (A.fml) {
        for (int i = threadIdx.x; i < nl; i += POSE_THREADS) {
            const int m = A.fml[(size_t)f * A.capl + i];
            if (m < 0 || m >= A.nml || A.line_outlier[(size_t)f * A.capl + i]) continue;
            const double* l = A.lineeq + ((size_t)f * A.capl + i) * 3;
            for (int s = 0; s < 2; s++) {
                const double* X = A.mlpos + (size_t)m * 6 + 3 * s;
                double J[6];
                const double e = line_edge(P, X, l, A, kSystem ? J : nullptr);
                const double chi2 = e * e;
                double r0 = chi2, r1 = 1.0;
                if (robust) huber(chi2, dLine, r0, r1);
                acc[NV - 1] += r0;
                if constexpr (kSystem) accum(acc, J, r1, r1 * e);
            }
        }
    }
    block_sum<NV>(acc, s_red, s_out);
}

// Dense LDLT of the 6 x 6 system (H + lambda I) x = b without pivoting; false when a pivot is not positive (x left as it was)
__device__ __noinline__ bool ldlt6(const double* H, double lambda, const double* b, double* x) {
    double L[6][6], D[6];
    int k = 0;
    double M[6][6];
    for (int r = 0; r < 6; r++) for (int c = r; c < 6; c++) { M[r][c] = H[k]; M[c][r] = H[k]; k++; }
    for (int r = 0; r < 6; r++) M[r][r] += lambda;
    for (int j = 0; j < 6; j++) {
        double d = M[j][j];
        for (int p = 0; p < j; p++) d -= L[j][p] * L[j][p] * D[p];
        if (!(d > 0) || !isfinite(d)) return false;
        D[j] = d;
        for (int i = j + 1; i < 6; i++) {
            double s = M[i][j];
            for (int p = 0; p < j; p++) s -= L[i][p] * L[j][p] * D[p];
            L[i][j] = s / d;
        }
    }
    double y[6];
    for (int i = 0; i < 6; i++) { double s = b[i]; for (int p = 0; p < i; p++) s -= L[i][p] * y[p]; y[i] = s; }
    for (int i = 5; i >= 0; i--) { double s = y[i] / D[i]; for (int p = i + 1; p < 6; p++) s -= L[p][i] * x[p]; x[i] = s; }
    return true;
}

// Block-wide count of an int per thread (fixed order)
__device__ __forceinline__ int block_count(int v, int* s_cnt) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    __syncthreads();
    if (lane == 0) s_cnt[wid] = v;
    __syncthreads();
    int s = 0;
    for (int w = 0; w < POSE_THREADS / 32; w++) s += s_cnt[w];
    return s;
}

// Shared state of one frame's solve: thread 0 runs the Levenberg bookkeeping and publishes it here
struct PoseShared {
    double red[(POSE_THREADS / 32) * 28];
    double sys[28];                    // H (21), b (6), chi2 of the last pass
    double x[6];
    SE3 est, trial, last, init;        // estimate, trial, pose of the last computeActiveErrors, toSE3Quat(mTcw)
    double lambda, ni, cur, ini, rho;
    int nbad_lm, go, cnt[POSE_THREADS / 32];
};

__global__ void __launch_bounds__(POSE_THREADS) k_pose_opt(const __grid_constant__ PoseArgs A) {
    __shared__ PoseShared S;
    const int f = blockIdx.x, tid = threadIdx.x;
    const int n = min(max(A.n[f], 0), A.cap);
    const int nl = A.fml ? min(max(A.nl[f], 0), A.capl) : 0;
    const float* kp = A.kps + (size_t)f * A.cap * 7;
    uint8_t* out = A.outlier + (size_t)f * A.cap;
    uint8_t* lout = A.fml ? A.line_outlier + (size_t)f * A.capl : nullptr;
    const float* T = A.Tcw + 12 * f;

    // edges: one per point with a MapPoint, two per line with a MapLine; an octave outside the pyramid rejects the frame
    int np = 0, nln = 0, badoct = 0;
    for (int i = tid; i < n; i += POSE_THREADS) {
        const int m = A.fmp[(size_t)f * A.cap + i];
        if (m < 0 || m >= A.nmp) continue;
        np++;
        const int o = __float_as_int(kp[7 * i + 5]);
        badoct |= (o < 0 || o >= A.nlevels);
    }
    for (int i = tid; i < nl; i += POSE_THREADS) {
        const int m = A.fml[(size_t)f * A.capl + i];
        nln += (m >= 0 && m < A.nml);
    }
    const int nbadoct = block_count(badoct, S.cnt);
    const int Np = block_count(np, S.cnt), Nl = block_count(nln, S.cnt);
    if (nbadoct) {
        if (tid < 12) A.Tcw_out[12 * f + tid] = T[tid];
        if (tid == 0) A.ninlier[f] = -1;
        return;
    }
    // adding the edges clears mvbOutlier / mvbLineOutlier (Optimizer.cc:716, :814): level 0
    for (int i = tid; i < n; i += POSE_THREADS) { const int m = A.fmp[(size_t)f * A.cap + i]; if (m >= 0 && m < A.nmp) out[i] = 0; }
    for (int i = tid; i < nl; i += POSE_THREADS) { const int m = A.fml[(size_t)f * A.capl + i]; if (m >= 0 && m < A.nml) lout[i] = 0; }
    const int nInit = Np + Nl, E = Np + 2 * Nl;
    if (nInit < 3) {
        if (tid < 12) A.Tcw_out[12 * f + tid] = T[tid];
        if (tid == 0) A.ninlier[f] = 0;
        return;
    }
    if (tid == 0) se3_from_f32(T, S.init);
    __syncthreads();

    int nBad = 0, nActive = E;
    for (int it = 0; it < POSE_ROUNDS; it++) {
        const bool robust = it < 3;                                        // kernels removed after the classification of round 2
        if (tid == 0) { S.est = S.init; S.last = S.init; for (int k = 0; k < 6; k++) S.x[k] = 0; }
        __syncthreads();
        // OptimizationAlgorithmLevenberg::solve, its[it] times; nothing to optimise without a level-0 edge
        for (int iter = 0; nActive > 0 && iter < POSE_ITERS; iter++) {
            pose_pass<true>(A, f, n, nl, S.est, robust, S.red, S.sys);
            if (tid == 0) {
                S.cur = S.sys[27]; S.ini = S.cur;
                if (iter == 0) {
                    double mx = 0;
                    for (int r = 0, k = 0; r < 6; k += 6 - r, r++) mx = fmax(fabs(S.sys[k]), mx);
                    S.lambda = 1e-5 * mx; S.ni = 2; S.nbad_lm = 0;
                }
            }
            int q = 0;
            double rho;
            do {
                if (tid == 0) {
                    S.go = ldlt6(S.sys, S.lambda, S.sys + 21, S.x);
                    se3_exp_mul(S.x, S.est, S.trial);
                    S.last = S.trial;
                }
                __syncthreads();
                pose_pass<false>(A, f, n, nl, S.trial, robust, S.red, S.red + (POSE_THREADS / 32));
                if (tid == 0) {
                    double tmp = S.red[POSE_THREADS / 32];
                    if (!S.go) tmp = DBL_MAX;
                    double scale = 0;
                    for (int k = 0; k < 6; k++) scale += S.x[k] * (S.lambda * S.x[k] + S.sys[21 + k]);
                    scale += 1e-3;
                    const double r = (S.cur - tmp) / scale;
                    if (r > 0 && isfinite(tmp)) {
                        const double alpha = fmin(1. - pow(2 * r - 1, 3), 2. / 3.);
                        S.lambda *= fmax(1. / 3., alpha);
                        S.ni = 2; S.cur = tmp; S.est = S.trial;
                    } else {
                        S.lambda *= S.ni; S.ni *= 2;
                    }
                    S.rho = r;
                }
                __syncthreads();
                rho = S.rho;
                q++;
            } while (rho < 0 && q < POSE_TRIALS);
            if (q == POSE_TRIALS || rho == 0) break;
            if (tid == 0) {
                if ((S.ini - S.cur) * 1e3 < S.ini) S.nbad_lm++; else S.nbad_lm = 0;
            }
            __syncthreads();
            if (S.nbad_lm >= 3) break;
        }
        __syncthreads();
        // classification (Optimizer.cc:886-996): an active point keeps the error of the last computeActiveErrors, an inactive one and
        // every line are recomputed at the estimate
        const SE3 est = S.est, last = S.last;
        int bad = 0, act = 0;
        for (int i = tid; i < n; i += POSE_THREADS) {
            const int m = A.fmp[(size_t)f * A.cap + i];
            if (m < 0 || m >= A.nmp) continue;
            const double X[3] = {A.mp[(size_t)m * 9], A.mp[(size_t)m * 9 + 1], A.mp[(size_t)m * 9 + 2]};
            const double inv = A.invs2[__float_as_int(kp[7 * i + 5])];
            double e0, e1;
            mono_edge(out[i] ? est : last, X, kp[7 * i], kp[7 * i + 1], A, e0, e1, nullptr);
            const float chi2 = (float)(e0 * (inv * e0) + e1 * (inv * e1));
            const bool o = chi2 > POSE_CHI2_MONO;
            out[i] = o; bad += o; act += !o;
        }
        for (int i = tid; i < nl; i += POSE_THREADS) {
            const int m = A.fml[(size_t)f * A.capl + i];
            if (m < 0 || m >= A.nml) continue;
            const double* l = A.lineeq + ((size_t)f * A.capl + i) * 3;
            const double es = line_edge(est, A.mlpos + (size_t)m * 6, l, A, nullptr);
            const double ee = line_edge(est, A.mlpos + (size_t)m * 6 + 3, l, A, nullptr);
            const float cs = (float)(es * es), ce = (float)(ee * ee);
            const bool o = cs > 2 * POSE_CHI2_MONO || ce > 2 * POSE_CHI2_MONO;
            lout[i] = o; bad += o; act += 2 * !o;
        }
        nBad = block_count(bad, S.cnt);
        nActive = block_count(act, S.cnt);
        if (E < 10) break;
    }
    // SetPose(Converter::toCvMat(SE3quat_recov))
    if (tid == 0) {
        double R[3][3]; quat_to_matrix(S.est.q, R);
        float* o = A.Tcw_out + 12 * f;
        for (int r = 0; r < 3; r++) { for (int c = 0; c < 3; c++) o[4 * r + c] = (float)R[r][c]; o[4 * r + 3] = (float)S.est.t[r]; }
        A.ninlier[f] = nInit - nBad;
    }
}

}  // namespace sslpl
