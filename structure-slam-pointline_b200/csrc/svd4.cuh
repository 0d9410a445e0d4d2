// svd4.cuh — the 4x4 linear triangulation of LocalMapping::CreateNewMapPoints (LocalMapping.cc:500-509) on the device, bit for bit:
//   glibc_hypot  glibc >= 2.35's hypot (sysdeps/ieee754/dbl-64/e_hypot.c: Borges' corrected algorithm, the kernel without FMA, with its
//                power-of-two scaling of extreme operands).  CUDA's hypot is a different function.
//   svd4_jacobi  OpenCV 4.13's one-sided Jacobi JacobiSVDImpl_<float> (modules/core/src/lapack.cpp), which cv::SVD::compute runs for a
//                4x4 CV_32F matrix: At = A^T in float; column norms and inner products accumulated in double; eps = 2 FLT_EPSILON,
//                30 sweeps over (i < j) at most; c / s narrowed to float; float rotations of At and Vt; W = sqrt(sum t^2); selection sort
//                by strict <.  U (and its random completion for zero singular values) never touches Vt and is not computed.
// Every operation is an explicit _rn intrinsic: the file is included by match.cu, which is not built with -fmad=false.
#pragma once

namespace sslpl {

__device__ __forceinline__ double hypot_kernel(double ax, double ay) {
    double h = __dsqrt_rn(__dadd_rn(__dmul_rn(ax, ax), __dmul_rn(ay, ay)));
    double t1, t2;
    if (h <= __dmul_rn(2.0, ay)) {
        const double delta = __dsub_rn(h, ay);
        t1 = __dmul_rn(ax, __dsub_rn(__dmul_rn(2.0, delta), ax));
        t2 = __dmul_rn(__dsub_rn(delta, __dmul_rn(2.0, __dsub_rn(ax, ay))), delta);
    } else {
        const double delta = __dsub_rn(h, ax);
        t1 = __dmul_rn(__dmul_rn(2.0, delta), __dsub_rn(ax, __dmul_rn(2.0, ay)));
        t2 = __dadd_rn(__dmul_rn(__dsub_rn(__dmul_rn(4.0, delta), ay), ay), __dmul_rn(delta, delta));
    }
    return __dsub_rn(h, __ddiv_rn(__dadd_rn(t1, t2), __dmul_rn(2.0, h)));
}

__device__ __forceinline__ double glibc_hypot(double x, double y) {
    constexpr double SCALE = 0x1p-600, LARGE_VAL = 0x1p+511, TINY_VAL = 0x1p-459, EPS = 0x1p-54;
    if (!isfinite(x) || !isfinite(y)) return (isinf(x) || isinf(y)) ? __longlong_as_double(0x7ff0000000000000LL) : __dadd_rn(x, y);
    x = fabs(x); y = fabs(y);
    const double ax = x < y ? y : x, ay = x < y ? x : y;
    if (ax > LARGE_VAL) {
        if (ay <= __dmul_rn(ax, EPS)) return __dadd_rn(ax, ay);
        return __ddiv_rn(hypot_kernel(__dmul_rn(ax, SCALE), __dmul_rn(ay, SCALE)), SCALE);
    }
    if (ay < TINY_VAL) {
        if (ax >= __ddiv_rn(ay, EPS)) return __dadd_rn(ax, ay);
        return __dmul_rn(hypot_kernel(__ddiv_rn(ax, SCALE), __ddiv_rn(ay, SCALE)), SCALE);
    }
    if (ay <= __dmul_rn(ax, EPS)) return __dadd_rn(ax, ay);
    return hypot_kernel(ax, ay);
}

__device__ __forceinline__ double sq4(const float* t) {            // sum of (double)t[k] * t[k] in k order
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < 4; k++) s = __dadd_rn(s, __dmul_rn((double)t[k], (double)t[k]));
    return s;
}

// A row-major 4x4 -> W (descending) and Vt (row-major); A is destroyed (MODIFY_A).
__device__ __forceinline__ void svd4_jacobi(float A[16], float Wout[4], float Vt[16]) {
    float At[16];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int k = 0; k < 4; k++) { At[4 * i + k] = A[4 * k + i]; Vt[4 * i + k] = i == k ? 1.f : 0.f; }
    double W[4];
#pragma unroll
    for (int i = 0; i < 4; i++) W[i] = sq4(At + 4 * i);
    const double eps = (double)(2.0f * 1.1920928955078125e-07f);
    for (int iter = 0; iter < 30; iter++) {
        bool changed = false;
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = i + 1; j < 4; j++) {
                const double a = W[i], b = W[j];
                double p = 0.0;
#pragma unroll
                for (int k = 0; k < 4; k++) p = __dadd_rn(p, __dmul_rn((double)At[4 * i + k], (double)At[4 * j + k]));
                if (fabs(p) <= __dmul_rn(eps, __dsqrt_rn(__dmul_rn(a, b)))) continue;
                p = __dmul_rn(p, 2.0);
                const double beta = __dsub_rn(a, b), gamma = glibc_hypot(p, beta);
                float c, s;
                if (beta < 0) {
                    const double delta = __dmul_rn(__dsub_rn(gamma, beta), 0.5);
                    s = __double2float_rn(__dsqrt_rn(__ddiv_rn(delta, gamma)));
                    c = __double2float_rn(__ddiv_rn(p, __dmul_rn(__dmul_rn(gamma, (double)s), 2.0)));
                } else {
                    c = __double2float_rn(__dsqrt_rn(__ddiv_rn(__dadd_rn(gamma, beta), __dmul_rn(gamma, 2.0))));
                    s = __double2float_rn(__ddiv_rn(p, __dmul_rn(__dmul_rn(gamma, (double)c), 2.0)));
                }
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const float ai = At[4 * i + k], aj = At[4 * j + k];
                    At[4 * i + k] = __fadd_rn(__fmul_rn(c, ai), __fmul_rn(s, aj));
                    At[4 * j + k] = __fadd_rn(__fmul_rn(-s, ai), __fmul_rn(c, aj));
                    const float vi = Vt[4 * i + k], vj = Vt[4 * j + k];
                    Vt[4 * i + k] = __fadd_rn(__fmul_rn(c, vi), __fmul_rn(s, vj));
                    Vt[4 * j + k] = __fadd_rn(__fmul_rn(-s, vi), __fmul_rn(c, vj));
                }
                W[i] = sq4(At + 4 * i); W[j] = sq4(At + 4 * j);
                changed = true;
            }
        if (!changed) break;
    }
#pragma unroll
    for (int i = 0; i < 4; i++) W[i] = __dsqrt_rn(sq4(At + 4 * i));
#pragma unroll
    for (int i = 0; i < 3; i++) {
        int j = i;
        double wj = W[i];
#pragma unroll
        for (int k = i + 1; k < 4; k++) if (wj < W[k]) { j = k; wj = W[k]; }
        // swap rows i and j with compile-time indices only (a dynamic index would put W / Vt in local memory)
#pragma unroll
        for (int k = i + 1; k < 4; k++) {
            if (j != k) continue;
            const double w = W[i]; W[i] = W[k]; W[k] = w;
#pragma unroll
            for (int q = 0; q < 4; q++) { const float t = Vt[4 * i + q]; Vt[4 * i + q] = Vt[4 * k + q]; Vt[4 * k + q] = t; }
        }
    }
#pragma unroll
    for (int i = 0; i < 4; i++) Wout[i] = __double2float_rn(W[i]);
}

}  // namespace sslpl
