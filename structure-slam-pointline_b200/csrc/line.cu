// line.cu — H100 (sm_90a) line path: LSD (OpenCV 4.13 LineSegmentDetector, LSD_REFINE_ADV) + KeyLine packaging +
// LBD 256-bit descriptors + line equations.  Replaces LineSegment::ExtractLineSegment
// (reference src/ExtractLineSegment.cpp:18-69, which delegates to cv::line_descriptor / cv::LineSegmentDetector).
//
// Per-pixel stages are ordinary data-parallel kernels (k_lsd_prep: both blurs, resize, ll_angle and Sobel in one pass; k_lsd_seeds, k_lsd_nfa_*).
// The region stage (k_lsd_regions) is order-dependent by definition (seeds in descending gradient bins, shared
// `used` map, incrementally updated region angle): one warp walks one frame; the warp's lanes cooperate on neighbour
// fetches and on the rectangle scans of rect_nfa, frames of a batch run on different SMs.  It is latency-bound,
// not HBM-bound, and is reported separately (SURVEY.md 7.3 item 1).
//
// This file is compiled with -fmad=false: every float/double expression is evaluated as separate IEEE operations,
// in the same order as the CPU restatement, so that discrete decisions (alignment tests, density, NFA) agree.
#include "common.cuh"
#include "mathx.cuh"
#include "ddtrig.h"
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <vector>

namespace sslpl {

constexpr double L_PI = 3.14159265358979323846;
constexpr double L_DEG = L_PI / 180;
constexpr double L_3_2_PI = (3 * L_PI) / 2;
constexpr double L_2PI = 2 * L_PI;
constexpr float NOTDEF_F = -1024.f;
constexpr int NBINS = 1024;

struct LineGeom {
    int w, h, pitch;            // input frame (pitch of the staging / view)
    int sw, sh;                 // LSD detection scale (0.8x)
    int tiles_x, tiles_y;       // tiles of k_lsd_prep
    int xtab_off, ytab_off;     // INTER_LINEAR_EXACT tables (int2: index, w1)
    int seg_cap;                // raw segments per frame
    int kl_cap;                 // lsdNFeatures
    long long in_stride, pix_stride /* sw*sh */, full_stride /* w*h */;
    double rho, prec, p, log_nt;
    int min_reg_size;
    int trace_cap;              // rows of the debug trace per frame (0 = off)
    int dbg;                    // SSLPL_WALKER_DBG bit mask (bring-up switches of the region walker)
    int dbg_seed;               // SSLPL_WALKER_SEED: pixel index whose first region list is printed (bring-up)
};

// What region growing reads per neighbour, in one 16-byte load: level-line angle (degrees, NOTDEF_F when undefined),
// (float)cos / sin of (float)(angle in radians) — the values region_grow sums — and the mutable `used` flag.
struct __align__(16) LPix { float ang, cx, cy; unsigned used; };   // `used` = ticket of the region-growing attempt holding the pixel (0 = none)

struct LineWs {
    float* angdeg; LPix* pix; float2* cs0; double* modgrad;
    unsigned long long* maxgrad; unsigned* seeds; int* nseeds;
    int* prep_next;             // k_lsd_prep's tile counter (zeroed before every launch)
    unsigned* reg;              // region pixel list (x | y << 16) of the turn holder (whole-frame capacity)
    unsigned* sreg;             // per frame: WALK_RING speculation slots x WALK_SLOT_CAP list entries (v3: one list of V3_LIST entries per worker)
    unsigned* dlist;            // v3, per frame: V3_DPOOL entries (see V3Shared::dl_off)
    unsigned char* rcode;       // v3, per frame: one byte per rank: the try it committed with | 0x80 if it released pixels, 0xff = none
    double* sjob;               // per frame: one pending NFA job (13 doubles) per speculation slot
    unsigned long long* wstat;  // walker statistics (whole launch): see sslpl_line_walker_stats
    double* seg;                // raw rectangles: x1,y1,x2,y2 (detection scale, before +0.5)
    int* nseg;
    double* jobs; int* njobs; int* jobflag;   // NFA jobs: 13 doubles per candidate region (LRect + log_nfa), in walker order
    int2* jobnk; double* jobnfa;              // per job: (total, aligned) pixel counts and NFA of the unmodified rectangle
    int2* rej; int* rejctl;                   // work list of rejected jobs (frame, job); rejctl[0] = count, rejctl[1] = cursor, rejctl[2] = walker frame cursor
    int16_t* dx; int16_t* dy;
    int2* tab;
    float* resp; float4* ext;   // per raw segment: response and clamped extremes
    sslpl_keyline* kl; uint8_t* ldesc; double* lineeq; int* nl;
    int* err;
    double* trace; int* ntrace;
    const double* lgam;         // lgam[n] = log_gamma(n + 1) of lsd.cpp (Lanczos / Windschitl), tabulated by the host's libm
};

struct LView { const uint8_t* base; int pitch; long long frame_stride; };

// sin / cos of x in [0, 2 pi] to ~1 ulp (double): Cody-Waite reduction by pi/2 and the fdlibm kernel polynomials.
// Branch-free and table-free (libm's sincos drags its large-argument path and constant-bank tables through the
// memory pipe); the callers round the results to float, which hides the last-ulp freedom.
__device__ __forceinline__ void l_sincos_2pi(double x, double* s_out, double* c_out) {
    const double k = rint(x * 0.6366197723675814);
    const double r = (x - k * 1.57079632673412561417e+00) - k * 6.07710050650619224932e-11;
    const double z = r * r;
    double ps = 1.58969099521155010221e-10;
    ps = -2.50507602534068634195e-08 + z * ps; ps = 2.75573137070700676789e-06 + z * ps; ps = -1.98412698298579493134e-04 + z * ps;
    ps = 8.33333333332248946124e-03 + z * ps; ps = -1.66666666666666324348e-01 + z * ps;
    const double s = r + r * (z * ps);
    double pc = -1.13596475577881948265e-11;
    pc = 2.08757232129817482790e-09 + z * pc; pc = -2.75573143513906633035e-07 + z * pc; pc = 2.48015872894767294178e-05 + z * pc;
    pc = -1.38888888888741095749e-03 + z * pc; pc = 4.16666666666666019037e-02 + z * pc;
    const double c = (1.0 - 0.5 * z) + z * (z * pc);
    const int q = (int)k & 3;
    *s_out = (q == 0) ? s : (q == 1) ? c : (q == 2) ? -s : -c;
    *c_out = (q == 0) ? c : (q == 1) ? -s : (q == 2) ? -c : s;
}

// -------------------------------------------------------------------------------------------------
// The per-pixel pre-pass of LSD and LBD in one kernel, one CTA per tile.  From one staged box of the input frame it computes
//   blur5  GaussianBlur(5x5, sigma 1) of BinaryDescriptor  -> Sobel 3x3 -> dx, dy (s16, input resolution)
//   blur7  GaussianBlur(sigma 0.6/0.8) of lsd.cpp          -> resize 0.8x (INTER_LINEAR_EXACT) -> ll_angle -> pix, angdeg, cs0, modgrad, maxgrad
// and keeps blur5, blur7 and the resized image in shared memory: none of the three is written to global memory.
// 0.8 = 4/5, so a PT_W x PT_H tile of input pixels maps exactly onto PT_SW x PT_SH detection-scale pixels (the 4 resized pixels of
// a group of 5 input columns or rows read only those 5).  Halos are recomputed by each CTA.
// Both blurs are OpenCV 4.13's GaussianBlur 8U fixed point, out = (sum_j k_j sum_i k_i p + 32768) >> 16 with BORDER_REFLECT_101, and
// have five non-zero taps (lsd.cpp's 7-tap kernel rounds its end taps to 0).  The horizontal pass is two dp4a per output on byte
// windows of three aligned words, the vertical pass dp2a on (row r | row r+1 << 16) pairs: all taps are < 256 and every partial
// sum of the horizontal pass < 65536, so the packed forms are exact.
// -------------------------------------------------------------------------------------------------
constexpr int PT_W = 160, PT_H = 40, PT_SW = 128, PT_SH = 32;    // input tile and its 0.8x image
constexpr int PT_NT = 128;                                      // threads per CTA
constexpr int PI_X = 4, PI_Y = 3;                               // staged box origin (X0 - 4, Y0 - 3): X0 % 32 == 0, so the origin is word aligned
constexpr int PI_W = 172, PI_H = 47;                            // staged box: columns X0-4 .. X0+167, rows Y0-3 .. Y0+43
constexpr int PB_W = 164, PB_H = 42;                            // blurred box (162 columns used): blur5 from (X0-1, Y0-1), blur7 from (X0, Y0)
constexpr int PH_H = PB_H + 4;                                  // rows of the horizontal pass
constexpr int PS_W = 132, PS_H = PT_SH + 1;                     // resized box from (SX0, SY0): the tile + one column and one row (129 columns used)
constexpr unsigned BL7_T0 = 4u | 56u << 8 | 136u << 16 | 56u << 24, BL7_T4 = 4u;      // lsd.cpp: {0, 4, 56, 136, 56, 4, 0}
constexpr unsigned BL5_T0 = 14u | 62u << 8 | 104u << 16 | 62u << 24, BL5_T4 = 14u;    // BinaryDescriptor: {14, 62, 104, 62, 14}

// bytes s .. s+3 of the 12-byte string w0:w1:w2 (bytes past the string read as 0)
__device__ __forceinline__ unsigned byte_window(unsigned w0, unsigned w1, unsigned w2, int s) {
    return s < 4 ? __funnelshift_r(w0, w1, 8 * s) : s < 8 ? __funnelshift_r(w1, w2, 8 * (s - 4)) : w2 >> (8 * (s - 8));
}

// Horizontal pass over the staged box: s_h[r][c] = sum_t k_t in[r + ROFF][c + SH + t] (u16), for PH_H rows and PB_W columns.
template <int SH, int ROFF>
__device__ __forceinline__ void prep_hpass(const unsigned* s_in, unsigned short* s_h, unsigned T0, unsigned T4) {
    for (int i = threadIdx.x; i < PH_H * (PB_W / 4); i += PT_NT) {
        const int r = i / (PB_W / 4), c4 = i - r * (PB_W / 4);
        const unsigned* w = s_in + (r + ROFF) * (PI_W / 4) + c4;
        const unsigned w0 = w[0], w1 = w[1], w2 = w[2];
        unsigned o[4];
#pragma unroll
        for (int k = 0; k < 4; k++) o[k] = __dp4a(byte_window(w0, w1, w2, SH + k), T0, __dp4a(byte_window(w0, w1, w2, SH + k + 4), T4, 0u));
        *reinterpret_cast<uint2*>(s_h + r * PB_W + 4 * c4) = make_uint2(o[0] | o[1] << 16, o[2] | o[3] << 16);
    }
}

// Vertical pass: s_b[r][c] = (sum_t k_t s_h[r + t][c] + 32768) >> 16, for PB_H rows and PB_W columns.
__device__ __forceinline__ void prep_vpass(const unsigned short* s_h, uint8_t* s_b, unsigned T0, unsigned T4) {
    const unsigned C01 = T0 & 0xffffu, C23 = T0 >> 16, C4L = T4, C4H = T4 << 8;
    for (int i = threadIdx.x; i < PB_H * (PB_W / 4); i += PT_NT) {
        const int r = i / (PB_W / 4), c4 = i - r * (PB_W / 4);
        const uint2* p = reinterpret_cast<const uint2*>(s_h + r * PB_W) + c4;
        const uint2 h0 = p[0], h1 = p[PB_W / 4], h2 = p[2 * (PB_W / 4)], h3 = p[3 * (PB_W / 4)], h4 = p[4 * (PB_W / 4)];
        // __byte_perm(a, b, 0x5410) pairs the low halves of rows a, b (column 2m), 0x7632 the high halves (column 2m + 1)
        const unsigned a0 = __dp2a_lo(__byte_perm(h0.x, h1.x, 0x5410), C01, __dp2a_lo(__byte_perm(h2.x, h3.x, 0x5410), C23, __dp2a_lo(h4.x, C4L, 32768u)));
        const unsigned a1 = __dp2a_lo(__byte_perm(h0.x, h1.x, 0x7632), C01, __dp2a_lo(__byte_perm(h2.x, h3.x, 0x7632), C23, __dp2a_lo(h4.x, C4H, 32768u)));
        const unsigned a2 = __dp2a_lo(__byte_perm(h0.y, h1.y, 0x5410), C01, __dp2a_lo(__byte_perm(h2.y, h3.y, 0x5410), C23, __dp2a_lo(h4.y, C4L, 32768u)));
        const unsigned a3 = __dp2a_lo(__byte_perm(h0.y, h1.y, 0x7632), C01, __dp2a_lo(__byte_perm(h2.y, h3.y, 0x7632), C23, __dp2a_lo(h4.y, C4H, 32768u)));
        reinterpret_cast<unsigned*>(s_b + r * PB_W)[c4] = (a0 >> 16) | ((a1 >> 16) << 8) | ((a2 >> 16) << 16) | ((a3 >> 16) << 24);
    }
}

// ll_angle (lsd.cpp) of one pixel from its 2x2 differences DA = D - A, BC = B - C: the gradient norm and, where it exceeds rho, the
// level-line angle in degrees (NOTDEF_F elsewhere), (float)cos / sin of (float)(angle in radians) — the values region_grow sums — and
// float(cos / sin) of the angle in radians taken as double — region_grow's seed values (both 0 where undefined).  k_lsd_prep and the
// debug table k_ll_table both evaluate it, so the table checks the kernel's own arithmetic.
struct LLPix { double norm; float ang; float2 cs, cs0; };
__device__ __forceinline__ LLPix ll_pixel(int DA, int BC, double rho) {
    LLPix o;
    o.ang = NOTDEF_F; o.cs = make_float2(0.f, 0.f); o.cs0 = make_float2(0.f, 0.f);
    const int gx = DA + BC, gy = DA - BC;
    o.norm = sqrt((double)(gx * gx + gy * gy) / 4.0);
    if (o.norm > rho) {
        o.ang = fast_atan2_deg((float)gx, (float)-gy);
        const double ad = (double)o.ang * L_DEG;
        double sn, cn;
        l_sincos_2pi((double)(float)ad, &sn, &cn);
        o.cs = make_float2((float)cn, (float)sn);
        // region_grow's seed values float(cos(ad)), float(sin(ad)) get their own reduction.  A second-order Taylor step from (cn, sn)
        // is accurate to a few double ulps in absolute terms only: near a zero of cos or sin (90 and 180 degrees) that is a relative
        // error of ~1e-7, which survives the narrowing to float.  (Redoing the reduction only there was slower: more registers.)
        l_sincos_2pi(ad, &sn, &cn);
        o.cs0 = make_float2((float)cn, (float)sn);
    }
    return o;
}

// Stage the input box of tile (X0, Y0) of frame f into s_in: aligned words where the view allows and the word lies inside the row, as
// 4-byte cp.async copies that complete at the next cp.async.wait_all; reflected bytes elsewhere, loaded and stored synchronously.
// Not unrolled: a copy in flight holds no register, and unrolling took the kernel past 70 registers.
__device__ __forceinline__ void prep_stage(unsigned* s_in, const LineGeom& g, const LView& v, int f, int X0, int Y0) {
    const uint8_t* img = v.base + f * v.frame_stride;
    const bool aligned = (((size_t)img | (size_t)v.pitch) & 3) == 0;
#pragma unroll 1
    for (int i = threadIdx.x; i < PI_H * (PI_W / 4); i += PT_NT) {
        const int r = i / (PI_W / 4), x = X0 - PI_X + 4 * (i - r * (PI_W / 4));
        const uint8_t* src = img + (long long)reflect101(Y0 - PI_Y + r, g.h) * v.pitch;
        if (aligned && x >= 0 && x + 3 < g.w)
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((unsigned)__cvta_generic_to_shared(s_in + i)), "l"(src + x) : "memory");
        else s_in[i] = (unsigned)__ldg(src + reflect101(x, g.w)) | (unsigned)__ldg(src + reflect101(x + 1, g.w)) << 8 |
                       (unsigned)__ldg(src + reflect101(x + 2, g.w)) << 16 | (unsigned)__ldg(src + reflect101(x + 3, g.w)) << 24;
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
}

// A persistent tile loop: the grid holds as many CTAs as fit on the device at once (fewer when the tiles are fewer), and every CTA
// takes tile after tile (frame-major) from the counter ws.prep_next (zeroed before every launch) until they run out.  A CTA that
// becomes resident late finds the work taken and exits.  The next tile's input box is requested as soon as the current tile's last
// read of s_in (blur7's horizontal pass) is done, so its load overlaps blur7's vertical pass, the resize and ll_angle.  Outputs go to
// fixed places and maxgrad is an atomicMax: which CTA runs a tile, and in what order, changes no result.
// ll_angle over the tile: 2x2 gradient, level-line angle, gradient norm, max over defined pixels.  Four horizontally adjacent pixels
// per thread and item: 9 vector stores per 4 pixels (the scalar form was limited by the memory-instruction queue, not by HBM or by
// the trigonometry).
__global__ void __launch_bounds__(PT_NT) k_lsd_prep(const __grid_constant__ LineGeom g, LView v, LineWs ws, int nframes) {
    __shared__ __align__(16) unsigned s_in[PI_H * (PI_W / 4)];     // staged input, reflected at the frame's borders
    __shared__ __align__(16) unsigned short s_h[PH_H * PB_W];      // horizontal pass; then the resized box (PS_H x PS_W bytes)
    __shared__ __align__(16) uint8_t s_b[PB_H * PB_W];             // blur5, then blur7
    __shared__ int s_next;
    unsigned* s_sc = reinterpret_cast<unsigned*>(s_h);
    const int tid = threadIdx.x, per_frame = g.tiles_x * g.tiles_y, ntiles = per_frame * nframes;
    if (tid == 0) s_next = atomicAdd(ws.prep_next, 1);
    __syncthreads();
    int t = s_next;
    if (t >= ntiles) return;
    prep_stage(s_in, g, v, t / per_frame, (t % per_frame % g.tiles_x) * PT_W, (t % per_frame / g.tiles_x) * PT_H);
    for (;;) {
        const int f = t / per_frame, tile = t - f * per_frame;
        const int trow = tile / g.tiles_x, tcol = tile - trow * g.tiles_x;
        const int X0 = tcol * PT_W, Y0 = trow * PT_H, SX0 = tcol * PT_SW, SY0 = trow * PT_SH;
        asm volatile("cp.async.wait_all;" ::: "memory");
        __syncthreads();                                 // the staged box is complete; the previous tile is done with s_h and s_next
        if (tid == 0) s_next = atomicAdd(ws.prep_next, 1);
        prep_hpass<1, 0>(s_in, s_h, BL5_T0, BL5_T4);     // blur5 column c = input column X0-1+c: window X0-3+c .. X0+1+c = staged c+1 ..
        __syncthreads();
        prep_vpass(s_h, s_b, BL5_T0, BL5_T4);
        __syncthreads();
        // Sobel 3x3 of blur5 with BORDER_REFLECT_101 -> dx, dy; four pixels per item
        for (int i = tid; i < PT_H * (PT_W / 4); i += PT_NT) {
            const int r = i / (PT_W / 4), q = i - r * (PT_W / 4);
            const int y = Y0 + r, x0 = X0 + 4 * q;
            if (y >= g.h || x0 >= g.w) continue;
            const int rows[3] = {reflect101(y - 1, g.h) - Y0 + 1, r + 1, reflect101(y + 1, g.h) - Y0 + 1};
            int vv[3][6];                                            // columns x0-1 .. x0+4 of the three rows (blur5 column c is s_b column c-X0+1)
#pragma unroll
            for (int k = 0; k < 3; k++) {
                const unsigned* p = reinterpret_cast<const unsigned*>(s_b + rows[k] * PB_W) + q;
                const unsigned a = p[0], b = p[1];
                vv[k][0] = x0 ? a & 0xff : (a >> 16) & 0xff;         // column -1 reflects to column 1
                vv[k][1] = (a >> 8) & 0xff; vv[k][2] = (a >> 16) & 0xff; vv[k][3] = a >> 24; vv[k][4] = b & 0xff; vv[k][5] = (b >> 8) & 0xff;
            }
            short dxs[4], dys[4];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const int x = x0 + k;
                int m0 = vv[0][k], m1 = vv[1][k], m2 = vv[2][k], c0 = vv[0][k + 1], c2 = vv[2][k + 1], p0 = vv[0][k + 2], p1 = vv[1][k + 2], p2 = vv[2][k + 2];
                if (x == g.w - 1) { p0 = m0; p1 = m1; p2 = m2; }    // reflect101(w) = w - 2 = x - 1
                dxs[k] = (short)((p0 - m0) + 2 * (p1 - m1) + (p2 - m2));
                dys[k] = (short)((m2 - m0) + 2 * (c2 - c0) + (p2 - p0));
            }
            const long long o = f * g.full_stride + (long long)y * g.w + x0;
            if ((g.w & 3) == 0 && (g.full_stride & 3) == 0) {
                *reinterpret_cast<short4*>(ws.dx + o) = make_short4(dxs[0], dxs[1], dxs[2], dxs[3]);
                *reinterpret_cast<short4*>(ws.dy + o) = make_short4(dys[0], dys[1], dys[2], dys[3]);
            } else {
#pragma unroll
                for (int k = 0; k < 4; k++) if (x0 + k < g.w) { ws.dx[o + k] = dxs[k]; ws.dy[o + k] = dys[k]; }
            }
        }
        prep_hpass<2, 1>(s_in, s_h, BL7_T0, BL7_T4);     // blur7 column c = input column X0+c: window X0-2+c .. X0+2+c = staged c+2 ..
        __syncthreads();                                 // s_in is free: request the next tile's box
        {
            const int tn = s_next;
            if (tn < ntiles) prep_stage(s_in, g, v, tn / per_frame, (tn % per_frame % g.tiles_x) * PT_W, (tn % per_frame / g.tiles_x) * PT_H);
        }
        prep_vpass(s_h, s_b, BL7_T0, BL7_T4);
        __syncthreads();
        // cv::resize(INTER_LINEAR_EXACT) 8U, 8.8 fixed point (SURVEY.md A.6 iii): the tables hold (i0, w1).  Resized columns past the tile's
        // one-column halo or the image are never read: they are written as 0.
        for (int i = tid; i < PS_H * (PS_W / 4); i += PT_NT) {
            const int r = i / (PS_W / 4), c4 = (i - r * (PS_W / 4)) * 4, y = SY0 + r;
            unsigned o = 0;
            if (y < g.sh) {
                const int2 ty = __ldg(&ws.tab[g.ytab_off + y]);
                const uint8_t* S0 = s_b + (ty.x - Y0) * PB_W;
                const uint8_t* S1 = s_b + (min(ty.x + 1, g.h - 1) - Y0) * PB_W;
                const int v1 = ty.y, v0 = 256 - v1;
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const int x = SX0 + c4 + k;
                    if (c4 + k > PT_SW || x >= g.sw) continue;
                    const int2 tx = __ldg(&ws.tab[g.xtab_off + x]);
                    const int i0 = tx.x - X0, i1 = min(tx.x + 1, g.w - 1) - X0, w1 = tx.y, w0 = 256 - w1;
                    const int r0 = w0 * S0[i0] + w1 * S0[i1], r1 = w0 * S1[i0] + w1 * S1[i1];
                    o |= (unsigned)((v0 * r0 + v1 * r1 + 32768) >> 16) << (8 * k);
                }
            }
            s_sc[i] = o;
        }
        __syncthreads();
        unsigned long long bits = 0ull;                    // max gradient norm of the defined pixels (positive doubles order like integers)
        for (int i = tid; i < PT_SH * (PT_SW / 4); i += PT_NT) {
            const int r = i / (PT_SW / 4), q = i - r * (PT_SW / 4);
            const int x0 = SX0 + 4 * q, y = SY0 + r;
            if (x0 >= g.sw || y >= g.sh) continue;
            float ang[4]; float2 cs[4], cs0[4]; double norm[4];
            unsigned r0 = 0, r1 = 0; int e0 = 0, e1 = 0;    // rows y, y+1: bytes x0..x0+3 and x0+4
            const bool row_ok = y < g.sh - 1;
            if (row_ok) {
                const unsigned* p = s_sc + r * (PS_W / 4) + q;
                r0 = p[0]; r1 = p[PS_W / 4]; e0 = p[1] & 0xff; e1 = p[PS_W / 4 + 1] & 0xff;
            }
#pragma unroll
            for (int k = 0; k < 4; k++) {
                ang[k] = NOTDEF_F; cs[k] = make_float2(0.f, 0.f); cs0[k] = make_float2(0.f, 0.f); norm[k] = 0;
                if (row_ok && x0 + k < g.sw - 1) {      // the last row and column stay NOTDEF with norm 0 (lsd.cpp)
                    const int A = (r0 >> (8 * k)) & 0xff, C = (r1 >> (8 * k)) & 0xff;
                    const int Bv = (k < 3) ? (int)((r0 >> (8 * k + 8)) & 0xff) : e0, D = (k < 3) ? (int)((r1 >> (8 * k + 8)) & 0xff) : e1;
                    const LLPix p = ll_pixel(D - A, Bv - C, g.rho);
                    norm[k] = p.norm; ang[k] = p.ang; cs[k] = p.cs; cs0[k] = p.cs0;
                    if (p.norm > g.rho) {
                        const unsigned long long nb = (unsigned long long)__double_as_longlong(p.norm);
                        bits = nb > bits ? nb : bits;
                    }
                }
            }
            const long long pi = f * g.pix_stride + (long long)y * g.sw + x0;
            if ((g.sw & 3) == 0 && (g.pix_stride & 3) == 0) {                  // rows start 16-byte aligned in every per-pixel array
                *reinterpret_cast<float4*>(ws.angdeg + pi) = make_float4(ang[0], ang[1], ang[2], ang[3]);
                float4* c4 = reinterpret_cast<float4*>(ws.cs0 + pi);
                c4[0] = make_float4(cs0[0].x, cs0[0].y, cs0[1].x, cs0[1].y); c4[1] = make_float4(cs0[2].x, cs0[2].y, cs0[3].x, cs0[3].y);
                double2* m2 = reinterpret_cast<double2*>(ws.modgrad + pi);
                m2[0] = make_double2(norm[0], norm[1]); m2[1] = make_double2(norm[2], norm[3]);
                uint4* px = reinterpret_cast<uint4*>(ws.pix + pi);
#pragma unroll
                for (int k = 0; k < 4; k++) px[k] = make_uint4(__float_as_uint(ang[k]), __float_as_uint(cs[k].x), __float_as_uint(cs[k].y), 0u);
            } else {
#pragma unroll
                for (int k = 0; k < 4; k++) if (x0 + k < g.sw) {
                    ws.angdeg[pi + k] = ang[k]; ws.cs0[pi + k] = cs0[k]; ws.modgrad[pi + k] = norm[k];
                    LPix px; px.ang = ang[k]; px.cx = cs[k].x; px.cy = cs[k].y; px.used = 0u;
                    ws.pix[pi + k] = px;
                }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { const unsigned long long b = __shfl_xor_sync(0xffffffffu, bits, o); bits = b > bits ? b : bits; }
        if ((threadIdx.x & 31) == 0 && bits) atomicMax(ws.maxgrad + f, bits);
        t = s_next;                                      // unchanged since the read above: it is rewritten only after the loop's first barrier
        if (t >= ntiles) break;
    }
}

// Debug (sslpl_line_debug_ll_table): ll_pixel on every (DA, BC) in [-255, 255]^2, entry (DA + 255) * LL_SPAN + (BC + 255).
constexpr int LL_SPAN = 511;
__global__ void k_ll_table(double rho, float* ang, float2* cs, float2* cs0, double* norm) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= LL_SPAN * LL_SPAN) return;
    const LLPix p = ll_pixel(i / LL_SPAN - 255, i % LL_SPAN - 255, rho);
    ang[i] = p.ang; cs[i] = p.cs; cs0[i] = p.cs0; norm[i] = p.norm;
}

__device__ __forceinline__ int lsd_bin(double norm, double max_grad) {
    const double bin_coef = (max_grad > 0) ? double(NBINS - 1) / max_grad : 0;
    return (int)(norm * bin_coef);
}

// Seed ordering of lsd.cpp in one kernel: the defined pixels sorted by gradient bin (descending), raster order inside
// a bin — a stable counting sort.  One CTA of 32 warps per frame; warp w owns the w-th contiguous pixel range (raster
// order), builds its own 1024-bin histogram in shared memory, the histograms are prefix-summed across warps and bins,
// and every warp then scatters its pixels in order (ranks inside a 32-group by __match_any_sync).
constexpr int SEED_WARPS = 8;                       // warps per frame: 32 KB of histograms and ~16k registers per CTA, so that
                                                    // seed CTAs fit on SMs that are busy with region walkers of other batches
__global__ void __launch_bounds__(SEED_WARPS * 32) k_lsd_seeds(const __grid_constant__ LineGeom g, LineWs ws) {
    __shared__ int s_wh[SEED_WARPS * NBINS];         // [warp][bin] running offsets
    __shared__ int s_warp[33];
    constexpr int NT = SEED_WARPS * 32, BPT = NBINS / NT;   // bins per thread in the prefix step
    const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    // a pixel is defined (angle != NOTDEF) exactly when its gradient norm exceeds rho (k_lsd_prep): one array to read
    const double* mod = ws.modgrad + f * g.pix_stride;
    const double mg = __longlong_as_double((long long)ws.maxgrad[f]), rho = g.rho;
    const double bin_coef = (mg > 0) ? double(NBINS - 1) / mg : 0;
    int* wh = s_wh + wid * NBINS;
    for (int i = tid; i < SEED_WARPS * NBINS; i += NT) s_wh[i] = 0;
    __syncthreads();
    const long long per = ((g.pix_stride + SEED_WARPS - 1) / SEED_WARPS + 31) / 32 * 32;   // pixels per warp, multiple of 32
    const long long b = wid * per, e = min(g.pix_stride, b + per);
    constexpr int U = 8;                                                       // groups of 32 pixels in flight per warp
    for (long long i0 = b; i0 < e; i0 += 32 * U) {
        double m[U];
#pragma unroll
        for (int u = 0; u < U; u++) { const long long i = i0 + u * 32 + lane; m[u] = i < e ? __ldg(mod + i) : 0.0; }
#pragma unroll
        for (int u = 0; u < U; u++) if (m[u] > rho) atomicAdd(&wh[NBINS - 1 - (int)(m[u] * bin_coef)], 1);
    }
    __syncthreads();
    {   // thread = BPT consecutive bins: exclusive prefix over the warps inside each bin, then over the bins
        int run[BPT], mine = 0;
#pragma unroll
        for (int k = 0; k < BPT; k++) {
            const int bin = tid * BPT + k;
            int r = 0;
            for (int w = 0; w < SEED_WARPS; w++) { const int c = s_wh[w * NBINS + bin]; s_wh[w * NBINS + bin] = r; r += c; }
            run[k] = r; mine += r;
        }
        int total;
        int base = block_exclusive_scan(mine, s_warp, &total);
#pragma unroll
        for (int k = 0; k < BPT; k++) {
            const int bin = tid * BPT + k;
            for (int w = 0; w < SEED_WARPS; w++) s_wh[w * NBINS + bin] += base;
            base += run[k];
        }
        if (tid == 0) ws.nseeds[f] = total;
    }
    __syncthreads();
    unsigned* seeds = ws.seeds + f * g.pix_stride;
    for (long long i0 = b; i0 < e; i0 += 32 * U) {
        double m[U];
#pragma unroll
        for (int u = 0; u < U; u++) { const long long i = i0 + u * 32 + lane; m[u] = i < e ? __ldg(mod + i) : 0.0; }
#pragma unroll
        for (int u = 0; u < U; u++) {                                          // groups in raster order: a stable sort
            const bool def = m[u] > rho;
            if (!__any_sync(0xffffffffu, def)) continue;
            const int key = def ? (NBINS - 1 - (int)(m[u] * bin_coef)) : (2048 + lane);
            const unsigned peers = __match_any_sync(0xffffffffu, key);
            const int leader = __ffs(peers) - 1, rank = __popc(peers & ((1u << lane) - 1));
            int off = 0;
            if (def && lane == leader) { off = wh[key]; wh[key] = off + __popc(peers); }
            off = __shfl_sync(0xffffffffu, off, leader);
            if (def) seeds[off + rank] = (unsigned)(i0 + u * 32 + lane);
            __syncwarp();
        }
    }
}

// -------------------------------------------------------------------------------------------------
// The sequential region walker.  All lanes run the same control flow on warp-uniform values; loads of 32
// region points / 9 neighbours are spread over the lanes and broadcast with shuffles; lane 0 does the writes.
// The walker's CTA is ONE warp; its per-frame context lives in shared memory (file scope) so that the big
// per-region routines can be real calls (__noinline__): inlined, the kernel was ~175 KB of SASS and the resident
// warps (each at a different place in it) spent most of their stall time on instruction fetch.
// -------------------------------------------------------------------------------------------------
struct LRect { double x1, y1, x2, y2, width, x, y, theta, dx, dy, prec, p; };

struct Walk {                   // context of the rectangle scans (k_lsd_nfa_*): registers
    int w, h;
    const float* ang;
    double log_nt;
    const double* lgam;
    int lane;
};

constexpr int WALK_MAXW = 16;          // warps of a walker CTA (one CTA per frame)
constexpr int WALK_RING = 64;          // region-growing attempts in flight per frame (speculation slots)
constexpr int WALK_SLOT_CAP = 2048;    // list entries of a slot: every pixel the attempt ever accepted + the pixels it assumed used
constexpr int WALK_SMALL = 32;         // attempts with at most this many list entries are committed from shared memory
constexpr int WALK_WIN = 64;           // seeds staged in shared memory for the claims

struct WalkCtx {                // context of one walker warp (k_lsd_regions): shared memory
    int w, h;
    const float* ang; const double* mod;
    LPix* pix;                  // packed per-pixel record; .used holds the ticket (global): who is growing over this pixel right now
    const unsigned* bits;       // the frame's COMMITTED `used` bitmap (shared memory); bits only ever go 0 -> 1
    unsigned* reg;              // current region list (x | y << 16)
    unsigned* base0;            // start of this attempt's list space
    const float2* cs0;          // per pixel: (float)cos / sin of the level-line angle taken as double (region seed values)
    int cap;                    // entries available at reg (the assumed-used list grows down from reg + cap)
    int nasm;                   // assumed-used pixels recorded so far
    int acc;                    // entries of base0[] that hold accepted-ever pixels (validated at commit)
    int seq;                    // rank of this attempt (claim order)
    int mode;                   // 0 = speculative, 1 = turn holder (everything of lower rank is committed)
    int dbg;
    int abort;                  // speculative attempt abandoned: 1 = capacity, 2 = a live attempt of LOWER rank holds a pixel it needs
    int conflict;               // abort == 2: that rank (the attempt can be repeated once it has been retired)
    unsigned ticket;
    int dirty, ndeps; unsigned dep[2];   // v3: released pixels; tickets of live lower attempts whose pixels were assumed used
};
struct FrameCtl {               // one per walker CTA
    unsigned cursor, nclaims, turn;
    int claim_lock, commit_lock, all_claimed, nj, frame, ns, win_base;
    unsigned win[WALK_WIN];
    int seqof[WALK_RING], seedpix[WALK_RING], state[WALK_RING], acc[WALK_RING], nasm[WALK_RING], finoff[WALK_RING], nfin[WALK_RING], job[WALK_RING], poison[WALK_RING];
    double jobv[WALK_RING][13];                 // the pending NFA job of the slot
    unsigned small[WALK_RING][WALK_SMALL];      // acc + nasm <= WALK_SMALL and finoff == 0: accepted list, then the assumed pixels (as indices)
};
__shared__ WalkCtx s_Wc[WALK_MAXW];
__shared__ FrameCtl s_F;
__shared__ __align__(16) double s_stc[WALK_MAXW][96];     // per warp: staging of a 32-point chunk: 3 quantities x 32
__shared__ WalkCtx s_W1;                                   // the one-warp throughput kernel keeps its own small context:
__shared__ __align__(16) double s_st1[96];                 // 28 of its CTAs share an SM
constexpr int SOLO = 0;                                    // (hidden by the template parameter of the same name inside the helpers)
// SOLO: 0 = multi-warp walker of round 2a (k_lsd_regions), 1 / 2 = one warp per frame (round-2a form / lean), 3 = multi-warp walker v3,
// 4 = lane-parallel walker (one warp per frame; the cooperative routines work on the region of one lane)
#define s_W (*((SOLO == 1 || SOLO == 2 || SOLO == 4) ? &s_W1 : &s_Wc[threadIdx.x >> 5]))
#define s_st ((SOLO == 1 || SOLO == 2 || SOLO == 4) ? s_st1 : s_stc[threadIdx.x >> 5])

// SLOT_PRESUMED: the seed was under the ticket of a live attempt of lower rank when its turn to be grown came: it is presumed
// swallowed; the commit checks (and grows it for real if it was not).  SLOT_ABORTED: to be redone by the turn holder.
enum { SLOT_EMPTY = 0, SLOT_RUNNING = 1, SLOT_DONE = 2, SLOT_ABORTED = 3, SLOT_PRESUMED = 4 };

// ticket = rank + 1 in bits 0..23, attempt number in bits 24..30, bit 31 = grown by the turn holder
__device__ __forceinline__ unsigned l_turn() { return *reinterpret_cast<volatile unsigned*>(&s_F.turn); }
__device__ __forceinline__ bool l_bit(const unsigned* bits, int q) { return (reinterpret_cast<const volatile unsigned*>(bits)[q >> 5] >> (q & 31)) & 1u; }
// Is ticket m (not mine) held by an attempt that has not been retired yet?  Ranks below `turn` are committed or discarded.
__device__ __forceinline__ bool l_live(unsigned m, int* seq_out) { const int s = (int)(m & 0xffffffu) - 1; *seq_out = s; return m != 0u && s >= (int)l_turn(); }
// (v3: a released pixel keeps the ticket with bit 31 set: it is free for everybody, but an attempt of LOWER rank that takes it still
//  poisons the releasing attempt, whose first growth went over a pixel that the sequential order gives to the lower rank)
template <int SOLO> __device__ __forceinline__ void l_release(const WalkCtx& W, int q) {
    if (SOLO == 1 || SOLO == 2) W.pix[q].used = 0u;
    else if (SOLO == 3 || SOLO == 4) atomicCAS(&W.pix[q].used, W.ticket, W.ticket | 0x80000000u);
    else atomicCAS(&W.pix[q].used, W.ticket, 0u);
}

__device__ __forceinline__ bool l_aligned(float angdeg, double theta, double prec) {
    if (angdeg == NOTDEF_F) return false;
    const double a = (double)angdeg * L_DEG;
    double n = theta - a;
    if (n < 0) n = -n;
    if (n > L_3_2_PI) { n -= L_2PI; if (n < 0) n = -n; }
    return n <= prec;
}

__device__ __forceinline__ bool l_aligned_rad(double a, double theta, double prec) {      // a = (double)angdeg * L_DEG, not NOTDEF
    double n = theta - a;
    if (n < 0) n = -n;
    if (n > L_3_2_PI) { n -= L_2PI; if (n < 0) n = -n; }
    return n <= prec;
}

// region_grow (lsd.cpp).  FOUR queue entries are expanded per step: lane = 8 * slot + neighbour (the centre pixel is
// always used, so the 3x3 scan has 8 live neighbours, kept in the reference's yy-outer / xx-inner order), i.e. the 32
// lanes hold the next 32 neighbour tests of the sequential algorithm in order.  Sequential semantics (each neighbour
// is tested once, in scan order, against the region angle as updated by the neighbours accepted before it) are kept
// in as many rounds as there are acceptances: all pending lanes test against the current angle; the first passing
// lane k0 is accepted, lanes < k0 are definitively rejected (they saw exactly the angle the sequential scan would have
// shown them), later lanes holding the same pixel drop out (the scan would find it used).
//
// "Used" is what the sequential algorithm would see: the frame's committed bitmap (regions of lower rank that are final) or
// my own ticket.  A pixel under the ticket of a LIVE attempt of lower rank is assumed used and recorded (checked at commit);
// one under a live ticket of higher rank counts as free (taking it poisons that attempt).  A pixel is taken with one atomic
// whose result is only looked at one step later (the round trip overlaps the next step's loads): a speculative attempt that
// lost a pixel to a live attempt of lower rank is abandoned then (abort = 2, conflict = that rank).
// Returns -1 when the attempt has to be abandoned (s_W.abort says why).
struct LTake { unsigned seen, old; int q; bool pend; };
__device__ __forceinline__ void l_take_issue(const WalkCtx& W, LTake& t, int q, unsigned seen) {
    t.q = q; t.seen = seen; t.pend = true;
    t.old = W.mode == 0 ? atomicCAS(&W.pix[q].used, seen, W.ticket) : atomicExch(&W.pix[q].used, W.ticket);
}
// Looks at the result of the atomic issued one step earlier.  Returns -1 when the pixel is mine, the rank of the live attempt of
// LOWER rank that holds it (the speculative attempt must be repeated after that rank retires), or -2 when a speculative attempt lost
// the compare-and-swap to anybody else: the word changed between this attempt's read and its atomic, so other lanes may have acted
// on the stale ticket during the step in between (the pixel could be in the list twice) — the attempt is simply repeated at once.
__device__ __forceinline__ int l_take_resolve(const WalkCtx& W, LTake& t) {
    if (!t.pend) return -1;
    t.pend = false;
    const unsigned old = t.old; int s;
    if (W.mode != 0 || old == t.seen) {                           // the pixel is mine; whoever held it alive (higher rank) is poisoned
        if (old != W.ticket && l_live(old, &s) && s != W.seq) s_F.poison[s % WALK_RING] = 1;
        return -1;
    }
    return (l_live(old, &s) && s < W.seq) ? s : -2;
}

template <int SOLO> __device__ __noinline__ int l_region_grow(int sx, int sy, double prec, double* reg_angle_out) {
    WalkCtx& W = s_W;
    const int lane = threadIdx.x & 31, w = W.w, h = W.h;
    LPix* pix = W.pix; unsigned* reg = W.reg; const unsigned* bits = W.bits;
    const unsigned T = W.ticket; const int myseq = W.seq; const bool spec = W.mode == 0;
    const int sq = sy * w + sx;                                   // 32-bit pixel indices (sw * sh < 2^31)
    LTake tk; tk.pend = false; tk.q = 0; tk.seen = 0u; tk.old = 0u;
    int failrank = -1;                                            // -1 fine, >= 0 rank to wait for, -2 repeat at once
    if (SOLO) { if (lane == 0) { reg[0] = (unsigned)sx | ((unsigned)sy << 16); pix[sq].used = 1u; } }
    else {
        int fail = 0;
        if (lane == 0) {
            reg[0] = (unsigned)sx | ((unsigned)sy << 16);
            const unsigned m0 = __ldcg(&pix[sq].used);
            int s0;
            if (m0 != T) {
                if (spec && l_live(m0, &s0) && s0 < myseq) fail = 3;          // an in-flight region of lower rank reached the seed first: presumed swallowed
                else { W.conflict = -1; l_take_issue(W, tk, sq, m0); const int r = l_take_resolve(W, tk); if (r >= 0) fail = 3; else if (r == -2) fail = 2; }
            }
        }
        fail = __shfl_sync(0xffffffffu, fail, 0);
        if (fail) { W.abort = fail; return -1; }
    }
    double reg_angle = (double)__ldg(W.ang + sq) * L_DEG;
    const float2 c0 = __ldg(W.cs0 + sq);
    float sumdx = c0.x, sumdy = c0.y;
    int n = 1, nasm = W.nasm;
    const int cap = W.cap;
    const int slot = lane >> 3, nb = (lane & 7) + ((lane & 7) >= 4 ? 1 : 0);   // neighbour 0..8 without the centre (4)
    const int ox = nb % 3 - 1, oy = nb / 3 - 1;
    __syncwarp();
    for (int i = 0; i < n;) {
        const int cnt = min(4, n - i);
        unsigned pk = 0, pkn = 0;
        if (slot < cnt) pk = reg[i + slot];
        const bool hasn = i + 4 + slot < n;                      // the next step's entries, where they already exist:
        if (hasn) pkn = reg[i + 4 + slot];                       // pull their neighbour records towards L2 now
        const int xx = (int)(pk & 0xffff) + ox, yy = (int)(pk >> 16) + oy, q = yy * w + xx;
        const bool valid = slot < cnt && (unsigned)xx < (unsigned)w && (unsigned)yy < (unsigned)h;
        {
            const int xn = (int)(pkn & 0xffff) + ox, yn = (int)(pkn >> 16) + oy;
            if (hasn && (unsigned)xn < (unsigned)w && (unsigned)yn < (unsigned)h)
                asm volatile("prefetch.global.L2 [%0];" :: "l"(pix + (yn * w + xn)));
        }
        uint4 v = make_uint4(__float_as_uint(NOTDEF_F), 0u, 0u, 0u);
        if (valid) v = SOLO ? *reinterpret_cast<const uint4*>(pix + q) : __ldcg(reinterpret_cast<const uint4*>(pix + q));   // record + ticket in one load (L2: the ticket is mutable)
        if (!SOLO) { const int r = l_take_resolve(W, tk); if (r != -1) failrank = (r >= 0 && r > failrank) ? r : (failrank >= 0 ? failrank : r); }   // last step's atomic, while this step's loads fly
        const float a = __uint_as_float(v.x), cx = __uint_as_float(v.y), cy = __uint_as_float(v.z);
        const unsigned m = v.w;
        bool cand = false, assumed = false;
        if (SOLO) cand = valid && a != NOTDEF_F && m == 0u;
        else if (valid && a != NOTDEF_F && m != T && !l_bit(bits, q)) {
            int s;
            if (spec && l_live(m, &s) && s < myseq) { assumed = true; if (W.dbg & 16) failrank = s > failrank ? s : failrank; }
            else cand = true;
        }
        const unsigned lt = (1u << lane) - 1u;
        const unsigned am = __ballot_sync(0xffffffffu, assumed);
        if (am) {                                                 // remember what was assumed: the commit checks these bits are set
            if (n + nasm + __popc(am) > cap) { W.abort = 1; return -1; }
            if (assumed) reg[cap - 1 - nasm - __popc(am & lt)] = (unsigned)q;
            nasm += __popc(am);
        }
        const double ad = (double)a * L_DEG;
        unsigned pending = __ballot_sync(0xffffffffu, cand);
        while (pending) {
            const bool mep = (pending >> lane) & 1u;
            const unsigned S0 = __ballot_sync(0xffffffffu, mep && l_aligned_rad(ad, reg_angle, prec));
            if (!S0) break;                                       // nobody passes at the current angle: all rejected
            if (n + nasm + __popc(S0) > cap) { W.abort = 1; return -1; }
            if ((S0 & (S0 - 1u)) == 0u) {
                // exactly one candidate: the plain sequential step
                const int k0 = __ffs(S0) - 1;
                const float kx = __shfl_sync(0xffffffffu, cx, k0), ky = __shfl_sync(0xffffffffu, cy, k0);
                const int q0 = __shfl_sync(0xffffffffu, q, k0);
                if (lane == k0) { reg[n] = (unsigned)xx | ((unsigned)yy << 16); if (SOLO) pix[q].used = 1u; else l_take_issue(W, tk, q, m); }
                n++;
                sumdx += kx; sumdy += ky;
                reg_angle = (double)fast_atan2_deg(sumdy, sumdx) * L_DEG;
                pending &= ~((2u << k0) - 1u);
                pending &= ~__ballot_sync(0xffffffffu, q == q0);  // the same pixel seen from another queue entry
                continue;
            }
            // Several candidates: SPECULATE that exactly the lanes passing at the current angle (first holder of each
            // pixel only) will be accepted.  Every lane then forms the running sums the sequential scan would hold when
            // it reaches that lane (ordered float adds over the earlier members), ONE SIMT atan2 gives every member's
            // "angle after me", each pending lane re-tests itself against the angle of the member just before it, and
            // the speculation is accepted up to the first lane whose verified outcome differs from the guess (that
            // lane's verified outcome is the true one, because everything before it was right).
            const unsigned peers = __match_any_sync(0xffffffffu, mep ? q : ~lane);
            const bool inS0 = (S0 >> lane) & 1u;
            const unsigned S = S0 & ~__ballot_sync(0xffffffffu, inS0 && (peers & S0 & lt) != 0u);
            const bool inS = (S >> lane) & 1u;
            float bx = sumdx, by = sumdy;
            for (unsigned Tm = S; Tm; Tm &= Tm - 1u) {
                const int mm = __ffs(Tm) - 1;
                const float mx = __shfl_sync(0xffffffffu, cx, mm), my = __shfl_sync(0xffffffffu, cy, mm);
                if (lane > mm) { bx += mx; by += my; }
            }
            const float ax = bx + cx, ay = by + cy;
            const double aft = (double)fast_atan2_deg(ay, ax) * L_DEG;
            const unsigned prevm = S & lt;
            double bef = __shfl_sync(0xffffffffu, aft, (31 - __clz(prevm)) & 31);
            if (!prevm) bef = reg_angle;
            const bool dup_e = (peers & S & lt) != 0u;            // an earlier member holds my pixel: the scan finds it used
            const bool actual = mep && !dup_e && l_aligned_rad(ad, bef, prec);
            const unsigned mism = __ballot_sync(0xffffffffu, mep && (actual != inS));
            int src; unsigned A;
            if (!mism) { A = S; src = 31 - __clz(S); }
            else {
                src = __ffs(mism) - 1;
                const unsigned acc = __ballot_sync(0xffffffffu, actual);
                A = (S & ((1u << src) - 1u)) | (acc & (1u << src));
            }
            if ((A >> lane) & 1u) { reg[n + __popc(A & lt)] = (unsigned)xx | ((unsigned)yy << 16); if (SOLO) pix[q].used = 1u; else l_take_issue(W, tk, q, m); }
            n += __popc(A);
            const float selx = actual ? ax : bx, sely = actual ? ay : by;
            const double sela = actual ? aft : bef;
            sumdx = __shfl_sync(0xffffffffu, selx, src); sumdy = __shfl_sync(0xffffffffu, sely, src);
            reg_angle = __shfl_sync(0xffffffffu, sela, src);
            if (!mism) break;                                     // every pending lane is resolved
            pending &= ~((2u << src) - 1u);
            pending &= ~__ballot_sync(0xffffffffu, mep && (peers & A) != 0u);   // later holders of accepted pixels
        }
        __syncwarp();
        if (!SOLO && spec && __any_sync(0xffffffffu, failrank != -1)) break;   // lost a pixel: stop growing now
        i += cnt;
    }
    if (SOLO) { *reg_angle_out = reg_angle; return n; }
    { const int r = l_take_resolve(W, tk); if (r != -1) failrank = (r >= 0 && r > failrank) ? r : (failrank >= 0 ? failrank : r); }
    const bool lostany = __any_sync(0xffffffffu, failrank != -1);
    failrank = __reduce_max_sync(0xffffffffu, failrank);          // the highest rank to wait for (-1 / -2 lanes do not count)
    W.nasm = nasm;
    if (lostany) { W.abort = 2; W.conflict = failrank >= 0 ? failrank : -1; return -1; }
    *reg_angle_out = reg_angle;
    return n;
}


// -------------------------------------------------------------------------------------------------
// region_grow, LEAN form (one warp per frame, round 2b).  Same sequential semantics as l_region_grow<1>, restructured around
// the dependent-chain latencies of the GPU (tools/lat_probe.cu measures SHFL, MATCH, FDIV, the double alignment test, L1 and L2
// hits and LDS), because the walker is one warp following one chain:
//   * the region list's tail lives in a shared-memory ring (the frontier is read with LDS, not through L1/L2; the full list
//     still goes to global memory for region2rect / refine, fire and forget);
//   * the alignment test runs on the float DEGREES that both operands come from (|theta - a| <= prec is decided in float
//     when it is further than 2e-3 deg from the threshold or from the 270-degree fold; closer than that the reference's
//     double formula decides) — no FP64 and no conversions on the chain;
//   * the region angle is LAZY: a round tests every pending lane against the exact current angle; the first passing lane k0
//     is accepted (exact), and every later lane whose outcome cannot change while at most K = popc(passing) more unit
//     vectors are added to the sums is decided in the same round without recomputing the angle.  The bound is rigorous:
//     the scan reaches lane l after accepting at most K_l = (first holders among the passing lanes before l) unit vectors, each
//     within prec + E of S, so S has turned by at most atan(sum |sin phi_i| / |S|) <= 57.3 deg * sin(prec + E) * K_l / |S|;
//     cv::fastAtan2 is within E = 0.00956 deg of atan2 (measured over 5e8 inputs; 2E = 0.0202 used), float rounding of the
//     sums is < 3e-4 deg, the rest of the 0.0215 deg is slack.  tools/sim_lean_grow.cpp runs this lane by lane against the
//     oracle's sequential region_grow (every call of four frames identical).
//     The round stops before the first lane that is not robust in that sense; only then is the angle recomputed on the
//     chain.  For big regions (|S| ~ n) nearly every step is ONE round with no atan2 before the next step's loads;
//   * the angle of the next step is recomputed after that step's loads have been issued (it overlaps their latency);
//   * duplicates (the same pixel seen from two queue entries) come from one MATCH issued under the record load;
//   * accepted pixels warm L1 with the six sectors of their 3x3 neighbourhood (consumed one step later).
// -------------------------------------------------------------------------------------------------
__device__ int l_region_grow_v3(int sx, int sy, double prec, double* reg_angle_out);
constexpr int LEAN_RING = 1024;
__shared__ unsigned s_ring1[LEAN_RING];

__device__ __noinline__ int l_region_grow_lean(int sx, int sy, double prec, double* reg_angle_out) {
    WalkCtx& W = s_W1;
    const int lane = threadIdx.x & 31, w = W.w, h = W.h;
    LPix* pix = W.pix; unsigned* reg = W.reg;
    const int sq = sy * w + sx;
    if (lane == 0) { const unsigned pk0 = (unsigned)sx | ((unsigned)sy << 16); reg[0] = pk0; s_ring1[0] = pk0; pix[sq].used = 1u; }
    float th = __ldg(W.ang + sq);                                // degrees; the region angle is (double)th * L_DEG throughout
    const float2 c0 = __ldg(W.cs0 + sq);
    float sumdx = c0.x, sumdy = c0.y;
    float rM = rsqrtf(sumdx * sumdx + sumdy * sumdy);
    bool dirty = false;                                          // th / rM are older than the sums
    int n = 1;
    const float pdeg = (float)(prec * (180.0 / L_PI));
    const float coef = (float)(57.2958 * 1.0002 * sin(prec + 0.0006));     // degrees the sums can turn per (accepted vector / |S|): see above
    const bool rob_ok = prec < 0.78;                             // <= 45 deg: then prec + B <= 75.2 deg < 90 and the reference's fold at 270 deg is the circular distance
    const int slot = lane >> 3, nb = (lane & 7) + ((lane & 7) >= 4 ? 1 : 0);
    const int ox = nb % 3 - 1, oy = nb / 3 - 1;
    const unsigned lt = (1u << lane) - 1u;
    unsigned sink = 0u, wu0 = 0u, wu1 = 0u, wu2 = 0u, wu3 = 0u, wu4 = 0u, wu5 = 0u;
    __syncwarp();
    for (int i = 0; i < n;) {
        const int cnt = min(4, n - i);
        unsigned pk = 0;
        { const int j = i + slot; if (slot < cnt) pk = (n - j <= LEAN_RING) ? s_ring1[j & (LEAN_RING - 1)] : reg[j]; }
        const int xx = (int)(pk & 0xffff) + ox, yy = (int)(pk >> 16) + oy, q = yy * w + xx;
        const bool valid = slot < cnt && (unsigned)xx < (unsigned)w && (unsigned)yy < (unsigned)h;
        uint4 v = make_uint4(__float_as_uint(NOTDEF_F), 0u, 0u, 1u);
        if (valid) v = *reinterpret_cast<const uint4*>(pix + q);
        const unsigned peers = __match_any_sync(0xffffffffu, valid ? q : ~lane);     // under the load
        sink ^= wu0 ^ wu1 ^ wu2 ^ wu3 ^ wu4 ^ wu5;                                   // last step's warm-up loads have landed by now
        if (dirty) { th = fast_atan2_deg(sumdy, sumdx); rM = rsqrtf(sumdx * sumdx + sumdy * sumdy); dirty = false; }
        const float a = __uint_as_float(v.x), cx = __uint_as_float(v.y), cy = __uint_as_float(v.z);
        unsigned pending = __ballot_sync(0xffffffffu, valid && a != NOTDEF_F && v.w == 0u);
        while (pending) {
            const bool mep = (pending >> lane) & 1u;
            const float d = fabsf(th - a);
            const float e = d > 270.f ? 360.f - d : d;
            bool pass = e <= pdeg;
            const bool near = fabsf(e - pdeg) < 2e-3f || fabsf(d - 270.f) < 2e-3f;
            if (__any_sync(0xffffffffu, mep && near)) { if (near) pass = l_aligned_rad((double)a * L_DEG, (double)th * L_DEG, prec); }
            const unsigned P = __ballot_sync(0xffffffffu, mep && pass);
            if (!P) break;                                        // nobody passes at the current angle: all rejected
            const int k0 = __ffs(P) - 1;
            const unsigned P1 = P & ~__ballot_sync(0xffffffffu, pass && mep && (peers & P & lt) != 0u);   // first holders among the passing lanes
            const float x = (float)__popc(P1 & lt) * rM;          // (vectors the scan can have added before this lane) / |S|
            bool robust = false;
            if (rob_ok && x <= 0.5f) { const float B = coef * x + 0.0215f; robust = pass ? (e <= pdeg - B) : (e >= pdeg + B); }
            const unsigned NR = __ballot_sync(0xffffffffu, mep && lane > k0 && !robust);
            const unsigned below = NR ? ((NR & (0u - NR)) - 1u) : 0xffffffffu;       // lanes before the first non-robust one
            const unsigned A = P1 & below;                        // accepted in this round, in scan order
            for (unsigned Tm = A; Tm; Tm &= Tm - 1u) {            // the sums, in scan order
                const int mm = __ffs(Tm) - 1;
                sumdx += __shfl_sync(0xffffffffu, cx, mm); sumdy += __shfl_sync(0xffffffffu, cy, mm);
            }
            if ((A >> lane) & 1u) {
                const int pos = n + __popc(A & lt);
                const unsigned me = (unsigned)xx | ((unsigned)yy << 16);
                s_ring1[pos & (LEAN_RING - 1)] = me; reg[pos] = me; pix[q].used = 1u;
                const int xa = max(xx - 1, 0), xb = min(xx + 1, w - 1), ya = max(yy - 1, 0), yb = min(yy + 1, h - 1);
                const unsigned* r0 = reinterpret_cast<const unsigned*>(pix + ya * w), * r1 = reinterpret_cast<const unsigned*>(pix + yy * w), * r2 = reinterpret_cast<const unsigned*>(pix + yb * w);
                asm volatile("ld.global.ca.u32 %0, [%1];" : "=r"(wu0) : "l"(r0 + 4 * xa));
                asm volatile("ld.global.ca.u32 %0, [%1];" : "=r"(wu1) : "l"(r0 + 4 * xb));
                asm volatile("ld.global.ca.u32 %0, [%1];" : "=r"(wu2) : "l"(r1 + 4 * xa));
                asm volatile("ld.global.ca.u32 %0, [%1];" : "=r"(wu3) : "l"(r1 + 4 * xb));
                asm volatile("ld.global.ca.u32 %0, [%1];" : "=r"(wu4) : "l"(r2 + 4 * xa));
                asm volatile("ld.global.ca.u32 %0, [%1];" : "=r"(wu5) : "l"(r2 + 4 * xb));
            }
            n += __popc(A);
            pending &= ~below;                                    // everything before the first non-robust lane is resolved
            pending &= ~__ballot_sync(0xffffffffu, mep && (peers & A) != 0u);        // later holders of accepted pixels
            dirty = true;
            if (pending) { th = fast_atan2_deg(sumdy, sumdx); rM = rsqrtf(sumdx * sumdx + sumdy * sumdy); dirty = false; }
        }
        __syncwarp();
        i += cnt;
    }
    if (dirty) th = fast_atan2_deg(sumdy, sumdx);
    if (sink == 0x9e3779b9u && n < 0) reg[0] = sink;             // keeps the warm-up loads alive (never true)
    *reg_angle_out = (double)th * L_DEG;
    return n;
}

__device__ __forceinline__ double l_angle_diff_signed(double a, double b) {
    double d = a - b;
    while (d <= -L_PI) d += L_2PI;
    while (d > L_PI) d -= L_2PI;
    return d;
}

// Sum of the three staged quantities of one chunk, in list order: lane c (c = lane % 3) owns accumulator c, so a
// point costs one shared load and one add per warp instead of three of each.
template <int SOLO> __device__ __noinline__ double l_chunk_sum(const double* sp, int m, double acc) {
    if (m == 32) {
        const double2* s2 = reinterpret_cast<const double2*>(sp);
#pragma unroll
        for (int j = 0; j < 16; j++) { const double2 v = s2[j]; acc += v.x; acc += v.y; }
    } else {
#pragma unroll 1
        for (int j = 0; j < m; j++) acc += sp[j];
    }
    return acc;
}

// region2rect + get_theta (lsd.cpp).  The weighted sums must be accumulated in list order to stay bit-identical with
// the CPU, but only the ADDS are sequential: each lane forms the products of its own point, stages them in shared
// memory, and lanes 0..2 (replicated over the warp) each walk one of the three staged rows.  The extents are exact
// min/max.
template <int SOLO> __device__ __noinline__ void l_region2rect(int n, double reg_angle, double prec, double p, LRect* out) {
    const int lane = threadIdx.x & 31, w = s_W.w;
    const unsigned* reg = s_W.reg; const double* __restrict__ mod = s_W.mod;
    double* s0 = s_st; double* s1 = s_st + 32; double* s2 = s_st + 64;
    const double* sp = s_st + (lane % 3) * 32;
    double acc = 0;
#pragma unroll 1
    for (int b = 0; b < n; b += 32) {
        const int i = b + lane;
        if (i < n) {
            const unsigned pk = reg[i]; const int rx = pk & 0xffff, ry = pk >> 16;
            const double wg = mod[ry * w + rx];
            s0[lane] = (double)rx * wg; s1[lane] = (double)ry * wg; s2[lane] = wg;
        }
        __syncwarp();
        acc = l_chunk_sum<SOLO>(sp, min(32, n - b), acc);
        __syncwarp();
    }
    double x = __shfl_sync(0xffffffffu, acc, 0), y = __shfl_sync(0xffffffffu, acc, 1);
    const double sum = __shfl_sync(0xffffffffu, acc, 2);
    x /= sum; y /= sum;
    acc = 0;
#pragma unroll 1
    for (int b = 0; b < n; b += 32) {
        const int i = b + lane;
        if (i < n) {
            const unsigned pk = reg[i]; const int rx = pk & 0xffff, ry = pk >> 16;
            const double wg = mod[ry * w + rx];
            const double dx = (double)rx - x, dy = (double)ry - y;
            s0[lane] = dy * dy * wg; s1[lane] = dx * dx * wg; s2[lane] = -(dx * dy * wg);      // Ixy -= v  ==  Ixy += -v
        }
        __syncwarp();
        acc = l_chunk_sum<SOLO>(sp, min(32, n - b), acc);
        __syncwarp();
    }
    const double Ixx = __shfl_sync(0xffffffffu, acc, 0), Iyy = __shfl_sync(0xffffffffu, acc, 1), Ixy = __shfl_sync(0xffffffffu, acc, 2);
    const double lambda = 0.5 * (Ixx + Iyy - sqrt((Ixx - Iyy) * (Ixx - Iyy) + 4.0 * Ixy * Ixy));
    double theta = (fabs(Ixx) > fabs(Iyy)) ? (double)fast_atan2_deg((float)(lambda - Ixx), (float)Ixy)
                                           : (double)fast_atan2_deg((float)Ixy, (float)(lambda - Iyy));
    theta *= L_DEG;
    if (fabs(l_angle_diff_signed(theta, reg_angle)) > prec) theta += L_PI;
    // correctly-rounded cos/sin (see ddtrig.h): the extreme region pixels sit exactly on the rectangle's end edges
    double dx, dy;
    ddtrig::sincos_cr(theta, &dy, &dx);
    double l_min = 0, l_max = 0, w_min = 0, w_max = 0;           // max(0, max l), min(0, min l): order-independent
#pragma unroll 2
    for (int i = lane; i < n; i += 32) {                         // (no NaNs here: plain compares instead of fmax/fmin)
        const unsigned pk = reg[i];
        const double rdx = (double)(pk & 0xffff) - x, rdy = (double)(pk >> 16) - y;
        const double l = rdx * dx + rdy * dy, ww = -rdx * dy + rdy * dx;
        l_max = l > l_max ? l : l_max; l_min = l < l_min ? l : l_min; w_max = ww > w_max ? ww : w_max; w_min = ww < w_min ? ww : w_min;
    }
#pragma unroll 1
    for (int o = 16; o > 0; o >>= 1) {
        const double a = __shfl_xor_sync(0xffffffffu, l_max, o), b = __shfl_xor_sync(0xffffffffu, l_min, o);
        const double c = __shfl_xor_sync(0xffffffffu, w_max, o), d = __shfl_xor_sync(0xffffffffu, w_min, o);
        l_max = a > l_max ? a : l_max; l_min = b < l_min ? b : l_min; w_max = c > w_max ? c : w_max; w_min = d < w_min ? d : w_min;
    }
    LRect rec;
    rec.x1 = x + l_min * dx; rec.y1 = y + l_min * dy; rec.x2 = x + l_max * dx; rec.y2 = y + l_max * dy;
    rec.width = w_max - w_min; rec.x = x; rec.y = y; rec.theta = theta; rec.dx = dx; rec.dy = dy; rec.prec = prec; rec.p = p;
    if (rec.width < 1.0) rec.width = 1.0;
    *out = rec;
}

__device__ __forceinline__ double l_dist(double x1, double y1, double x2, double y2) { return sqrt((x2 - x1) * (x2 - x1) + (y2 - y1) * (y2 - y1)); }
__device__ __forceinline__ double l_distsq(double x1, double y1, double x2, double y2) { return (x2 - x1) * (x2 - x1) + (y2 - y1) * (y2 - y1); }

// reduce_region_radius (lsd.cpp).  The reference removes far points by swap-with-last while scanning forward, which
// leaves the kept points in a definite order (it matters: region2rect sums in list order): every kept point below the
// new size m' stays where it is, and the holes below m' (ascending) receive the kept points from positions >= m'
// in DESCENDING position order.  That is computed here chunk-wise with ballots: a descending cursor collects
// "fillers", an ascending one "holes", matched through a 32-entry shared buffer.  The removed tail's order is
// irrelevant (those points are only un-marked).
template <int SOLO> __device__ __noinline__ bool l_reduce_region_radius(int* n_io, double reg_angle, double prec, double p, LRect* rec, double density, double density_th) {
    const int lane = threadIdx.x & 31, w = s_W.w;
    int n = *n_io;
    if ((SOLO == 0 || SOLO == 3 || SOLO == 4) && s_W.mode == 0) {  // speculative attempt: keep the list as it is (the commit validates every pixel ever accepted) and work on a copy
        if (2 * n + s_W.nasm > s_W.cap) { s_W.abort = 1; return false; }
        for (int i = lane; i < n; i += 32) s_W.reg[n + i] = s_W.reg[i];
        s_W.reg += n; s_W.cap -= n;
        __syncwarp();
    }
    unsigned* reg = s_W.reg;
    unsigned* s_fill = reinterpret_cast<unsigned*>(s_st);             // 32 filler values (s_st is free between region2rect calls)
    const unsigned p0 = reg[0];
    const double xc = (double)(p0 & 0xffff), yc = (double)(p0 >> 16);
    double radSq = fmax(l_distsq(xc, yc, rec->x1, rec->y1), l_distsq(xc, yc, rec->x2, rec->y2));
    while (density < density_th) {
        radSq *= 0.75 * 0.75;
        // pass 1: count the kept points, un-mark the removed ones
        int kept = 0;
#pragma unroll 1
        for (int b = 0; b < n; b += 32) {
            const int i = b + lane;
            bool keep = false;
            if (i < n) {
                const unsigned pk = reg[i];
                keep = !(l_distsq(xc, yc, (double)(pk & 0xffff), (double)(pk >> 16)) > radSq);
                if (!keep) l_release<SOLO>(s_W, (int)(pk >> 16) * w + (int)(pk & 0xffff));
            }
            kept += __popc(__ballot_sync(0xffffffffu, keep));
        }
        const int m2 = kept;
        // pass 2: fill the holes below m2 (ascending) with the kept points at or above m2 (descending)
        int lo = 0;                      // next hole chunk start (ascending, < m2)
        int hi = n;                      // filler cursor: positions [m2, hi) not yet consumed
        int nfill = 0, fpos = 0;         // fillers staged in s_fill[fpos .. nfill)
        while (lo < m2) {
            const int i = lo + lane;
            unsigned pk = 0; bool hole = false;
            if (i < m2) { pk = reg[i]; hole = l_distsq(xc, yc, (double)(pk & 0xffff), (double)(pk >> 16)) > radSq; }
            unsigned hm = __ballot_sync(0xffffffffu, hole);
            while (hm) {
                if (fpos == nfill) {     // stage the next (up to 32) fillers, descending from hi
                    nfill = 0; fpos = 0;
                    while (nfill == 0 && hi > m2) {
                        const int j = hi - 1 - lane;
                        unsigned fk = 0; bool isf = false;
                        if (j >= m2) { fk = reg[j]; isf = !(l_distsq(xc, yc, (double)(fk & 0xffff), (double)(fk >> 16)) > radSq); }
                        const unsigned fm = __ballot_sync(0xffffffffu, isf);
                        if (isf) s_fill[__popc(fm & ((1u << lane) - 1u))] = fk;
                        nfill = __popc(fm);
                        hi -= 32;
                    }
                    __syncwarp();
                    if (nfill == 0) break;                      // cannot happen (holes below m2 == kept at/above m2)
                }
                const int t = min(__popc(hm), nfill - fpos);    // holes served in this step
                const int r = __popc(hm & ((1u << lane) - 1u)); // this lane's rank among the pending holes
                if (((hm >> lane) & 1u) && r < t) reg[i] = s_fill[fpos + r];
                fpos += t;
                // drop the t lowest set bits of hm
                unsigned served = __ballot_sync(0xffffffffu, ((hm >> lane) & 1u) && r < t);
                hm &= ~served;
                __syncwarp();
            }
            lo += 32;
        }
        n = m2;
        __syncwarp();
        if (n < 2) { *n_io = n; return false; }
        l_region2rect<SOLO>(n, reg_angle, prec, p, rec);
        density = (double)n / (l_dist(rec->x1, rec->y1, rec->x2, rec->y2) * rec->width);
    }
    *n_io = n;
    return true;
}

template <int SOLO> __device__ __noinline__ bool l_refine(int* n_io, double* reg_angle_io, double prec, double p, LRect* rec, double density_th) {
    const int lane = threadIdx.x & 31, w = s_W.w;
    int n = *n_io;
    double density = (double)n / (l_dist(rec->x1, rec->y1, rec->x2, rec->y2) * rec->width);
    if (density >= density_th) return true;
    if constexpr (SOLO == 3) { if (lane == 0) s_W.dirty = 1; }      // pixels get released: attempts that assumed them used cannot be validated
    const unsigned* reg = s_W.reg; const float* __restrict__ ang = s_W.ang;
    const unsigned p0 = reg[0];
    const int sx = p0 & 0xffff, sy = p0 >> 16;
    const double xc = (double)sx, yc = (double)sy;
    const double ang_c = (double)ang[sy * w + sx] * L_DEG;
    const double width = rec->width;
    double* s0 = s_st; double* s1 = s_st + 32;
    const double* sp = s_st + (lane & 1) * 32;        // lane parity picks the accumulator: sum of d / sum of d*d
    double acc = 0; int cnt = 0;
#pragma unroll 1
    for (int b = 0; b < n; b += 32) {
        const int i = b + lane;
        bool in = false;
        if (i < n) {
            const unsigned pk = reg[i]; const int rx = pk & 0xffff, ry = pk >> 16;
            const float ad = ang[ry * w + rx];
            l_release<SOLO>(s_W, ry * w + rx);
            in = l_dist(xc, yc, (double)rx, (double)ry) < width;
            const double d = l_angle_diff_signed((double)ad * L_DEG, ang_c);
            // skipped points contribute +0.0, which leaves a running sum unchanged (the sums are never -0.0)
            s0[lane] = in ? d : 0.0; s1[lane] = in ? d * d : 0.0;
        }
        cnt += __popc(__ballot_sync(0xffffffffu, in));
        __syncwarp();
        acc = l_chunk_sum<SOLO>(sp, min(32, n - b), acc);
        __syncwarp();
    }
    const double sum = __shfl_sync(0xffffffffu, acc, 0), s_sum = __shfl_sync(0xffffffffu, acc, 1);
    const double mean_angle = sum / (double)cnt;
    const double tau = 2.0 * sqrt((s_sum - 2.0 * mean_angle * sum) / (double)cnt + mean_angle * mean_angle);
    __syncwarp();
    if ((SOLO == 0 || SOLO == 3) && s_W.mode == 0) { s_W.reg += n; s_W.cap -= n; }   // speculative: the first list stays (validated at commit), the regrown one follows it
    if constexpr (SOLO == 2) n = l_region_grow_lean(sx, sy, tau, reg_angle_io);
    else if constexpr (SOLO == 3) n = l_region_grow_v3(sx, sy, tau, reg_angle_io);
    else n = l_region_grow<SOLO>(sx, sy, tau, reg_angle_io);
    if (n < 0) { *n_io = 0; return false; }
    if ((SOLO == 0 || SOLO == 3) && s_W.mode == 0) s_W.acc += n;
    *n_io = n;
    if (n < 2) return false;
    l_region2rect<SOLO>(n, *reg_angle_io, prec, p, rec);
    density = (double)n / (l_dist(rec->x1, rec->y1, rec->x2, rec->y2) * rec->width);
    if (density < density_th) return l_reduce_region_radius<SOLO>(n_io, *reg_angle_io, prec, p, rec, density, density_th);
    return true;
}

__device__ double l_log_gamma(double x) {
    if (x > 15.0) return 0.918938533204673 + (x - 0.5) * log(x) - x + 0.5 * x * log(x * sinh(1 / x) + 1 / (810.0 * pow(x, 6.0)));
    const double q[7] = {75122.6331530, 80916.6278952, 36308.2951477, 8687.24529705, 1168.92649479, 83.8676043424, 2.50662827511};
    double a = (x + 0.5) * log(x + 5.5) - (x + 5.5), b = 0;
    for (int n = 0; n < 7; ++n) { a -= log(x + (double)n); b += q[n] * pow(x, (double)n); }
    return a + log(b);
}

__device__ __noinline__ double l_log(double x) { return log(x); }          // one copy of each libm routine per kernel
__device__ __noinline__ double l_log10(double x) { return log10(x); }
__device__ __noinline__ double l_exp(double x) { return exp(x); }
// (a real call everywhere: log / exp / pow / log10 inline to ~10 KB of SASS, and the NFA kernels keep thousands of
// warps at different program counters — code size is what their instruction cache sees)
__device__ __noinline__ double l_nfa(int n, int k, double p, double LOG_NT, const double* lgam) {
    if (n == 0 || k == 0) return -LOG_NT;
    if (n == k) return -LOG_NT - (double)n * l_log10(p);
    const double p_term = p / (1 - p);
    const double log1term = lgam[n] - lgam[k] - lgam[n - k] +
                            (double)k * l_log(p) + (double)(n - k) * l_log(1.0 - p);
    double term = l_exp(log1term);
    {   // double_equal(term, 0)
        bool eq = term == 0.0;
        if (!eq) { double abs_max = fabs(term); if (abs_max < 2.2250738585072014e-308) abs_max = 2.2250738585072014e-308; eq = (fabs(term) / abs_max) <= (100.0 * 2.220446049250313e-16); }
        if (eq) {
            if ((double)k > (double)n * p) return -log1term / 2.30258509299404568402 - LOG_NT;
            return -LOG_NT;
        }
    }
    double bin_tail = term;
    for (int i = k + 1; i <= n; i++) {
        const double bin_term = (double)(n - i + 1) / (double)i;
        const double mult_term = bin_term * p_term;
        term *= mult_term;
        bin_tail += term;
        if (bin_term < 1) {
            // pow(mult_term, m) < 2^-56 whenever mult_term < 1/4 and m >= 28; then 1 - pow rounds to exactly 1.0: skipping
            // the call is bit-identical (mult_term = bin_term * p / (1 - p) < 1/7 here for every p <= 1/8)
            const int m = n - i + 1;
            const double pw = (m >= 28 && mult_term < 0.25) ? 0.0 : pow(mult_term, (double)m);
            const double err = term * ((1 - pw) / (1 - mult_term) - 1);
            // threshold 0.1 * |-l_log10(bin_tail) - LOG_NT| * bin_tail: bracket log10 by the binary exponent first and
            // evaluate the logarithm only when the bracket cannot decide (same decision as the plain test, always)
            bool stop;
            const int e2 = ilogb(bin_tail);
            if (e2 > -1000 && e2 < 1000) {
                const double l_lo = -((double)(e2 + 1) * 0.30102999566398120) - LOG_NT, l_hi = -((double)e2 * 0.30102999566398120) - LOG_NT;  // L in [l_lo, l_hi]
                const double a_lo = (l_lo > 0) ? l_lo : ((l_hi < 0) ? -l_hi : 0.0), a_hi = fmax(fabs(l_lo), fabs(l_hi));
                if (err < 0.1 * a_lo * bin_tail * (1 - 1e-9)) stop = true;
                else if (err >= 0.1 * a_hi * bin_tail * (1 + 1e-9)) stop = false;
                else stop = err < 0.1 * fabs(-l_log10(bin_tail) - LOG_NT) * bin_tail;
            } else stop = err < 0.1 * fabs(-l_log10(bin_tail) - LOG_NT) * bin_tail;
            if (stop) break;
        }
    }
    return -l_log10(bin_tail) - LOG_NT;
}

__device__ __forceinline__ int l_x86_d2i(double v) {                 // cvttsd2si semantics
    if (!(v > -2147483649.0 && v < 2147483648.0)) return INT_MIN;
    return (int)v;
}

// rect_nfa of OpenCV 4.13 (see oracle/line_oracle.cpp): rows are distributed over the lanes (or, for flat
// rectangles, the pixels of a row); the two counts are exact integers, so the reduction order is irrelevant.
__device__ void l_rect_count(const Walk& W, const LRect& rec, int& total_out, int& alg_out) {
    const double half_width = 0.5 * rec.width, dyhw = rec.dy * half_width, dxhw = rec.dx * half_width;
    const double vx[4] = {rec.x1 - dyhw, rec.x2 - dyhw, rec.x2 + dyhw, rec.x1 + dyhw};
    const double vy[4] = {rec.y1 + dxhw, rec.y2 + dxhw, rec.y2 - dxhw, rec.y1 - dxhw};
    int off = 0;
#pragma unroll
    for (int i = 1; i < 4; i++) if (vy[i] < vy[off] || (vy[i] == vy[off] && vx[i] < vx[off])) off = i;
    const double Mx = vx[off], My = vy[off], Ax = vx[(off + 1) & 3], Ay = vy[(off + 1) & 3];
    const double Bx = vx[(off + 2) & 3], By = vy[(off + 2) & 3], Cx = vx[(off + 3) & 3], Cy = vy[(off + 3) & 3];
    const int cM = l_x86_d2i(ceil(My)), cA = l_x86_d2i(ceil(Ay)), cB = l_x86_d2i(ceil(By)), cC = l_x86_d2i(ceil(Cy));
    const double s1 = (cA != cM) ? (Ax - Mx) / (Ay - My) : 0.0;
    const double s2 = (cB != cA) ? (Bx - Ax) / (By - Ay) : 0.0;
    const double s3 = (cC != cM) ? (Cx - Mx) / (Cy - My) : 0.0;
    const double s4 = (cB != cC) ? (Bx - Cx) / (By - Cy) : 0.0;
    int total = 0, alg = 0;
    const int y0 = max(cM, 0), y1 = min(cB, W.h - 1);
    const bool by_rows = (y1 - y0) >= 16;
    for (int yb = y0; yb <= y1; yb += by_rows ? 32 : 1) {
        const int y = by_rows ? yb + W.lane : yb;
        if (y > y1) continue;
        const double xl = (cA < y) ? ((double)y - Ay) * s2 + Ax : ((double)y - My) * s1 + Mx;
        const double xr = (cC <= y) ? ((double)y - Cy) * s4 + Cx : ((double)y - My) * s3 + Mx;
        int xs = l_x86_d2i(ceil(xl));
        int xe = l_x86_d2i(xr);
        if (xe < xs) continue;
        if (xs < 0) xs = 0;
        if (xe > W.w - 1) xe = W.w - 1;
        const float* row = W.ang + (long long)y * W.w;
        if (by_rows) {
            for (int x = xs; x <= xe; ++x) { ++total; if (l_aligned(row[x], rec.theta, rec.prec)) ++alg; }
        } else {
            for (int x = xs + W.lane; x <= xe; x += 32) { ++total; if (l_aligned(row[x], rec.theta, rec.prec)) ++alg; }
        }
    }
    total_out = __reduce_add_sync(0xffffffffu, total);
    alg_out = __reduce_add_sync(0xffffffffu, alg);
}

__device__ double l_rect_nfa(const Walk& W, const LRect& rec) {
    int total, alg;
    l_rect_count(W, rec, total, alg);
    return l_nfa(total, alg, rec.p, W.log_nt, W.lgam);
}

// Five candidate rectangles of one rect_improve phase at once: lane group g = lane / 6 (6 lanes each, lanes 30-31 idle)
// scans candidate g's rows, the counts are combined through shared-memory atomics (exact integers), and the five
// scalar NFA evaluations run side by side in lanes 0, 6, 12, 18, 24.  s_cnt: 10 ints of this warp.
__device__ __noinline__ void l_rect_nfa5(const Walk& W, const LRect& mine, bool valid, int* s_cnt, double* out5) {
    const int lane = W.lane, grp = lane / 6, sub = lane - grp * 6;
    if (lane < 10) s_cnt[lane] = 0;
    __syncwarp();
    if (grp < 5 && valid) {
        const LRect& rec = mine;
        const double half_width = 0.5 * rec.width, dyhw = rec.dy * half_width, dxhw = rec.dx * half_width;
        const double vx[4] = {rec.x1 - dyhw, rec.x2 - dyhw, rec.x2 + dyhw, rec.x1 + dyhw};
        const double vy[4] = {rec.y1 + dxhw, rec.y2 + dxhw, rec.y2 - dxhw, rec.y1 - dxhw};
        int off = 0;
#pragma unroll
        for (int i = 1; i < 4; i++) if (vy[i] < vy[off] || (vy[i] == vy[off] && vx[i] < vx[off])) off = i;
        const double Mx = vx[off], My = vy[off], Ax = vx[(off + 1) & 3], Ay = vy[(off + 1) & 3];
        const double Bx = vx[(off + 2) & 3], By = vy[(off + 2) & 3], Cx = vx[(off + 3) & 3], Cy = vy[(off + 3) & 3];
        const int cM = l_x86_d2i(ceil(My)), cA = l_x86_d2i(ceil(Ay)), cB = l_x86_d2i(ceil(By)), cC = l_x86_d2i(ceil(Cy));
        const double s1 = (cA != cM) ? (Ax - Mx) / (Ay - My) : 0.0;
        const double s2 = (cB != cA) ? (Bx - Ax) / (By - Ay) : 0.0;
        const double s3 = (cC != cM) ? (Cx - Mx) / (Cy - My) : 0.0;
        const double s4 = (cB != cC) ? (Bx - Cx) / (By - Cy) : 0.0;
        int total = 0, alg = 0;
        const int y0 = max(cM, 0), y1 = min(cB, W.h - 1);
        for (int y = y0 + sub; y <= y1; y += 6) {
            const double xl = (cA < y) ? ((double)y - Ay) * s2 + Ax : ((double)y - My) * s1 + Mx;
            const double xr = (cC <= y) ? ((double)y - Cy) * s4 + Cx : ((double)y - My) * s3 + Mx;
            int xs = l_x86_d2i(ceil(xl));
            int xe = l_x86_d2i(xr);
            if (xe < xs) continue;
            if (xs < 0) xs = 0;
            if (xe > W.w - 1) xe = W.w - 1;
            const float* row = W.ang + (long long)y * W.w;
            for (int x = xs; x <= xe; ++x) { ++total; if (l_aligned(__ldg(row + x), rec.theta, rec.prec)) ++alg; }
        }
        if (total) atomicAdd(&s_cnt[2 * grp], total);
        if (alg) atomicAdd(&s_cnt[2 * grp + 1], alg);
    }
    __syncwarp();
    double v = 0.0;
    if (grp < 5 && sub == 0 && valid) v = l_nfa(s_cnt[2 * grp], s_cnt[2 * grp + 1], mine.p, W.log_nt, W.lgam);
#pragma unroll
    for (int g5 = 0; g5 < 5; g5++) out5[g5] = __shfl_sync(0xffffffffu, v, g5 * 6);
    __syncwarp();
}

// rect_improve (lsd.cpp): each of the five refinement phases tries a fixed sequence of five candidate rectangles that
// does not depend on the NFA values inside the phase, so the five are evaluated at once (l_rect_nfa5) and the
// reference's "first strict improvement wins" rule is then replayed in order.
__device__ double l_rect_improve(const Walk& W, LRect& rec, int* s_cnt, double log_nfa) {
    const double delta = 0.5, delta_2 = delta / 2.0;
    const int lane = W.lane, grp = lane / 6, k = min(grp, 4) + 1;     // this lane's candidate = k-th step of the phase
    if (log_nfa > 0.0) return log_nfa;           // log_nfa = NFA of the unmodified rectangle (k_lsd_nfa_first)
    double v[5];
#pragma unroll 1
    for (int phase = 0; phase < 5; phase++) {
        // candidate k of the phase, built exactly as the sequential loop would have built it
        LRect r = rec;
        bool valid = true;
        if (phase == 0 || phase == 4) {
            if (phase == 4) valid = (r.width - delta) >= 0.5;          // the guard does not change inside the loop
            for (int i = 0; i < k; i++) { r.p /= 2; r.prec = r.p * L_PI; }
        } else {
            for (int i = 0; i < k; i++) {
                if ((r.width - delta) >= 0.5) {
                    if (phase == 2) { r.x1 += -r.dy * delta_2; r.y1 += r.dx * delta_2; r.x2 += -r.dy * delta_2; r.y2 += r.dx * delta_2; }
                    if (phase == 3) { r.x1 -= -r.dy * delta_2; r.y1 -= r.dx * delta_2; r.x2 -= -r.dy * delta_2; r.y2 -= r.dx * delta_2; }
                    r.width -= delta;
                } else valid = false;                                   // this step (and all later ones) is skipped
            }
        }
        l_rect_nfa5(W, r, valid, s_cnt, v);
        // replay: for n = 1..5: if (candidate n exists && v_n > log_nfa) { log_nfa = v_n; rec = candidate n; }
        int best = -1;
        for (int n = 0; n < 5; n++) {
            const bool vn = __shfl_sync(0xffffffffu, valid ? 1 : 0, n * 6) != 0;
            if (vn && v[n] > log_nfa) { log_nfa = v[n]; best = n; }
        }
        if (best >= 0) {                                                // broadcast the winning candidate's fields
            const int src = best * 6;
            rec.x1 = __shfl_sync(0xffffffffu, r.x1, src); rec.y1 = __shfl_sync(0xffffffffu, r.y1, src);
            rec.x2 = __shfl_sync(0xffffffffu, r.x2, src); rec.y2 = __shfl_sync(0xffffffffu, r.y2, src);
            rec.width = __shfl_sync(0xffffffffu, r.width, src);
            rec.p = __shfl_sync(0xffffffffu, r.p, src); rec.prec = __shfl_sync(0xffffffffu, r.prec, src);
        }
        if (log_nfa > 0.0) return log_nfa;
    }
    return log_nfa;
}

// The order-dependent core: seeds in order, region growing, rectangle fit and the density refinement (the only steps
// that read or write the `used` map).  rect_improve / NFA of a region is a pure function of its rectangle and of the
// immutable angle map, so it is NOT done here: the walker emits one job per candidate region and k_lsd_nfa evaluates
// all jobs of all frames in parallel (one warp per job).
//
// ONE CTA PER FRAME, several warps, exact sequential semantics.  The regions of a frame form a sparse dependency graph
// (tools/sim_spec_walker.cpp: critical path 1/17 of the work at 640x480, 1/100 at 1280x960), but which regions exist and
// what they depend on is only known by running them.  So the warps run region growing AHEAD of the sequential order and
// the results are committed strictly IN that order:
//   * claim  (claim_lock, shared memory only): the next seed, in seed order, that is not in the committed bitmap gets the
//     next rank `seq` and a slot of a ring (its own list buffer);
//   * attempt (any warp, speculative): grow / fit / refine exactly as the sequential code would, reading "used" as
//     committed bitmap | my ticket | live ticket of lower rank (the last one recorded as an assumption), writing only
//     tickets (LPix.used, global) and its private lists.  A seed already under a live ticket of lower rank is presumed
//     swallowed; an attempt that loses a pixel to a live attempt of lower rank waits for that rank to retire and starts over;
//   * commit (commit_lock, in rank order, by whichever warp is idle): the attempt is VALID iff it was not poisoned, none
//     of the pixels it ever accepted is in the committed bitmap and all the pixels it assumed used are.  Then every
//     membership test it made had the sequential outcome, so its lists are the sequential ones: its final pixels are
//     published to the bitmap and its job appended.  Otherwise (and for presumed seeds that were not swallowed after all)
//     the region is grown on the spot by the "turn holder": everything of lower rank is final, nothing can invalidate it.
// Bits only go 0 -> 1 and are written only under commit_lock; tickets of retired ranks are garbage by construction.
__device__ __forceinline__ void l_unlock(int* l) { __threadfence_block(); atomicExch(l, 0); }

struct WalkFrame { const LineGeom* g; const LineWs* ws; int f; unsigned* bits; };

// grow + fit + refine one seed.  Returns 1 = candidate rectangle in *rec, 0 = no job (small or rejected by refine), -1 = abandoned.
// *n0 = size of the first region, *nfin = pixels that stay used (the list at s_W.reg).
__device__ __noinline__ int l_one_region(const LineGeom& g, unsigned idx, LRect* rec, int* n0, int* nfin) {
    WalkCtx& W = s_W;
    double reg_angle;
    int n = l_region_grow<0>((int)(idx % (unsigned)g.sw), (int)(idx / (unsigned)g.sw), g.prec, &reg_angle);
    if (n < 0) return -1;
    W.acc = n;
    *n0 = n; *nfin = n;
    if (n < g.min_reg_size) return 0;
    l_region2rect<0>(n, reg_angle, g.prec, g.p, rec);
    const bool okr = l_refine<0>(&n, &reg_angle, g.prec, g.p, rec, 0.7);
    if (W.abort) return -1;
    *nfin = n;
    return okr ? 1 : 0;
}

__device__ __forceinline__ void l_emit_job(const LineGeom& g, double* dst, const LRect& rec, unsigned idx, int n0, int lane) {
    if (lane < 13) {
        const double v[13] = {rec.x1, rec.y1, rec.x2, rec.y2, rec.width, rec.x, rec.y, rec.theta, rec.dx, rec.dy, rec.prec, rec.p, (double)idx * 65536.0 + (double)min(n0, 65535)};
        double out = v[0];
#pragma unroll
        for (int k = 1; k < 13; k++) if (lane == k) out = v[k];
        dst[lane] = out;
    }
}

__device__ __forceinline__ void l_set_bit(unsigned* bits, unsigned pk, int w) { const int q = (int)(pk >> 16) * w + (int)(pk & 0xffff); atomicOr(bits + (q >> 5), 1u << (q & 31)); }

// The turn holder grows the region of seed `idx` for real (commit_lock held, every lower rank committed).
__device__ __noinline__ void l_turn_region(const WalkFrame& F, unsigned idx, int seq) {
    const LineGeom& g = *F.g; const LineWs& ws = *F.ws;
    const int lane = threadIdx.x & 31;
    const long long t0 = clock64();
    WalkCtx& W = s_W;
    __syncwarp();
    if (lane == 0) {
        W.mode = 1; W.abort = 0; W.seq = seq; W.ticket = (unsigned)(seq + 1) | 0x80000000u;
        W.reg = ws.reg + (long long)F.f * g.pix_stride; W.base0 = W.reg; W.cap = (int)g.pix_stride; W.nasm = 0; W.acc = 0;
    }
    __syncwarp();
    LRect rec; int n0 = 0, nfin = 0;
    const int r = l_one_region(g, idx, &rec, &n0, &nfin);
    __syncwarp();
    for (int i = lane; i < nfin; i += 32) l_set_bit(F.bits, W.reg[i], g.sw);
    if (r == 1) {
        const int nj = s_F.nj;
        if (nj < g.seg_cap) l_emit_job(g, ws.jobs + ((long long)F.f * g.seg_cap + nj) * 13, rec, idx, n0, lane);
        __syncwarp();
        if (lane == 0) s_F.nj = nj + 1;
    }
    __syncwarp();
    if (lane == 0 && (g.dbg & 32)) { atomicAdd(ws.wstat + 0, 1ull); atomicAdd(ws.wstat + 1, (unsigned long long)(clock64() - t0)); atomicAdd(ws.wstat + 2, (unsigned long long)nfin); }
}

// commit slot `k` (rank `seq`); commit_lock held
__device__ __noinline__ void l_commit_slot(const WalkFrame& F, int k, int seq) {
    const LineGeom& g = *F.g; const LineWs& ws = *F.ws;
    const int lane = threadIdx.x & 31;
    const int st = s_F.state[k];
    if (s_F.seedpix[k] < 0) return;                               // the sentinel claim that closes the frame
    const unsigned idx = (unsigned)s_F.seedpix[k];
    if (l_bit(F.bits, (int)idx)) { if (lane == 0 && (g.dbg & 32)) atomicAdd(ws.wstat + 4, 1ull); return; }     // swallowed by a region of lower rank: nothing to do
    bool ok = st == SLOT_DONE && !s_F.poison[k];
    const int acc = s_F.acc[k], nasm = s_F.nasm[k], finoff = s_F.finoff[k], nfin = s_F.nfin[k];
    const bool small = finoff == 0 && acc + nasm <= WALK_SMALL && !(g.dbg & 2);    // everything needed is in shared memory
    const unsigned* list = ws.sreg + ((long long)F.f * WALK_RING + k) * WALK_SLOT_CAP;
    if (ok) {
        bool bad = false;
        if (small) {
            if (lane < acc) { const unsigned pk = s_F.small[k][lane]; bad = l_bit(F.bits, (int)(pk >> 16) * g.sw + (int)(pk & 0xffff)); }
            else if (lane < acc + nasm) bad = !l_bit(F.bits, (int)s_F.small[k][lane]);
        } else {
            for (int i = lane; i < acc; i += 32) { const unsigned pk = __ldcg(list + i); bad |= l_bit(F.bits, (int)(pk >> 16) * g.sw + (int)(pk & 0xffff)); }
            for (int i = lane; i < nasm; i += 32) bad |= !l_bit(F.bits, (int)__ldcg(list + WALK_SLOT_CAP - 1 - i));
        }
        ok = !__any_sync(0xffffffffu, bad);
    }
    if (!ok) {
        if (lane == 0 && (g.dbg & 32)) atomicAdd(ws.wstat + 5 + (st == SLOT_PRESUMED ? 3 : (st != SLOT_DONE ? 0 : (s_F.poison[k] ? 1 : 2))), 1ull);
        l_turn_region(F, idx, seq);
        return;
    }
    if (lane == 0 && (g.dbg & 32)) { atomicAdd(ws.wstat + 9, 1ull); atomicAdd(ws.wstat + 10, (unsigned long long)nfin); }
    if (small) { if (lane < nfin) l_set_bit(F.bits, s_F.small[k][lane], g.sw); }
    else for (int i = lane; i < nfin; i += 32) l_set_bit(F.bits, __ldcg(list + finoff + i), g.sw);
    if (s_F.job[k]) {
        const int nj = s_F.nj;
        if (nj < g.seg_cap && lane < 13) ws.jobs[((long long)F.f * g.seg_cap + nj) * 13 + lane] = s_F.jobv[k][lane];
        __syncwarp();
        if (lane == 0) s_F.nj = nj + 1;
    }
    __syncwarp();
}

// claim the next seed (claim_lock held by this warp): returns the slot, -1 when the ring is full, -2 for the closing sentinel
__device__ __noinline__ int l_claim(const WalkFrame& F) {
    const LineGeom& g = *F.g; const LineWs& ws = *F.ws;
    const int lane = threadIdx.x & 31;
    const unsigned* seeds = ws.seeds + (long long)F.f * g.pix_stride;
    const int ns = s_F.ns;
    const unsigned nclaims = s_F.nclaims;
    if (s_F.all_claimed || nclaims - l_turn() >= (unsigned)WALK_RING) return -1;
    const int k = (int)(nclaims % WALK_RING);
    if (*reinterpret_cast<volatile int*>(&s_F.state[k]) != SLOT_EMPTY) return -1;
    int cur = (int)s_F.cursor, found = ns;
    unsigned pixidx = 0;
    while (cur < ns) {
        int wb = s_F.win_base;
        if (cur < wb || cur >= wb + WALK_WIN) {                    // stage the next window of the ordered seed list
            wb = cur & ~31;
            for (int i = lane; i < WALK_WIN; i += 32) s_F.win[i] = wb + i < ns ? seeds[wb + i] : 0u;
            if (lane == 0) s_F.win_base = wb;
            __syncwarp();
        }
        const int i = cur + lane;
        const bool have = i < ns && i < wb + WALK_WIN;
        const unsigned mine = have ? s_F.win[i - wb] : 0u;
        const unsigned fm = __ballot_sync(0xffffffffu, have && !l_bit(F.bits, (int)mine));
        if (fm) { const int j = __ffs(fm) - 1; found = cur + j; pixidx = __shfl_sync(0xffffffffu, mine, j); break; }
        cur = min(cur + 32, wb + WALK_WIN);
    }
    if (lane == 0) {
        s_F.seqof[k] = (int)nclaims; s_F.seedpix[k] = found >= ns ? -1 : (int)pixidx; s_F.poison[k] = 0; s_F.job[k] = 0;
        *reinterpret_cast<volatile int*>(&s_F.state[k]) = found >= ns ? SLOT_ABORTED : SLOT_RUNNING;     // the sentinel has nothing to grow
        s_F.cursor = (unsigned)min(found + 1, ns);
        if (found >= ns) s_F.all_claimed = 1;
        __threadfence_block();
        s_F.nclaims = nclaims + 1;
    }
    __syncwarp();
    return found >= ns ? -2 : k;
}

// 128 registers: a build held to 80 (three 8-warp CTAs per SM) spills
__global__ void __launch_bounds__(WALK_MAXW * 32) k_lsd_regions(const __grid_constant__ LineGeom g, LineWs ws, int nframes) {
    extern __shared__ unsigned s_bits[];                       // committed `used` bitmap of the frame
    const int lane = threadIdx.x & 31;
    const int nwords = (int)((g.pix_stride + 31) >> 5);
  for (;;) {
    // frames are pulled from a counter: the grid may be smaller than the batch (sslpl_line_set_max_walkers)
    __syncthreads();
    if (threadIdx.x == 0) {
        const int f = atomicAdd(ws.rejctl + 2, 1);
        s_F.frame = f; s_F.cursor = 0; s_F.nclaims = 0; s_F.turn = 0; s_F.claim_lock = 0; s_F.commit_lock = 0; s_F.all_claimed = 0; s_F.nj = 0; s_F.win_base = -(1 << 30);
        s_F.ns = f < nframes ? ws.nseeds[f] : 0;
        for (int k = 0; k < WALK_RING; k++) { s_F.state[k] = SLOT_EMPTY; s_F.poison[k] = 0; }
    }
    for (int i = threadIdx.x; i < nwords; i += blockDim.x) s_bits[i] = 0u;
    __syncthreads();
    const int f = s_F.frame;
    if (f >= nframes) break;
    const long long tf0 = clock64();
    WalkFrame F; F.g = &g; F.ws = &ws; F.f = f; F.bits = s_bits;
    WalkCtx& W = s_W;
    if (lane == 0) {
        W.w = g.sw; W.h = g.sh;
        W.ang = ws.angdeg + f * g.pix_stride; W.mod = ws.modgrad + f * g.pix_stride;
        W.pix = ws.pix + f * g.pix_stride; W.cs0 = ws.cs0 + f * g.pix_stride; W.bits = s_bits; W.dbg = g.dbg;
    }
    __syncwarp();
    int myslot = -1, tries = 0, waitfor = -1;                  // an attempt of this warp waiting for rank `waitfor` to retire
    for (;;) {
        // ---- 1. commits, by whoever finds the head of the ring finished
        int did = 0;
        {
            int go = 0;
            if (lane == 0) {
                const unsigned t = l_turn();
                if (t < *reinterpret_cast<volatile unsigned*>(&s_F.nclaims)) {
                    const int st = *reinterpret_cast<volatile int*>(&s_F.state[t % WALK_RING]);
                    if (st >= SLOT_DONE && atomicCAS(&s_F.commit_lock, 0, 1) == 0) { __threadfence_block(); go = 1; }
                }
            }
            go = __shfl_sync(0xffffffffu, go, 0);
            if (go) {
                const long long tc0 = clock64();
                for (;;) {
                    const unsigned t = l_turn();
                    if (t >= *reinterpret_cast<volatile unsigned*>(&s_F.nclaims)) break;
                    const int k = (int)(t % WALK_RING);
                    if (*reinterpret_cast<volatile int*>(&s_F.state[k]) < SLOT_DONE) break;
                    __syncwarp();
                    l_commit_slot(F, k, (int)t);
                    __syncwarp();
                    if (lane == 0) { __threadfence_block(); *reinterpret_cast<volatile int*>(&s_F.state[k]) = SLOT_EMPTY; __threadfence_block(); *reinterpret_cast<volatile unsigned*>(&s_F.turn) = t + 1; }
                    __syncwarp();
                    did = 1;
                }
                if (lane == 0) { if (g.dbg & 32) atomicAdd(ws.wstat + 11, (unsigned long long)(clock64() - tc0)); l_unlock(&s_F.commit_lock); }
                __syncwarp();
            }
        }
        if (did) continue;
        // ---- 2. an attempt: a new claim, or the repetition of one that had to wait for a lower rank
        if (myslot < 0) {
            int go = 0;
            if (lane == 0 && !*reinterpret_cast<volatile int*>(&s_F.all_claimed) &&
                *reinterpret_cast<volatile unsigned*>(&s_F.nclaims) - l_turn() < (unsigned)WALK_RING && atomicCAS(&s_F.claim_lock, 0, 1) == 0) { __threadfence_block(); go = 1; }
            go = __shfl_sync(0xffffffffu, go, 0);
            if (go) {
                const long long tk0 = clock64();
                const int k = l_claim(F);
                if (lane == 0) { if (g.dbg & 32) atomicAdd(ws.wstat + 12, (unsigned long long)(clock64() - tk0)); l_unlock(&s_F.claim_lock); }
                __syncwarp();
                if (k >= 0) { myslot = k; tries = 0; waitfor = -1; }
            }
        }
        if (myslot >= 0 && (waitfor < 0 || (int)l_turn() > waitfor)) {
            const int k = myslot;
            const unsigned idx = (unsigned)s_F.seedpix[k];
            if (lane == 0) {
                W.mode = 0; W.abort = 0; W.conflict = -1; W.nasm = 0; W.acc = 0; W.seq = s_F.seqof[k];
                W.ticket = (unsigned)(W.seq + 1) | ((unsigned)(tries & 127) << 24);
                W.reg = ws.sreg + ((long long)f * WALK_RING + k) * WALK_SLOT_CAP; W.base0 = W.reg; W.cap = WALK_SLOT_CAP;
            }
            __syncwarp();
            LRect rec; int n0 = 0, nfin = 0;
            int r = -1;
            if (l_bit(s_bits, (int)idx)) { if (lane == 0) W.abort = 3; __syncwarp(); }     // swallowed while this attempt waited
            else r = l_one_region(g, idx, &rec, &n0, &nfin);
            __syncwarp();
            if (r < 0 && W.abort == 2 && tries < 100 && !(g.dbg & 1)) {           // a live attempt of lower rank holds a pixel this one needs: repeat after it retires
                waitfor = W.conflict; tries++;
                if (lane == 0 && (g.dbg & 32)) atomicAdd(ws.wstat + 13, 1ull);
                __syncwarp();
                continue;
            }
            if (r == 1) l_emit_job(g, s_F.jobv[k], rec, idx, n0, lane);
            int st = SLOT_DONE;
            if (r < 0) st = W.abort == 3 ? SLOT_PRESUMED : SLOT_ABORTED;
            else {
                const int acc = W.acc, nasm = W.nasm, finoff = (int)(W.reg - W.base0);
                if (finoff == 0 && acc + nasm <= WALK_SMALL && !(g.dbg & 2)) {   // small attempt: its lists travel through shared memory
                    if (lane < acc) s_F.small[k][lane] = W.base0[lane];
                    else if (lane < acc + nasm) s_F.small[k][lane] = W.base0[WALK_SLOT_CAP - 1 - (lane - acc)];
                }
                if (lane == 0) { s_F.acc[k] = acc; s_F.nasm[k] = nasm; s_F.finoff[k] = finoff; s_F.nfin[k] = nfin; s_F.job[k] = r == 1; }
            }
            __syncwarp();
            if (lane == 0) { __threadfence(); *reinterpret_cast<volatile int*>(&s_F.state[k]) = st; }
            __syncwarp();
            myslot = -1;
            continue;
        }
        // ---- 3. done?
        if (myslot < 0 && *reinterpret_cast<volatile int*>(&s_F.all_claimed) && l_turn() >= *reinterpret_cast<volatile unsigned*>(&s_F.nclaims)) break;
        __nanosleep(100);
    }
    __syncthreads();
    if (threadIdx.x == 0) { if (g.dbg & 32) { atomicAdd(ws.wstat + 14, (unsigned long long)(clock64() - tf0)); atomicAdd(ws.wstat + 15, (unsigned long long)s_F.nclaims); }
        ws.njobs[f] = min(s_F.nj, g.seg_cap); if (s_F.nj > g.seg_cap) atomicOr(ws.err, DERR_LSD_OVERFLOW); }
  }
}

// THROUGHPUT form of the same stage for big batches: ONE WARP PER FRAME, no speculation (every instruction is useful work, 72
// registers, ~28 frames resident per SM; latency-bound per frame, amortised when thousands of frames are in flight).
// sslpl picks it when a call brings at least two frames per SM; smaller calls use the multi-warp walker above.
#ifndef SSLPL_SOLO_MINB
#define SSLPL_SOLO_MINB 28
#endif
__global__ void __launch_bounds__(32, SSLPL_SOLO_MINB) k_lsd_regions_solo(const __grid_constant__ LineGeom g, LineWs ws, int nframes) {
    const int lane = threadIdx.x;
  for (;;) {
    int f = 0;
    if (lane == 0) f = atomicAdd(ws.rejctl + 2, 1);
    f = __shfl_sync(0xffffffffu, f, 0);
    if (f >= nframes) break;
    __syncwarp();
    WalkCtx& W = s_W1;
    if (lane == 0) {
        W.w = g.sw; W.h = g.sh; W.mode = 2; W.abort = 0; W.nasm = 0; W.acc = 0; W.cap = (int)g.pix_stride; W.ticket = 1u; W.seq = 0;
        W.ang = ws.angdeg + f * g.pix_stride; W.mod = ws.modgrad + f * g.pix_stride;
        W.pix = ws.pix + f * g.pix_stride; W.reg = ws.reg + f * g.pix_stride; W.base0 = W.reg; W.cs0 = ws.cs0 + f * g.pix_stride; W.bits = nullptr;
    }
    __syncwarp();
    const LPix* pix = ws.pix + f * g.pix_stride;
    const unsigned* seeds = ws.seeds + f * g.pix_stride;
    const int ns = ws.nseeds[f];
    double* jobs = ws.jobs + (long long)f * g.seg_cap * 13;
    int nj = 0;
    for (int sb = 0; sb < ns; sb += 32) {
        const bool have = sb + lane < ns;
        const unsigned mine = have ? seeds[sb + lane] : 0u;                   // 32 seeds per coalesced load
        unsigned umask = __ballot_sync(0xffffffffu, !have || pix[mine].used != 0u); // their `used` state, one round trip
        while (~umask) {                                    // angle != NOTDEF holds for every seed
            const int j = __ffs(~umask) - 1;
            umask |= (2u << j) - 1u;                        // seeds up to j are done
            const unsigned idx = __shfl_sync(0xffffffffu, mine, j);
            double reg_angle;
            int n = l_region_grow<1>((int)(idx % (unsigned)g.sw), (int)(idx / (unsigned)g.sw), g.prec, &reg_angle);
            umask |= __ballot_sync(0xffffffffu, !have || pix[mine].used != 0u);    // the region may have swallowed later seeds
            if (n < g.min_reg_size) continue;
            LRect rec;
            l_region2rect<1>(n, reg_angle, g.prec, g.p, &rec);
            const int n0 = n;
            const bool okr = l_refine<1>(&n, &reg_angle, g.prec, g.p, &rec, 0.7);
            umask = ((2u << j) - 1u) | __ballot_sync(0xffffffffu, !have || pix[mine].used != 0u);   // refine can release and re-take pixels
            if (!okr) continue;
            if (nj < g.seg_cap) l_emit_job(g, jobs + (long long)nj * 13, rec, idx, n0, lane);
            nj++;
        }
    }
    if (lane == 0) { ws.njobs[f] = min(nj, g.seg_cap); if (nj > g.seg_cap) atomicOr(ws.err, DERR_LSD_OVERFLOW); }
    __syncwarp();
  }
}

// The same loop over the frame's seeds with the LEAN region growing (l_region_grow_lean).  It is not faster than
// k_lsd_regions_solo: it executes slightly MORE warp instructions (the lazy-angle bookkeeping costs what the removed FP64 saved), and a
// lone warp's time is its instruction count times the dependent-issue latency.  Kept for A/B runs (SSLPL_WALKER_LEAN=1) and as the base of the v3 and lane-parallel growth.
__global__ void __launch_bounds__(32, 28) k_lsd_regions_lean(const __grid_constant__ LineGeom g, LineWs ws, int nframes) {
    const int lane = threadIdx.x;
  for (;;) {
    int f = 0;
    if (lane == 0) f = atomicAdd(ws.rejctl + 2, 1);
    f = __shfl_sync(0xffffffffu, f, 0);
    if (f >= nframes) break;
    __syncwarp();
    WalkCtx& W = s_W1;
    if (lane == 0) {
        W.w = g.sw; W.h = g.sh; W.mode = 2; W.abort = 0; W.nasm = 0; W.acc = 0; W.cap = (int)g.pix_stride; W.ticket = 1u; W.seq = 0;
        W.ang = ws.angdeg + f * g.pix_stride; W.mod = ws.modgrad + f * g.pix_stride;
        W.pix = ws.pix + f * g.pix_stride; W.reg = ws.reg + f * g.pix_stride; W.base0 = W.reg; W.cs0 = ws.cs0 + f * g.pix_stride; W.bits = nullptr;
    }
    __syncwarp();
    const LPix* pix = ws.pix + f * g.pix_stride;
    const unsigned* seeds = ws.seeds + f * g.pix_stride;
    const int ns = ws.nseeds[f];
    double* jobs = ws.jobs + (long long)f * g.seg_cap * 13;
    int nj = 0;
    for (int sb = 0; sb < ns; sb += 32) {
        const bool have = sb + lane < ns;
        const unsigned mine = have ? seeds[sb + lane] : 0u;                   // 32 seeds per coalesced load
        unsigned umask = __ballot_sync(0xffffffffu, !have || pix[mine].used != 0u); // their `used` state, one round trip
        while (~umask) {                                    // angle != NOTDEF holds for every seed
            const int j = __ffs(~umask) - 1;
            umask |= (2u << j) - 1u;                        // seeds up to j are done
            const unsigned idx = __shfl_sync(0xffffffffu, mine, j);
            double reg_angle;
            int n = l_region_grow_lean((int)(idx % (unsigned)g.sw), (int)(idx / (unsigned)g.sw), g.prec, &reg_angle);
#ifdef SSLPL_V3_DEBUG
            if ((int)idx == g.dbg_seed) { __syncwarp(); for (int i = lane; i < n; i += 32) printf("L1 %d %u %u\n", i, W.reg[i] & 0xffff, W.reg[i] >> 16); __syncwarp(); }
#endif
            umask |= __ballot_sync(0xffffffffu, !have || pix[mine].used != 0u);    // the region may have swallowed later seeds
            if (n < g.min_reg_size) continue;
            LRect rec;
            l_region2rect<2>(n, reg_angle, g.prec, g.p, &rec);
            const int n0 = n;
            const bool okr = l_refine<2>(&n, &reg_angle, g.prec, g.p, &rec, 0.7);
            umask = ((2u << j) - 1u) | __ballot_sync(0xffffffffu, !have || pix[mine].used != 0u);   // refine can release and re-take pixels
            if (!okr) continue;
            if (nj < g.seg_cap) l_emit_job(g, jobs + (long long)nj * 13, rec, idx, n0, lane);
            nj++;
        }
    }
    if (lane == 0) { ws.njobs[f] = min(nj, g.seg_cap); if (nj > g.seg_cap) atomicOr(ws.err, DERR_LSD_OVERFLOW); }
    __syncwarp();
  }
}


// =================================================================================================
// Multi-warp region walker, v3 (round 2b).  Same idea as k_lsd_regions — regions are grown AHEAD of the sequential order
// by several warps and retired strictly IN that order — with the two costs that dominated it removed (much of a frame's
// cycles under the commit lock, every invalid attempt regrown under that lock while 15 warps wait):
//   * RETIRING AN ATTEMPT IS O(1).  "Used" is not a bitmap that a commit has to fill but a property of the ticket found in
//     LPix.used: a ticket (rank, try) of a retired rank is USED iff that try is the one the rank committed with.  That
//     is try 0 unless the rank's bit is set in a 64k-bit exception map in shared memory (then one byte per rank in global
//     memory says which try, if any).  So a commit writes one byte, maybe one bit, advances `turn`; there are no lists to
//     validate, no bits to set, no list storage per slot (the lists belong to the worker and die with the attempt);
//   * validity is tracked where it is decided: an attempt that takes a pixel from a live attempt of higher rank POISONS it;
//     an attempt that meets a pixel held by a live attempt of LOWER rank assumes it used and records that attempt as a
//     dependency (two at most), valid iff it commits with that very try without ever having released a pixel;
//   * warp 0 is the CONTROL warp (claims seeds in order into a ring of 256 tiny slots (more ranks in flight only add wasted speculation), retires the head); the others are
//     workers that pick the lowest runnable slot.  No locks.  An invalid attempt goes back to the ring with try + 1; the
//     head of the ring can neither meet a live lower rank nor be poisoned, so its attempt always commits.
// Region growing is the lean form (float-degree test, lazy angle, list tail in shared memory) with tickets taken by CAS whose
// result is looked at one step later.
// =================================================================================================
constexpr int V3_MAXW = 16;            // warps per CTA: 1 control + up to 15 workers
#ifndef SSLPL_V3_RING
#define SSLPL_V3_RING 256
#endif
constexpr int V3_RING = SSLPL_V3_RING; // ranks in flight (claimed, not retired)
constexpr int V3_LIST = 8192;          // list entries of a worker (ws.sreg); bigger regions are regrown as head with the frame-sized list
constexpr int V3_LRING = 512;          // tail of the worker's list kept in shared memory
constexpr int V3_RANKS = 65536;        // ranks per frame (exception bits, rcode bytes)
constexpr int V3_DPOOL = 131072;       // per frame: list entries of the attempts that released pixels, kept until they retire
static_assert(V3_MAXW * V3_LIST <= WALK_RING * WALK_SLOT_CAP, "the workers' lists live in ws.sreg");
enum { V3_EMPTY = 0, V3_READY = 1, V3_RUNNING = 2, V3_DONE = 3, V3_PRESUMED = 4, V3_VOID = 5 };
enum { V3F_JOB = 1, V3F_DIRTY = 2, V3F_RAN = 4 };      // slot flags; bits 4..5 = number of dependencies

struct V3Shared {
    volatile unsigned turn, nclaims;     // ranks [turn, nclaims) are live; slot of rank r = r % V3_RING
    unsigned cursor;
    int ns, nj, all_claimed, frame, done, nready, scanhint, win_base, overflow;
    unsigned win[WALK_WIN];
    int state[V3_RING];
    int seed[V3_RING];
    int wait[V3_RING];                   // READY: runnable once turn > wait
    int dl_off[V3_RING], dl_n[V3_RING];  // DONE, dirty: where the pixels it ever accepted are kept until it retires (ws.dlist)
    int dl_used;
    int nblocked;                        // READY slots that wait for an attempt of lower rank (they do not count against the claim throttle)
    unsigned dep[V3_RING][2];
    unsigned char tryno[V3_RING], poison[V3_RING], flag[V3_RING];
    unsigned excbits[V3_RANKS / 32];     // rank retired with something else than "try 0 committed" although a try ran
    unsigned lring[1];                   // [warps][V3_LRING] follows
};
extern __shared__ __align__(16) unsigned char s_v3raw[];
__device__ __forceinline__ V3Shared& v3s() { return *reinterpret_cast<V3Shared*>(s_v3raw); }

__device__ __forceinline__ int v3_rank(unsigned m) { return (int)(m & 0xffffffu) - 1; }
__device__ __forceinline__ int v3_try(unsigned m) { return (int)((m >> 24) & 0x7fu); }
// What is a foreign, non-zero ticket to the attempt of rank `myseq`?  0 free (stale), 1 used (committed), 2 held by a live attempt
// of lower rank, 3 held by a live attempt of higher rank.
__device__ __forceinline__ int v3_classify(unsigned m, int myseq, const unsigned char* __restrict__ rcode) {
    V3Shared& S = v3s();
    if (m & 0x80000000u) return 0;                                // released by its attempt
    const int r = v3_rank(m), y = v3_try(m);
    if (r >= (int)S.turn) {
        const int yy = *reinterpret_cast<volatile unsigned char*>(&S.tryno[r & (V3_RING - 1)]);
        if (r >= (int)S.turn) {                                   // still live: the slot was rank r's when it was read
            if (yy != y) return 0;                                // an earlier, abandoned try of a live rank
            return r < myseq ? 2 : 3;
        }
    }
    if (!((reinterpret_cast<volatile unsigned*>(S.excbits)[r >> 5] >> (r & 31)) & 1u)) return y == 0 ? 1 : 0;
    const unsigned code = __ldcg(rcode + r);
    return (code != 0xffu && (int)(code & 0x7fu) == y) ? 1 : 0;
}
__device__ __forceinline__ void v3_poison(unsigned m) {
    V3Shared& S = v3s();
    const int r = v3_rank(m);
    if (r >= (int)S.turn) *reinterpret_cast<volatile unsigned char*>(&S.poison[r & (V3_RING - 1)]) = (unsigned char)(v3_try(m) + 1);
}
// Result of the atomic issued one step earlier: -1 the pixel is mine, >= 0 the live attempt of lower rank that holds it (repeat after
// it has retired), -2 lost to anybody else (repeat at once).
__device__ __forceinline__ int v3_take_resolve(const WalkCtx& W, LTake& t, const unsigned char* rcode) {
    if (!t.pend) return -1;
    t.pend = false;
    const unsigned old = t.old;
#ifdef SSLPL_V3_DEBUG
    if ((W.dbg & 16) && t.q == W.nasm) printf("RES T %x seen %x old %x mode %d turn %u\n", W.ticket, t.seen, old, W.mode, v3s().turn);
#endif
    if (W.mode != 0 || old == t.seen) {
        // mine now.  Whoever held it alive, or had held and released it, with a higher rank grew over a pixel that is mine: poisoned
        const unsigned o = old & 0x7fffffffu;
        if (o != 0u && o != W.ticket && v3_classify(o, W.seq, rcode) == 3) v3_poison(o);
        return -1;
    }
    if (old != 0u && v3_classify(old, W.seq, rcode) == 2) return v3_rank(old);
    return -2;
}

__device__ __noinline__ int l_region_grow_v3(int sx, int sy, double prec, double* reg_angle_out) {
    WalkCtx& W = s_Wc[threadIdx.x >> 5];
    V3Shared& S = v3s();
    unsigned* ring = S.lring + (threadIdx.x >> 5) * V3_LRING;
    const int lane = threadIdx.x & 31, w = W.w, h = W.h;
    LPix* pix = W.pix; unsigned* reg = W.reg;
    const unsigned char* rcode = reinterpret_cast<const unsigned char*>(W.bits);      // per-rank commit codes of this frame (global)
    const unsigned T = W.ticket; const int myseq = W.seq; const bool spec = W.mode == 0;
    const int cap = W.cap;
    const int sq = sy * w + sx;
    LTake tk; tk.pend = false; tk.q = 0; tk.seen = 0u; tk.old = 0u;
    int failrank = -1;
    {
        int fail = 0;
        if (lane == 0) {
            const unsigned pk0 = (unsigned)sx | ((unsigned)sy << 16);
            reg[0] = pk0; ring[0] = pk0;
            const unsigned m0 = __ldcg(&pix[sq].used);
            if (m0 != T) {
                const int c = m0 == 0u ? 0 : v3_classify(m0, myseq, rcode);
                if (c == 1) fail = 4;                                          // committed meanwhile: nothing to grow
                else if (c == 2) { fail = 3; W.conflict = (int)m0; }           // under a live attempt of lower rank: presumed swallowed
                else {
                    l_take_issue(W, tk, sq, m0);
                    const int r = v3_take_resolve(W, tk, rcode);
                    if (r != -1) { fail = 2; W.conflict = r >= 0 ? r : -1; }
                }
            }
        }
        fail = __shfl_sync(0xffffffffu, fail, 0);
        if (fail) { if (lane == 0) W.abort = fail; __syncwarp(); return -1; }
    }
    float th = __ldg(W.ang + sq);
    const float2 c0 = __ldg(W.cs0 + sq);
    float sumdx = c0.x, sumdy = c0.y;
    float rM = rsqrtf(sumdx * sumdx + sumdy * sumdy);
    bool dirty = false;
    int n = 1;
    const float pdeg = (float)(prec * (180.0 / L_PI));
    const float coef = (float)(57.2958 * 1.0002 * sin(prec + 0.0006));
    const bool rob_ok = prec < 0.78;
    const int slot = lane >> 3, nb = (lane & 7) + ((lane & 7) >= 4 ? 1 : 0);
    const int ox = nb % 3 - 1, oy = nb / 3 - 1;
    const unsigned lt = (1u << lane) - 1u;
    __syncwarp();
    for (int i = 0; i < n;) {
        const int cnt = min(4, n - i);
        unsigned pk = 0;
        { const int j = i + slot; if (slot < cnt) pk = (n - j <= V3_LRING) ? ring[j & (V3_LRING - 1)] : reg[j]; }
        const int xx = (int)(pk & 0xffff) + ox, yy = (int)(pk >> 16) + oy, q = yy * w + xx;
        const bool valid = slot < cnt && (unsigned)xx < (unsigned)w && (unsigned)yy < (unsigned)h;
        uint4 v = make_uint4(__float_as_uint(NOTDEF_F), 0u, 0u, 0u);
        if (valid) v = __ldcg(reinterpret_cast<const uint4*>(pix + q));          // record + ticket (tickets change under atomics: L2)
        const unsigned peers = __match_any_sync(0xffffffffu, valid ? q : ~lane);
        { const int r = v3_take_resolve(W, tk, rcode); if (r != -1) failrank = (r >= 0 && r > failrank) ? r : (failrank >= 0 ? failrank : r); }
        if (dirty) { th = fast_atan2_deg(sumdy, sumdx); rM = rsqrtf(sumdx * sumdx + sumdy * sumdy); dirty = false; }
        const float a = __uint_as_float(v.x), cx = __uint_as_float(v.y), cy = __uint_as_float(v.z);
        const unsigned m = v.w;
        bool cand = false, lower = false;
        if (valid && a != NOTDEF_F && m != T) {
            if (m == 0u) cand = true;
            else { const int c = v3_classify(m, myseq, rcode); cand = c == 0 || c == 3; lower = c == 2; }
        }
#ifdef SSLPL_V3_DEBUG
        if ((W.dbg & 16) && valid && q == W.nasm) printf("SEE T %x m %x cand %d lower %d turn %u\n", T, m, (int)cand, (int)lower, S.turn);
#endif
        for (unsigned lm = __ballot_sync(0xffffffffu, lower); lm;) {              // remember whose pixels were assumed used
            const unsigned t = __shfl_sync(0xffffffffu, m, __ffs(lm) - 1);
            if (lane == 0) {
                const int nd = W.ndeps;
                if (!((nd > 0 && W.dep[0] == t) || (nd > 1 && W.dep[1] == t))) { if (nd < 2) { W.dep[nd] = t; W.ndeps = nd + 1; } else W.abort = 5; }
            }
            lm &= ~__ballot_sync(0xffffffffu, lower && m == t);
        }
        unsigned pending = __ballot_sync(0xffffffffu, cand);
        while (pending) {
            const bool mep = (pending >> lane) & 1u;
            const float d = fabsf(th - a);
            const float e = d > 270.f ? 360.f - d : d;
            bool pass = e <= pdeg;
            const bool near = fabsf(e - pdeg) < 2e-3f || fabsf(d - 270.f) < 2e-3f;
            if (__any_sync(0xffffffffu, mep && near)) { if (near) pass = l_aligned_rad((double)a * L_DEG, (double)th * L_DEG, prec); }
            const unsigned P = __ballot_sync(0xffffffffu, mep && pass);
            if (!P) break;
            const int k0 = __ffs(P) - 1;
            const unsigned P1 = P & ~__ballot_sync(0xffffffffu, pass && mep && (peers & P & lt) != 0u);
            const float x = (float)__popc(P1 & lt) * rM;
            bool robust = false;
            if (rob_ok && x <= 0.5f) { const float B = coef * x + 0.0215f; robust = pass ? (e <= pdeg - B) : (e >= pdeg + B); }
            const unsigned NR = __ballot_sync(0xffffffffu, mep && lane > k0 && !robust);
            const unsigned below = NR ? ((NR & (0u - NR)) - 1u) : 0xffffffffu;
            const unsigned A = P1 & below;
            if (n + __popc(A) > cap) { if (lane == 0) W.abort = 1; __syncwarp(); return -1; }
            for (unsigned Tm = A; Tm; Tm &= Tm - 1u) {
                const int mm = __ffs(Tm) - 1;
                sumdx += __shfl_sync(0xffffffffu, cx, mm); sumdy += __shfl_sync(0xffffffffu, cy, mm);
            }
            if ((A >> lane) & 1u) {
                const int pos = n + __popc(A & lt);
                const unsigned me = (unsigned)xx | ((unsigned)yy << 16);
                ring[pos & (V3_LRING - 1)] = me; reg[pos] = me;
#ifdef SSLPL_V3_DEBUG
                if ((W.dbg & 16) && q == W.nasm) printf("TAKE T %x q (%d,%d) seen %x mode %d pos %d turn %u\n", T, xx, yy, m, W.mode, pos, S.turn);
#endif
                l_take_issue(W, tk, q, m);
            }
            n += __popc(A);
            pending &= ~below;
            pending &= ~__ballot_sync(0xffffffffu, mep && (peers & A) != 0u);
            dirty = true;
            if (pending) { th = fast_atan2_deg(sumdy, sumdx); rM = rsqrtf(sumdx * sumdx + sumdy * sumdy); dirty = false; }
        }
        __syncwarp();
        if (spec && (__any_sync(0xffffffffu, failrank != -1) || W.abort)) break;    // lost a pixel / too many dependencies: stop now
        if (spec && !(W.dbg & 64) && *reinterpret_cast<volatile unsigned char*>(&S.poison[myseq & (V3_RING - 1)]) == (unsigned char)((T >> 24) + 1u)) { if (lane == 0) { W.abort = 2; W.conflict = -1; } __syncwarp(); return -1; }   // a lower rank took one of my pixels: this try is void
        i += cnt;
    }
    { const int r = v3_take_resolve(W, tk, rcode); if (r != -1) failrank = (r >= 0 && r > failrank) ? r : (failrank >= 0 ? failrank : r); }
    const bool lostany = __any_sync(0xffffffffu, failrank != -1);
    failrank = __reduce_max_sync(0xffffffffu, failrank);
    if (W.abort) return -1;
    if (lostany) { if (lane == 0) { W.abort = 2; W.conflict = failrank >= 0 ? failrank : -1; } __syncwarp(); return -1; }
    if (dirty) th = fast_atan2_deg(sumdy, sumdx);
    *reg_angle_out = (double)th * L_DEG;
    return n;
}

// grow + fit + refine one seed as attempt (W.seq, try): 1 = candidate rectangle in *rec, 0 = no job, -1 = abandoned (W.abort)
__device__ __noinline__ int v3_one_region(const LineGeom& g, unsigned idx, LRect* rec, int* n0) {
    WalkCtx& W = s_Wc[threadIdx.x >> 5];
    double reg_angle;
    int n = l_region_grow_v3((int)(idx % (unsigned)g.sw), (int)(idx / (unsigned)g.sw), g.prec, &reg_angle);
    if (n < 0) return -1;
    *n0 = n;
    W.acc = n;
#ifdef SSLPL_V3_DEBUG
    if ((int)idx == g.dbg_seed) { __syncwarp(); for (int i = (threadIdx.x & 31); i < n; i += 32) printf("L3 %d %u %u %u\n", i, W.reg[i] & 0xffff, W.reg[i] >> 16, W.ticket); __syncwarp(); }
#endif
    if (n < g.min_reg_size) return 0;
    l_region2rect<3>(n, reg_angle, g.prec, g.p, rec);
    const bool okr = l_refine<3>(&n, &reg_angle, g.prec, g.p, rec, 0.7);
    if (W.abort) return -1;
    return okr ? 1 : 0;
}

// One pass of the RETIRER over the head of the ring (a whole warp; returns whether anything moved).  Runs of PRESUMED slots — the
// seeds a region swallowed while it was live come right behind it in seed order — are looked at 32 at a time (one ticket load per
// lane) and retired together; DONE / VOID slots one by one (their validity can depend on the slot before).
__device__ bool v3_retire_pass(const LineGeom& g, const LineWs& ws, int f, unsigned char* rcode, unsigned long long* cnt) {
    V3Shared& S = v3s();
    const int lane = threadIdx.x & 31;
    const LPix* pix = ws.pix + (long long)f * g.pix_stride;
    bool progress = false;
    for (;;) {
        const unsigned t = S.turn, nc = S.nclaims;
        if (t >= nc) break;
        const int k = (int)(t & (V3_RING - 1));
        const int st = *reinterpret_cast<volatile int*>(&S.state[k]);
        if (st == V3_PRESUMED) {
            const unsigned r = t + (unsigned)lane;
            const int kk = (int)(r & (V3_RING - 1));
            const bool pres = r < nc && *reinterpret_cast<volatile int*>(&S.state[kk]) == V3_PRESUMED;
            const unsigned pm = __ballot_sync(0xffffffffu, pres);
            const int len = __ffs(~pm) - 1 < 0 ? 32 : __ffs(~pm) - 1;            // leading PRESUMED slots
            __threadfence_block();
            int c = 0;
            if (lane < len) { const unsigned m = __ldcg(&pix[S.seed[kk]].used); c = m == 0u ? 0 : v3_classify(m, (int)r, rcode); }
            const unsigned sw = __ballot_sync(0xffffffffu, lane < len && c == 1);
            const int nsw = __ffs(~sw) - 1 < 0 ? 32 : __ffs(~sw) - 1;             // leading swallowed ones: they retire together
            bool ran = false;
            if (lane < nsw) {
                rcode[r] = 0xffu;
                ran = (S.flag[kk] & V3F_RAN) != 0;
                if (ran) atomicOr(&S.excbits[r >> 5], 1u << (r & 31));
                *reinterpret_cast<volatile int*>(&S.state[kk]) = V3_EMPTY;
            }
            if (__any_sync(0xffffffffu, ran)) __threadfence(); else __threadfence_block();
            __syncwarp();
            if (nsw > 0) { if (lane == 0) S.turn = t + (unsigned)nsw; cnt[4] += (unsigned long long)nsw; progress = true; }
            if (nsw < len) {                                                       // the new head was not swallowed after all: it grows now
                if (lane == nsw) { S.wait[kk] = -1; atomicMin(&S.scanhint, (int)r); __threadfence_block(); atomicAdd(&S.nready, 1); *reinterpret_cast<volatile int*>(&S.state[kk]) = V3_READY; }
                cnt[5]++; progress = true;
                __syncwarp();
                break;
            }
            __syncwarp();
            continue;
        }
        if (st != V3_DONE && st != V3_VOID) break;
        __threadfence_block();
        bool relbad = false;                                      // a pixel it accepted and released is used by a region of lower rank
        if (st == V3_DONE && (S.flag[k] & V3F_DIRTY) && S.dl_n[k] > 0) {
            const unsigned* dl = ws.dlist + (long long)f * V3_DPOOL + S.dl_off[k];
            const int nn = S.dl_n[k];
            bool bad = false;
            for (int i = lane; i < nn; i += 32) {
                const unsigned pk = __ldcg(dl + i);
                const unsigned tg = __ldcg(&pix[(int)(pk >> 16) * g.sw + (int)(pk & 0xffff)].used);
                if (tg != 0u && !(tg & 0x80000000u) && v3_rank(tg) != (int)t && v3_classify(tg, (int)t, rcode) == 1) bad = true;
            }
            relbad = __any_sync(0xffffffffu, bad);
        }
        int act = 0;                                              // 1 retire (| 4 with a job, | 8 exception), 2 back to READY
        if (lane == 0) {
            const int y = S.tryno[k], fl = S.flag[k];
            if (st == V3_DONE) {
                const bool pois = *reinterpret_cast<volatile unsigned char*>(&S.poison[k]) == (unsigned char)(y + 1);
                bool ok = !pois && !relbad;
                const int nd = (fl >> 4) & 3;
                for (int d = 0; d < nd && ok; d++) { const unsigned tk = S.dep[k][d]; ok = __ldcg(rcode + v3_rank(tk)) == (unsigned)v3_try(tk); }   // committed with that try, nothing released
#ifdef SSLPL_V3_DEBUG
                if ((g.dbg & 16) && t < 64) printf("RET rank %u try %d flags %x poison %d -> %s\n", t, y, fl, (int)S.poison[k], ok ? "commit" : "redo");
#endif
                if (ok) {
                    rcode[t] = (unsigned char)(y | ((fl & V3F_DIRTY) ? 0x80 : 0));
                    if (y != 0) S.excbits[t >> 5] |= 1u << (t & 31);
                    act = 1 | ((fl & V3F_JOB) ? 4 : 0) | (y != 0 ? 8 : 0);
                    cnt[0]++;
                } else {
                    S.tryno[k] = (unsigned char)min(y + 1, 126); S.poison[k] = 0; S.flag[k] = V3F_RAN; S.wait[k] = -1;
                    act = 2;
                    cnt[pois ? 1 : 2]++;
                }
            } else {
                rcode[t] = 0xffu;
                if (fl & V3F_RAN) S.excbits[t >> 5] |= 1u << (t & 31);
                act = 1 | ((fl & V3F_RAN) ? 8 : 0);
                cnt[3]++;
            }
        }
        act = __shfl_sync(0xffffffffu, act, 0);
        if (act & 1) {
            if (act & 4) {
                const int nj = S.nj;
                if (nj < g.seg_cap && lane < 13) ws.jobs[((long long)f * g.seg_cap + nj) * 13 + lane] = __ldcg(ws.sjob + ((long long)f * V3_RING + k) * 13 + lane);
                if (lane == 0) S.nj = nj + 1;
            }
            __syncwarp();
            if (lane == 0) { if (act & 8) __threadfence(); *reinterpret_cast<volatile int*>(&S.state[k]) = V3_EMPTY; __threadfence_block(); S.turn = t + 1; }
        } else {
            if (lane == 0) { atomicMin(&S.scanhint, (int)t); __threadfence_block(); atomicAdd(&S.nready, 1); *reinterpret_cast<volatile int*>(&S.state[k]) = V3_READY; }
        }
        __syncwarp();
        progress = true;
        if (!(act & 1)) break;                                    // the head runs again: nothing behind it can retire
    }
    return progress;
}

// One pass of the CLAIMER: the next 32 seeds of the ordered list are looked at together (one ticket load per lane) and every one
// that is not used by a committed region gets the next rank and a slot — READY, or PRESUMED swallowed if it is under a live ticket.
__device__ bool v3_claim_pass(const LineGeom& g, const LineWs& ws, int f, unsigned char* rcode, int limit = 0) {
    V3Shared& S = v3s();
    const int lane = threadIdx.x & 31;
    const LPix* pix = ws.pix + (long long)f * g.pix_stride;
    const unsigned* seeds = ws.seeds + (long long)f * g.pix_stride;
    const int ns = S.ns;
    if (S.all_claimed) return false;
    const unsigned nc = S.nclaims;
    if (nc - S.turn >= (unsigned)(V3_RING - 33)) { if ((g.dbg & 32) && (threadIdx.x & 31) == 0) atomicAdd(ws.wstat + 6, 1ull); return false; }
    if (*reinterpret_cast<volatile int*>(&S.nready) - *reinterpret_cast<volatile int*>(&S.nblocked) >= (limit ? limit : (((g.dbg >> 8) & 0xff) ? ((g.dbg >> 8) & 0xff) : 1) * (int)(blockDim.x >> 5))) return false;
    if (nc >= (unsigned)(V3_RANKS - 33)) { if (lane == 0) { S.overflow = 1; S.all_claimed = 1; } __syncwarp(); return true; }
    const int cur = (int)S.cursor;
    if (cur >= ns) { if (lane == 0) S.all_claimed = 1; __syncwarp(); return true; }
    const int i = cur + lane;
    const bool have = i < ns;
    const unsigned mine = have ? seeds[i] : 0u;
    unsigned m = 0; int cls = 1;
    if (have) { m = __ldcg(&pix[mine].used); cls = m == 0u ? 0 : v3_classify(m, 0x7fffffff, rcode); }     // any live ticket is of lower rank than a new claim
    const unsigned fm = __ballot_sync(0xffffffffu, have && cls != 1);
    const int nfree = __popc(__ballot_sync(0xffffffffu, have && cls == 0));
    if (have && cls != 1) {
        const unsigned r = nc + (unsigned)__popc(fm & ((1u << lane) - 1u));
        const int k = (int)(r & (V3_RING - 1));
        S.seed[k] = (int)mine; S.tryno[k] = 0; S.poison[k] = 0; S.flag[k] = 0; S.wait[k] = -1;
        if (cls != 0) S.dep[k][0] = m;
        __threadfence_block();
        *reinterpret_cast<volatile int*>(&S.state[k]) = cls != 0 ? V3_PRESUMED : V3_READY;
    }
    __threadfence_block();
    __syncwarp();
    if (lane == 0) {
        if (nfree) atomicAdd(&S.nready, nfree);
        S.cursor = (unsigned)min(cur + 32, ns);
        __threadfence_block();
        S.nclaims = nc + (unsigned)__popc(fm);
    }
    __syncwarp();
    return true;
}

__device__ void v3_worker(const LineGeom& g, const LineWs& ws, int f, unsigned char* rcode) {
    V3Shared& S = v3s();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    WalkCtx& W = s_Wc[wid];
    unsigned idle = 0;
    const bool stat = (g.dbg & 32) != 0;
    unsigned long long c_busy = 0, c_idle = 0, n_conf = 0, n_cap = 0, n_head = 0, c_abort = 0, c_idle_wait = 0;
    for (;;) {
        if (*reinterpret_cast<volatile int*>(&S.done)) break;
        const long long tw0 = stat ? clock64() : 0;
        // ---- pick the lowest runnable slot
        const unsigned t = S.turn, nc = S.nclaims;
        int from = max((int)t, *reinterpret_cast<volatile int*>(&S.scanhint));
        int got = -1; bool sawready = false;
        for (int b = from; b < (int)nc && got < 0; b += 32) {
            const int r = b + lane;
            bool ready = false, run = false;
            if (r < (int)nc) {
                const int k = r & (V3_RING - 1);
                ready = *reinterpret_cast<volatile int*>(&S.state[k]) == V3_READY;
                if (ready) {
                    // an attempt that lost a pixel to a live attempt of lower rank runs again once that one has finished GROWING (its
                    // tickets are then what it will commit with, and become a dependency) — not only after it has retired
                    const int wt = *reinterpret_cast<volatile int*>(&S.wait[k]);
                    if (wt == r) run = r == (int)t;                            // (out of list space / too many dependencies: only as head)
                    else {
                        run = wt < (int)t;
                        if (!run && !(g.dbg & 128)) { const int sw = *reinterpret_cast<volatile int*>(&S.state[wt & (V3_RING - 1)]); run = sw != V3_READY && sw != V3_RUNNING; }
                    }
                }
            }
            const unsigned rm = __ballot_sync(0xffffffffu, run);
            if (!sawready) {
                const unsigned am = __ballot_sync(0xffffffffu, ready);
                if (am) sawready = true;
                else if (lane == 0 && b == from && b + 32 <= (int)nc) atomicCAS(&S.scanhint, from, b + 32);     // nothing READY here: later scans start further on
            }
            if (rm) {
                const int r0 = b + __ffs(rm) - 1;
                int ok = 0;
                if (lane == 0) ok = atomicCAS(&S.state[r0 & (V3_RING - 1)], V3_READY, V3_RUNNING) == V3_READY;
                ok = __shfl_sync(0xffffffffu, ok, 0);
                if (ok) got = r0; else break;                     // somebody else took it: scan again
            }
        }
        if (got < 0) { idle = min(idle + 1, 8u); __nanosleep(32u << min(idle, 4u)); if (stat) { const long long dd = clock64() - tw0; c_idle += dd; if (sawready) c_idle_wait += dd; } continue; }
        idle = 0;
        const long long tw1 = stat ? clock64() : 0;
        if (stat) c_idle += tw1 - tw0;
        const int r = got, k = r & (V3_RING - 1);
        __threadfence_block();
        const unsigned idx = (unsigned)S.seed[k];
        const int y = S.tryno[k];
        const bool head = r == (int)S.turn;                       // nothing of lower rank is live: the frame-sized list is free for it
        if (lane == 0) {
            atomicSub(&S.nready, 1);
            if (S.wait[k] >= 0) atomicSub(&S.nblocked, 1);
            W.mode = head ? 1 : 0; W.abort = 0; W.conflict = -1; W.seq = r; W.ticket = (unsigned)(r + 1) | ((unsigned)y << 24);
            W.dirty = 0; W.ndeps = 0; W.nasm = g.dbg_seed; W.acc = 0;
            if (head) { W.reg = ws.reg + (long long)f * g.pix_stride; W.cap = (int)g.pix_stride; }
            else { W.reg = ws.sreg + ((long long)f * V3_MAXW + wid) * V3_LIST; W.cap = V3_LIST; }
            W.base0 = W.reg;
        }
        __syncwarp();
        LRect rec; int n0 = 0;
        const int res = v3_one_region(g, idx, &rec, &n0);
        __syncwarp();
#ifdef SSLPL_V3_DEBUG
        if ((g.dbg & 16) && lane == 0 && r < 64) printf("W%02d rank %d try %d seed (%d,%d) %s res %d abort %d conflict %d n0 %d ndeps %d [%x %x] dirty %d turn %u\n", wid, r, y, (int)(idx % (unsigned)g.sw), (int)(idx / (unsigned)g.sw), head ? "HEAD" : "spec", res, W.abort, W.conflict, n0, W.ndeps, W.dep[0], W.dep[1], W.dirty, S.turn);
#endif
        int res2 = res;
        if (res >= 0 && W.dirty && W.mode == 0) {
            // it released pixels: whether one of them belongs to a region of lower rank can only be told when it retires — the pixels
            // it ever accepted (first growth + re-growth, W.base0[0 .. W.acc)) wait in the frame's pool
            const int nacc = W.acc;
            int off = 0;
            if (lane == 0) off = atomicAdd(&S.dl_used, nacc);
            off = __shfl_sync(0xffffffffu, off, 0);
            if (off + nacc > V3_DPOOL) { if (lane == 0) W.abort = 1; res2 = -1; }        // pool exhausted: run it again as head
            else {
                unsigned* dst = ws.dlist + (long long)f * V3_DPOOL + off;
                for (int i = lane; i < nacc; i += 32) dst[i] = W.base0[i];
                if (lane == 0) { S.dl_off[k] = off; S.dl_n[k] = nacc; }
            }
            __syncwarp();
        } else if (lane == 0) S.dl_n[k] = 0;
        __syncwarp();
        if (res2 >= 0) {
            if (res == 1) l_emit_job(g, ws.sjob + ((long long)f * V3_RING + k) * 13, rec, idx, n0, lane);
            __syncwarp();
            if (lane == 0) {
                const int nd = W.ndeps;
                for (int d = 0; d < nd; d++) S.dep[k][d] = W.dep[d];
                S.flag[k] = (unsigned char)(V3F_RAN | (res == 1 ? V3F_JOB : 0) | (W.dirty ? V3F_DIRTY : 0) | (nd << 4));
                __threadfence();
                *reinterpret_cast<volatile int*>(&S.state[k]) = V3_DONE;
            }
        } else if (lane == 0) {
            const int ab = W.abort;
            // (both can also come out of refine's re-growth, after this try has put tickets on pixels: the try number moves on)
            if (ab == 4) { S.tryno[k] = (unsigned char)min(y + 1, 126); S.flag[k] = V3F_RAN; __threadfence_block(); *reinterpret_cast<volatile int*>(&S.state[k]) = V3_VOID; }   // the seed is used by a committed region
            else if (ab == 3) { S.tryno[k] = (unsigned char)min(y + 1, 126); S.poison[k] = 0; S.flag[k] = V3F_RAN; S.dep[k][0] = (unsigned)W.conflict; __threadfence_block(); *reinterpret_cast<volatile int*>(&S.state[k]) = V3_PRESUMED; }
            else {
                // 2: lost a pixel to a live attempt of lower rank (run again after it has retired) or to a race (run again at once);
                // 1 / 5: out of list space / more than two dependencies: run again as head
                S.tryno[k] = (unsigned char)min(y + 1, 126); S.poison[k] = 0; S.flag[k] = V3F_RAN;
                int wt = ab == 2 ? W.conflict : r;            // wait == r: only as head (turn > r - 1 is checked as wait - 1 < turn below)
                if (y >= 100) wt = r;
                S.wait[k] = wt;
                if (wt >= 0) atomicAdd(&S.nblocked, 1);
                atomicMin(&S.scanhint, r);
                __threadfence_block();
                atomicAdd(&S.nready, 1);
                *reinterpret_cast<volatile int*>(&S.state[k]) = V3_READY;
                n_conf++;
            }
        }
        __syncwarp();
        if (stat) { const long long d = clock64() - tw1; c_busy += d; if (res < 0) c_abort += d; if (head) n_head++; }
    }
    if (stat && lane == 0) {
        atomicAdd(ws.wstat + 6, n_conf); atomicAdd(ws.wstat + 7, n_cap); atomicAdd(ws.wstat + 10, c_busy); atomicAdd(ws.wstat + 11, c_idle);
        atomicAdd(ws.wstat + 12, c_abort); atomicAdd(ws.wstat + 15, n_head); atomicAdd(ws.wstat + 7, c_idle_wait);
    }
}

__global__ void __launch_bounds__(V3_MAXW * 32) k_lsd_regions_v3(const __grid_constant__ LineGeom g, LineWs ws, int nframes) {
    V3Shared& S = v3s();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (;;) {
    __syncthreads();
    if (threadIdx.x == 0) {
        const int f = atomicAdd(ws.rejctl + 2, 1);
        S.frame = f; S.turn = 0; S.nclaims = 0; S.cursor = 0; S.nj = 0; S.all_claimed = 0; S.done = 0; S.nready = 0; S.nblocked = 0; S.dl_used = 0; S.scanhint = 0; S.win_base = -(1 << 30); S.overflow = 0;
        S.ns = f < nframes ? ws.nseeds[f] : 0;
    }
    for (int i = threadIdx.x; i < V3_RING; i += blockDim.x) { S.state[i] = V3_EMPTY; S.wait[i] = -1; S.tryno[i] = 0; S.poison[i] = 0; S.flag[i] = 0; }
    for (int i = threadIdx.x; i < V3_RANKS / 32; i += blockDim.x) S.excbits[i] = 0u;
    __syncthreads();
    const int f = S.frame;
    if (f >= nframes) break;
    unsigned char* rcode = ws.rcode + (long long)f * V3_RANKS;
    if (lane == 0) {
        WalkCtx& W = s_Wc[wid];
        W.w = g.sw; W.h = g.sh; W.dbg = g.dbg;
        W.ang = ws.angdeg + f * g.pix_stride; W.mod = ws.modgrad + f * g.pix_stride;
        W.pix = ws.pix + f * g.pix_stride; W.cs0 = ws.cs0 + f * g.pix_stride; W.bits = reinterpret_cast<const unsigned*>(rcode);
    }
    __syncwarp();
    {
        // warp 0 claims (and works once every seed has been claimed), warp 1 retires, the others work; with two warps, warp 0 does both
        const bool two = blockDim.x == 64;
        const bool stat = (g.dbg & 32) != 0;
        unsigned long long cnt[6] = {0, 0, 0, 0, 0, 0}, c_ret = 0, c_claim = 0, c_idle = 0;
        if (wid == 0 || (wid == 1 && !two)) {
            for (;;) {
                const long long t0 = stat ? clock64() : 0;
                bool p1 = false, p2 = false;
                if (wid == 0) p1 = v3_claim_pass(g, ws, f, rcode);
                const long long t1 = stat ? clock64() : 0;
                if (wid == 1 || two) {
                    p2 = v3_retire_pass(g, ws, f, rcode, cnt);
                    if (S.all_claimed && S.turn >= S.nclaims) { if (lane == 0) { __threadfence_block(); S.done = 1; } __syncwarp(); break; }
                }
                if (stat) { const long long t2 = clock64(); if (p1) c_claim += t1 - t0; else c_idle += t1 - t0; if (p2) c_ret += t2 - t1; else c_idle += t2 - t1; }
                if (wid == 0 && !two && S.all_claimed) break;       // nothing left to claim: become a worker
                if (!p1 && !p2) __nanosleep(32);
            }
            if (stat && lane == 0) {
                for (int i = 0; i < 6; i++) atomicAdd(ws.wstat + i, cnt[i]);
                atomicAdd(ws.wstat + 8, c_ret); atomicAdd(ws.wstat + 9, c_claim); atomicAdd(ws.wstat + 14, c_idle);
                if (wid == 0) atomicAdd(ws.wstat + 13, (unsigned long long)S.nclaims);
            }
            if (wid == 0 && !two) v3_worker(g, ws, f, rcode);
        } else v3_worker(g, ws, f, rcode);
    }
    __syncthreads();
    if (threadIdx.x == 0) { ws.njobs[f] = min(S.nj, g.seg_cap); if (S.nj > g.seg_cap || S.overflow) atomicOr(ws.err, DERR_LSD_OVERFLOW); }
  }
}

// =================================================================================================
// LANE-PARALLEL region walker (round 2b, k_lsd_regions_lanes): ONE WARP PER FRAME, every LANE grows its own region.
// The one-warp walkers spend hundreds of warp instructions per growth step on 32 neighbour tests of ONE region, almost all of it
// warp-uniform bookkeeping: a lone warp retires one instruction every several cycles, so the stage is bound by instruction count.
// Here region growing is the plain scalar loop of lsd.cpp run by each lane on a different seed (same protocol as the multi-warp
// walker v3: ranks in seed order, tickets in LPix.used, poison / dependencies / released-pixel lists, strictly ordered retire —
// v3_retire_pass and v3_claim_pass are used as they are), so that one warp instruction serves up to 32 regions.  A neighbour is
// accepted with a SYNCHRONOUS compare-and-swap (nothing to roll back, no "lost a pixel" aborts).  The region angle is lazy per
// lane (exact fastAtan2 only when a test is within the drift bound of the threshold).  What is cheap per region but long in code
// — rectangle fit with its ordered double sums, density, refine's release and tau, reduce_region_radius — runs warp-cooperatively
// with the existing routines (template mode 4) for one finished lane at a time.
// =================================================================================================
constexpr int LN_LIST = 4096;          // list entries per lane (32 lanes x 4096 = ws.sreg of a frame); bigger regions run as head on ws.reg
enum { LN_IDLE = 0, LN_GROW = 1, LN_POST = 2 };

template <int SOLO> __device__ __forceinline__ bool l4_exact_pass(float a, float th, float pdeg, double prec) {
    const float d = fabsf(th - a);
    const float e = d > 270.f ? 360.f - d : d;
    bool pass = e <= pdeg;
    if (fabsf(e - pdeg) < 2e-3f || fabsf(d - 270.f) < 2e-3f) pass = l_aligned_rad((double)a * L_DEG, (double)th * L_DEG, prec);
    return pass;
}

// refine, first half (lsd.cpp refine up to the re-growth): nothing to do if the density is fine (returns true); otherwise every
// pixel is released, tau is formed from the angles near the seed and, for a speculative attempt, the list pointer moves behind the
// first list (which stays: every pixel ever accepted is looked at when the attempt retires).
__device__ __noinline__ bool l4_refine_begin(int n, const LRect* rec, double density_th, double* tau_out) {
    constexpr int SOLO = 4;
    const int lane = threadIdx.x & 31, w = s_W.w;
    const double density = (double)n / (l_dist(rec->x1, rec->y1, rec->x2, rec->y2) * rec->width);
    if (density >= density_th) return true;
    if (lane == 0) s_W.dirty = 1;
    const unsigned* reg = s_W.reg; const float* __restrict__ ang = s_W.ang;
    const unsigned p0 = reg[0];
    const int sx = p0 & 0xffff, sy = p0 >> 16;
    const double xc = (double)sx, yc = (double)sy;
    const double ang_c = (double)ang[sy * w + sx] * L_DEG;
    const double width = rec->width;
    double* s0 = s_st; double* s1 = s_st + 32;
    const double* sp = s_st + (lane & 1) * 32;
    double acc = 0; int cnt = 0;
#pragma unroll 1
    for (int b = 0; b < n; b += 32) {
        const int i = b + lane;
        bool in = false;
        if (i < n) {
            const unsigned pk = reg[i]; const int rx = pk & 0xffff, ry = pk >> 16;
            const float ad = ang[ry * w + rx];
            l_release<SOLO>(s_W, ry * w + rx);
            in = l_dist(xc, yc, (double)rx, (double)ry) < width;
            const double d = l_angle_diff_signed((double)ad * L_DEG, ang_c);
            s0[lane] = in ? d : 0.0; s1[lane] = in ? d * d : 0.0;
        }
        cnt += __popc(__ballot_sync(0xffffffffu, in));
        __syncwarp();
        acc = l_chunk_sum<SOLO>(sp, min(32, n - b), acc);
        __syncwarp();
    }
    const double sum = __shfl_sync(0xffffffffu, acc, 0), s_sum = __shfl_sync(0xffffffffu, acc, 1);
    const double mean_angle = sum / (double)cnt;
    *tau_out = 2.0 * sqrt((s_sum - 2.0 * mean_angle * sum) / (double)cnt + mean_angle * mean_angle);
    __syncwarp();
    return false;
}

struct LaneAtt {
    int st, slot, rank, mode, phase, tryno;
    unsigned T;
    unsigned* list; int cap;          // the list being grown (behind the first list during a speculative re-growth)
    int i, n, kacc, n0, acc;
    float sx, sy, th, rM, pdeg, coefX; double prec; int robok;
    int ndeps; unsigned dep0, dep1;
    int abortc, conflict, dirty;
    unsigned seedidx;
};

struct LaneFrame { int w, h; LPix* pix; const float* ang; const float2* cs0; const unsigned char* rcode; };

// take pixel q (ticket seen in `m`) for the lane's attempt: 1 taken, 0 it is used after all (committed, or held by a live attempt of
// lower rank: recorded as a dependency), -1 give up (abortc set)
__device__ __forceinline__ int ln_take(LaneAtt& A, const LaneFrame& F, int q, unsigned m) {
    for (int tries = 0; tries < 8; tries++) {
        const unsigned old = A.mode ? atomicExch(&F.pix[q].used, A.T) : atomicCAS(&F.pix[q].used, m, A.T);
        if (A.mode || old == m) {
            const unsigned o = old & 0x7fffffffu;
            if (o != 0u && o != A.T && v3_classify(o, A.rank, F.rcode) == 3) v3_poison(o);
            return 1;
        }
        m = old;                                                  // somebody changed it in between: look again
        if (m == A.T) return 0;
        const int c = m == 0u ? 0 : v3_classify(m, A.rank, F.rcode);
        if (c == 1) return 0;
        if (c == 2) {
            if (!((A.ndeps > 0 && A.dep0 == m) || (A.ndeps > 1 && A.dep1 == m))) { if (A.ndeps == 0) A.dep0 = m; else if (A.ndeps == 1) A.dep1 = m; else { A.abortc = 5; return -1; } A.ndeps++; }
            return 0;
        }
    }
    A.abortc = 5;                                                 // contended: run it again as head
    return -1;
}

// start (or restart, for refine's re-growth) the growth of the lane's attempt from its seed with tolerance prec
__device__ __forceinline__ void ln_begin(LaneAtt& A, const LaneFrame& F, double prec) {
    const int sq = (int)A.seedidx;
    const unsigned m0 = __ldcg(&F.pix[sq].used);
    if (m0 != A.T) {
        const int c = m0 == 0u ? 0 : v3_classify(m0, A.rank, F.rcode);
        if (c == 1) { A.abortc = 4; return; }
        if (c == 2) { A.abortc = 3; A.conflict = (int)m0; return; }
        const int t = ln_take(A, F, sq, m0);
        if (t == 0) { A.abortc = 2; A.conflict = -1; return; }   // lost the seed between the look and the take: look again from the start
        if (t < 0) return;
    }
    A.list[0] = (unsigned)(sq % F.w) | ((unsigned)(sq / F.w) << 16);
    A.n = 1; A.i = 0; A.kacc = 0;
    A.th = __ldg(F.ang + sq);
    const float2 c0 = __ldg(F.cs0 + sq);
    A.sx = c0.x; A.sy = c0.y; A.rM = rsqrtf(c0.x * c0.x + c0.y * c0.y);
    A.prec = prec; A.pdeg = (float)(prec * (180.0 / L_PI));
    A.robok = prec < 0.78;
    A.coefX = (float)(57.2958 * 1.0002 * sin(prec + 0.17453 + 0.0006));     // vectors accepted within prec + 10 deg of the sums at the last exact angle
    A.st = LN_GROW;
}

// one queue entry of the lane's region: the 3x3 scan of lsd.cpp's region_grow, neighbour by neighbour, in order
__device__ __forceinline__ void ln_step(LaneAtt& A, const LaneFrame& F) {
    const unsigned pk = A.list[A.i];
    const int x0 = (int)(pk & 0xffff), y0 = (int)(pk >> 16);
    uint4 v[8]; int qq[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {                                  // the eight records in flight together
        const int nb = j + (j >= 4 ? 1 : 0);                       // 0..8 without the centre (4)
        const int xx = x0 + nb % 3 - 1, yy = y0 + nb / 3 - 1;
        const bool ok = (unsigned)xx < (unsigned)F.w && (unsigned)yy < (unsigned)F.h;
        qq[j] = ok ? yy * F.w + xx : -1;
        v[j] = make_uint4(__float_as_uint(NOTDEF_F), 0u, 0u, 0u);
        if (ok) v[j] = __ldcg(reinterpret_cast<const uint4*>(F.pix + qq[j]));
    }
#pragma unroll
    for (int j = 0; j < 8; j++) {
        if (A.abortc) break;
        const float a = __uint_as_float(v[j].x);
        const unsigned m = v[j].w;
        if (qq[j] < 0 || a == NOTDEF_F || m == A.T) continue;
        if (m != 0u) {
            const int c = v3_classify(m, A.rank, F.rcode);
            if (c == 1) continue;
            if (c == 2) {
                if (!((A.ndeps > 0 && A.dep0 == m) || (A.ndeps > 1 && A.dep1 == m))) { if (A.ndeps == 0) A.dep0 = m; else if (A.ndeps == 1) A.dep1 = m; else { A.abortc = 5; break; } A.ndeps++; }
                continue;
            }
        }
        // the alignment test against the region angle as the sequential scan has it now
        bool pass;
        if (A.kacc == 0) pass = l4_exact_pass<4>(a, A.th, A.pdeg, A.prec);
        else {
            const float d = fabsf(A.th - a);
            const float e = d > 270.f ? 360.f - d : d;
            const float B = A.coefX * (float)A.kacc * A.rM + 0.0215f;
            const bool ok = A.robok && B <= 10.f;
            if (ok && e <= A.pdeg - B) pass = true;
            else if (ok && e >= A.pdeg + B) pass = false;
            else {
                A.th = fast_atan2_deg(A.sy, A.sx); A.rM = rsqrtf(A.sx * A.sx + A.sy * A.sy); A.kacc = 0;
                pass = l4_exact_pass<4>(a, A.th, A.pdeg, A.prec);
            }
        }
        if (!pass) continue;
        if (A.n >= A.cap) { A.abortc = 1; break; }
        const int t = ln_take(A, F, qq[j], m);
        if (t < 0) break;
        if (t == 0) continue;
        const int nb = j + (j >= 4 ? 1 : 0);
        A.list[A.n++] = (unsigned)(x0 + nb % 3 - 1) | ((unsigned)(y0 + nb / 3 - 1) << 16);
        A.sx += __uint_as_float(v[j].y); A.sy += __uint_as_float(v[j].z);
        A.kacc++;
    }
    A.i++;
}

__global__ void __launch_bounds__(32, 8) k_lsd_regions_lanes(const __grid_constant__ LineGeom g, LineWs ws, int nframes) {
    constexpr int SOLO = 4;
    V3Shared& S = v3s();
    const int lane = threadIdx.x;
    const unsigned lt = (1u << lane) - 1u;
  for (;;) {
    __syncwarp();
    if (lane == 0) {
        const int f = atomicAdd(ws.rejctl + 2, 1);
        S.frame = f; S.turn = 0; S.nclaims = 0; S.cursor = 0; S.nj = 0; S.all_claimed = 0; S.done = 0; S.nready = 0; S.nblocked = 0; S.dl_used = 0; S.scanhint = 0; S.win_base = -(1 << 30); S.overflow = 0;
        S.ns = f < nframes ? ws.nseeds[f] : 0;
    }
    for (int i = lane; i < V3_RING; i += 32) { S.state[i] = V3_EMPTY; S.wait[i] = -1; S.tryno[i] = 0; S.poison[i] = 0; S.flag[i] = 0; S.dl_n[i] = 0; }
    for (int i = lane; i < V3_RANKS / 32; i += 32) S.excbits[i] = 0u;
    __syncwarp();
    const int f = S.frame;
    if (f >= nframes) break;
    unsigned char* rcode = ws.rcode + (long long)f * V3_RANKS;
    LaneFrame F; F.w = g.sw; F.h = g.sh; F.pix = ws.pix + f * g.pix_stride; F.ang = ws.angdeg + f * g.pix_stride; F.cs0 = ws.cs0 + f * g.pix_stride; F.rcode = rcode;
    if (lane == 0) {
        WalkCtx& W = s_W1;
        W.w = g.sw; W.h = g.sh; W.dbg = g.dbg;
        W.ang = F.ang; W.mod = ws.modgrad + f * g.pix_stride; W.pix = F.pix; W.cs0 = F.cs0; W.bits = reinterpret_cast<const unsigned*>(rcode);
    }
    __syncwarp();
    unsigned* const mylist = ws.sreg + ((long long)f * 32 + lane) * LN_LIST;
    unsigned* const biglist = ws.reg + (long long)f * g.pix_stride;
    LaneAtt A; A.st = LN_IDLE; A.abortc = 0; A.ndeps = 0; A.dep0 = A.dep1 = 0u; A.n = 0; A.i = 0; A.kacc = 0; A.mode = 0; A.phase = 0; A.dirty = 0; A.acc = 0; A.n0 = 0;
    A.slot = 0; A.rank = 0; A.tryno = 0; A.T = 0u; A.list = mylist; A.cap = LN_LIST; A.sx = A.sy = A.th = A.rM = A.pdeg = A.coefX = 0.f; A.prec = 0; A.robok = 0; A.conflict = -1; A.seedidx = 0u;
    unsigned long long dummy[6] = {0, 0, 0, 0, 0, 0};
    const bool stat = (g.dbg & 32) != 0;
    unsigned long long c_ret = 0, c_asg = 0, c_grow = 0, c_post = 0, n_iter = 0, n_round = 0, n_act = 0, n_post = 0;
    for (;;) {
        const long long q0 = stat ? clock64() : 0;
        // ---- retire the head of the ring while it is finished (the whole warp, cooperatively)
        {
            const unsigned t = S.turn;
            const int hs = t < S.nclaims ? *reinterpret_cast<volatile int*>(&S.state[t & (V3_RING - 1)]) : V3_EMPTY;
            if (hs == V3_DONE || hs == V3_PRESUMED || hs == V3_VOID) v3_retire_pass(g, ws, f, rcode, dummy);
        }
        if (S.all_claimed && S.turn >= S.nclaims) break;
        const long long q1 = stat ? clock64() : 0;
        // ---- finished lanes that need no cooperative work publish their own slot: regions below the minimum size, and every abort
        if (A.st == LN_POST && (A.abortc || (A.phase == 0 && A.n < g.min_reg_size))) {
            const int slot = A.slot, y = A.tryno;
            if (!A.abortc) {
                S.dep[slot][0] = A.dep0; S.dep[slot][1] = A.dep1; S.dl_n[slot] = 0;
                S.flag[slot] = (unsigned char)(V3F_RAN | (A.ndeps << 4));
                __threadfence_block();
                *reinterpret_cast<volatile int*>(&S.state[slot]) = V3_DONE;
            } else if (A.abortc == 4) { S.tryno[slot] = (unsigned char)min(y + 1, 126); S.flag[slot] = V3F_RAN; __threadfence_block(); *reinterpret_cast<volatile int*>(&S.state[slot]) = V3_VOID; }
            else if (A.abortc == 3) { S.tryno[slot] = (unsigned char)min(y + 1, 126); S.poison[slot] = 0; S.flag[slot] = V3F_RAN; S.dep[slot][0] = (unsigned)A.conflict; __threadfence_block(); *reinterpret_cast<volatile int*>(&S.state[slot]) = V3_PRESUMED; }
            else {
                S.tryno[slot] = (unsigned char)min(y + 1, 126); S.poison[slot] = 0; S.flag[slot] = V3F_RAN;
                int wt = A.abortc == 2 ? A.conflict : A.rank;
                if (y >= 100) wt = A.rank;
                S.wait[slot] = wt;
                if (wt >= 0) atomicAdd(&S.nblocked, 1);
                atomicMin(&S.scanhint, A.rank);
                __threadfence_block();
                atomicAdd(&S.nready, 1);
                *reinterpret_cast<volatile int*>(&S.state[slot]) = V3_READY;
            }
            A.st = LN_IDLE; A.abortc = 0;
        }
        __syncwarp();
        const unsigned idle = __ballot_sync(0xffffffffu, A.st == LN_IDLE);
        if (idle) {
            for (int pass = 0; pass < 3 && !S.all_claimed && *reinterpret_cast<volatile int*>(&S.nready) - *reinterpret_cast<volatile int*>(&S.nblocked) < __popc(idle) + 8; pass++)
                if (!v3_claim_pass(g, ws, f, rcode, 1 << 20)) break;
            // ---- hand runnable slots to the idle lanes, lowest ranks first
            const unsigned t = S.turn, nc = S.nclaims;
            int from = max((int)t, *reinterpret_cast<volatile int*>(&S.scanhint));
            unsigned left = idle;
            bool sawready = false;
            for (int b = from; b < (int)nc && left; b += 32) {
                const int r = b + lane;
                bool ready = false, run = false;
                if (r < (int)nc) {
                    const int k = r & (V3_RING - 1);
                    ready = *reinterpret_cast<volatile int*>(&S.state[k]) == V3_READY;
                    if (ready) {
                        const int wt = *reinterpret_cast<volatile int*>(&S.wait[k]);
                        if (wt == r) run = r == (int)t;
                        else { run = wt < (int)t; if (!run) { const int sw = *reinterpret_cast<volatile int*>(&S.state[wt & (V3_RING - 1)]); run = sw != V3_READY && sw != V3_RUNNING; } }
                    }
                }
                const unsigned rm = __ballot_sync(0xffffffffu, run);
                if (!sawready) { if (__ballot_sync(0xffffffffu, ready)) sawready = true; else if (lane == 0 && b == from && b + 32 <= (int)nc) atomicCAS(&S.scanhint, from, b + 32); }
                // the j-th idle lane takes the j-th runnable slot of this block
                const int take = min(__popc(rm), __popc(left));
                if (take) {
                    const bool mine = ((left >> lane) & 1u) && __popc(left & lt) < take;
                    if (mine) {
                        const int r0 = b + (int)__fns(rm, 0, __popc(left & lt) + 1);
                        const int k = r0 & (V3_RING - 1);
                        *reinterpret_cast<volatile int*>(&S.state[k]) = V3_RUNNING;       // one warp per frame: nobody competes for the slot
                        atomicSub(&S.nready, 1);
                        if (S.wait[k] >= 0) atomicSub(&S.nblocked, 1);
                        A.slot = k; A.rank = r0; A.tryno = S.tryno[k]; A.seedidx = (unsigned)S.seed[k];
                        A.T = (unsigned)(r0 + 1) | ((unsigned)A.tryno << 24);
                        A.mode = r0 == (int)t ? 1 : 0;
                        A.list = A.mode ? biglist : mylist; A.cap = A.mode ? (int)g.pix_stride : LN_LIST;
                        A.phase = 0; A.abortc = 0; A.conflict = -1; A.ndeps = 0; A.dirty = 0; A.acc = 0; A.n0 = 0; A.n = 0; A.i = 0;
                        ln_begin(A, F, g.prec);
                        if (A.abortc) A.st = LN_POST;              // (settled at the top of the next iteration)
                    }
                    left &= ~__ballot_sync(0xffffffffu, mine);
                }
            }
        }
        const long long q2 = stat ? clock64() : 0;
        // ---- growth: every busy lane expands one queue entry of its own region
        {
            if (stat) { n_round++; n_act += __popc(__ballot_sync(0xffffffffu, A.st == LN_GROW)); }
            if (A.st == LN_GROW) {
                if (A.mode == 0 && *reinterpret_cast<volatile unsigned char*>(&S.poison[A.slot]) == (unsigned char)(A.tryno + 1)) { A.abortc = 2; A.conflict = -1; }
                if (!A.abortc && A.i < A.n) ln_step(A, F);
                if (A.abortc || A.i >= A.n) A.st = LN_POST;
            }
            __syncwarp();
        }
        const long long q3 = stat ? clock64() : 0;
        if (stat) { c_ret += q1 - q0; c_asg += q2 - q1; c_grow += q3 - q2; n_iter++; }
        // ---- post: one finished lane at a time, the warp works on its region together (lowest rank first)
        for (;;) {
            const bool coop = A.st == LN_POST && !A.abortc && !(A.phase == 0 && A.n < g.min_reg_size);
            const unsigned pm = __ballot_sync(0xffffffffu, coop);
            if (!pm) { if (stat) c_post += clock64() - q3; break; }
            n_post++;
            int best = coop ? A.rank : 0x7fffffff;
            best = __reduce_min_sync(0xffffffffu, best);
            const int L = __ffs(__ballot_sync(0xffffffffu, coop && A.rank == best)) - 1;
            // the lane's attempt, broadcast
            const int abortc = __shfl_sync(0xffffffffu, A.abortc, L), slot = __shfl_sync(0xffffffffu, A.slot, L), rank = __shfl_sync(0xffffffffu, A.rank, L);
            const int mode = __shfl_sync(0xffffffffu, A.mode, L), phase = __shfl_sync(0xffffffffu, A.phase, L), tryno = __shfl_sync(0xffffffffu, A.tryno, L);
            int n = __shfl_sync(0xffffffffu, A.n, L);
            const unsigned long long lp = __shfl_sync(0xffffffffu, (unsigned long long)A.list, L);
            unsigned* list = reinterpret_cast<unsigned*>(lp);
            const int cap = __shfl_sync(0xffffffffu, A.cap, L);
            const unsigned T = __shfl_sync(0xffffffffu, A.T, L), seedidx = __shfl_sync(0xffffffffu, A.seedidx, L);
            int res = -1;            // -1 aborted, 0 no job, 1 job, 2 keeps growing (re-growth started)
            LRect rec;
            if (!abortc) {
                // region angle at the end of the growth: exact
                float th = __shfl_sync(0xffffffffu, A.th, L);
                { const float sx = __shfl_sync(0xffffffffu, A.sx, L), sy = __shfl_sync(0xffffffffu, A.sy, L); if (__shfl_sync(0xffffffffu, A.kacc, L) > 0) th = fast_atan2_deg(sy, sx); }
                double reg_angle = (double)th * L_DEG;
                __syncwarp();
                if (lane == 0) { WalkCtx& W = s_W1; W.reg = list; W.base0 = mode ? biglist : (ws.sreg + ((long long)f * 32 + L) * LN_LIST); W.cap = cap; W.mode = mode; W.ticket = T; W.seq = rank; W.abort = 0; W.dirty = 0; W.nasm = 0; }
                __syncwarp();
                int n0 = __shfl_sync(0xffffffffu, A.n0, L), acc = __shfl_sync(0xffffffffu, A.acc, L);
                if (phase == 0) {
                    n0 = n; acc = n;
                    if (lane == 0) s_W1.acc = acc;
                    __syncwarp();
                    if (n < g.min_reg_size) res = 0;
                    else {
                        l_region2rect<SOLO>(n, reg_angle, g.prec, g.p, &rec);
                        double tau;
                        if (l4_refine_begin(n, &rec, 0.7, &tau)) res = 1;
                        else {
                            // re-growth from the seed with tolerance tau: the lane goes back to growing (behind its first list if speculative)
                            if (lane == L) {
                                A.dirty = 1; A.phase = 1; A.n0 = n0; A.acc = acc;
                                if (mode == 0) { A.list += n; A.cap -= n; }
                                if (A.cap < 8) A.abortc = 1; else ln_begin(A, F, tau);
                                if (A.abortc) A.st = LN_POST;         // settled in the next round of this loop
                            }
                            res = 2;
                        }
                    }
                } else {
                    if (mode == 0) acc += n;
                    if (lane == 0) { s_W1.acc = acc; s_W1.dirty = 1; }
                    __syncwarp();
                    if (n < 2) res = 0;
                    else {
                        l_region2rect<SOLO>(n, reg_angle, g.prec, g.p, &rec);
                        const double density = (double)n / (l_dist(rec.x1, rec.y1, rec.x2, rec.y2) * rec.width);
                        bool okr = true;
                        if (density < 0.7) { int nn = n; okr = l_reduce_region_radius<SOLO>(&nn, reg_angle, g.prec, g.p, &rec, density, 0.7); if (s_W1.abort) okr = false; }
                        res = s_W1.abort ? -1 : (okr ? 1 : 0);
                    }
                }
                __syncwarp();
                if (res == 2) continue;
                // publish
                const int dirty = phase == 1 ? 1 : 0;
                int res2 = res;
                if (res >= 0 && dirty && mode == 0) {
                    int off = 0;
                    if (lane == 0) off = atomicAdd(&S.dl_used, acc);
                    off = __shfl_sync(0xffffffffu, off, 0);
                    if (off + acc > V3_DPOOL) res2 = -2;
                    else {
                        unsigned* dst = ws.dlist + (long long)f * V3_DPOOL + off;
                        const unsigned* src = ws.sreg + ((long long)f * 32 + L) * LN_LIST;
                        for (int i = lane; i < acc; i += 32) dst[i] = src[i];
                        if (lane == 0) { S.dl_off[slot] = off; S.dl_n[slot] = acc; }
                    }
                } else if (lane == 0) S.dl_n[slot] = 0;
                __syncwarp();
                if (res2 >= 0) {
                    if (res == 1) l_emit_job(g, ws.sjob + ((long long)f * V3_RING + slot) * 13, rec, seedidx, n0, lane);
                    __syncwarp();
                    const int nd = __shfl_sync(0xffffffffu, A.ndeps, L);
                    const unsigned d0 = __shfl_sync(0xffffffffu, A.dep0, L), d1 = __shfl_sync(0xffffffffu, A.dep1, L);
                    if (lane == 0) {
                        S.dep[slot][0] = d0; S.dep[slot][1] = d1;
                        S.flag[slot] = (unsigned char)(V3F_RAN | (res == 1 ? V3F_JOB : 0) | (dirty ? V3F_DIRTY : 0) | (nd << 4));
                        __threadfence();
                        *reinterpret_cast<volatile int*>(&S.state[slot]) = V3_DONE;
                    }
                    __syncwarp();
                    if (lane == L) A.st = LN_IDLE;
                    continue;
                }
            }
            // aborted (by the growth, by the cooperative part, or no room for its released-pixel list)
            {
                int ab = abortc ? abortc : (res == -1 ? (s_W1.abort ? s_W1.abort : 1) : 1);
                const int conflict = __shfl_sync(0xffffffffu, A.conflict, L);
                if (lane == 0) {
                    const int y = tryno;
                    if (ab == 4) { S.tryno[slot] = (unsigned char)min(y + 1, 126); S.flag[slot] = V3F_RAN; __threadfence_block(); *reinterpret_cast<volatile int*>(&S.state[slot]) = V3_VOID; }
                    else if (ab == 3) { S.tryno[slot] = (unsigned char)min(y + 1, 126); S.poison[slot] = 0; S.flag[slot] = V3F_RAN; S.dep[slot][0] = (unsigned)conflict; __threadfence_block(); *reinterpret_cast<volatile int*>(&S.state[slot]) = V3_PRESUMED; }
                    else {
                        S.tryno[slot] = (unsigned char)min(y + 1, 126); S.poison[slot] = 0; S.flag[slot] = V3F_RAN;
                        int wt = ab == 2 ? conflict : rank;
                        if (y >= 100) wt = rank;
                        S.wait[slot] = wt;
                        if (wt >= 0) atomicAdd(&S.nblocked, 1);
                        atomicMin(&S.scanhint, rank);
                        __threadfence_block();
                        atomicAdd(&S.nready, 1);
                        *reinterpret_cast<volatile int*>(&S.state[slot]) = V3_READY;
                    }
                }
                __syncwarp();
                if (lane == L) { A.st = LN_IDLE; A.abortc = 0; }
            }
        }
    }
    __syncwarp();
    if (stat && lane == 0) {
        atomicAdd(ws.wstat + 0, n_iter); atomicAdd(ws.wstat + 1, n_round); atomicAdd(ws.wstat + 2, n_act); atomicAdd(ws.wstat + 3, n_post);
        atomicAdd(ws.wstat + 8, c_ret); atomicAdd(ws.wstat + 9, c_asg); atomicAdd(ws.wstat + 10, c_grow); atomicAdd(ws.wstat + 11, c_post); atomicAdd(ws.wstat + 13, (unsigned long long)S.nclaims);
    }
    if (lane == 0) { ws.njobs[f] = min(S.nj, g.seg_cap); if (S.nj > g.seg_cap || S.overflow) atomicOr(ws.err, DERR_LSD_OVERFLOW); }
  }
}

// NFA of every candidate region of every frame, in three data-parallel steps (grids are sized by the work, not by the
// per-frame capacity seg_cap, which is ~13k slots of which a few hundred are used):
//   k_lsd_nfa_count   one warp per job: the rectangle scan (total / aligned pixel counts)
//   k_lsd_nfa_first   one THREAD per job: the scalar NFA formula (32 jobs per warp side by side); most jobs are accepted
//                     here, the others are appended to a global work list
//   k_lsd_nfa_improve persistent warps pull rejected jobs from that list: the five refinement phases of rect_improve
constexpr int NFA_COUNT_CTAS = 16;          // CTAs (4 warps) per frame in k_lsd_nfa_count
constexpr int NFA_FIRST_CTAS = 2;           // CTAs (128 threads) per frame in k_lsd_nfa_first

__device__ __forceinline__ void l_trace_row(const LineGeom& g, const LineWs& ws, int f, int j, const double* job, double tag, double log_nfa) {
    if (g.trace_cap && j < g.trace_cap) {
        double* t = ws.trace + ((long long)f * g.trace_cap + j) * 10;
        const double idx = floor(tag / 65536.0);
        t[0] = idx; t[1] = tag - idx * 65536.0; t[2] = 0; t[3] = log_nfa;
        t[4] = job[0]; t[5] = job[1]; t[6] = job[2]; t[7] = job[3]; t[8] = job[4]; t[9] = job[11];
    }
}

__global__ void __launch_bounds__(128) k_lsd_nfa_count(const __grid_constant__ LineGeom g, LineWs ws) {
    const int f = blockIdx.y, nj = ws.njobs[f];
    Walk W;
    W.w = g.sw; W.h = g.sh; W.lane = threadIdx.x & 31; W.ang = ws.angdeg + f * g.pix_stride; W.log_nt = g.log_nt; W.lgam = ws.lgam;
    for (int j = blockIdx.x * 4 + (threadIdx.x >> 5); j < nj; j += NFA_COUNT_CTAS * 4) {
        const double* job = ws.jobs + ((long long)f * g.seg_cap + j) * 13;
        LRect rec;
        rec.x1 = job[0]; rec.y1 = job[1]; rec.x2 = job[2]; rec.y2 = job[3]; rec.width = job[4]; rec.theta = job[7]; rec.dx = job[8]; rec.dy = job[9]; rec.prec = job[10];
        int total, alg;
        l_rect_count(W, rec, total, alg);
        if (W.lane == 0) ws.jobnk[(long long)f * g.seg_cap + j] = make_int2(total, alg);
    }
}

__global__ void __launch_bounds__(128) k_lsd_nfa_first(const __grid_constant__ LineGeom g, LineWs ws) {
    const int f = blockIdx.y, nj = ws.njobs[f];
    for (int j = blockIdx.x * 128 + threadIdx.x; j < nj; j += NFA_FIRST_CTAS * 128) {
        const long long q = (long long)f * g.seg_cap + j;
        const int2 nk = ws.jobnk[q];
        double* job = ws.jobs + q * 13;
        const double v = l_nfa(nk.x, nk.y, job[11], g.log_nt, ws.lgam);
        if (v > 0.0) {
            const double tag = job[12];
            ws.jobflag[q] = 1; job[12] = v;
            l_trace_row(g, ws, f, j, job, tag, v);
        } else {
            ws.jobflag[q] = 0; ws.jobnfa[q] = v;
            ws.rej[atomicAdd(ws.rejctl, 1)] = make_int2(f, j);     // order is irrelevant: results go back to the job slot
        }
    }
}

__global__ void __launch_bounds__(128) k_lsd_nfa_improve(const __grid_constant__ LineGeom g, LineWs ws) {
    __shared__ int s_cnt[4][10];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int nrej = ws.rejctl[0];
    for (;;) {
        int r = 0;
        if (lane == 0) r = atomicAdd(ws.rejctl + 1, 1);
        r = __shfl_sync(0xffffffffu, r, 0);
        if (r >= nrej) break;
        const int2 fj = ws.rej[r];
        const int f = fj.x, j = fj.y;
        const long long q = (long long)f * g.seg_cap + j;
        double log_nfa = ws.jobnfa[q];
        double* job = ws.jobs + q * 13;
        Walk W;
        W.w = g.sw; W.h = g.sh; W.lane = lane;
        W.ang = ws.angdeg + f * g.pix_stride; W.log_nt = g.log_nt; W.lgam = ws.lgam;
        LRect rec;
        rec.x1 = job[0]; rec.y1 = job[1]; rec.x2 = job[2]; rec.y2 = job[3]; rec.width = job[4]; rec.x = job[5]; rec.y = job[6];
        rec.theta = job[7]; rec.dx = job[8]; rec.dy = job[9]; rec.prec = job[10]; rec.p = job[11];
        const double tag = job[12];
        __syncwarp();
        log_nfa = l_rect_improve(W, rec, s_cnt[wid], log_nfa);
        __syncwarp();
        if (lane == 0) {
            job[0] = rec.x1; job[1] = rec.y1; job[2] = rec.x2; job[3] = rec.y2; job[4] = rec.width; job[11] = rec.p;
            ws.jobflag[q] = log_nfa > 0.0 ? 1 : 0;
            job[12] = log_nfa;
            l_trace_row(g, ws, f, j, job, tag, log_nfa);
        }
        __syncwarp();
    }
}

// cv::LineIterator(img, p1, p2, 8).count: the endpoints are cvRound()ed floats from [0, lim), so 639.6 becomes 640 — one past
// the last column — and OpenCV clips the segment to the image (cv::clipLine, 64-bit integer arithmetic) before counting.
// Pinned to cv2.clipLine in tests/test_line_oracle_cpu.py through the oracle's identical restatement.
__device__ __forceinline__ int line_iterator_count(int w, int h, int ax, int ay, int bx, int by) {
    long long x1 = ax, y1 = ay, x2 = bx, y2 = by;
    if ((unsigned)ax < (unsigned)w && (unsigned)bx < (unsigned)w && (unsigned)ay < (unsigned)h && (unsigned)by < (unsigned)h)
        return max(abs(bx - ax), abs(by - ay)) + 1;
    const long long right = w - 1, bottom = h - 1;
    int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
    int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
        long long a;
        if (c1 & 12) { a = c1 < 8 ? 0 : bottom; x1 += (a - y1) * (x2 - x1) / (y2 - y1); y1 = a; c1 = (x1 < 0) + (x1 > right) * 2; }
        if (c2 & 12) { a = c2 < 8 ? 0 : bottom; x2 += (a - y2) * (x2 - x1) / (y2 - y1); y2 = a; c2 = (x2 < 0) + (x2 > right) * 2; }
        if ((c1 & c2) == 0 && (c1 | c2) != 0) {
            if (c1) { a = c1 == 1 ? 0 : right; y1 += (a - x1) * (y2 - y1) / (x2 - x1); x1 = a; c1 = 0; }
            if (c2) { a = c2 == 1 ? 0 : right; y2 += (a - x2) * (y2 - y1) / (x2 - x1); x2 = a; c2 = 0; }
        }
    }
    if ((c1 | c2) != 0) return 0;
    const long long dx = x2 > x1 ? x2 - x1 : x1 - x2, dy = y2 > y1 ? y2 - y1 : y1 - y2;
    return (int)(dx > dy ? dx : dy) + 1;
}

// -------------------------------------------------------------------------------------------------
// KeyLine packaging (line_descriptor LSDDetector::detectImpl), top-N by response (ExtractLineSegment.cpp:45-51),
// line equations (:56-68).  One CTA per frame.
// -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_keylines(const __grid_constant__ LineGeom g, LineWs ws) {
    __shared__ int s_warp[33];
    const int f = blockIdx.x, tid = threadIdx.x;
    // accepted jobs -> raw segment list, in detection order
    const int nj = ws.njobs[f];
    int* flag = ws.jobflag + (long long)f * g.seg_cap;
    const int n = block_scan_array(flag, nj, s_warp);              // exclusive offsets in place
    double* segw = ws.seg + (long long)f * g.seg_cap * 4;
    const double* jobs = ws.jobs + (long long)f * g.seg_cap * 13;
    for (int j = tid; j < nj; j += 256)
        if (jobs[(long long)j * 13 + 12] > 0.0) { const int o = flag[j]; for (int k = 0; k < 4; k++) segw[4 * o + k] = jobs[(long long)j * 13 + k]; }
    if (tid == 0) { ws.nseg[f] = n; if (g.trace_cap) ws.ntrace[f] = min(nj, g.trace_cap); }
    __syncthreads();
    const double* seg = segw;
    float* resp = ws.resp + (long long)f * g.seg_cap;
    float4* ext = ws.ext + (long long)f * g.seg_cap;
    const double SCALE = 0.8;
    for (int i = tid; i < n; i += 256) {
        float e[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            double v = seg[4 * i + k] + 0.5;
            v /= SCALE;
            float fv = (float)v;
            const int lim = (k & 1) ? g.h : g.w;                       // checkLineExtremes
            if (fv < 0) fv = 0;
            if (fv >= (float)lim) fv = (float)lim - 1.0f;
            e[k] = fv;
        }
        ext[i] = make_float4(e[0], e[1], e[2], e[3]);
        const float ddx = e[0] - e[2], ddy = e[1] - e[3];
        const float len = (float)sqrt((double)ddx * (double)ddx + (double)ddy * (double)ddy);
        resp[i] = len / (float)max(g.w, g.h);
    }
    __syncthreads();
    const int keep = min(n, g.kl_cap);
    sslpl_keyline* KL = ws.kl + (long long)f * g.kl_cap;
    double* EQ = ws.lineeq + (long long)f * g.kl_cap * 3;
    for (int i = tid; i < n; i += 256) {
        int pos = i;
        if (n > g.kl_cap) {                       // stable rank by descending response
            const float r = resp[i];
            int rank = 0;
            for (int j = 0; j < n; j++) { const float rj = resp[j]; rank += (rj > r) || (rj == r && j < i); }
            pos = rank;
        }
        if (pos >= keep) continue;
        const float4 e = ext[i];
        sslpl_keyline k;
        k.startPointX = e.x; k.startPointY = e.y; k.endPointX = e.z; k.endPointY = e.w;
        k.sPointInOctaveX = e.x; k.sPointInOctaveY = e.y; k.ePointInOctaveX = e.z; k.ePointInOctaveY = e.w;
        const float ddx = e.x - e.z, ddy = e.y - e.w;
        k.lineLength = (float)sqrt((double)ddx * (double)ddx + (double)ddy * (double)ddy);
        const int ax = __float2int_rn(e.x), ay = __float2int_rn(e.y), bx = __float2int_rn(e.z), by = __float2int_rn(e.w);
        k.numOfPixels = line_iterator_count(g.w, g.h, ax, ay, bx, by);  // cv::LineIterator(8-connected).count (after cv::clipLine)
        k.angle = (float)atan2((double)(e.w - e.y), (double)(e.z - e.x));
        k.class_id = pos; k.octave = 0;
        k.size = (e.z - e.x) * (e.w - e.y);
        k.response = resp[i];
        k.pt_x = (e.z + e.x) / 2; k.pt_y = (e.w + e.y) / 2;
        KL[pos] = k;
        const double sx = e.x, sy = e.y, ex = e.z, ey = e.w;
        const double l0 = sy * 1.0 - 1.0 * ey, l1 = 1.0 * ex - sx * 1.0, l2 = sx * ey - sy * ex;
        const double nrm = sqrt(l0 * l0 + l1 * l1);
        EQ[3 * pos] = l0 / nrm; EQ[3 * pos + 1] = l1 / nrm; EQ[3 * pos + 2] = l2 / nrm;
    }
    if (tid == 0) ws.nl[f] = keep;
}

// LBD (BinaryDescriptor::computeLBD, binary_descriptor.cpp) — one CTA (64 threads) per line: thread h walks row h
// of the 63-row line support region sequentially (float sums keep the reference's order), thread 0 folds the rows
// into the 9 bands in row order, then builds the 72-float vector and the 32 pair-comparison bytes.
struct LbdCoef { float G[63]; float L[21]; };
__constant__ int c_comb[32][2] = {{0, 1}, {0, 2}, {0, 3}, {0, 4}, {0, 5}, {0, 6}, {1, 2}, {1, 3}, {1, 4}, {1, 5}, {1, 6}, {2, 3}, {2, 4}, {2, 5}, {2, 6}, {2, 7},
                                  {2, 8}, {3, 4}, {3, 5}, {3, 6}, {3, 7}, {3, 8}, {4, 5}, {4, 6}, {4, 7}, {4, 8}, {5, 6}, {5, 7}, {5, 8}, {6, 7}, {6, 8}, {7, 8}};

__global__ void __launch_bounds__(64) k_lbd(const __grid_constant__ LineGeom g, LineWs ws, const __grid_constant__ LbdCoef C) {
    __shared__ float s_row[63][8];
    __shared__ float s_des[72];
    const int li = blockIdx.x, f = blockIdx.y, h = threadIdx.x;
    if (li >= ws.nl[f]) return;
    const sslpl_keyline kl = ws.kl[(long long)f * g.kl_cap + li];
    const int16_t* dxI = ws.dx + f * g.full_stride; const int16_t* dyI = ws.dy + f * g.full_stride;
    const short imageWidth = (short)(g.w - 1), imageHeight = (short)(g.h - 1);
    const short lengthOfLSP = (short)kl.numOfPixels, halfWidth = (short)((lengthOfLSP - 1) / 2), halfHeight = 31;
    const float mx = (float)(0.5 * (double)(kl.sPointInOctaveX + kl.ePointInOctaveX));
    const float my = (float)(0.5 * (double)(kl.sPointInOctaveY + kl.ePointInOctaveY));
    const float dL0 = (float)cos((double)kl.angle), dL1 = (float)sin((double)kl.angle);
    const float dO0 = -dL1, dO1 = dL0;
    if (h < 63) {
        // sCorX0 after h steps of (sCorX0 -= dL[1]; sCorY0 += dL[0]) — replay the float recurrence exactly
        float sx0 = -dL0 * halfWidth + dL1 * halfHeight + mx;
        float sy0 = -dL1 * halfWidth - dL0 * halfHeight + my;
        for (int k = 0; k < h; k++) { sx0 -= dL1; sy0 += dL0; }
        float sx = sx0, sy = sy0, pL = 0, nL = 0, pO = 0, nO = 0;
        for (short wID = 0; wID < lengthOfLSP; wID++) {
            short t = (short)roundf(sx);
            const short xc = (t < 0) ? 0 : (t > imageWidth) ? imageWidth : t;
            t = (short)roundf(sy);
            const short yc = (t < 0) ? 0 : (t > imageHeight) ? imageHeight : t;
            const short dx = dxI[(int)yc * g.w + xc], dy = dyI[(int)yc * g.w + xc];
            const float gDL = dx * dL0 + dy * dL1, gDO = dx * dO0 + dy * dO1;
            if (gDL > 0) pL += gDL; else nL -= gDL;
            if (gDO > 0) pO += gDO; else nO -= gDO;
            sx += dL0; sy += dL1;
        }
        const float cg = C.G[h];
        pL = cg * pL; nL = cg * nL; pO = cg * pO; nO = cg * nO;
        s_row[h][0] = pL; s_row[h][1] = nL; s_row[h][2] = pL * pL; s_row[h][3] = nL * nL;
        s_row[h][4] = pO; s_row[h][5] = nO; s_row[h][6] = pO * pO; s_row[h][7] = nO * nO;
    }
    __syncthreads();
    if (h < 8) {      // thread q accumulates quantity q of every band, rows in order (same add order as the reference)
        float band[9];
#pragma unroll
        for (int b = 0; b < 9; b++) band[b] = 0;
        const bool sq = (h & 2) != 0;           // quantities 2,3,6,7 use squared local weights
        for (int r = 0; r < 63; r++) {
            const float v = s_row[r][h];
            int b = r / 7;
            float c = C.L[r % 7 + 7];
            band[b] += (sq ? c * c : c) * v;
            b--;
            if (b >= 0) { c = C.L[r % 7 + 14]; band[b] += (sq ? c * c : c) * v; }
            b += 2;
            if (b < 9) { c = C.L[r % 7]; band[b] += (sq ? c * c : c) * v; }
        }
        for (int b = 0; b < 9; b++) s_row[b][h] = band[b];      // reuse rows 0..8 as band sums (all reads are done: see sync)
    }
    __syncthreads();
    if (h == 0) {
        const float invN2 = (float)(1.0 / (7 * 2.0)), invN3 = (float)(1.0 / (7 * 3.0));
        float* d = s_des;
        for (int b = 0; b < 9; b++) {
            const float invN = (b == 0 || b == 8) ? invN2 : invN3;
            float t = s_row[b][0] * invN; d[8 * b] = t; d[8 * b + 4] = sqrtf(s_row[b][2] * invN - t * t);
            t = s_row[b][1] * invN; d[8 * b + 1] = t; d[8 * b + 5] = sqrtf(s_row[b][3] * invN - t * t);
            t = s_row[b][4] * invN; d[8 * b + 2] = t; d[8 * b + 6] = sqrtf(s_row[b][6] * invN - t * t);
            t = s_row[b][5] * invN; d[8 * b + 3] = t; d[8 * b + 7] = sqrtf(s_row[b][7] * invN - t * t);
        }
        float tM = 0, tS = 0;
        for (int b = 0; b < 9; b++) {
            for (int i = 0; i < 4; i++) tM += d[8 * b + i] * d[8 * b + i];
            for (int i = 4; i < 8; i++) tS += d[8 * b + i] * d[8 * b + i];
        }
        tM = 1 / sqrtf(tM); tS = 1 / sqrtf(tS);
        for (int b = 0; b < 9; b++) {
            for (int i = 0; i < 4; i++) d[8 * b + i] = d[8 * b + i] * tM;
            for (int i = 4; i < 8; i++) d[8 * b + i] = d[8 * b + i] * tS;
        }
        for (int i = 0; i < 72; i++) if ((double)d[i] > 0.4) d[i] = (float)0.4;
        float t = 0;
        for (int i = 0; i < 72; i++) t += d[i] * d[i];
        t = 1 / sqrtf(t);
        for (int i = 0; i < 72; i++) d[i] = d[i] * t;
    }
    __syncthreads();
    if (h < 32) {
        const float* f1 = &s_des[8 * c_comb[h][0]]; const float* f2 = &s_des[8 * c_comb[h][1]];
        unsigned r = 0;
#pragma unroll
        for (int i = 0; i < 8; i++) if (f1[i] > f2[i]) r += 0x80u >> i;
        // 32 bytes -> two coalesced 16-byte stores
        uint32_t w = r << (8 * (h & 3));
        w |= __shfl_xor_sync(0xffffffffu, w, 1);
        w |= __shfl_xor_sync(0xffffffffu, w, 2);
        const uint32_t w0 = __shfl_sync(0xffffffffu, w, (h & 16) + 0), w1 = __shfl_sync(0xffffffffu, w, (h & 16) + 4),
                       w2 = __shfl_sync(0xffffffffu, w, (h & 16) + 8), w3 = __shfl_sync(0xffffffffu, w, (h & 16) + 12);
        if ((h & 15) == 0) reinterpret_cast<uint4*>(ws.ldesc + ((long long)f * g.kl_cap + li) * 32)[h >> 4] = make_uint4(w0, w1, w2, w3);
    }
}

}  // namespace sslpl

// =================================================================================================
using namespace sslpl;

struct sslpl_line {
    sslpl_line_params p;
    cudaStream_t stream = nullptr, own_stream = nullptr;
    uint8_t* arena = nullptr; size_t arena_size = 0;
    LineGeom g; LineWs ws; LView view;
    uint8_t* d_input = nullptr;
    LbdCoef coef;
    bool trace = false;
    int used_smem = 0;
    int sm_count = 132;         // replaced by the device's count at creation
    int prep_ctas = 0;          // k_lsd_prep CTAs resident on the whole device at once (occupancy x SMs), at creation
    int max_walkers = 0;        // 0 = one walker CTA per frame
    int walker_warps = 0;       // 0 = automatic (8 or 16 warps per frame)
    int walker_v3 = 0;          // multi-warp walker: 0 = the round-2a form (shipped), 1 = v3 (control warps + workers, O(1) retire), -1 = v3 by frame size
    int used_smem3 = 0, used_smem4 = 0;
    int walker_lanes = 0;       // one warp per frame, lane-parallel region growing (SSLPL_WALKER_LANES=1)
    int walker_lean = 0;        // one-warp walker: 0 = the round-2a form (shipped: faster when several launches overlap), 1 = lean region growing (SSLPL_WALKER_LEAN=1)
    int cur_w = 0, cur_h = 0, cur_frames = 0;
    long long launches = 0;
    int* h_err = nullptr;
    bool profiling = false;
    std::vector<cudaEvent_t> ev; std::vector<const char*> ev_name; int ev_n = 0;
};

namespace {

void lmark(sslpl_line* h, const char* name) {
    if (!h->profiling) return;
    if ((int)h->ev.size() <= h->ev_n) { cudaEvent_t e; cudaEventCreate(&e); h->ev.push_back(e); h->ev_name.push_back(name); }
    h->ev_name[h->ev_n] = name;
    cudaEventRecord(h->ev[h->ev_n++], h->stream);
}

// gradient threshold of lsd.cpp: quant / sin(ang_th) with quant 2, ang_th 22.5 degrees
double lsd_rho() { return 2.0 / std::sin(L_PI * 22.5 / 180); }

void make_geometry(const sslpl_line* h, int W, int H, LineGeom& g, std::vector<int2>* tab) {
    memset(&g, 0, sizeof(g));
    g.w = W; g.h = H; g.pitch = (int)align_up(W, 16);
    g.sw = (int)lrint(W * 0.8); g.sh = (int)lrint(H * 0.8);
    // a tile covers PT_W x PT_H input and PT_SW x PT_SH detection-scale pixels (both counts agree for every size; max() for clarity)
    g.tiles_x = std::max((W + PT_W - 1) / PT_W, (g.sw + PT_SW - 1) / PT_SW); g.tiles_y = std::max((H + PT_H - 1) / PT_H, (g.sh + PT_SH - 1) / PT_SH);
    g.xtab_off = 0; g.ytab_off = g.sw;
    g.in_stride = (long long)g.pitch * H;
    g.pix_stride = (long long)g.sw * g.sh;
    g.full_stride = (long long)W * H;
    g.kl_cap = h->p.lsdNFeatures;
    // lsd.cpp constants (ANG_TH 22.5, QUANT 2.0); host libm, exactly as the CPU implementation evaluates them
    g.prec = L_PI * 22.5 / 180; g.p = 22.5 / 180; g.rho = lsd_rho();
    g.log_nt = 5 * (std::log10(double(g.sw)) + std::log10(double(g.sh))) / 2 + std::log10(11.0);
    g.min_reg_size = (int)size_t(-g.log_nt / std::log10(g.p));
    g.seg_cap = (int)(g.pix_stride / std::max(g.min_reg_size, 1)) + 16;
    g.trace_cap = h->trace ? g.seg_cap : 0;
    g.dbg = getenv("SSLPL_WALKER_DBG") ? atoi(getenv("SSLPL_WALKER_DBG")) : 0;
    g.dbg_seed = getenv("SSLPL_WALKER_SEED") ? atoi(getenv("SSLPL_WALKER_SEED")) : -1;
    if (tab) {
        tab->assign(g.sw + g.sh, make_int2(0, 0));
        for (int axis = 0; axis < 2; axis++) {
            const int dn = axis ? g.sh : g.sw, sn = axis ? H : W, off = axis ? g.ytab_off : g.xtab_off;
            // cv::resize(..., Size(), 0.8, 0.8, INTER_LINEAR_EXACT) maps with scale = 1 / fx = 1.25, not sn / dn (resize.cpp)
            const double sc = 1.0 / 0.8; (void)sn;
            for (int d = 0; d < dn; d++) {
                double s = (d + 0.5) * sc - 0.5;
                int i0 = (int)floor(s);
                double f = s - i0;
                if (i0 < 0) { i0 = 0; f = 0; }
                if (i0 >= sn - 1) { i0 = sn - 1; f = 0; }
                (*tab)[off + d] = make_int2(i0, (int)lrint(f * 256));
            }
        }
    }
}

void carve(sslpl_line* h, Arena& A, const LineGeom& g, int B) {
    LineWs& ws = h->ws;
    h->d_input = A.take<uint8_t>((size_t)B * g.in_stride + 256);
    ws.angdeg = A.take<float>((size_t)B * g.pix_stride); ws.pix = A.take<LPix>((size_t)B * g.pix_stride);
    ws.modgrad = A.take<double>((size_t)B * g.pix_stride); ws.cs0 = A.take<float2>((size_t)B * g.pix_stride);
    ws.maxgrad = A.take<unsigned long long>(B); ws.prep_next = A.take<int>(1);
    ws.seeds = A.take<unsigned>((size_t)B * g.pix_stride); ws.nseeds = A.take<int>(B);
    ws.reg = A.take<unsigned>((size_t)B * g.pix_stride);
    ws.sreg = A.take<unsigned>((size_t)B * WALK_RING * WALK_SLOT_CAP); ws.sjob = A.take<double>((size_t)B * V3_RING * 13); ws.rcode = A.take<unsigned char>((size_t)B * V3_RANKS); ws.dlist = A.take<unsigned>((size_t)B * V3_DPOOL);
    ws.wstat = A.take<unsigned long long>(16);
    ws.seg = A.take<double>((size_t)B * g.seg_cap * 4); ws.nseg = A.take<int>(B);
    ws.jobs = A.take<double>((size_t)B * g.seg_cap * 13); ws.njobs = A.take<int>(B); ws.jobflag = A.take<int>((size_t)B * g.seg_cap);
    ws.jobnk = A.take<int2>((size_t)B * g.seg_cap); ws.jobnfa = A.take<double>((size_t)B * g.seg_cap);
    ws.rej = A.take<int2>((size_t)B * g.seg_cap); ws.rejctl = A.take<int>(4);

    ws.dx = A.take<int16_t>((size_t)B * g.full_stride); ws.dy = A.take<int16_t>((size_t)B * g.full_stride);
    ws.tab = A.take<int2>(g.sw + g.sh);
    ws.resp = A.take<float>((size_t)B * g.seg_cap); ws.ext = A.take<float4>((size_t)B * g.seg_cap);
    ws.kl = A.take<sslpl_keyline>((size_t)B * g.kl_cap); ws.ldesc = A.take<uint8_t>((size_t)B * g.kl_cap * 32);
    ws.lineeq = A.take<double>((size_t)B * g.kl_cap * 3); ws.nl = A.take<int>(B);
    ws.err = A.take<int>(1);
    ws.trace = A.take<double>((size_t)B * g.trace_cap * 10 + 16); ws.ntrace = A.take<int>(B);
    ws.lgam = A.take<double>((size_t)g.pix_stride + 2);
}

// log_gamma of lsd.cpp on the host (same libm as the CPU implementation): Lanczos for x <= 15, Windschitl above
double host_log_gamma(double x) {
    if (x > 15.0) return 0.918938533204673 + (x - 0.5) * std::log(x) - x + 0.5 * x * std::log(x * std::sinh(1 / x) + 1 / (810.0 * std::pow(x, 6.0)));
    static const double q[7] = {75122.6331530, 80916.6278952, 36308.2951477, 8687.24529705, 1168.92649479, 83.8676043424, 2.50662827511};
    double a = (x + 0.5) * std::log(x + 5.5) - (x + 5.5), b = 0;
    for (int n = 0; n < 7; ++n) { a -= std::log(x + double(n)); b += q[n] * std::pow(x, double(n)); }
    return a + std::log(b);
}

int configure(sslpl_line* h, int W, int H) {
    if (W == h->cur_w && H == h->cur_h) return SSLPL_OK;
    SSLPL_REQUIRE(W <= h->p.max_width && H <= h->p.max_height, SSLPL_ERR_ARG, "frame larger than the handle's max_width/max_height");
    SSLPL_REQUIRE(W >= 16 && H >= 16 && W < 32768 && H < 32768, SSLPL_ERR_ARG, "frame size out of range");
    std::vector<int2> tab;
    make_geometry(h, W, H, h->g, &tab);
    Arena A; A.base = h->arena; A.size = h->arena_size;
    carve(h, A, h->g, h->p.max_batch);
    SSLPL_REQUIRE(A.used <= h->arena_size, SSLPL_ERR_CAPACITY, "internal: arena too small for this frame size");
    SSLPL_CUDA(cudaStreamSynchronize(h->stream));
    SSLPL_CUDA(cudaMemcpy(h->ws.tab, tab.data(), tab.size() * sizeof(int2), cudaMemcpyHostToDevice));
    SSLPL_CUDA(cudaMemset(h->ws.err, 0, sizeof(int)));
    {
        std::vector<double> lg((size_t)h->g.pix_stride + 2);
        for (size_t n = 0; n < lg.size(); n++) lg[n] = host_log_gamma((double)n + 1.0);
        SSLPL_CUDA(cudaMemcpy(const_cast<double*>(h->ws.lgam), lg.data(), lg.size() * sizeof(double), cudaMemcpyHostToDevice));
    }
    h->cur_w = W; h->cur_h = H;
    return SSLPL_OK;
}

int run_pipeline(sslpl_line* h, int B) {
    const LineGeom& g = h->g;
    cudaStream_t st = h->stream;
    h->ev_n = 0;
    lmark(h, "start");
    SSLPL_CUDA(cudaMemsetAsync(h->ws.maxgrad, 0, sizeof(unsigned long long) * B, st));
    SSLPL_CUDA(cudaMemsetAsync(h->ws.prep_next, 0, sizeof(int), st));
    k_lsd_prep<<<std::min(h->prep_ctas, g.tiles_x * g.tiles_y * B), PT_NT, 0, st>>>(g, h->view, h->ws, B);      // blurs, resize, ll_angle, Sobel
    lmark(h, "lsd_prep");
    k_lsd_seeds<<<B, SEED_WARPS * 32, 0, st>>>(g, h->ws);
    lmark(h, "lsd_seeds");
    SSLPL_CUDA(cudaMemsetAsync(h->ws.rejctl, 0, 4 * sizeof(int), st));
    SSLPL_CUDA(cudaMemsetAsync(h->ws.wstat, 0, 16 * sizeof(unsigned long long), st));
    {   // one CTA per frame; few frames -> more warps per frame (latency), many frames -> more CTAs per SM (throughput)
        // automatic choice: big batches -> one warp per frame (throughput); one or a few frames -> a multi-warp CTA per frame, the
        // round-2a walker with 16 warps.  v3 (SSLPL_WALKER_V3=1, 8 warps) is at best level with it on 640x480 frames and behind on
        // 1280x960 (its deeper speculation loses more work than it overlaps), so it is not the default; SSLPL_WALKER_V3=-1 picks it by
        // frame size (up to ~0.3 M detection-scale pixels)
        const bool small = g.pix_stride <= 300000;
        const bool v3 = h->walker_v3 > 0 || (h->walker_v3 < 0 && small);
        const int ww = h->walker_warps < 0 ? 0 : h->walker_warps > 0 ? std::min(h->walker_warps, WALK_MAXW) : (B >= 2 * h->sm_count ? 0 : (v3 ? 8 : WALK_MAXW));
        const size_t smem = (size_t)((g.pix_stride + 31) / 32) * sizeof(unsigned);
        if ((int)smem > h->used_smem) { SSLPL_CUDA(cudaFuncSetAttribute(k_lsd_regions, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); h->used_smem = (int)smem; }
        if (h->walker_lanes && ww == 0) {
            const size_t sm4 = sizeof(V3Shared);
            if ((int)sm4 > h->used_smem4) { SSLPL_CUDA(cudaFuncSetAttribute(k_lsd_regions_lanes, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm4)); h->used_smem4 = (int)sm4; }
            k_lsd_regions_lanes<<<(h->max_walkers > 0 ? std::min(B, h->max_walkers) : B), 32, sm4, st>>>(g, h->ws, B);
        }
        else if (ww >= 2 && v3) {
            const size_t sm3 = sizeof(V3Shared) + (size_t)ww * V3_LRING * sizeof(unsigned);
            if ((int)sm3 > h->used_smem3) { SSLPL_CUDA(cudaFuncSetAttribute(k_lsd_regions_v3, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm3)); h->used_smem3 = (int)sm3; }
            k_lsd_regions_v3<<<(h->max_walkers > 0 ? std::min(B, h->max_walkers) : B), ww * 32, sm3, st>>>(g, h->ws, B);
        }
        else if (ww == 0 && h->walker_lean) k_lsd_regions_lean<<<(h->max_walkers > 0 ? std::min(B, h->max_walkers) : B), 32, 0, st>>>(g, h->ws, B);   // one warp per frame
        else if (ww == 0) k_lsd_regions_solo<<<(h->max_walkers > 0 ? std::min(B, h->max_walkers) : B), 32, 0, st>>>(g, h->ws, B);              // round-2a form (A/B)
        else k_lsd_regions<<<(h->max_walkers > 0 ? std::min(B, h->max_walkers) : B), ww * 32, smem, st>>>(g, h->ws, B);
    }
    lmark(h, "lsd_regions");
    k_lsd_nfa_count<<<dim3(NFA_COUNT_CTAS, B), 128, 0, st>>>(g, h->ws);
    k_lsd_nfa_first<<<dim3(NFA_FIRST_CTAS, B), 128, 0, st>>>(g, h->ws);
    k_lsd_nfa_improve<<<std::min(h->sm_count * 8, (B * 64 + 3) / 4), 128, 0, st>>>(g, h->ws);
    lmark(h, "lsd_nfa");
    k_keylines<<<B, 256, 0, st>>>(g, h->ws);
    k_lbd<<<dim3(g.kl_cap, B), 64, 0, st>>>(g, h->ws, h->coef);
    lmark(h, "keylines_lbd");
    h->launches += 8;      // kernels only (the three small memsets are not counted)
    SSLPL_CUDA(cudaGetLastError());
    return SSLPL_OK;
}

int check_device_err(sslpl_line* h) {
    if (h->cur_w == 0) { SSLPL_CUDA(cudaStreamSynchronize(h->stream)); return SSLPL_OK; }     // never used yet: no workspace, nothing to report
    SSLPL_CUDA(cudaMemcpyAsync(h->h_err, h->ws.err, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    SSLPL_CUDA(cudaStreamSynchronize(h->stream));
    if (*h->h_err) {
        set_error("device-side capacity overflow in the line path, flags=0x%x", *h->h_err);
        cudaMemsetAsync(h->ws.err, 0, sizeof(int), h->stream);
        return SSLPL_ERR_CAPACITY;
    }
    return SSLPL_OK;
}

}  // namespace

extern "C" {

int sslpl_line_create(const sslpl_line_params* p, sslpl_line** out) {
    SSLPL_REQUIRE(p && out, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(p->lsdNFeatures >= 1 && p->lsdNFeatures <= 65536, SSLPL_ERR_ARG, "lsdNFeatures out of range");
    SSLPL_REQUIRE(p->max_batch >= 1 && p->max_width >= 16 && p->max_height >= 16, SSLPL_ERR_ARG, "bad max_batch / max size");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { set_error("no CUDA device available: libsslpl_b200 has no CPU fallback"); return SSLPL_ERR_CUDA; }
    SSLPL_CUDA(cudaSetDevice(p->device));
    sslpl_line* h = new sslpl_line();
    h->p = *p;
    { int v = 0; if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, p->device) == cudaSuccess && v > 0) h->sm_count = v; }
    {   // the persistent pre-pass fills the device once; tiles beyond that are taken from its counter
        int occ = 0;
        const cudaError_t oe = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_lsd_prep, PT_NT, 0);
        if (oe != cudaSuccess || occ < 1) { set_error("k_lsd_prep occupancy query failed: %s", cudaGetErrorString(oe)); delete h; return SSLPL_ERR_CUDA; }
        h->prep_ctas = occ * h->sm_count;
    }
    h->trace = getenv("SSLPL_LINE_TRACE") != nullptr;
    if (const char* e = getenv("SSLPL_WALKER_LANES")) h->walker_lanes = atoi(e) != 0;
    if (const char* e = getenv("SSLPL_WALKER_V3")) h->walker_v3 = atoi(e) < 0 ? -1 : (atoi(e) != 0 ? 1 : 0);
    if (const char* e = getenv("SSLPL_WALKER_LEAN")) h->walker_lean = atoi(e) != 0;
    if (const char* e = getenv("SSLPL_WALKER_WARPS")) h->walker_warps = std::max(-1, std::min(WALK_MAXW, atoi(e)));   // tuning knob (tests sweep it); -1 = the one-warp throughput kernel
    {   // BinaryDescriptor constructor: local (F_l) and global (F_g) Gaussian weights, widthOfBand 7, 9 bands
        double u = (7 * 3 - 1) / 2, sigma = (7 * 2 + 1) / 2, inv = -1 / (2 * sigma * sigma);
        for (int i = 0; i < 21; i++) { const double d = i - u; h->coef.L[i] = (float)exp(d * d * inv); }
        u = (9 * 7 - 1) / 2; sigma = u; inv = -1 / (2 * sigma * sigma);
        for (int i = 0; i < 63; i++) { const double d = i - u; h->coef.G[i] = (float)exp(d * d * inv); }
    }
    LineGeom g;
    make_geometry(h, p->max_width, p->max_height, g, nullptr);
    Arena A; carve(h, A, g, p->max_batch);
    h->arena_size = A.used + (1 << 20);
    cudaError_t e = cudaMalloc(&h->arena, h->arena_size);
    if (e != cudaSuccess) { set_error("cudaMalloc(%zu) failed: %s", h->arena_size, cudaGetErrorString(e)); delete h; return SSLPL_ERR_CUDA; }
    SSLPL_CUDA(cudaMemset(h->arena, 0, h->arena_size));
    SSLPL_CUDA(cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking));
    h->stream = h->own_stream;
    SSLPL_CUDA(cudaHostAlloc((void**)&h->h_err, sizeof(int), cudaHostAllocDefault));
    *out = h;
    return SSLPL_OK;
}

void sslpl_line_destroy(sslpl_line* h) {
    if (!h) return;
    cudaSetDevice(h->p.device);
    // an external stream may already be gone (its owner was destroyed first): never touch it here
    if (h->stream && h->stream == h->own_stream) cudaStreamSynchronize(h->own_stream); else cudaDeviceSynchronize();
    if (h->own_stream) cudaStreamDestroy(h->own_stream);
    for (auto e : h->ev) cudaEventDestroy(e);
    if (h->arena) cudaFree(h->arena);
    if (h->h_err) cudaFreeHost(h->h_err);
    delete h;
}

int sslpl_line_sync(sslpl_line* h) { SSLPL_REQUIRE(h, SSLPL_ERR_ARG, "null handle"); SSLPL_CUDA(cudaSetDevice(h->p.device)); return check_device_err(h); }
void* sslpl_line_stream(sslpl_line* h) { return h ? (void*)h->stream : nullptr; }
int sslpl_line_set_stream(sslpl_line* h, void* s) {
    SSLPL_REQUIRE(h, SSLPL_ERR_ARG, "null handle");
    SSLPL_CUDA(cudaSetDevice(h->p.device));
    SSLPL_CUDA(cudaStreamSynchronize(h->stream));
    h->stream = s ? (cudaStream_t)s : h->own_stream;
    return SSLPL_OK;
}
long long sslpl_line_launch_count(const sslpl_line* h) { return h ? h->launches : 0; }
int sslpl_line_set_max_walkers(sslpl_line* h, int max_concurrent) {
    SSLPL_REQUIRE(h && max_concurrent >= 0, SSLPL_ERR_ARG, "bad argument");
    h->max_walkers = max_concurrent;
    return SSLPL_OK;
}
int sslpl_line_set_profiling(sslpl_line* h, int on) { SSLPL_REQUIRE(h, SSLPL_ERR_ARG, "null handle"); h->profiling = on != 0; return SSLPL_OK; }
int sslpl_line_stage_ms(sslpl_line* h, float* ms, int cap, const char** names, int* nstages) {
    SSLPL_REQUIRE(h && nstages, SSLPL_ERR_ARG, "null argument");
    SSLPL_CUDA(cudaStreamSynchronize(h->stream));
    int k = 0;
    for (int i = 1; i < h->ev_n; i++, k++)
        if (k < cap) { float t = 0; cudaEventElapsedTime(&t, h->ev[i - 1], h->ev[i]); if (ms) ms[k] = t; if (names) names[k] = h->ev_name[i]; }
    *nstages = k;
    return SSLPL_OK;
}

int sslpl_line_extract_batch_device(sslpl_line* h, const uint8_t* d_imgs, int nframes, int width, int height, int pitch, size_t frame_stride) {
    SSLPL_REQUIRE(h && d_imgs, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(nframes >= 1 && nframes <= h->p.max_batch && pitch >= width, SSLPL_ERR_ARG, "bad nframes / pitch");
    SSLPL_CUDA(cudaSetDevice(h->p.device));
    int rc = configure(h, width, height);
    if (rc) return rc;
    h->view.base = d_imgs; h->view.pitch = pitch; h->view.frame_stride = (long long)frame_stride;
    h->cur_frames = nframes;
    return run_pipeline(h, nframes);
}

int sslpl_line_device_results(sslpl_line* h, const sslpl_keyline** d_kl, const uint8_t** d_ldesc, const double** d_lineeq, const int** d_n, int* cap) {
    SSLPL_REQUIRE(h, SSLPL_ERR_ARG, "null handle");
    if (d_kl) *d_kl = h->ws.kl;
    if (d_ldesc) *d_ldesc = h->ws.ldesc;
    if (d_lineeq) *d_lineeq = h->ws.lineeq;
    if (d_n) *d_n = h->ws.nl;
    if (cap) *cap = h->p.lsdNFeatures;
    return SSLPL_OK;
}

int sslpl_line_extract_batch_begin(sslpl_line* h, const uint8_t* imgs, int nframes, int width, int height, int pitch, size_t frame_stride,
                                   sslpl_keyline* kl, uint8_t* ldesc, double* lineeq, int cap, int* n) {
    SSLPL_REQUIRE(h && kl && ldesc && lineeq && n && imgs, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(nframes >= 1 && nframes <= h->p.max_batch && pitch >= width, SSLPL_ERR_ARG, "bad nframes / pitch");
    SSLPL_REQUIRE(cap >= h->p.lsdNFeatures, SSLPL_ERR_CAPACITY, "caller line capacity smaller than lsdNFeatures");
    SSLPL_CUDA(cudaSetDevice(h->p.device));
    int rc = configure(h, width, height);
    if (rc) return rc;
    const LineGeom& g = h->g;
    if (frame_stride == (size_t)pitch * height)
        SSLPL_CUDA(cudaMemcpy2DAsync(h->d_input, g.pitch, imgs, pitch, width, (size_t)height * nframes, cudaMemcpyHostToDevice, h->stream));
    else
        for (int f = 0; f < nframes; f++)
            SSLPL_CUDA(cudaMemcpy2DAsync(h->d_input + f * g.in_stride, g.pitch, imgs + f * frame_stride, pitch, width, height, cudaMemcpyHostToDevice, h->stream));
    h->view.base = h->d_input; h->view.pitch = g.pitch; h->view.frame_stride = g.in_stride;
    h->cur_frames = nframes;
    rc = run_pipeline(h, nframes);
    if (rc) return rc;
    const int kc = g.kl_cap;
    SSLPL_CUDA(cudaMemcpyAsync(n, h->ws.nl, sizeof(int) * nframes, cudaMemcpyDeviceToHost, h->stream));
    SSLPL_CUDA(cudaMemcpy2DAsync(kl, (size_t)cap * sizeof(sslpl_keyline), h->ws.kl, (size_t)kc * sizeof(sslpl_keyline), (size_t)kc * sizeof(sslpl_keyline), nframes, cudaMemcpyDeviceToHost, h->stream));
    SSLPL_CUDA(cudaMemcpy2DAsync(ldesc, (size_t)cap * 32, h->ws.ldesc, (size_t)kc * 32, (size_t)kc * 32, nframes, cudaMemcpyDeviceToHost, h->stream));
    SSLPL_CUDA(cudaMemcpy2DAsync(lineeq, (size_t)cap * 24, h->ws.lineeq, (size_t)kc * 24, (size_t)kc * 24, nframes, cudaMemcpyDeviceToHost, h->stream));
    return SSLPL_OK;
}

int sslpl_line_extract_batch(sslpl_line* h, const uint8_t* imgs, int nframes, int width, int height, int pitch, size_t frame_stride,
                             sslpl_keyline* kl, uint8_t* ldesc, double* lineeq, int cap, int* n) {
    int rc = sslpl_line_extract_batch_begin(h, imgs, nframes, width, height, pitch, frame_stride, kl, ldesc, lineeq, cap, n);
    if (rc) return rc;
    return check_device_err(h);
}

int sslpl_line_extract(sslpl_line* h, const uint8_t* img, int width, int height, int pitch, sslpl_keyline* kl, uint8_t* ldesc, double* lineeq, int cap, int* n) {
    return sslpl_line_extract_batch(h, img, 1, width, height, pitch, (size_t)pitch * height, kl, ldesc, lineeq, cap, n);
}

int sslpl_line_download_segments(sslpl_line* h, int frame, float* seg4, int cap, int* n) {
    SSLPL_REQUIRE(h && n && frame >= 0 && frame < h->cur_frames, SSLPL_ERR_ARG, "bad argument");
    SSLPL_CUDA(cudaSetDevice(h->p.device));
    SSLPL_CUDA(cudaStreamSynchronize(h->stream));
    int cnt = 0;
    SSLPL_CUDA(cudaMemcpy(&cnt, h->ws.nseg + frame, sizeof(int), cudaMemcpyDeviceToHost));
    std::vector<double> s((size_t)std::max(cnt, 1) * 4);
    if (cnt) SSLPL_CUDA(cudaMemcpy(s.data(), h->ws.seg + (size_t)frame * h->g.seg_cap * 4, sizeof(double) * 4 * cnt, cudaMemcpyDeviceToHost));
    for (int i = 0; i < cnt && i < cap; i++)
        for (int k = 0; k < 4; k++) { double v = s[4 * i + k] + 0.5; v /= 0.8; seg4[4 * i + k] = (float)v; }
    *n = cnt;
    return SSLPL_OK;
}

// Region growing changes only LPix.used after k_lsd_prep / k_lsd_seeds, so these planes are still the pre-pass's after a full call.
int sslpl_line_download_prep(sslpl_line* h, int frame, int* w, int* hgt, int* sw, int* sh, int16_t* dx, int16_t* dy, float* angdeg,
                             float* pix_cs, float* cs0, double* modgrad, double* maxgrad, uint32_t* seeds, int* nseeds) {
    SSLPL_REQUIRE(h && frame >= 0 && frame < h->cur_frames, SSLPL_ERR_ARG, "bad argument");
    SSLPL_CUDA(cudaSetDevice(h->p.device));
    SSLPL_CUDA(cudaStreamSynchronize(h->stream));
    const LineGeom& g = h->g;
    const size_t np = (size_t)g.pix_stride, nf = (size_t)g.full_stride, po = (size_t)frame * np, fo = (size_t)frame * nf;
    if (w) *w = g.w;
    if (hgt) *hgt = g.h;
    if (sw) *sw = g.sw;
    if (sh) *sh = g.sh;
    if (dx) SSLPL_CUDA(cudaMemcpy(dx, h->ws.dx + fo, nf * sizeof(int16_t), cudaMemcpyDeviceToHost));
    if (dy) SSLPL_CUDA(cudaMemcpy(dy, h->ws.dy + fo, nf * sizeof(int16_t), cudaMemcpyDeviceToHost));
    if (angdeg) SSLPL_CUDA(cudaMemcpy(angdeg, h->ws.angdeg + po, np * sizeof(float), cudaMemcpyDeviceToHost));
    if (pix_cs) SSLPL_CUDA(cudaMemcpy2D(pix_cs, 2 * sizeof(float), &h->ws.pix[po].cx, sizeof(LPix), 2 * sizeof(float), np, cudaMemcpyDeviceToHost));
    if (cs0) SSLPL_CUDA(cudaMemcpy(cs0, h->ws.cs0 + po, np * sizeof(float2), cudaMemcpyDeviceToHost));
    if (modgrad) SSLPL_CUDA(cudaMemcpy(modgrad, h->ws.modgrad + po, np * sizeof(double), cudaMemcpyDeviceToHost));
    if (maxgrad) {
        unsigned long long bits = 0;
        SSLPL_CUDA(cudaMemcpy(&bits, h->ws.maxgrad + frame, sizeof(bits), cudaMemcpyDeviceToHost));
        memcpy(maxgrad, &bits, sizeof(double));
    }
    int cnt = 0;
    SSLPL_CUDA(cudaMemcpy(&cnt, h->ws.nseeds + frame, sizeof(int), cudaMemcpyDeviceToHost));
    if (seeds && cnt > 0) SSLPL_CUDA(cudaMemcpy(seeds, h->ws.seeds + po, (size_t)cnt * sizeof(unsigned), cudaMemcpyDeviceToHost));
    if (nseeds) *nseeds = cnt;
    return SSLPL_OK;
}

int sslpl_line_debug_ll_table(sslpl_line* h, float* angdeg, float* cs, float* cs0, double* modgrad) {
    SSLPL_REQUIRE(h, SSLPL_ERR_ARG, "null handle");
    SSLPL_CUDA(cudaSetDevice(h->p.device));
    SSLPL_CUDA(cudaStreamSynchronize(h->stream));
    constexpr size_t N = (size_t)LL_SPAN * LL_SPAN;
    uint8_t* buf = nullptr;
    SSLPL_CUDA(cudaMalloc(&buf, N * (sizeof(float) + 2 * sizeof(float2) + sizeof(double))));
    double* d_norm = reinterpret_cast<double*>(buf);
    float2* d_cs = reinterpret_cast<float2*>(d_norm + N);
    float2* d_cs0 = d_cs + N;
    float* d_ang = reinterpret_cast<float*>(d_cs0 + N);
    k_ll_table<<<(unsigned)((N + 255) / 256), 256, 0, h->stream>>>(lsd_rho(), d_ang, d_cs, d_cs0, d_norm);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e == cudaSuccess && angdeg) e = cudaMemcpy(angdeg, d_ang, N * sizeof(float), cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && cs) e = cudaMemcpy(cs, d_cs, N * sizeof(float2), cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && cs0) e = cudaMemcpy(cs0, d_cs0, N * sizeof(float2), cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && modgrad) e = cudaMemcpy(modgrad, d_norm, N * sizeof(double), cudaMemcpyDeviceToHost);
    cudaFree(buf);
    SSLPL_CUDA(e);
    return SSLPL_OK;
}

/* debug (SSLPL_LINE_TRACE=1 at handle creation): one row of 10 doubles per region that reached region2rect */
/* Statistics of the last region-walker launch (16 values; collected with SSLPL_WALKER_DBG=32).  For the round-2a multi-warp walker as
   listed below; the v3 and lane-parallel walkers fill the same array with their own counters (tools/v3_stats.py, tools/lanes_stats.py
   name them).  Round-2a: [0] regions grown by the turn holder, [1] their clock cycles, [2] their
   pixels, [3] -, [4] claims whose seed had been swallowed by commit time, [5] redone by the turn holder: abandoned, [6] poisoned,
   [7] failed validation, [8] presumed swallowed but not, [9] attempts committed as speculated, [10] their pixels, [11] cycles
   under the commit lock, [12] under the claim lock, [13] attempts repeated after a lower rank retired, [14] cycles per frame
   (summed), [15] claims. */
int sslpl_line_walker_stats(sslpl_line* h, unsigned long long* out16) {
    SSLPL_REQUIRE(h && out16, SSLPL_ERR_ARG, "null argument");
    SSLPL_CUDA(cudaSetDevice(h->p.device));
    SSLPL_CUDA(cudaStreamSynchronize(h->stream));
    SSLPL_CUDA(cudaMemcpy(out16, h->ws.wstat, 16 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return SSLPL_OK;
}
int sslpl_line_debug_trace(sslpl_line* h, int frame, double* out, int cap_rows, int* n) {
    SSLPL_REQUIRE(h && n && frame >= 0 && frame < h->cur_frames, SSLPL_ERR_ARG, "bad argument");
    SSLPL_REQUIRE(h->g.trace_cap > 0, SSLPL_ERR_UNSUPPORTED, "tracing is off (set SSLPL_LINE_TRACE=1 before creating the handle)");
    SSLPL_CUDA(cudaSetDevice(h->p.device));
    SSLPL_CUDA(cudaStreamSynchronize(h->stream));
    int cnt = 0;
    SSLPL_CUDA(cudaMemcpy(&cnt, h->ws.ntrace + frame, sizeof(int), cudaMemcpyDeviceToHost));
    const int m = std::min(cnt, cap_rows);
    if (m > 0) SSLPL_CUDA(cudaMemcpy(out, h->ws.trace + (size_t)frame * h->g.trace_cap * 10, sizeof(double) * 10 * m, cudaMemcpyDeviceToHost));
    *n = cnt;
    return SSLPL_OK;
}

}  // extern "C"
