// oracle/refshim/minicv.cpp — TEST INFRASTRUCTURE ONLY.  Implementation of the OpenCV stand-in (see minicv.hpp):
// image primitives forward to the cv2-pinned oracle primitives (oracle/oracle.h), Mat arithmetic follows cv::gemm as
// probed on cv2 4.13 (tools/probe_cv_gemm.py).
#include "minicv.hpp"
#include "opencv2/line_descriptor/descriptor.hpp"
#include "../oracle.h"

namespace cv {

double Mat::getd(int r, int c) const {
    switch (depth()) {
        case CV_8U: return at<uchar>(r, c);
        case CV_16S: return at<short>(r, c);
        case CV_32S: return at<int>(r, c);
        case CV_32F: return at<float>(r, c);
        case CV_64F: return at<double>(r, c);
    }
    assert(!"minicv: unsupported depth"); return 0;
}
void Mat::setd(int r, int c, double v) {
    switch (depth()) {
        case CV_8U: at<uchar>(r, c) = (uchar)std::min(255, std::max(0, cvRound(v))); return;
        case CV_16S: at<short>(r, c) = (short)std::min(32767, std::max(-32768, cvRound(v))); return;
        case CV_32S: at<int>(r, c) = cvRound(v); return;
        case CV_32F: at<float>(r, c) = (float)v; return;
        case CV_64F: at<double>(r, c) = v; return;
    }
    assert(!"minicv: unsupported depth");
}
Mat& Mat::setTo(const Scalar& s) { for (int r = 0; r < rows; r++) for (int c = 0; c < cols; c++) setd(r, c, s.val[0]); return *this; }
void Mat::convertTo(Mat& dst, int rtype, double alpha, double beta) const {
    Mat out(rows, cols, rtype < 0 ? type() : rtype);
    for (int r = 0; r < rows; r++) for (int c = 0; c < cols; c++) out.setd(r, c, getd(r, c) * alpha + beta);
    dst = out;
}
Mat Mat::transposed() const { Mat m(cols, rows, type()); for (int r = 0; r < rows; r++) for (int c = 0; c < cols; c++) m.setd(c, r, getd(r, c)); return m; }
double Mat::dot(const Mat& m) const {        // cv::Mat::dot: double accumulator over the elements in order
    assert(total() == m.total());
    double s = 0; const int n = (int)total();
    for (int i = 0; i < n; i++) s += getd(i / cols, i % cols) * m.getd(i / m.cols, i % m.cols);
    return s;
}
Mat Mat::cross(const Mat& m) const {
    assert(total() == 3 && m.total() == 3);
    Mat o(rows, cols, type());
    auto g = [](const Mat& a, int i) { return a.getd(i / a.cols, i % a.cols); };
    const double v[3] = {g(*this, 1) * g(m, 2) - g(*this, 2) * g(m, 1), g(*this, 2) * g(m, 0) - g(*this, 0) * g(m, 2), g(*this, 0) * g(m, 1) - g(*this, 1) * g(m, 0)};
    for (int i = 0; i < 3; i++) o.setd(i / cols, i % cols, v[i]);
    return o;
}
Mat Mat::mul(const Mat& m, double scale) const {
    Mat o(rows, cols, type());
    for (int r = 0; r < rows; r++) for (int c = 0; c < cols; c++) o.setd(r, c, getd(r, c) * m.getd(r, c) * scale);
    return o;
}
Mat Mat::inv(int) const {                     // Gauss-Jordan in double; only reached from code outside the tested path
    assert(rows == cols);
    const int n = rows; std::vector<double> a((size_t)n * 2 * n, 0.0);
    for (int r = 0; r < n; r++) { for (int c = 0; c < n; c++) a[(size_t)r * 2 * n + c] = getd(r, c); a[(size_t)r * 2 * n + n + r] = 1; }
    for (int i = 0; i < n; i++) {
        int p = i; for (int r = i + 1; r < n; r++) if (fabs(a[(size_t)r * 2 * n + i]) > fabs(a[(size_t)p * 2 * n + i])) p = r;
        if (a[(size_t)p * 2 * n + i] == 0) return Mat::zeros(n, n, type());
        for (int c = 0; c < 2 * n; c++) std::swap(a[(size_t)i * 2 * n + c], a[(size_t)p * 2 * n + c]);
        const double d = a[(size_t)i * 2 * n + i];
        for (int c = 0; c < 2 * n; c++) a[(size_t)i * 2 * n + c] /= d;
        for (int r = 0; r < n; r++) if (r != i) { const double f = a[(size_t)r * 2 * n + i]; for (int c = 0; c < 2 * n; c++) a[(size_t)r * 2 * n + c] -= f * a[(size_t)i * 2 * n + c]; }
    }
    Mat o(n, n, type());
    for (int r = 0; r < n; r++) for (int c = 0; c < n; c++) o.setd(r, c, a[(size_t)r * 2 * n + n + c]);
    return o;
}

// cv::gemm as observed on cv2 4.13 (tools/probe_cv_gemm.py, 3000 random cases per shape, all bit-equal):
//  CV_32F with inner length 2..4 equal to the output width or height: float products summed left to right in float,
//  then (float)(sum*alpha + c*beta) (alpha = +-1 probed); otherwise — other shapes, or a transposed operand (GEMM_1_T / GEMM_2_T,
//  e.g. -Rcw.t()*tcw) — double accumulation and one rounding.
Mat gemm_eval(const Mat& a0, const Mat& b0, double alpha, const Mat* c, double beta, int flags) {
    const Mat a = (flags & 1) ? a0.transposed() : a0, b = (flags & 2) ? b0.transposed() : b0;
    assert(a.cols == b.rows && a.type() == b.type());
    const int m = a.rows, len = a.cols, n = b.cols;
    Mat d(m, n, a.type());
    if (c) assert(c->rows == m && c->cols == n);
    if (a.depth() == CV_32F) {
        const bool small = flags == 0 && len >= 2 && len <= 4 && (len == n || len == m);   // transposed operands take the general path
        for (int i = 0; i < m; i++) for (int j = 0; j < n; j++) {
            if (small) {
                float s = a.at<float>(i, 0) * b.at<float>(0, j);
                for (int k = 1; k < len; k++) s = s + a.at<float>(i, k) * b.at<float>(k, j);
                d.at<float>(i, j) = (float)((double)s * alpha + (c ? (double)c->at<float>(i, j) * beta : 0.0));
            } else {
                double s = 0;
                for (int k = 0; k < len; k++) s += (double)a.at<float>(i, k) * (double)b.at<float>(k, j);
                d.at<float>(i, j) = (float)(s * alpha + (c ? (double)c->at<float>(i, j) * beta : 0.0));
            }
        }
    } else {
        assert(a.depth() == CV_64F);
        for (int i = 0; i < m; i++) for (int j = 0; j < n; j++) {
            double s = 0;
            for (int k = 0; k < len; k++) s += a.at<double>(i, k) * b.at<double>(k, j);
            d.at<double>(i, j) = s * alpha + (c ? c->at<double>(i, j) * beta : 0.0);
        }
    }
    return d;
}
void gemm(const Mat& a, const Mat& b, double alpha, const Mat& c, double beta, Mat& dst, int flags) {
    dst = gemm_eval(a, b, alpha, c.empty() ? nullptr : &c, beta, flags);
}

static Mat binop(const Mat& a, const Mat& b, int sign) {
    assert(a.rows == b.rows && a.cols == b.cols && a.type() == b.type());
    Mat o(a.rows, a.cols, a.type());
    if (a.depth() == CV_32F) { for (int r = 0; r < a.rows; r++) for (int c = 0; c < a.cols; c++) o.at<float>(r, c) = sign > 0 ? a.at<float>(r, c) + b.at<float>(r, c) : a.at<float>(r, c) - b.at<float>(r, c); }
    else for (int r = 0; r < a.rows; r++) for (int c = 0; c < a.cols; c++) o.setd(r, c, a.getd(r, c) + sign * b.getd(r, c));
    return o;
}
Mat operator+(const Mat& a, const Mat& b) { return binop(a, b, 1); }
Mat operator-(const Mat& a, const Mat& b) { return binop(a, b, -1); }
Mat negate(const Mat& a) { Mat o(a.rows, a.cols, a.type()); for (int r = 0; r < a.rows; r++) for (int c = 0; c < a.cols; c++) o.setd(r, c, -a.getd(r, c)); return o; }
Mat operator*(const Mat& a, double s) { Mat o(a.rows, a.cols, a.type()); for (int r = 0; r < a.rows; r++) for (int c = 0; c < a.cols; c++) o.setd(r, c, a.getd(r, c) * s); return o; }
Mat operator/(const Mat& a, double s) { return a * (1.0 / s); }
Mat operator+(const Mat& a, const Scalar& s) { Mat o(a.rows, a.cols, a.type()); for (int r = 0; r < a.rows; r++) for (int c = 0; c < a.cols; c++) o.setd(r, c, a.getd(r, c) + s.val[0]); return o; }
std::ostream& operator<<(std::ostream& os, const Mat& m) {
    os << "[";
    for (int r = 0; r < m.rows; r++) { for (int c = 0; c < m.cols; c++) os << (c ? ", " : "") << m.getd(r, c); os << (r + 1 < m.rows ? ";\n " : ""); }
    return os << "]";
}

static inline int popc_row(const uchar* a, const uchar* b, int n) { int d = 0; for (int i = 0; i < n; i++) d += __builtin_popcount(a[i] ^ b[i]); return d; }
double norm(const Mat& a, int normType) {
    assert(normType == NORM_L2);
    double s = 0;                               // double accumulation of squares, element order
    for (int r = 0; r < a.rows; r++) for (int c = 0; c < a.cols; c++) { const double v = a.getd(r, c); s += v * v; }
    return std::sqrt(s);
}
double norm(const Mat& a, const Mat& b, int normType) {
    assert(a.rows == b.rows && a.cols == b.cols);
    if (normType == NORM_HAMMING) { int d = 0; for (int r = 0; r < a.rows; r++) d += popc_row(a.ptr(r), b.ptr(r), a.cols * (int)a.elemSize()); return d; }
    return norm(a - b, normType);
}

float fastAtan2(float y, float x) { return orc_fast_atan2(y, x); }

// ------------------------------------------------------------------------------------------------
void FAST(InputArray image, std::vector<KeyPoint>& keypoints, int threshold, bool nonmaxSuppression) {
    assert(nonmaxSuppression);
    const Mat img = image.getMat();
    assert(img.type() == CV_8UC1);
    const int cap = img.rows * img.cols / 2 + 16;
    std::vector<int> xs(cap), ys(cap), sc(cap);
    const int n = orc_fast9_16(img.data, img.cols, img.rows, (int)img.step, threshold, xs.data(), ys.data(), sc.data(), cap);
    keypoints.clear();
    for (int i = 0; i < n; i++) keypoints.push_back(KeyPoint((float)xs[i], (float)ys[i], 7.f, -1.f, (float)sc[i]));
}
void resize(InputArray src, OutputArray dst, Size dsize, double fx, double fy, int interpolation) {
    assert(interpolation == INTER_LINEAR && fx == 0 && fy == 0);
    const Mat s = src.getMat();
    dst.create(dsize, s.type());
    Mat d = dst.getMat();
    orc_resize_linear_u8(s.data, s.cols, s.rows, (int)s.step, d.data, d.cols, d.rows, (int)d.step);
}
void copyMakeBorder(InputArray src, OutputArray dst, int top, int bottom, int left, int right, int borderType, const Scalar&) {
    assert((borderType & ~BORDER_ISOLATED) == BORDER_REFLECT_101 && top == bottom && left == right && top == left);
    const Mat s = src.getMat();
    dst.create(s.rows + top + bottom, s.cols + left + right, s.type());
    Mat d = dst.getMat();
    // the source may be the interior ROI of the destination (ORBextractor.cc:1122): the primitive reads the source rows
    // before it writes the border of each row, and interior bytes are copied onto themselves
    Mat tmp = (s.data >= d.data && s.data < d.data + (size_t)d.rows * d.step) ? s.clone() : s;
    orc_border_reflect101_u8(tmp.data, tmp.cols, tmp.rows, (int)tmp.step, d.data, (int)d.step, top);
}
void GaussianBlur(InputArray src, OutputArray dst, Size ksize, double sigmaX, double sigmaY, int borderType) {
    assert(ksize.width == 7 && ksize.height == 7 && sigmaX == 2 && sigmaY == 2 && borderType == BORDER_REFLECT_101);
    const Mat s = src.getMat().clone();
    dst.create(s.rows, s.cols, s.type());
    Mat d = dst.getMat();
    orc_gauss7_sigma2_u8(s.data, s.cols, s.rows, (int)s.step, d.data, (int)d.step);
}
void cvtColor(InputArray src, OutputArray dst, int code, int) {
    // 8-bit RGB/BGR(A) -> gray, OpenCV 4.13's fixed-point weights: (R*9798 + G*19235 + B*3735 + 16384) >> 15  (pinned to cv2 in tests)
    const Mat s = src.getMat();
    const int cn = s.channels();
    assert(s.depth() == CV_8U && (cn == 3 || cn == 4));
    const bool rgb = (code == COLOR_RGB2GRAY || code == COLOR_RGBA2GRAY);
    Mat d(s.rows, s.cols, CV_8UC1);
    for (int y = 0; y < s.rows; y++) for (int x = 0; x < s.cols; x++) {
        const uchar* p = s.ptr(y) + (size_t)x * cn;
        const int r = rgb ? p[0] : p[2], g = p[1], b = rgb ? p[2] : p[0];
        d.at<uchar>(y, x) = (uchar)((r * 9798 + g * 19235 + b * 3735 + 16384) >> 15);
    }
    *dst.m = d;
}
void meanStdDev(InputArray, OutputArray, OutputArray, InputArray) { assert(!"minicv: meanStdDev is outside the tested path"); abort(); }
void Laplacian(InputArray, OutputArray, int, int, double, double, int) { assert(!"minicv: Laplacian is outside the tested path"); abort(); }
void convertScaleAbs(InputArray, OutputArray, double, double) { assert(!"minicv: convertScaleAbs is outside the tested path"); abort(); }
Mat imread(const std::string&, int) { return Mat(); }
SVD::SVD(InputArray, int) { assert(!"minicv: SVD is outside the tested path"); abort(); }
void SVD::compute(InputArray, OutputArray, OutputArray, OutputArray, int) { assert(!"minicv: SVD is outside the tested path"); abort(); }

// cv::undistortPoints(src, dst, K, D, noArray(), P=K) for N x 2 CV_32F points (Frame.cc:492-501, :519-527): iterative
// inverse of the radial/tangential model (k1 k2 p1 p2 [k3]), 5 iterations as in OpenCV 4.13, computed in double: on the first iteration
// whose distortion factor icdist is negative the point goes back to its normalised start and the iteration stops.
void undistortPoints(InputArray src, OutputArray dst, InputArray cameraMatrix, InputArray distCoeffs, InputArray R, InputArray P) {
    const Mat s = src.getMat().clone(), K = cameraMatrix.getMat(), D = distCoeffs.getMat(), Pm = P.getMat();
    assert(R.empty() && s.depth() == CV_32F);
    const bool two_ch = s.channels() == 2;                 // N x 1 CV_32FC2 or N x 2 CV_32FC1
    const int n = s.rows;
    double k[5] = {0, 0, 0, 0, 0};
    for (int i = 0; i < (int)D.total() && i < 5; i++) k[i] = D.getd(i / D.cols, i % D.cols);
    const double fx = K.getd(0, 0), fy = K.getd(1, 1), cx = K.getd(0, 2), cy = K.getd(1, 2), ifx = 1. / fx, ify = 1. / fy;
    Mat out(s.rows, s.cols, s.type());
    for (int i = 0; i < n; i++) {
        const float* sp = s.ptr<float>(i); float* op = out.ptr<float>(i);
        double x = sp[0], y = sp[1];
        x = (x - cx) * ifx; y = (y - cy) * ify;
        const double x0 = x, y0 = y;
        for (int j = 0; j < 5; j++) {
            const double r2 = x * x + y * y, icdist = 1. / (1 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2);
            if (icdist < 0) { x = x0; y = y0; break; }
            const double dx = 2 * k[2] * x * y + k[3] * (r2 + 2 * x * x), dy = k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y;
            x = (x0 - dx) * icdist; y = (y0 - dy) * icdist;
        }
        if (!Pm.empty()) {
            const double xx = Pm.getd(0, 0) * x + Pm.getd(0, 1) * y + Pm.getd(0, 2), yy = Pm.getd(1, 0) * x + Pm.getd(1, 1) * y + Pm.getd(1, 2);
            const double ww = 1. / (Pm.getd(2, 0) * x + Pm.getd(2, 1) * y + Pm.getd(2, 2));
            x = xx * ww; y = yy * ww;
        }
        op[0] = (float)x; op[1] = (float)y;
    }
    (void)two_ch;
    *dst.m = out;
}

void KeyPointsFilter::retainBest(std::vector<KeyPoint>& kps, int n) {      // only reached from ComputeKeyPointsOld (dead code)
    if (n >= 0 && (int)kps.size() > n) {
        std::stable_sort(kps.begin(), kps.end(), [](const KeyPoint& a, const KeyPoint& b) { return a.response > b.response; });
        kps.resize(n);
    }
}

void BFMatcher::knnMatch(InputArray query, InputArray train, std::vector<std::vector<DMatch> >& matches, int k, InputArray, bool) const {
    assert(normType == NORM_HAMMING && !crossCheck && k == 2);
    const Mat q = query.getMat(), t = train.getMat();
    assert(q.empty() || t.empty() || (q.cols == 32 && t.cols == 32 && q.isContinuous() && t.isContinuous()));
    matches.clear();
    std::vector<int32_t> out((size_t)q.rows * 4 + 4);
    orc_knn2(q.data, q.rows, t.data, t.rows, out.data());
    for (int i = 0; i < q.rows; i++) {
        std::vector<DMatch> m;
        if (t.rows >= 1 && out[4 * i] >= 0) m.push_back(DMatch(i, out[4 * i], 0, (float)out[4 * i + 1]));
        if (t.rows >= 2 && out[4 * i + 2] >= 0) m.push_back(DMatch(i, out[4 * i + 2], 0, (float)out[4 * i + 3]));
        matches.push_back(m);
    }
}

namespace line_descriptor {
void LSDDetector::detect(const Mat& image, std::vector<KeyLine>& keylines, int scale, int numOctaves, const Mat&) {
    assert(scale == 1 && numOctaves == 1 && image.type() == CV_8UC1);
    const int cap = orc_lsd_keylines(image.data, image.cols, image.rows, (int)image.step, nullptr, 0);
    std::vector<orc_keyline> kl(cap + 1);
    const int n = orc_lsd_keylines(image.data, image.cols, image.rows, (int)image.step, kl.data(), cap);
    keylines.resize(n);
    static_assert(sizeof(orc_keyline) == sizeof(KeyLine), "layout");
    if (n) memcpy((void*)keylines.data(), kl.data(), (size_t)n * sizeof(KeyLine));
}
void BinaryDescriptor::compute(const Mat& image, std::vector<KeyLine>& keylines, Mat& descriptors, bool) const {
    assert(image.type() == CV_8UC1);
    const int n = (int)keylines.size();
    if (n == 0) { descriptors.release(); return; }
    descriptors.create(n, 32, CV_8UC1);
    orc_lbd_compute(image.data, image.cols, image.rows, (int)image.step, (const orc_keyline*)keylines.data(), n, descriptors.data);
}
}  // namespace line_descriptor

}  // namespace cv
