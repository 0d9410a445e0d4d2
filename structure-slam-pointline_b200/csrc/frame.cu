// frame.cu — the frame-level entry point of libsslpl_b200 (sm_90a): what Frame::Frame(imGray, ...) does with the two
// extractors (reference src/Frame.cc:69-131), plus the colour conversion in front of it (src/Tracking.cc:148-161) and the keypoint
// undistortion behind it (Frame::UndistortKeyPoints / ComputeImageBounds, src/Frame.cc:483-543 — SURVEY.md 8(f) row 4):
//   * ONE host->device copy of the frame (the reference's two extractors each read the same cv::Mat; the per-extractor host entry
//     points of this library each upload it);
//   * 3- and 4-channel input is turned into the grey frame on the device (bit-exact cv::cvtColor, 8-bit fixed point);
//   * ORB and LSD+LBD run on two streams fed by that one grey frame (Frame.cc:86-87 runs them back to back);
//   * the undistorted keypoints (mvKeysUn) are computed from the device-resident keypoints, no second upload.
// Product code: no oracle, no CPU fallback.
#include "common.cuh"
#include <new>

namespace sslpl {
namespace {

// cv::cvtColor(RGB/BGR[A] -> GRAY) for CV_8U as OpenCV 4.13 computes it: (R*9798 + G*19235 + B*3735 + 16384) >> 15
// (pinned to cv2.cvtColor in tests/test_frame_gpu.py and, through the oracle's restatement, in tests/test_oracle_cpu.py).
__global__ void __launch_bounds__(256) k_cvt_gray(const uint8_t* __restrict__ src, int w, int h, int spitch, int cn, int rgb,
                                                  uint8_t* __restrict__ dst, int dpitch, long long sstride, long long dstride) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, f = blockIdx.z;
    if (x >= w) return;
    const uint8_t* p = src + f * sstride + (long long)y * spitch + (long long)x * cn;
    const int c0 = p[0], c1 = p[1], c2 = p[2];
    const int r = rgb ? c0 : c2, b = rgb ? c2 : c0;
    dst[f * dstride + (long long)y * dpitch + x] = (uint8_t)((r * 9798 + c1 * 19235 + b * 3735 + 16384) >> 15);
}

struct Camera { double fx, fy, cx, cy, k[5]; int distorted; };

// cv::undistortPoints(src, dst, K, D, noArray(), K) on the keypoint coordinates (Frame.cc:492-501): five fixed-point iterations of
// the radial / tangential model in double, re-projection with K, narrowing to float (bit-equal to cv2 4.13 in the tests).
__device__ __forceinline__ void undistort_pt(const Camera& c, float xin, float yin, float* xo, float* yo) {
    double x = ((double)xin - c.cx) * (1.0 / c.fx), y = ((double)yin - c.cy) * (1.0 / c.fy);
    const double x0 = x, y0 = y;
#pragma unroll 1
    for (int j = 0; j < 5; j++) {
        const double r2 = __dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y));
        const double icdist = 1.0 / __dadd_rn(1.0, __dmul_rn(__dadd_rn(__dmul_rn(__dadd_rn(__dmul_rn(c.k[4], r2), c.k[1]), r2), c.k[0]), r2));
        const double dx = __dadd_rn(__dmul_rn(__dmul_rn(__dmul_rn(2.0, c.k[2]), x), y), __dmul_rn(c.k[3], __dadd_rn(r2, __dmul_rn(__dmul_rn(2.0, x), x))));
        const double dy = __dadd_rn(__dmul_rn(c.k[2], __dadd_rn(r2, __dmul_rn(__dmul_rn(2.0, y), y))), __dmul_rn(__dmul_rn(__dmul_rn(2.0, c.k[3]), x), y));
        x = __dmul_rn(__dadd_rn(x0, -dx), icdist); y = __dmul_rn(__dadd_rn(y0, -dy), icdist);
    }
    *xo = (float)__dadd_rn(__dmul_rn(c.fx, x), c.cx); *yo = (float)__dadd_rn(__dmul_rn(c.fy, y), c.cy);
}

__global__ void __launch_bounds__(256) k_undistort(const sslpl_keypoint* __restrict__ in, const int* __restrict__ n, int cap, Camera cam,
                                                   sslpl_keypoint* __restrict__ out) {
    const int f = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n[f]) return;
    sslpl_keypoint k = in[(long long)f * cap + i];
    if (cam.distorted) undistort_pt(cam, k.x, k.y, &k.x, &k.y);
    out[(long long)f * cap + i] = k;
}

}  // namespace
}  // namespace sslpl

using namespace sslpl;

struct sslpl_frame {
    sslpl_frame_params p;
    sslpl_orb* orb = nullptr; sslpl_line* line = nullptr;
    cudaStream_t s_orb = nullptr, s_line = nullptr;
    cudaEvent_t ev_in = nullptr, ev_line = nullptr;
    uint8_t* d_raw = nullptr; size_t raw_bytes = 0;       // multi-channel input staging
    uint8_t* d_gray = nullptr; int gpitch = 0; size_t gstride = 0;
    sslpl_keypoint* d_un = nullptr;                        // undistorted keypoints [max_batch][cap]
    Camera cam;
    int cap = 0, last_pitch = 0; size_t last_stride = 0;
    bool last_undistorted = false;                         // the last call wrote mvKeysUn to d_un (k1 != 0)
    long long launches = 0;
};

extern "C" {

int sslpl_frame_create(const sslpl_frame_params* p, sslpl_frame** out) {
    SSLPL_REQUIRE(p && out, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(p->orb.device == p->line.device && p->orb.max_batch == p->line.max_batch && p->orb.max_width == p->line.max_width &&
                  p->orb.max_height == p->line.max_height, SSLPL_ERR_ARG, "the ORB and line parameters must agree on device, max_batch and maximum frame size");
    sslpl_frame* h = new (std::nothrow) sslpl_frame();
    SSLPL_REQUIRE(h, SSLPL_ERR_ARG, "out of host memory");
    h->p = *p;
    int rc = sslpl_orb_create(&p->orb, &h->orb);
    if (rc == SSLPL_OK) rc = sslpl_line_create(&p->line, &h->line);
    if (rc != SSLPL_OK) { sslpl_frame_destroy(h); return rc; }
    cudaError_t e = cudaSetDevice(p->orb.device);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->s_orb, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->s_line, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->ev_in, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->ev_line, cudaEventDisableTiming);
    h->gpitch = (int)align_up((size_t)p->orb.max_width, 64); h->gstride = (size_t)h->gpitch * p->orb.max_height;
    h->cap = sslpl_orb_max_keypoints(h->orb);
    if (e == cudaSuccess) e = cudaMalloc(&h->d_gray, h->gstride * p->orb.max_batch + 256);
    if (e == cudaSuccess) e = cudaMalloc(&h->d_un, sizeof(sslpl_keypoint) * (size_t)h->cap * p->orb.max_batch);
    if (e != cudaSuccess) { set_error("sslpl_frame_create: %s", cudaGetErrorString(e)); sslpl_frame_destroy(h); return SSLPL_ERR_CUDA; }
    sslpl_orb_set_stream(h->orb, h->s_orb); sslpl_line_set_stream(h->line, h->s_line);
    memset(&h->cam, 0, sizeof(h->cam)); h->cam.fx = h->cam.fy = 1.0;
    *out = h;
    return SSLPL_OK;
}

void sslpl_frame_destroy(sslpl_frame* h) {
    if (!h) return;
    if (h->orb) sslpl_orb_destroy(h->orb);
    if (h->line) sslpl_line_destroy(h->line);
    if (h->d_raw) cudaFree(h->d_raw);
    if (h->d_gray) cudaFree(h->d_gray);
    if (h->d_un) cudaFree(h->d_un);
    if (h->ev_in) cudaEventDestroy(h->ev_in);
    if (h->ev_line) cudaEventDestroy(h->ev_line);
    if (h->s_orb) cudaStreamDestroy(h->s_orb);
    if (h->s_line) cudaStreamDestroy(h->s_line);
    delete h;
}

void* sslpl_frame_stream(sslpl_frame* h, int which) { return h ? (which ? (void*)h->s_line : (void*)h->s_orb) : nullptr; }
sslpl_orb* sslpl_frame_orb(sslpl_frame* h) { return h ? h->orb : nullptr; }
sslpl_line* sslpl_frame_line(sslpl_frame* h) { return h ? h->line : nullptr; }
long long sslpl_frame_launch_count(const sslpl_frame* h) { return h ? h->launches + sslpl_orb_launch_count(h->orb) + sslpl_line_launch_count(h->line) : 0; }

int sslpl_frame_set_camera(sslpl_frame* h, float fx, float fy, float cx, float cy, const float* dist, int ndist) {
    SSLPL_REQUIRE(h && ndist >= 0 && ndist <= 5 && (ndist == 0 || dist), SSLPL_ERR_ARG, "bad camera");
    h->cam.fx = fx; h->cam.fy = fy; h->cam.cx = cx; h->cam.cy = cy;
    for (int i = 0; i < 5; i++) h->cam.k[i] = i < ndist ? dist[i] : 0.0;
    h->cam.distorted = ndist > 0 && dist[0] != 0.0f;          // Frame.cc:485: only k1 decides
    return SSLPL_OK;
}

/* Frame::ComputeImageBounds (Frame.cc:515-543): mnMinX, mnMaxX, mnMinY, mnMaxY of a cols x rows image */
int sslpl_frame_image_bounds(sslpl_frame* h, int cols, int rows, float* bounds4) {
    SSLPL_REQUIRE(h && bounds4, SSLPL_ERR_ARG, "null argument");
    if (!h->cam.distorted) { bounds4[0] = 0.f; bounds4[1] = (float)cols; bounds4[2] = 0.f; bounds4[3] = (float)rows; return SSLPL_OK; }
    SSLPL_CUDA(cudaSetDevice(h->p.orb.device));
    sslpl_keypoint c[4]; int n4 = 4;
    memset(c, 0, sizeof(c));
    c[1].x = (float)cols; c[2].y = (float)rows; c[3].x = (float)cols; c[3].y = (float)rows;
    sslpl_keypoint* d = nullptr; int* dn = nullptr;
    SSLPL_CUDA(cudaMalloc(&d, sizeof(c) * 2)); 
    cudaError_t e = cudaMalloc(&dn, sizeof(int));
    if (e != cudaSuccess) { cudaFree(d); set_error("cudaMalloc: %s", cudaGetErrorString(e)); return SSLPL_ERR_CUDA; }
    cudaMemcpyAsync(d, c, sizeof(c), cudaMemcpyHostToDevice, h->s_orb); cudaMemcpyAsync(dn, &n4, sizeof(int), cudaMemcpyHostToDevice, h->s_orb);
    k_undistort<<<dim3(1, 1), 256, 0, h->s_orb>>>(d, dn, 4, h->cam, d + 4);
    h->launches++;
    cudaMemcpyAsync(c, d + 4, sizeof(c), cudaMemcpyDeviceToHost, h->s_orb);
    e = cudaStreamSynchronize(h->s_orb);
    cudaFree(d); cudaFree(dn);
    if (e != cudaSuccess) { set_error("sslpl_frame_image_bounds: %s", cudaGetErrorString(e)); return SSLPL_ERR_CUDA; }
    bounds4[0] = fminf(c[0].x, c[2].x); bounds4[1] = fmaxf(c[1].x, c[3].x); bounds4[2] = fminf(c[0].y, c[1].y); bounds4[3] = fmaxf(c[2].y, c[3].y);
    return SSLPL_OK;
}

/* enqueue only: the upload, both extractions and the result copies; finish with sslpl_frame_sync.  With pinned host buffers
   (sslpl_host_alloc) nothing here waits for the device, so consecutive calls on different handles overlap. */
int sslpl_frame_extract_batch_begin(sslpl_frame* h, const uint8_t* imgs, int nframes, int width, int height, int pitch, size_t frame_stride,
                                    int channels, int rgb_order,
                                    sslpl_keypoint* kps, sslpl_keypoint* kps_un, uint8_t* desc, int cap, int* nkp,
                                    sslpl_keyline* kl, uint8_t* ldesc, double* lineeq, int lcap, int* nl) {
    SSLPL_REQUIRE(h && imgs && nkp && nl, SSLPL_ERR_ARG, "null argument");
    SSLPL_REQUIRE(nframes >= 1 && nframes <= h->p.orb.max_batch, SSLPL_ERR_ARG, "nframes exceeds max_batch");
    SSLPL_REQUIRE(width >= 16 && height >= 16 && width <= h->p.orb.max_width && height <= h->p.orb.max_height, SSLPL_ERR_ARG, "frame size out of range");
    SSLPL_REQUIRE(channels == 1 || channels == 3 || channels == 4, SSLPL_ERR_ARG, "channels must be 1, 3 or 4");
    SSLPL_REQUIRE(pitch >= width * channels, SSLPL_ERR_ARG, "pitch smaller than a row");
    SSLPL_REQUIRE(cap >= h->cap || !kps, SSLPL_ERR_CAPACITY, "keypoint buffers smaller than sslpl_orb_max_keypoints()");
    SSLPL_REQUIRE(lcap >= h->p.line.lsdNFeatures || !kl, SSLPL_ERR_CAPACITY, "line buffers smaller than lsdNFeatures");
    SSLPL_CUDA(cudaSetDevice(h->p.orb.device));
    const int gp = (int)align_up((size_t)width, 64); const size_t gs = (size_t)gp * height;
    h->last_pitch = gp; h->last_stride = gs;
    // ---- one upload
    if (channels == 1) {
        if (nframes == 1 || frame_stride == (size_t)pitch * height)      // contiguous frames: one 2-D copy over all rows
            SSLPL_CUDA(cudaMemcpy2DAsync(h->d_gray, gp, imgs, pitch, width, (size_t)height * nframes, cudaMemcpyHostToDevice, h->s_orb));
        else for (int f = 0; f < nframes; f++)
            SSLPL_CUDA(cudaMemcpy2DAsync(h->d_gray + f * gs, gp, imgs + f * frame_stride, pitch, width, height, cudaMemcpyHostToDevice, h->s_orb));
    } else {
        const size_t rowb = (size_t)width * channels, need = rowb * height * nframes;
        if (need > h->raw_bytes) {
            SSLPL_CUDA(cudaStreamSynchronize(h->s_orb));
            if (h->d_raw) cudaFree(h->d_raw);
            h->d_raw = nullptr; h->raw_bytes = 0;
            SSLPL_CUDA(cudaMalloc(&h->d_raw, need)); h->raw_bytes = need;
        }
        for (int f = 0; f < nframes; f++)
            SSLPL_CUDA(cudaMemcpy2DAsync(h->d_raw + f * rowb * height, rowb, imgs + f * frame_stride, pitch, rowb, height, cudaMemcpyHostToDevice, h->s_orb));
        k_cvt_gray<<<dim3((width + 255) / 256, height, nframes), 256, 0, h->s_orb>>>(h->d_raw, width, height, (int)rowb, channels, rgb_order ? 1 : 0,
                                                                                 h->d_gray, gp, (long long)(rowb * height), (long long)gs);
        h->launches++;
    }
    SSLPL_CUDA(cudaEventRecord(h->ev_in, h->s_orb));
    SSLPL_CUDA(cudaStreamWaitEvent(h->s_line, h->ev_in, 0));
    // ---- ORB and LSD+LBD on two streams, from the same device frame
    int rc = sslpl_orb_extract_batch_device(h->orb, h->d_gray, nframes, width, height, gp, gs);
    if (rc != SSLPL_OK) return rc;
    rc = sslpl_line_extract_batch_device(h->line, h->d_gray, nframes, width, height, gp, gs);
    if (rc != SSLPL_OK) return rc;
    const sslpl_keypoint* d_kps; const uint8_t* d_desc; const int* d_n; int c2;
    rc = sslpl_orb_device_results(h->orb, &d_kps, &d_desc, &d_n, &c2);
    if (rc != SSLPL_OK) return rc;
    // mvKeysUn: always computed with k1 != 0 (the device consumers read it through sslpl_frame_device_keypoints_un); with k1 == 0 it
    // equals the ORB keypoints and is only copied for the host output
    h->last_undistorted = h->cam.distorted != 0;
    if (kps_un || h->last_undistorted) {
        k_undistort<<<dim3((c2 + 255) / 256, nframes), 256, 0, h->s_orb>>>(d_kps, d_n, c2, h->cam, h->d_un);
        h->launches++;
    }
    // ---- results
    SSLPL_CUDA(cudaMemcpyAsync(nkp, d_n, sizeof(int) * nframes, cudaMemcpyDeviceToHost, h->s_orb));
    if (cap == c2) {                                                     // same stride on both sides: one copy per array
        if (kps) SSLPL_CUDA(cudaMemcpyAsync(kps, d_kps, sizeof(sslpl_keypoint) * (size_t)c2 * nframes, cudaMemcpyDeviceToHost, h->s_orb));
        if (kps_un) SSLPL_CUDA(cudaMemcpyAsync(kps_un, h->d_un, sizeof(sslpl_keypoint) * (size_t)c2 * nframes, cudaMemcpyDeviceToHost, h->s_orb));
        if (desc) SSLPL_CUDA(cudaMemcpyAsync(desc, d_desc, (size_t)c2 * 32 * nframes, cudaMemcpyDeviceToHost, h->s_orb));
    } else for (int f = 0; f < nframes; f++) {
        if (kps) SSLPL_CUDA(cudaMemcpyAsync(kps + (size_t)f * cap, d_kps + (size_t)f * c2, sizeof(sslpl_keypoint) * c2, cudaMemcpyDeviceToHost, h->s_orb));
        if (kps_un) SSLPL_CUDA(cudaMemcpyAsync(kps_un + (size_t)f * cap, h->d_un + (size_t)f * c2, sizeof(sslpl_keypoint) * c2, cudaMemcpyDeviceToHost, h->s_orb));
        if (desc) SSLPL_CUDA(cudaMemcpyAsync(desc + (size_t)f * cap * 32, d_desc + (size_t)f * c2 * 32, (size_t)c2 * 32, cudaMemcpyDeviceToHost, h->s_orb));
    }
    const sslpl_keyline* d_kl; const uint8_t* d_ld; const double* d_eq; const int* d_nl; int cl;
    rc = sslpl_line_device_results(h->line, &d_kl, &d_ld, &d_eq, &d_nl, &cl);
    if (rc != SSLPL_OK) return rc;
    SSLPL_CUDA(cudaMemcpyAsync(nl, d_nl, sizeof(int) * nframes, cudaMemcpyDeviceToHost, h->s_line));
    if (lcap == cl) {
        if (kl) SSLPL_CUDA(cudaMemcpyAsync(kl, d_kl, sizeof(sslpl_keyline) * (size_t)cl * nframes, cudaMemcpyDeviceToHost, h->s_line));
        if (ldesc) SSLPL_CUDA(cudaMemcpyAsync(ldesc, d_ld, (size_t)cl * 32 * nframes, cudaMemcpyDeviceToHost, h->s_line));
        if (lineeq) SSLPL_CUDA(cudaMemcpyAsync(lineeq, d_eq, sizeof(double) * 3 * (size_t)cl * nframes, cudaMemcpyDeviceToHost, h->s_line));
    } else for (int f = 0; f < nframes; f++) {
        if (kl) SSLPL_CUDA(cudaMemcpyAsync(kl + (size_t)f * lcap, d_kl + (size_t)f * cl, sizeof(sslpl_keyline) * cl, cudaMemcpyDeviceToHost, h->s_line));
        if (ldesc) SSLPL_CUDA(cudaMemcpyAsync(ldesc + (size_t)f * lcap * 32, d_ld + (size_t)f * cl * 32, (size_t)cl * 32, cudaMemcpyDeviceToHost, h->s_line));
        if (lineeq) SSLPL_CUDA(cudaMemcpyAsync(lineeq + (size_t)f * lcap * 3, d_eq + (size_t)f * cl * 3, sizeof(double) * 3 * cl, cudaMemcpyDeviceToHost, h->s_line));
    }
    return SSLPL_OK;
}

int sslpl_frame_sync(sslpl_frame* h) {
    SSLPL_REQUIRE(h, SSLPL_ERR_ARG, "null handle");
    const int rc = sslpl_orb_sync(h->orb);
    const int rc2 = sslpl_line_sync(h->line);
    return rc != SSLPL_OK ? rc : rc2;
}

int sslpl_frame_extract_batch(sslpl_frame* h, const uint8_t* imgs, int nframes, int width, int height, int pitch, size_t frame_stride,
                              int channels, int rgb_order,
                              sslpl_keypoint* kps, sslpl_keypoint* kps_un, uint8_t* desc, int cap, int* nkp,
                              sslpl_keyline* kl, uint8_t* ldesc, double* lineeq, int lcap, int* nl) {
    const int rc = sslpl_frame_extract_batch_begin(h, imgs, nframes, width, height, pitch, frame_stride, channels, rgb_order, kps, kps_un, desc, cap, nkp,
                                                   kl, ldesc, lineeq, lcap, nl);
    return rc != SSLPL_OK ? rc : sslpl_frame_sync(h);
}

int sslpl_frame_extract(sslpl_frame* h, const uint8_t* img, int width, int height, int pitch, int channels, int rgb_order,
                        sslpl_keypoint* kps, sslpl_keypoint* kps_un, uint8_t* desc, int cap, int* nkp,
                        sslpl_keyline* kl, uint8_t* ldesc, double* lineeq, int lcap, int* nl) {
    return sslpl_frame_extract_batch(h, img, 1, width, height, pitch, 0, channels, rgb_order, kps, kps_un, desc, cap, nkp, kl, ldesc, lineeq, lcap, nl);
}

/* the grey frame of the last call (device), e.g. for a caller that keeps the image resident */
int sslpl_frame_device_gray(sslpl_frame* h, const uint8_t** d_gray, int* pitch, size_t* frame_stride) {
    SSLPL_REQUIRE(h && d_gray, SSLPL_ERR_ARG, "null argument");
    *d_gray = h->d_gray; if (pitch) *pitch = h->last_pitch; if (frame_stride) *frame_stride = h->last_stride;
    return SSLPL_OK;
}

/* mvKeysUn of the last call (device): d_un when it was undistorted, the ORB handle's keypoints when k1 == 0 (Frame.cc:485) */
int sslpl_frame_device_keypoints_un(sslpl_frame* h, const sslpl_keypoint** d_kps_un, int* cap) {
    SSLPL_REQUIRE(h && d_kps_un, SSLPL_ERR_ARG, "null argument");
    const sslpl_keypoint* d_kps; const uint8_t* d_desc; const int* d_n; int c2;
    const int rc = sslpl_orb_device_results(h->orb, &d_kps, &d_desc, &d_n, &c2);
    if (rc != SSLPL_OK) return rc;
    *d_kps_un = h->last_undistorted ? h->d_un : d_kps;
    if (cap) *cap = c2;
    return SSLPL_OK;
}

}  // extern "C"
