// common.cuh — shared helpers of libsslpl_b200 (sm_90a).  Product code: no oracle, no CPU fallback.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include "../../include/sslpl.h"

namespace sslpl {

void set_error(const char* fmt, ...);
const char* get_error();

#define SSLPL_CUDA(call)                                                                         \
    do {                                                                                         \
        cudaError_t e__ = (call);                                                                \
        if (e__ != cudaSuccess) {                                                                \
            sslpl::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
            return SSLPL_ERR_CUDA;                                                               \
        }                                                                                        \
    } while (0)

#define SSLPL_REQUIRE(cond, code, msg)                                                           \
    do {                                                                                         \
        if (!(cond)) { sslpl::set_error("%s:%d: %s", __FILE__, __LINE__, msg); return code; }    \
    } while (0)

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Simple bump allocator over one cudaMalloc'ed arena (device workspace is sized once per handle).
struct Arena {
    uint8_t* base = nullptr;
    size_t size = 0, used = 0;
    template <class T> T* take(size_t count) {
        used = align_up(used, 256);
        T* p = base ? reinterpret_cast<T*>(base + used) : nullptr;
        used += count * sizeof(T);
        return p;
    }
};

// a workspace of the handle allocated by the first call that needs it (a handle that never gets there never pays for it), freed with it
template <class T> int first_use(T*& p, size_t bytes) {
    if (p) return SSLPL_OK;
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) { p = nullptr; set_error("cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e)); return SSLPL_ERR_CUDA; }
    return SSLPL_OK;
}

// carve `count` elements out of a scratch arena and start their upload
template <class T> T* stage(Arena& A, const T* host, size_t count, cudaStream_t st, cudaError_t& err) {
    T* d = A.take<T>(count + 8);
    if (host && count && err == cudaSuccess) err = cudaMemcpyAsync(d, host, sizeof(T) * count, cudaMemcpyHostToDevice, st);
    return d;
}

// What every handle with a stream shares (sslpl_orb, sslpl_line, sslpl_matcher, sslpl_frame): its device and stream, the kernel
// count, the profiling events, a pinned word block, the workspace arena and a grow-only scratch.  A handle is created with open(),
// then alloc_arena() if it has one; its destroy calls close(), frees its own buffers and deletes it.  Nothing here calls CUDA from a
// constructor or destructor: sslpl_orb_tables_host builds an sslpl_orb on the stack.
struct StreamHandle {
    int device = 0;
    cudaStream_t stream = nullptr, own_stream = nullptr;   // `stream` is own_stream unless the caller set one
    long long launches = 0;                                // kernels launched through launch()
    int32_t* h_small = nullptr;                            // 64 pinned words; [0] receives the device-side error flags in sync()
    uint8_t* arena = nullptr; size_t arena_size = 0;
    uint8_t* scratch = nullptr; size_t scratch_size = 0;   // see ensure_scratch
    bool profiling = false;
    std::vector<cudaEvent_t> ev; std::vector<const char*> ev_name; int ev_n = 0;

    int open(int dev) {
        device = dev;
        int ndev = 0;
        if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { set_error("no CUDA device available: libsslpl_b200 has no CPU fallback"); return SSLPL_ERR_CUDA; }
        SSLPL_CUDA(cudaSetDevice(dev));
        SSLPL_CUDA(cudaStreamCreateWithFlags(&own_stream, cudaStreamNonBlocking));
        stream = own_stream;
        SSLPL_CUDA(cudaHostAlloc((void**)&h_small, 64 * sizeof(int32_t), cudaHostAllocDefault));
        return SSLPL_OK;
    }

    void close() {
        cudaSetDevice(device);
        // an external stream may already be gone (its owner was destroyed first): never touch it here
        if (stream != own_stream) cudaDeviceSynchronize();
        else if (own_stream) cudaStreamSynchronize(own_stream);
        if (own_stream) cudaStreamDestroy(own_stream);
        for (auto e : ev) cudaEventDestroy(e);
        if (arena) cudaFree(arena);
        if (scratch) cudaFree(scratch);
        if (h_small) cudaFreeHost(h_small);
    }

    int alloc_arena(size_t bytes) {
        if (int rc = first_use(arena, bytes)) return rc;
        arena_size = bytes;
        SSLPL_CUDA(cudaMemset(arena, 0, bytes));
        return SSLPL_OK;
    }

    int set_stream(void* s) {
        SSLPL_CUDA(cudaSetDevice(device));
        SSLPL_CUDA(cudaStreamSynchronize(stream));
        stream = s ? (cudaStream_t)s : own_stream;
        return SSLPL_OK;
    }

    // Wait for the stream.  d_err is the device-side error word (DERR_* bits), or null when there is none yet (the handle has not
    // run): non-zero flags are reported as SSLPL_ERR_CAPACITY in `what` and cleared.
    int sync(int* d_err, const char* what) {
        SSLPL_CUDA(cudaSetDevice(device));
        if (d_err) SSLPL_CUDA(cudaMemcpyAsync(h_small, d_err, sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
        SSLPL_CUDA(cudaStreamSynchronize(stream));
        if (!d_err || !h_small[0]) return SSLPL_OK;
        set_error("device-side capacity overflow in %s, flags=0x%x", what, h_small[0]);
        cudaMemsetAsync(d_err, 0, sizeof(int32_t), stream);
        return SSLPL_ERR_CAPACITY;
    }

    // profiling: an event after each stage of a call when on; the call resets ev_n and marks "start" first
    void mark(const char* name) {
        if (!profiling) return;
        if ((int)ev.size() <= ev_n) { cudaEvent_t e; cudaEventCreate(&e); ev.push_back(e); ev_name.push_back(name); }
        ev_name[ev_n] = name;
        cudaEventRecord(ev[ev_n++], stream);
    }

    int stage_ms(float* ms, int cap, const char** names, int* nstages) {
        SSLPL_REQUIRE(nstages, SSLPL_ERR_ARG, "null argument");
        SSLPL_CUDA(cudaStreamSynchronize(stream));
        int k = 0;
        for (int i = 1; i < ev_n; i++, k++)
            if (k < cap) { float t = 0; cudaEventElapsedTime(&t, ev[i - 1], ev[i]); if (ms) ms[k] = t; if (names) names[k] = ev_name[i]; }
        *nstages = k;
        return SSLPL_OK;
    }

    // nframes host frames of rows x row_bytes (frame f at src + f * sstride) into dst + f * dstride (dstride == dpitch * rows)
    int upload_frames(uint8_t* dst, size_t dpitch, size_t dstride, const uint8_t* src, size_t spitch, size_t sstride, size_t row_bytes,
                      int rows, int nframes) {
        if (nframes == 1 || sstride == spitch * rows)                  // contiguous frames: one 2-D copy over all rows
            SSLPL_CUDA(cudaMemcpy2DAsync(dst, dpitch, src, spitch, row_bytes, (size_t)rows * nframes, cudaMemcpyHostToDevice, stream));
        else for (int f = 0; f < nframes; f++)
            SSLPL_CUDA(cudaMemcpy2DAsync(dst + f * dstride, dpitch, src + f * sstride, spitch, row_bytes, rows, cudaMemcpyHostToDevice, stream));
        return SSLPL_OK;
    }
};

// Grow-only scratch shared by a handle's entry points.  Growing waits for the stream first: enqueued work may still read the old one.
inline int ensure_scratch(StreamHandle* h, size_t need) {
    if (need <= h->scratch_size) return SSLPL_OK;
    SSLPL_CUDA(cudaStreamSynchronize(h->stream));
    if (h->scratch) cudaFree(h->scratch);
    h->scratch = nullptr; h->scratch_size = 0;
    if (int rc = first_use(h->scratch, need)) return rc;
    h->scratch_size = need;
    return SSLPL_OK;
}

// every kernel launch of the library: on the handle's stream, counted by sslpl_*_launch_count
template <class T> struct same_type { using type = T; };
template <class... KArgs>
void launch(StreamHandle* h, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, typename same_type<KArgs>::type... args) {
    kernel<<<grid, block, smem, h->stream>>>(args...);
    h->launches++;
}

// device-side error flag bits
enum : int { DERR_POOL_OVERFLOW = 1, DERR_KEY_OVERFLOW = 2, DERR_SORT_OVERFLOW = 4, DERR_KP_OVERFLOW = 8,
             DERR_LSD_OVERFLOW = 16 };

#ifdef __CUDACC__
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

// Exclusive scan of one value per thread across the block (blockDim.x <= 1024, multiple of 32).
// s_warp must hold 33 ints. Returns the exclusive prefix; *total gets the block sum.
__device__ __forceinline__ int block_exclusive_scan(int v, int* s_warp, int* total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    __syncthreads();                        // protect s_warp reuse
    if (lane == 31) s_warp[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        int w = lane < nw ? s_warp[lane] : 0;
        int winc = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, winc, o); if (lane >= o) winc += t; }
        if (lane < nw) s_warp[lane] = winc - w;
        if (lane == 31) s_warp[32] = winc;
    }
    __syncthreads();
    if (total) *total = s_warp[32];
    return s_warp[wid] + inc - v;
}

// In-place exclusive scan of an int array (global or shared) of length n by the whole block.
// Thread t owns the contiguous chunk [t*chunk, (t+1)*chunk). Returns the total. s_warp: 33 ints.
__device__ __forceinline__ int block_scan_array(int* data, int n, int* s_warp) {
    const int T = blockDim.x, chunk = (n + T - 1) / T;
    const int b = min(n, (int)threadIdx.x * chunk), e = min(n, b + chunk);
    int s = 0;
    for (int i = b; i < e; i++) s += data[i];
    int total;
    int pre = block_exclusive_scan(s, s_warp, &total);
    for (int i = b; i < e; i++) { int v = data[i]; data[i] = pre; pre += v; }
    __syncthreads();
    return total;
}

__device__ __forceinline__ int popc256(const uint4& a0, const uint4& a1, const uint4& b0, const uint4& b1) {
    return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
           __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}
#endif

}  // namespace sslpl
