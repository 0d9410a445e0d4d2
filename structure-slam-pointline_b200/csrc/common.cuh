// common.cuh — shared helpers of libsslpl_b200 (sm_90a).  Product code: no oracle, no CPU fallback.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
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
