// tools/lat_probe2.cu — does prefetch.global.L1 warm the L1 on sm_90a?  (time of a dependent load after different warm-ups)
#include <cstdio>
#include <cuda_runtime.h>
__global__ void k(const unsigned* g, unsigned* out, long long* cyc, int mode, int stride) {
    // each trial touches a fresh 128-B line (never touched before in this launch)
    unsigned acc = 0; long long tot = 0;
    for (int i = 0; i < 256; i++) {
        const unsigned* p = g + (size_t)(i * stride + threadIdx.x * 8);        // 32 B per lane: one sector each
        if (mode == 1) asm volatile("prefetch.global.L1 [%0];" :: "l"(p));
        if (mode == 2) asm volatile("prefetch.global.L2 [%0];" :: "l"(p));
        if (mode == 3) { unsigned s; asm volatile("ld.global.ca.u32 %0, [%1];" : "=r"(s) : "l"(p)); acc ^= s; }
        // burn ~2000 cycles so that the warm-up has landed
        long long t = clock64(); while (clock64() - t < 2000) { }
        __syncwarp();
        const long long t0 = clock64();
        unsigned v; asm volatile("ld.global.ca.u32 %0, [%1];" : "=r"(v) : "l"(p));
        acc += v;
        asm volatile("" :: "r"(acc) : "memory");
        const long long t1 = clock64() + (acc & 0);
        tot += t1 - t0;
    }
    out[threadIdx.x] = acc;
    if (threadIdx.x == 0) *cyc = tot / 256;
}
int main() {
    unsigned* g; unsigned* out; long long* cyc;
    const size_t bytes = 512ull << 20;
    cudaMalloc(&g, bytes); cudaMemset(g, 0, bytes); cudaMalloc(&out, 256); cudaMalloc(&cyc, 8);
    const char* names[] = {"cold (DRAM/L2 miss)", "after prefetch.global.L1", "after prefetch.global.L2", "after ld.global.ca warm-up"};
    for (int mode = 0; mode < 4; mode++) {
        // different region per mode so that lines are fresh: offset by mode * 64 MB (in words: stride 64 KB per trial)
        k<<<1, 32>>>(g + (size_t)mode * (16u << 20), out, cyc, mode, 16384);
        cudaDeviceSynchronize();
        long long h; cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
        printf("%-30s %lld cycles\n", names[mode], h);
    }
    printf("%s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
