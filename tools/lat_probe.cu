// tools/lat_probe.cu — dependent-chain latencies on sm_90a (one warp): what the sequential LSD walker is made of.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -fmad=false -o /tmp/lat_probe tools/lat_probe.cu && /tmp/lat_probe
#include <cstdio>
#include <cuda_runtime.h>
#define N 4096
template <int OP> __global__ void k(double* out, long long* cyc, double seed, float fseed, unsigned* gm) {
    double a = seed + threadIdx.x; float f = fseed + threadIdx.x; unsigned u = threadIdx.x; int lane = threadIdx.x;
    __shared__ double sm[64];
    sm[lane] = seed; sm[lane + 32] = seed; __syncwarp();
    long long t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < N; i++) {
        if (OP == 0) a = a + seed;
        if (OP == 1) a = a * seed;
        if (OP == 2) f = f + fseed;
        if (OP == 3) f = __fdiv_rn(fseed, f + 1.0f);
        if (OP == 4) u = __shfl_sync(0xffffffffu, u, (u + 1) & 31);
        if (OP == 5) u = __match_any_sync(0xffffffffu, u & 7) + i;
        if (OP == 6) u = __ballot_sync(0xffffffffu, (u >> (i & 3)) & 1) + lane;
        if (OP == 7) u = gm[u & 1023];                       // dependent global loads (L1 hit)
        if (OP == 8) u = __ldcg(gm + (u & 1023));            // dependent L2 loads
        if (OP == 9) a = a + sm[(i & 31)];                   // DADD fed from smem (independent loads)
        if (OP == 10) u = ((unsigned*)sm)[u & 63] + 1;       // dependent LDS
        if (OP == 11) u = __reduce_add_sync(0xffffffffu, u);
        if (OP == 12) a = fma(a, seed, seed);
        if (OP == 13) u = __float_as_uint((float)((double)__uint_as_float(u | 0x3f800000u) * seed));   // F2D DMUL D2F
        if (OP == 14) { double n = a - seed; if (n < 0) n = -n; if (n > 4.71) { n -= 6.28; if (n < 0) n = -n; } a = n + (n <= 0.39 ? 1.0 : 2.0); }
    }
    long long t1 = clock64();
    out[threadIdx.x] = a + f + u;
    if (threadIdx.x == 0) *cyc = t1 - t0;
}
int main() {
    double* out; long long* cyc; unsigned* gm;
    cudaMalloc(&out, 256); cudaMalloc(&cyc, 8); cudaMalloc(&gm, 4096); cudaMemset(gm, 0, 4096);
    const char* names[] = {"DADD", "DMUL", "FADD", "FDIV_RN(+FADD)", "SHFL", "MATCH.ANY", "VOTE.BALLOT(+ops)", "LDG L1 chain", "LDG.CG L2 chain", "DADD smem-fed", "LDS chain", "REDUX", "DFMA", "F2D+DMUL+D2F", "aligned_rad double"};
    for (int op = 0; op < 15; op++) {
        for (int rep = 0; rep < 2; rep++) {
            switch (op) {
#define C(o) case o: k<o><<<1, 32>>>(out, cyc, 1.0000001, 1.0000001f, gm); break;
                C(0) C(1) C(2) C(3) C(4) C(5) C(6) C(7) C(8) C(9) C(10) C(11) C(12) C(13) C(14)
            }
            cudaDeviceSynchronize();
        }
        long long h; cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
        printf("%-22s %.1f cycles/iter\n", names[op], (double)h / N);
    }
    return 0;
}
