// Micro-benchmark: how fast can W warps of ONE SM run the accumulate step of bucket_mul_v4_kernel when the staged rows
// already sit in shared memory?  Separates the warp-level dependency chain (W = 1) from the SM-level shared-memory
// pipe limit (W = 8, 16).  Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -I effort_b200/csrc -o acc_rate acc_rate.cu
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "bucket_mul_v2.cuh"
using namespace effort;

template <int N>
__device__ __forceinline__ void acc_rows(uint32_t base_lane, float val, uint32_t a0) {
    if constexpr (N <= 4) accumulate_unit_fp16<4, N, 256>(base_lane, val, a0);
    else {
        uint32_t w[N][2];
#pragma unroll
        for (int r = 0; r < N; r++) asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(w[r][0]), "=r"(w[r][1]) : "r"(a0 + r * 256));
        uint32_t a[N][4];
        float f[N][4], acc[N][4];
#pragma unroll
        for (int r = 0; r < N; r++) AccFp16<4, 0>::addr(w[r], base_lane, a[r], f[r]);
#pragma unroll
        for (int r = 0; r < N; r++) RmwFp16<4, 0>::load(a[r], acc[r]);
#pragma unroll
        for (int r = 0; r < N; r++)
#pragma unroll
            for (int k = 0; k < 4; k++) acc[r][k] = fmaf(val, f[r][k], acc[r][k]);
#pragma unroll
        for (int r = 0; r < N; r++) RmwFp16<4, 0>::store(a[r], acc[r]);
    }
}

// mode 0: full accumulate; 1: only the staged LDS.64 + address math (no RMW); 2: RMW only (addresses from registers)
template <int N, int MODE>
__global__ void __launch_bounds__(512, 1) k(const uint32_t* __restrict__ words, int iters, int active, long long* cyc, float* sink) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t s0 = (uint32_t)__cvta_generic_to_shared(smem);
    const uint32_t s1 = (s0 + 8191u) & ~8191u;
    float* tiles = reinterpret_cast<float*>(smem + (s1 - s0));
    for (int i = tid; i < 16 * 2048; i += 512) tiles[i] = 0.f;
    unsigned char* stage = smem + (s1 - s0) + 16 * 8192;   // 16 warps x 4 KB (16 rows of 256 B)
    uint32_t* st32 = reinterpret_cast<uint32_t*>(stage);
    for (int i = tid; i < 16 * 1024; i += 512) st32[i] = words[i];
    __syncthreads();
    if (warp >= active) return;
    const uint32_t base_lane = (s1 + warp * 8192u) | (lane * 4u);
    const uint32_t sa = s1 + 16 * 8192u + warp * 4096u + lane * 8u;
    const long long t0 = clock64();
    float extra = 0.f;
    uint32_t wp[4][2] = {};
    for (int it = 0; it < iters; it++) {
        const float val = 1.0f + it * 1e-3f;
#pragma unroll
        for (int r = 0; r < 16; r += N) {
            if constexpr (MODE == 0) acc_rows<N>(base_lane, val, sa + r * 256);
            else if constexpr (MODE == 2) {  // software pipelined: the next four rows are fetched before this batch's RMW
                if (it == 0 && r == 0) {
#pragma unroll
                    for (int q = 0; q < 4; q++) asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(wp[q][0]), "=r"(wp[q][1]) : "r"(sa + q * 256));
                }
                uint32_t wn[4][2];
                const uint32_t na = sa + ((r + 4) & 15) * 256;
#pragma unroll
                for (int q = 0; q < 4; q++) asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(wn[q][0]), "=r"(wn[q][1]) : "r"(na + q * 256));
                {
                    uint32_t a[4][4];
                    float f[4][4], acc[4][4];
#pragma unroll
                    for (int q = 0; q < 4; q++) AccFp16<4, 0>::addr(wp[q], base_lane, a[q], f[q]);
#pragma unroll
                    for (int q = 0; q < 4; q++) RmwFp16<4, 0>::load(a[q], acc[q]);
#pragma unroll
                    for (int q = 0; q < 4; q++)
#pragma unroll
                        for (int k2 = 0; k2 < 4; k2++) acc[q][k2] = fmaf(val, f[q][k2], acc[q][k2]);
#pragma unroll
                    for (int q = 0; q < 4; q++) RmwFp16<4, 0>::store(a[q], acc[q]);
                }
#pragma unroll
                for (int q = 0; q < 4; q++) { wp[q][0] = wn[q][0]; wp[q][1] = wn[q][1]; }
            }
            else if constexpr (MODE == 1) {
#pragma unroll
                for (int q = 0; q < N; q++) {
                    uint32_t x, y;
                    asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(x), "=r"(y) : "r"(sa + (r + q) * 256));
                    extra += __uint_as_float((x & 0x3fffffffu) ^ (y >> 2));
                }
            }
        }
    }
    const long long t1 = clock64();
    if (lane == 0) cyc[blockIdx.x * 16 + warp] = t1 - t0;
    if (extra == 123.f) sink[0] = extra;
    __syncwarp();
    if (tid == 0) sink[1] = tiles[5];
}

template <int N, int MODE>
void run(const uint32_t* dw, long long* dc, float* ds, const char* name) {
    const size_t smem = 8192 + 16 * 8192 + 16 * 4096;
    cudaFuncSetAttribute(k<N, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const int iters = 200;
    for (int active : {1, 2, 4, 8, 12, 16}) {
        k<N, MODE><<<1, 512, smem>>>(dw, iters, active, dc, ds);
        cudaDeviceSynchronize();
        k<N, MODE><<<1, 512, smem>>>(dw, iters, active, dc, ds);
        cudaError_t e = cudaDeviceSynchronize();
        if (e != cudaSuccess) { printf("%s: %s\n", name, cudaGetErrorString(e)); return; }
        long long c[16];
        cudaMemcpy(c, dc, sizeof(c), cudaMemcpyDeviceToHost);
        long long mx = 0;
        for (int w = 0; w < active; w++) mx = c[w] > mx ? c[w] : mx;
        const double rows = (double)iters * 16;
        printf("%-22s warps %2d: %.1f cycles/row/warp, SM rate %.2f cycles/row (%.2f wavefront-cycles budget = 10)\n", name, active,
               mx / rows, mx / (rows * active), 0.0);
    }
}

int main() {
    std::vector<uint32_t> h(16 * 1024);
    srand(7);
    for (auto& x : h) x = ((uint32_t)rand() << 16) ^ (uint32_t)rand();
    uint32_t* dw; long long* dc; float* ds;
    cudaMalloc(&dw, h.size() * 4); cudaMalloc(&dc, 16 * 8 * 132); cudaMalloc(&ds, 64);
    cudaMemcpy(dw, h.data(), h.size() * 4, cudaMemcpyHostToDevice);
    run<4, 0>(dw, dc, ds, "rmw N=4");
    run<2, 0>(dw, dc, ds, "rmw N=2");
    run<8, 0>(dw, dc, ds, "rmw N=8");
    run<1, 0>(dw, dc, ds, "rmw N=1");
    run<4, 2>(dw, dc, ds, "rmw N=4 pipelined");
    return 0;
}
