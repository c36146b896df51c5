// Micro-benchmark: full-chip streaming + accumulate WITHOUT shared-memory staging.  16 warps per SM read their rows with
// 8-byte global loads into a register ring (B banks of 4 rows), an L2 prefetch runs PF units ahead, and every row goes
// through the same shared-memory read-modify-write as bucket_mul_v4_kernel.  Question: does the SM reach the 8
// wavefronts/row bound of the accumulate (instead of 12 with cp.async/TMA staging) and what DRAM rate results?
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -I effort_b200/csrc -o stream_acc stream_acc.cu
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "bucket_mul_v2.cuh"
using namespace effort;

__device__ __forceinline__ void ldg64(const void* p, uint32_t& x, uint32_t& y, uint64_t pol) {
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u32 {%0,%1}, [%2], %3;" : "=r"(x), "=r"(y) : "l"(p), "l"(pol));
}

template <int N>
__device__ __forceinline__ void acc_regs(uint32_t base_lane, float val, const uint32_t (&w)[N][2]) {
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

// unit = UR rows of 256 bytes, contiguous; unit u of (cta, warp) sits at a pseudo-random place of the buffer
template <int B, int UR, int PF, int NW>
__global__ void __launch_bounds__(NW * 32, 1) k(const unsigned char* __restrict__ buf, size_t n_units_total, int units_per_warp, float* sink) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t s0 = (uint32_t)__cvta_generic_to_shared(smem);
    const uint32_t s1 = (s0 + 8191u) & ~8191u;
    float* tiles = reinterpret_cast<float*>(smem + (s1 - s0));
    for (int i = tid; i < NW * 2048; i += NW * 32) tiles[i] = 0.f;
    __syncthreads();
    const uint32_t base_lane = (s1 + warp * 8192u) | (lane * 4u);
    const uint64_t pol = l2_policy_evict_first();
    const size_t stream = (size_t)blockIdx.x * NW + warp;
    auto unit_ptr = [&](int u) {
        const size_t g = (stream * (size_t)units_per_warp + (size_t)u) * 2654435761ull & (n_units_total - 1);
        return buf + g * (size_t)(UR * 256) + lane * 8;
    };
    constexpr int BANKS = B, GR = UR / 4;   // groups of 4 rows per unit
    static_assert(UR % 4 == 0, "");
    uint32_t w[BANKS][4][2];
    // prologue: prefetch, fill the banks
    if (PF > 0 && lane == 0)
        for (int u = 0; u < PF && u < units_per_warp; u++)
            asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(unit_ptr(u) - lane * 8), "r"(UR * 256) : "memory");
    // linear group index g = u*GR + gi; bank = g % BANKS
    const int total_groups = units_per_warp * GR;
    auto load_group = [&](int g, uint32_t (&dst)[4][2]) {
        const int u = g / GR, gi = g % GR;
        const unsigned char* p = unit_ptr(u) + gi * 1024;
#pragma unroll
        for (int r = 0; r < 4; r++) ldg64(p + r * 256, dst[r][0], dst[r][1], pol);
    };
#pragma unroll
    for (int b = 0; b < BANKS; b++)
        if (b < total_groups) load_group(b, w[b]);
    for (int g0 = 0; g0 < total_groups; g0 += BANKS) {
#pragma unroll
        for (int b = 0; b < BANKS; b++) {
            const int g = g0 + b;
            if (g < total_groups) {
                if (PF > 0 && (g % GR) == 0 && lane == 0 && g / GR + PF < units_per_warp)
                    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(unit_ptr(g / GR + PF)), "r"(UR * 256) : "memory");
                acc_regs<4>(base_lane, 1.0f + g * 1e-4f, w[b]);
                if (g + BANKS < total_groups) load_group(g + BANKS, w[b]);
            }
        }
    }
    __syncthreads();
    if (tid == 0) sink[blockIdx.x] = tiles[5];
}

template <int B, int UR, int PF, int NW>
void run(const unsigned char* buf, size_t bytes, float* ds, int units_per_warp) {
    const size_t smem = 8192 + NW * 8192;
    cudaFuncSetAttribute(k<B, UR, PF, NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const size_t n_units_total = bytes / (UR * 256);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    float best = 1e9f;
    for (int rep = 0; rep < 5; rep++) {
        cudaEventRecord(e0);
        k<B, UR, PF, NW><<<132, NW * 32, smem>>>(buf, n_units_total, units_per_warp, ds);
        cudaEventRecord(e1);
        cudaError_t e = cudaDeviceSynchronize();
        if (e != cudaSuccess) { printf("error %s\n", cudaGetErrorString(e)); return; }
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        if (rep > 0 && ms < best) best = ms;
    }
    const double total = 132.0 * NW * units_per_warp * UR * 256;
    printf("banks %d (rows in flight %2d/warp)  unit %2d rows  prefetch %d units  warps %2d: %7.1f us  %6.0f GB/s  (%.1f MB)\n", B, B * 4, UR, PF, NW,
           best * 1e3, total / (best * 1e-3) / 1e9, total / 1e6);
}

int main() {
    const size_t bytes = 1ull << 30;
    unsigned char* buf; float* ds;
    cudaMalloc(&buf, bytes); cudaMalloc(&ds, 4096);
    cudaMemset(buf, 0x3c, bytes);
    // ~117 MB per launch at 16-row units (effort 1.0 of a 4096x14336 matrix), ~29 MB at 4-row units
    run<2, 16, 0, 16>(buf, bytes, ds, 12);
    run<2, 16, 2, 16>(buf, bytes, ds, 12);
    run<3, 16, 0, 16>(buf, bytes, ds, 12);
    run<3, 16, 2, 16>(buf, bytes, ds, 12);
    run<4, 16, 0, 16>(buf, bytes, ds, 12);
    run<4, 16, 2, 16>(buf, bytes, ds, 12);
    run<4, 16, 4, 16>(buf, bytes, ds, 12);
    run<6, 16, 0, 16>(buf, bytes, ds, 12);
    run<6, 16, 4, 16>(buf, bytes, ds, 12);
    run<4, 16, 2, 8>(buf, bytes, ds, 24);
    run<6, 16, 4, 8>(buf, bytes, ds, 24);
    run<3, 4, 4, 16>(buf, bytes, ds, 12);
    run<4, 4, 8, 16>(buf, bytes, ds, 12);
    run<4, 8, 4, 16>(buf, bytes, ds, 12);
    return 0;
}
