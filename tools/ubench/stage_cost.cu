// Micro-benchmark: what do asynchronous copies INTO shared memory cost the shared-memory pipe?  8 consumer warps run the
// accumulate read-modify-write over rows that already sit in shared memory; 8 producer warps meanwhile stream 4 KB units
// from an L2-resident buffer into rings with (MODE 0) 16-byte cp.async or (MODE 1) cp.async.bulk, completion on mbarriers.
// Reports the consumers' cycles per row with the producers off / on and the bytes the producers moved per cycle.
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "bucket_mul_v4.cuh"
using namespace effort;

template <int MODE>
__global__ void __launch_bounds__(512, 1) k(const uint32_t* __restrict__ words, const unsigned char* __restrict__ src, size_t src_bytes,
                                            int iters, int producers_on, int unit_bytes, long long* out) {
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ unsigned long long bars[8][4];
    __shared__ int done_flag;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t s0 = (uint32_t)__cvta_generic_to_shared(smem);
    const uint32_t s1 = (s0 + 8191u) & ~8191u;
    float* tiles = reinterpret_cast<float*>(smem + (s1 - s0));
    for (int i = tid; i < 8 * 2048; i += 512) tiles[i] = 0.f;
    uint32_t* st32 = reinterpret_cast<uint32_t*>(smem + (s1 - s0) + 8 * 8192);  // 8 x 4 KB static rows
    for (int i = tid; i < 8 * 1024; i += 512) st32[i] = words[i];
    const uint32_t ring0 = s1 + 8 * 8192u + 8 * 4096u;                          // 8 x 16 KB rings
    if (tid < 32) {
        mbar_init((uint32_t)__cvta_generic_to_shared(&bars[0][0] + tid), MODE == 1 ? 1 : 32);
        if (tid == 0) done_flag = 0;
    }
    __syncthreads();
    if (warp < 8) {
        const uint32_t base_lane = (s1 + warp * 8192u) | (lane * 4u);
        const uint32_t sa = s1 + 8 * 8192u + warp * 4096u + lane * 8u;
        const long long t0 = clock64();
        for (int it = 0; it < iters; it++) {
            const float val = 1.0f + it * 1e-3f;
#pragma unroll
            for (int r = 0; r < 16; r += 4) accumulate_unit_fp16<4, 4, 256>(base_lane, val, sa + r * 256);
        }
        const long long t1 = clock64();
        if (lane == 0) out[blockIdx.x * 32 + warp] = t1 - t0;
        __syncwarp();
        if (lane == 0) atomicAdd(&done_flag, 1);
    } else if (producers_on) {
        const int p = warp - 8;
        const uint32_t ring = ring0 + p * 8192u;
        const uint64_t pol = l2_policy_evict_last();
        const int slots = 8192 / unit_bytes > 4 ? 4 : 8192 / unit_bytes;
        long long units = 0;
        const size_t n_units = src_bytes / unit_bytes;
        size_t u = ((size_t)blockIdx.x * 8 + p) * 977;
        const long long t0 = clock64();
        while (*(volatile int*)&done_flag < 8) {
            const int slot = (int)(units % slots);
            const uint32_t bar = (uint32_t)__cvta_generic_to_shared(&bars[p][slot]);
            if (units >= slots) mbar_wait(bar, (uint32_t)((units / slots - 1) & 1));
            const unsigned char* g = src + (u % n_units) * (size_t)unit_bytes;
            u += 131;
            const uint32_t dst = ring + slot * unit_bytes;
            if (MODE == 1) {
                if (lane == 0) { mbar_expect_tx(bar, unit_bytes); bulk_g2s(dst, g, unit_bytes, bar, pol); }
            } else {
                for (int q = lane; q < unit_bytes / 16; q += 32) cp_async16(dst + q * 16, g + q * 16, pol);
                cp_async_arrive_noinc(bar);
            }
            units++;
            __syncwarp();
        }
        const long long t1 = clock64();
        if (lane == 0) { out[blockIdx.x * 32 + 8 + p] = units; out[blockIdx.x * 32 + 16 + p] = t1 - t0; }
        // drain
        for (long long x = units > slots ? units - slots : 0; x < units; x++)
            mbar_wait((uint32_t)__cvta_generic_to_shared(&bars[p][x % slots]), (uint32_t)((x / slots) & 1));
    }
}

template <int MODE>
void run(const uint32_t* dw, const unsigned char* src, size_t src_bytes, long long* dout, int on, int unit_bytes, int grid) {
    const size_t smem = 8192 + 8 * 8192 + 8 * 4096 + 8 * 8192;
    cudaFuncSetAttribute(k<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const int iters = 400;
    cudaMemset(dout, 0, 132 * 32 * 8);
    k<MODE><<<grid, 512, smem>>>(dw, src, src_bytes, iters, on, unit_bytes, dout);
    cudaDeviceSynchronize();
    cudaMemset(dout, 0, 132 * 32 * 8);
    k<MODE><<<grid, 512, smem>>>(dw, src, src_bytes, iters, on, unit_bytes, dout);
    cudaError_t e = cudaDeviceSynchronize(); if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) { printf("error %s\n", cudaGetErrorString(e)); return; }
    std::vector<long long> h(132 * 32);
    cudaMemcpy(h.data(), dout, h.size() * 8, cudaMemcpyDeviceToHost);
    double cyc = 0, bytes = 0, pcyc = 0;
    for (int b = 0; b < grid; b++) {
        long long mx = 0;
        for (int w = 0; w < 8; w++) mx = h[b * 32 + w] > mx ? h[b * 32 + w] : mx;
        cyc += (double)mx / grid;
        for (int p = 0; p < 8; p++) { bytes += (double)h[b * 32 + 8 + p] * unit_bytes / grid; pcyc += (double)h[b * 32 + 16 + p] / (8.0 * grid); }
    }
    const double rows = iters * 16.0 * 8;
    printf("%s producers %s unit %5d B grid %3d: consumers %.2f cycles/row (SM);  staged %.1f B/cycle/SM = %.2f cycles per 256-B row"
           "  => pipe cycles per consumer row incl. staging share %.2f\n", MODE ? "bulk  " : "ldgsts", on ? "on " : "off", unit_bytes, grid,
           cyc / rows, on ? bytes / pcyc : 0.0, on ? 256.0 * pcyc / bytes : 0.0, cyc / rows);
}

int main() {
    std::vector<uint32_t> h(8 * 1024);
    srand(7);
    for (auto& x : h) x = (((uint32_t)rand() << 16) ^ (uint32_t)rand()) & 0x3fff3fffu;
    uint32_t* dw; long long* dout; unsigned char* src;
    const size_t src_bytes = 32u << 20;
    cudaMalloc(&dw, h.size() * 4); cudaMalloc(&dout, 132 * 32 * 8); cudaMalloc(&src, src_bytes);
    cudaMemset(src, 0x3c, src_bytes);
    cudaMemcpy(dw, h.data(), h.size() * 4, cudaMemcpyHostToDevice);
    for (int grid : {1, 132}) {
        run<0>(dw, src, src_bytes, dout, 0, 4096, grid);
        for (int ub : {4096, 2048, 1536, 512}) {
            run<0>(dw, src, src_bytes, dout, 1, ub, grid);
            run<1>(dw, src, src_bytes, dout, 1, ub, grid);
        }
    }
    return 0;
}
