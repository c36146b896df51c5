// common.cuh -- shared device helpers for the effort_b200 kernels (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace effort {

constexpr float kCutoffScale = 100000.0f;  // CUTOFF_SCALE, bucketMul.metal:33

// fp32 -> bfloat16 -> fp32, round-to-nearest-even; integer form so that it is bit-identical to the
// oracle (Metal `bfloat(x)`, bucketMul.metal:160).
__device__ __forceinline__ float bf16_round(float f) {
    uint32_t x = __float_as_uint(f);
    if ((x & 0x7FFFFFFFu) > 0x7F800000u) return __uint_as_float(x | 0x00400000u);
    uint32_t lsb = (x >> 16) & 1u;
    x += 0x7FFFu + lsb;
    x &= 0xFFFF0000u;
    return __uint_as_float(x);
}

__device__ __forceinline__ float half_bits_to_float(uint16_t b) {
    return __half2float(__ushort_as_half(b));
}

// Selection predicate of prepareDispatch (bucketMul.metal:66): cutoff < CUTOFF_SCALE*float(stat)*|v|
// evaluated left to right in fp32 (no fused contraction possible: two multiplies).
__device__ __forceinline__ bool row_selected(float cutoff, float stat, float v) {
    return cutoff < __fmul_rn(__fmul_rn(kCutoffScale, stat), fabsf(v));
}

// asynchronous global -> shared copy of BYTES (4, 8 or 16) with an L2 cache-policy hint; completion is tracked by
// the issuing thread's cp.async groups
template <int BYTES>
__device__ __forceinline__ void cp_async_hint(uint32_t dst_saddr, const void* src, uint64_t pol) {
    asm volatile("cp.async.ca.shared.global.L2::cache_hint [%0], [%1], %2, %3;" ::"r"(dst_saddr), "l"(src), "n"(BYTES), "l"(pol)
                 : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// streaming 8/16-byte loads that do not allocate in L1 (weights are read once)
__device__ __forceinline__ uint2 ldg_stream_u2(const void* p) {
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];"
                 : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}
__device__ __forceinline__ uint32_t ldg_stream_u1(const void* p) {
    uint32_t r;
    asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ uint4 ldg_stream_u4(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

// Programmatic dependent launch (PDL): a kernel launched with the programmatic-stream-serialization attribute
// may start while its predecessor still runs; everything that touches data the predecessor produces (or scratch it
// still reads) must come after pdl_wait().  pdl_trigger() lets the successor start its independent prologue
// (smem zeroing, loads of constant weight metadata) early.  Both are no-ops without the launch attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;"); }

// L2 eviction policies: bucket rows are read once per token (evict_first) while the small per-matrix
// metadata (stats, probes: ~41 MB for Mistral-7B) and the activations should stay L2 resident across the
// 14 GB that stream through between two uses (evict_last).
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint2 ldg_stream_u2(const void* p, uint64_t pol) {
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u32 {%0,%1}, [%2], %3;"
                 : "=r"(r.x), "=r"(r.y) : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ uint4 ldg_stream_u4(const void* p, uint64_t pol) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ uint32_t ldg_stream_u1(const void* p, uint64_t pol) {
    uint32_t r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(r) : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ uint4 ldg_keep_u4(const void* p, uint64_t pol) {
    uint4 r;
    asm volatile("ld.global.nc.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ uint16_t ldg_keep_u16(const void* p, uint64_t pol) {
    uint16_t r;
    asm volatile("ld.global.nc.L2::cache_hint.u16 %0, [%1], %2;" : "=h"(r) : "l"(p), "l"(pol));
    return r;
}

__device__ __forceinline__ int warp_sum_i(int x) { return __reduce_add_sync(0xffffffffu, x); }
__device__ __forceinline__ float warp_sum_f(float x) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    return x;
}

}  // namespace effort
