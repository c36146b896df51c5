// bucket_mul_v2.cuh -- round-2 fused bucketMul: ONE launch per group of approximate GEMVs.
//
// Reference steps replaced (all of BucketMul.fullMul, bucketMul.swift:34-88): findCutoff32 (bucketMul.metal:141-247),
// prepareDispatch (:47-79), roundUp / zeroRange32 (:11-31), bucketMul (:83-117), bucketIntegrate (:122-137);
// Q4: prepareDispatchQ4 / bucketMulQ4 (bucketMulQ4.metal:25-92).  What changed against bucket_mul.cuh (round 1):
//
//  * cutoff: an EXACT order statistic instead of the replayed 100-step bisection -- a radix descent over the 15-bit
//    bf16 keys of the 4096 probe products, all 16 warps, 8 keys per thread packed two per register, three thresholds
//    per round (HSET2.BF16 + HADD2.BF16 counts, REDUX, one shared atomic per warp, one barrier per round): 8 rounds.
//    c = (k+1)-th largest product (k = 4096 - q; c = 0 when k >= 4096), i.e. exactly k products lie above it
//    unless ties straddle the boundary -- inside the +-2 count slack the reference's own exit rule accepts
//    (bucketMul.metal:236).  kCutBisect keeps the bit-exact replay of the reference's loop (cutoff.cuh, four warps).
//  * selection list: 2 bytes per selected row ((local input << 4) | rank) written conflict-free with one ballot per
//    rank; the row's HBM offset is rebuilt at issue time from a per-input base (works for both row layouts).
//  * streaming: selected row slices are STAGED through a per-warp shared-memory ring by 16-byte cp.async copies
//    (completion by cp.async groups): units of up to kUnitRows consecutive ranks of one input, D units always in
//    flight per warp at no register cost, independent of how fast the accumulate loop drains them.  (A variant with
//    one cp.async.bulk per unit into the same per-warp rings measured 12-15 % slower and was dropped; the TMA
//    pipeline with a dedicated producer warp lives in bucket_mul_v3.cuh, the warp-pair design in bucket_mul_v4.cuh.)
//    This kernel is the generic path: any row layout (input-major, rank-major = NO_REPACK, slice-major) and Q4.
//  * cross-CTA reduction: no partial tiles, no integrate launch.  A CTA sums its 16 warp tiles and adds the result
//    into `out` with red.global.add.v4.f32 (one 16-byte reduction per thread).  Overwrite semantics (FP16 bucketMul
//    overwrites out, bucketMul.metal:133) are provided in-kernel: every CTA zeroes its share of its column slice
//    right after the dependency wait and arrives on a per-slice counter; the counter is checked only just before
//    the reductions, >= 5 us later (no stall in practice).  Accumulate semantics (Q4, residual stream) need neither.
//    The fp32 sum order across CTAs is therefore not fixed -- as in the reference (atomic dispatch order,
//    docs/gpu.html:196-198).
//  * glue on load: VMODE_NORM applies rmsNormFast(h) * w (aux.metal:113-152,269) to the input as it is loaded,
//    VMODE_SILU computes silu(x1) * x3 (matrix.metal:25-34), so the decode loop needs no separate kernels for them.
#pragma once
#include "bucket_mul.cuh"

namespace effort {

constexpr int kV2Warps = 16;
constexpr int kV2Threads = kV2Warps * 32;
constexpr int kUnitRows = 4;        // rows per streaming unit
template <int VEC> struct V2Unit {
    static constexpr int kRowStride = 32 * VEC * 2;                    // bytes reserved per staged row slice
    static constexpr int kUnitBytes = kUnitRows * kRowStride + 32;     // + header: the rows' multipliers [4], unit code
};
constexpr int kV2MaxInputs = kV2Threads;  // inputs per selection pass (one per thread)

enum VMode : int { kVPlain = 0, kVNorm = 1, kVSilu = 2 };
enum OutMode : int { kOutOverwrite = 0, kOutAccumulate = 1 };
enum CutMode : int { kCutSelect = 0, kCutBisect = 1 };

struct V2Problem {
    const float* v;          // [in] input (kVPlain); residual stream h (kVNorm); x1 (kVSilu)
    const float* v2;         // kVSilu: x3
    const float* v_cut;      // first n_probes entries of the full input vector (== v unless row-sharded); kVPlain only
    const __half* norm_w;    // kVNorm: [in] fp16
    const __half* st16;      // FP16 kind: one stat per row (fast-path row order)
    const float* st32;       // Q4 kind
    const uint16_t* bk;      // bucket rows [rows][C] 16-bit words
    const __half* probes;    // [E][4096]
    const uint32_t* exp_no;  // device scalar or null
    float* out;              // [C * SLOTS]
    const float* out_scale;  // optional device scalar g: out (+)= g * (W v)  (MoE gate value, runNetwork.swift:196)
    unsigned* sync;          // [CS][2] arrive / depart counters of the overwrite protocol (zero between launches)
    uint32_t* sel_counts;    // [RS] rows selected per row split (written by slice 0)
    float* cutoff_out;       // CTA 0 of the problem stores the cutoff
    float* cutoff_hint;      // [E] per-matrix memory of the last cutoff (x the rmsNorm denominator in kVNorm): where
                             // bucket_mul_v4's select starts looking (and what its optional L2 prefetch tests against)
    int* rounds_out;         // optional: CTA 0 stores the number of select rounds it needed
    unsigned* err_flag;      // set when the overwrite barrier times out
    unsigned long long* trace;
    float4* red_part;        // bucket_mul_v4: [grid][kV2Threads] per-CTA partial sums of the epilogue
    unsigned* red_sync;      // bucket_mul_v4: [CS][2] arrive / depart counters of the partial-sum exchange (zero between launches)
    unsigned long long* unit_trace;  // bucket_mul_v4's unit / prologue stamps of CTA 0: the 712 words after the per-CTA rows
    float norm_eps;
    int in, C, P, q, layout, out_mode;
    int CS, RS, W;           // column slices, row splits, columns per slice (W = 32 * VEC except when C is smaller)
    int R, lpr;              // rows per warp step / lanes per row when a row slice is narrower than a warp
};

struct V2Batch {
    int n;
    int list_cap;            // units
    int dynamic;             // 1: warps take units from a shared counter; 0: static round robin
    int ring_bytes;          // bucket_mul_v3_kernel: bytes of the producer's staging ring
    int prefetch;            // bucket_mul_v4_kernel: speculative L2 prefetch of the rows the hint selects
    int trace_cycles;        // EFFORT_TRACE=2: only the cheap SM-cycle stamps (the global-timer stamps perturb the phases)
    int cta_begin[kMulBatchMax + 1];
    V2Problem p[kMulBatchMax];
};

struct V2Header {
    CutoffSmem cut;               // bisect mode scratch
    unsigned sel_acc[8][2];       // select mode: per-round packed counts
    float red[kV2Warps];
    int warp_cnt[kV2Warps];
    int warp_rows[kV2Warps];
    int next_unit;                // streaming: next unit of the list nobody has taken yet
};

// dynamic smem: [pad][tiles 16 x 8 KB][header][sbase 512 x u32][sval 512 x f32][sstat (Q4) 512 x 8 x f32][list cap x u16][ring]
// list capacity is in UNITS (FP16: up to 8 per input, Q4: up to 4)
template <int SLOTS, int VEC>
struct V2Smem {
    static constexpr int kTileFloats = SLOTS * 32 * VEC;
    static constexpr int kTileBytes = kTileFloats * 4;
    static constexpr size_t kHdrBytes = (sizeof(V2Header) + 127) & ~size_t(127);
    static __host__ __device__ size_t list_bytes(int cap) { return ((size_t)cap * 2 + 127) & ~size_t(127); }
    static constexpr size_t kStatBytes = SLOTS == 16 ? 0 : (size_t)kV2MaxInputs * 8 * 4;
    static constexpr int kUnitsPerInput = SLOTS == 16 ? 8 : 4;
    static __host__ __device__ size_t fixed_bytes(int cap) {
        return (size_t)kTileBytes + (size_t)kV2Warps * kTileBytes + kHdrBytes + 2 * (size_t)kV2MaxInputs * 4 + kStatBytes +
               list_bytes(cap) + 128;
    }
    static __host__ __device__ size_t bytes(int cap, int ring_units) {
        return fixed_bytes(cap) + (size_t)kV2Warps * ring_units * V2Unit<VEC>::kUnitBytes;
    }
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint64_t pol) {
    asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "l"(pol) : "memory");
}
__device__ __forceinline__ void mbar_init(uint32_t bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, int bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, int bytes, uint32_t bar, uint64_t pol) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar), "l"(pol) : "memory");
}
// bounded: a copy that never completes (a bug, not a data condition) must not hang the GPU; returns false on give-up
__device__ __forceinline__ bool mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done = 0;
    for (int tries = 0; tries < (1 << 24) && !done; tries++) {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    }
    return done != 0;
}
__device__ __forceinline__ void red_add_v4(float* p, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

#define V2_TRACE(k)                                                                              \
    do {                                                                                         \
        if (pb.trace && !batch.trace_cycles && threadIdx.x == 0) pb.trace[(size_t)blockIdx.x * 16 + (k)] = gtime_ns(); \
    } while (0)

// ---- exact cutoff: (k+1)-th largest of the 4096 bf16 probe products ------------------------------------------------
// keys[4]: this thread's 8 products as bf16x2 (non-negative; the bf16 bit pattern orders like the value).
// G(x) = #{keys > x}.  Wanted: t = min{x : G(x) <= k} = the (k+1)-th largest key (0 when k >= n).  Equivalently
// u = max{x : G(x) >= k+1} and t = u + 1 (t = 0 when even G(0) <= k).  u is built digit by digit: round 0 decides bit
// 14 (and evaluates G(0)), rounds 1..7 two bits each, the counts at the candidate thresholds taken in one pass.
__device__ __forceinline__ uint32_t splat_bf16(uint32_t key) { return key | (key << 16); }
__device__ __forceinline__ uint32_t count_gt2(const uint32_t (&keys)[4], uint32_t th) {
    const __nv_bfloat162 t = as_bf162(splat_bf16(th));
    __nv_bfloat162 c = __hgt2(as_bf162(keys[0]), t);
#pragma unroll
    for (int i = 1; i < 4; i++) c = __hadd2(c, __hgt2(as_bf162(keys[i]), t));
    return (uint32_t)bf162_count(c);  // 0..8
}

__device__ __forceinline__ float select_cutoff(const uint32_t (&keys)[4], int k, V2Header& hdr, int tid) {
    const int lane = tid & 31;
    uint32_t u = 0;
    bool any = true;  // G(0) >= k+1
    const unsigned need = (unsigned)(k + 1);
#pragma unroll 1
    for (int round = 0; round < 8; round++) {
        const int b = (round == 0) ? 14 : 14 - 2 * round;  // round 0: bit 14;  round r: bits (b+1, b)
        uint32_t th1, th2, th3;
        if (round == 0) { th1 = 0u; th2 = 1u << 14; th3 = 0x7FFFu; }
        else { th1 = u | (1u << b); th2 = u | (2u << b); th3 = u | (3u << b); }
        const uint32_t c1 = count_gt2(keys, th1), c2 = count_gt2(keys, th2), c3 = count_gt2(keys, th3);
        const uint32_t a = __reduce_add_sync(0xffffffffu, c1 | (c2 << 16));
        const uint32_t bsum = __reduce_add_sync(0xffffffffu, c3);
        if (lane == 0) {
            atomicAdd(&hdr.sel_acc[round][0], a);
            atomicAdd(&hdr.sel_acc[round][1], bsum);
        }
        __syncthreads();
        const uint32_t A = hdr.sel_acc[round][0], B = hdr.sel_acc[round][1];
        const unsigned g1 = A & 0xFFFFu, g2 = A >> 16, g3 = B;
        if (round == 0) {
            any = g1 >= need;
            if (g2 >= need) u = 1u << 14;
        } else {
            const unsigned j = (g1 >= need ? 1u : 0u) + (g2 >= need ? 1u : 0u) + (g3 >= need ? 1u : 0u);
            u |= j << b;
        }
    }
    const uint32_t t = any ? (u + 1u) : 0u;
    return __uint_as_float(t << 16);
}

// products of thread tid: bfloat(|1e5 * v[i] * bfloat(probes[i])|), i = 8*tid .. 8*tid+7   (bucketMul.metal:158-163)
__device__ __forceinline__ void score8(const float (&vv)[8], const uint4 pw4, uint32_t (&keys)[4]) {
    const uint32_t pw[4] = {pw4.x, pw4.y, pw4.z, pw4.w};
#pragma unroll
    for (int m = 0; m < 4; m++) {
        const float2 pf = __half22float2(*reinterpret_cast<const __half2*>(&pw[m]));
        const uint32_t pb = bf162_bits(__floats2bfloat162_rn(pf.x, pf.y));  // bfloat(probe)
        const float x0 = fabsf(__fmul_rn(__fmul_rn(kCutoffScale, vv[2 * m]), __uint_as_float(pb << 16)));
        const float x1 = fabsf(__fmul_rn(__fmul_rn(kCutoffScale, vv[2 * m + 1]), __uint_as_float(pb & 0xFFFF0000u)));
        keys[m] = bf162_bits(__floats2bfloat162_rn(x0, x1));
    }
}

__device__ __forceinline__ float silu_mul(float x1, float x3) { return x3 * x1 / (1.f + expf(-x1)); }  // matrix.metal:25-34

// One unit of N rows (same input, consecutive ranks) staged at row stride RSTRIDE: the N*VEC read-modify-writes of a lane
// never alias (see the list build), so they are issued as four batches -- staged words, accumulator loads, FMAs, stores.
template <int IMM>
__device__ __forceinline__ void lds64_imm(uint32_t addr, uint32_t& x, uint32_t& y) {
    asm volatile("ld.shared.v2.u32 {%0,%1}, [%2+%3];" : "=r"(x), "=r"(y) : "r"(addr), "n"(IMM));
}
template <int VEC, int N, int RSTRIDE>
__device__ __forceinline__ void accumulate_unit_fp16(uint32_t base_lane, float val, uint32_t a0) {
    static_assert(VEC == 4 && N >= 1 && N <= 4, "FP16 tiles: 4 columns (8 bytes) per lane and row");
    uint32_t w[4][2];
    lds64_imm<0>(a0, w[0][0], w[0][1]);
    if constexpr (N > 1) lds64_imm<RSTRIDE>(a0, w[1][0], w[1][1]);
    if constexpr (N > 2) lds64_imm<2 * RSTRIDE>(a0, w[2][0], w[2][1]);
    if constexpr (N > 3) lds64_imm<3 * RSTRIDE>(a0, w[3][0], w[3][1]);
    uint32_t a[N][VEC];
    float f[N][VEC], acc[N][VEC];
#pragma unroll
    for (int r = 0; r < N; r++) AccFp16<VEC, 0>::addr(w[r], base_lane, a[r], f[r]);
#pragma unroll
    for (int r = 0; r < N; r++) RmwFp16<VEC, 0>::load(a[r], acc[r]);
#pragma unroll
    for (int r = 0; r < N; r++)
#pragma unroll
        for (int k = 0; k < VEC; k++) acc[r][k] = fmaf(val, f[r][k], acc[r][k]);
#pragma unroll
    for (int r = 0; r < N; r++) RmwFp16<VEC, 0>::store(a[r], acc[r]);
}

template <int SLOTS, int VEC, int CUT, int D>
__global__ void __launch_bounds__(kV2Threads, 1)
bucket_mul_v2_kernel(const __grid_constant__ V2Batch batch) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    using L = V2Smem<SLOTS, VEC>;
    constexpr int NT = kV2Threads, NW = kV2Warps;
    constexpr int TF = L::kTileFloats;
    constexpr int TW = 32 * VEC;           // column lanes of a tile
    constexpr int LB = VEC * 2;            // bytes a lane consumes per row
    constexpr int kRowStride = V2Unit<VEC>::kRowStride, kUnitBytes = V2Unit<VEC>::kUnitBytes;

    int pi = 0;
#pragma unroll
    for (int k = 1; k < kMulBatchMax; k++) pi += (k < batch.n && (int)blockIdx.x >= batch.cta_begin[k]) ? 1 : 0;
    const V2Problem& pb = batch.p[pi];
    const int lb = (int)blockIdx.x - batch.cta_begin[pi];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int slice = lb % pb.CS, rsp = lb / pb.CS;
    const int RS = pb.RS, P = pb.P, C = pb.C;

    // ---- carve shared memory ----
    const uint32_t s0 = (uint32_t)__cvta_generic_to_shared(smem_raw);
    const uint32_t s1 = (s0 + (uint32_t)L::kTileBytes - 1u) & ~((uint32_t)L::kTileBytes - 1u);
    unsigned char* p = smem_raw + (s1 - s0);
    float* tiles = reinterpret_cast<float*>(p);
    const uint32_t tiles_saddr = s1;
    p += (size_t)NW * L::kTileBytes;
    V2Header& hdr = *reinterpret_cast<V2Header*>(p);
    p += L::kHdrBytes;
    uint32_t* sbase = reinterpret_cast<uint32_t*>(p);   // per local input: offset of its rank-0 row slice, 16-byte units
    p += (size_t)kV2MaxInputs * 4;
    float* sval = reinterpret_cast<float*>(p);          // per local input: the multiplier v[i]
    p += (size_t)kV2MaxInputs * 4;
    float* sstat = reinterpret_cast<float*>(p);         // Q4: per local input its 8 row averages (payload = v * avg)
    p += L::kStatBytes;
    uint16_t* list = reinterpret_cast<uint16_t*>(p);
    p += L::list_bytes(batch.list_cap);
    const uint32_t ring_saddr = (uint32_t)__cvta_generic_to_shared(p) + (uint32_t)warp * (uint32_t)(D * kUnitBytes);
    static_assert((D & (D - 1)) == 0 && D <= 8, "ring depth: a power of two, at most 8 barriers per warp");

    pdl_trigger();
    if (pb.exp_no) pdl_wait();  // the expert index may be produced by the previous kernel (MoE gate)
    const uint32_t e_no = pb.exp_no ? *pb.exp_no : 0u;
    V2_TRACE(0);

    // ---- 0. constant metadata, before the dependency wait (overlaps the previous kernel's tail under PDL) ----
    const uint64_t keep = l2_policy_evict_last();
    const int n_in = (pb.in > rsp) ? (pb.in - 1 - rsp) / RS + 1 : 0;  // inputs of this row split: i = rsp + j*RS
    const int j_in = tid;                                            // pass 0 local input of this thread
    float sel_stat[16];
#pragma unroll
    for (int rho = 0; rho < 16; rho++) sel_stat[rho] = 0.f;
    auto load_stats = [&](int j, float (&st)[16]) {
        const int i = rsp + j * RS;
        if constexpr (SLOTS == 16) {
            if (pb.layout != kRankMajor && P == 16) {
                const uint4* sp = reinterpret_cast<const uint4*>(pb.st16 + ((size_t)e_no * pb.in + i) * 16);
                const uint4 a = ldg_keep_u4(sp, keep), b = ldg_keep_u4(sp + 1, keep);
                const uint32_t ws[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
                for (int q2 = 0; q2 < 8; q2++) {
                    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&ws[q2]));
                    st[2 * q2] = f.x;
                    st[2 * q2 + 1] = f.y;
                }
            } else {
#pragma unroll
                for (int rho = 0; rho < 16; rho++)
                    if (rho < P) {
                        const size_t row = (pb.layout != kRankMajor) ? ((size_t)e_no * pb.in + i) * P + rho
                                                                      : (size_t)e_no * P * pb.in + (size_t)rho * pb.in + i;
                        st[rho] = __half2float(pb.st16[row]);
                    }
            }
        } else {
#pragma unroll
            for (int rho = 0; rho < 16; rho++)
                if (rho < P) st[rho] = pb.st32[((size_t)e_no * pb.in + i) * P + rho];
        }
    };
    if (j_in < n_in) load_stats(j_in, sel_stat);
    uint4 prb = make_uint4(0u, 0u, 0u, 0u);
    if constexpr (CUT == kCutSelect) prb = ldg_keep_u4(reinterpret_cast<const uint4*>(pb.probes + (size_t)e_no * EFFORT_PROBES_MAX) + tid, keep);
    uint4 nwv = make_uint4(0u, 0u, 0u, 0u);
    if (pb.norm_w) nwv = *reinterpret_cast<const uint4*>(pb.norm_w + 8 * tid);
    // zero this warp's accumulator tile, the select counters, the ring barriers
    {
        float4* t4 = reinterpret_cast<float4*>(tiles + (size_t)warp * TF);
        for (int i = lane; i < TF / 4; i += 32) t4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        for (uint32_t a = ring_saddr + (uint32_t)lane * 16u; a < ring_saddr + (uint32_t)(D * kUnitBytes); a += 512u)
            asm volatile("st.shared.v4.u32 [%0], {%1,%1,%1,%1};" ::"r"(a), "r"(0u) : "memory");  // lanes past a narrow slice read zeros
        if (tid < 16) hdr.sel_acc[tid >> 1][tid & 1] = 0u;
    }
    __syncthreads();  // select counters / barriers initialised before any warp uses them
    V2_TRACE(1);
    pdl_wait();

    // ---- 1. the input vector: 8 consecutive entries per thread for the cutoff, plus the thread's own input dim ----
    const int vmode = pb.norm_w ? kVNorm : (pb.v2 ? kVSilu : kVPlain);
    float vv[8];
    {
        const float* src = (vmode == kVPlain) ? pb.v_cut : pb.v;
        const float4 a = *reinterpret_cast<const float4*>(src + 8 * tid), b = *reinterpret_cast<const float4*>(src + 8 * tid + 4);
        vv[0] = a.x; vv[1] = a.y; vv[2] = a.z; vv[3] = a.w; vv[4] = b.x; vv[5] = b.y; vv[6] = b.z; vv[7] = b.w;
        if (vmode == kVSilu) {
            const float4 c = *reinterpret_cast<const float4*>(pb.v2 + 8 * tid), d = *reinterpret_cast<const float4*>(pb.v2 + 8 * tid + 4);
            const float x3[8] = {c.x, c.y, c.z, c.w, d.x, d.y, d.z, d.w};
#pragma unroll
            for (int m = 0; m < 8; m++) vv[m] = silu_mul(vv[m], x3[m]);
        }
    }
    float my_v = 0.f, my_x3 = 0.f, my_nw = 1.f;
    if (j_in < n_in) {
        const int i = rsp + j_in * RS;
        my_v = pb.v[i];
        if (vmode == kVSilu) my_x3 = pb.v2[i];
        if (vmode == kVNorm) my_nw = __half2float(pb.norm_w[i]);
    }
    // overwrite semantics: zero this CTA's share of its column slice and arrive on the slice counter; the counter is
    // only inspected right before the reductions at the end of the kernel
    const int slice_cols = min(pb.W, C - slice * pb.W);
    if (pb.out_mode == kOutOverwrite) {
        const int n_out = slice_cols * SLOTS;  // outputs of this slice (a multiple of 16)
        const int n4 = n_out / 4, per = (n4 + RS - 1) / RS;
        float4* o4 = reinterpret_cast<float4*>(pb.out + (size_t)slice * pb.W * SLOTS);
        for (int x = rsp * per + tid; x < min(n4, (rsp + 1) * per); x += NT) o4[x] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float denom = 1.f;
    if (vmode == kVNorm) {  // rmsNorm32fast (aux.metal:113-152): x / sqrt(mean(x^2) + eps); in == 8 * NT
        float ss = 0.f;
#pragma unroll
        for (int m = 0; m < 8; m++) ss += vv[m] * vv[m];
        ss = warp_sum_f(ss);
        if (lane == 0) hdr.red[warp] = ss;
        __syncthreads();
        float t = (lane < NW) ? hdr.red[lane] : 0.f;
        t = warp_sum_f(t);
        denom = sqrtf(t / (float)pb.in + pb.norm_eps);
        const uint32_t nw[4] = {nwv.x, nwv.y, nwv.z, nwv.w};
#pragma unroll
        for (int m = 0; m < 4; m++) {
            const float2 wf = __half22float2(*reinterpret_cast<const __half2*>(&nw[m]));
            vv[2 * m] = (vv[2 * m] / denom) * wf.x;
            vv[2 * m + 1] = (vv[2 * m + 1] / denom) * wf.y;
        }
        my_v = (my_v / denom) * my_nw;
    } else if (vmode == kVSilu) {
        my_v = silu_mul(my_v, my_x3);
    }
    if (pb.out_mode == kOutOverwrite) {
        __syncthreads();  // all zero stores of the CTA issued
        if (tid == 0) {
            __threadfence();
            atomicAdd(pb.sync + 2 * slice, 1u);
        }
    }
    V2_TRACE(2);

    // ---- 2. cutoff ----
    float cutoff;
    if constexpr (CUT == kCutSelect) {
        uint32_t keys[4];
        score8(vv, prb, keys);
        V2_TRACE(3);
        cutoff = select_cutoff(keys, EFFORT_PROBES_MAX - pb.q, hdr, tid);
    } else {
        // bit-exact replay of the reference's bisection by four warps (cutoff.cuh); it loads its own operands
        float* vtmp = reinterpret_cast<float*>(p);  // ring memory is idle until the rows stream
        if (vmode == kVSilu) {  // the silu'd input exists only in registers: stage the 4096 cutoff entries
#pragma unroll
            for (int m = 0; m < 8; m++) vtmp[8 * tid + m] = vv[m];
            __syncthreads();
        }
        if (tid < kCutThreads) {
            GroupProbes gpr;
            group_load_probes(pb.probes + (size_t)e_no * EFFORT_PROBES_MAX, EFFORT_PROBES_MAX, tid, gpr, keep);
            GroupProducts gp;
            if (vmode == kVNorm) group_score<true>(pb.v, gpr, EFFORT_PROBES_MAX, tid, gp, pb.norm_w, denom);
            else if (vmode == kVPlain) group_score<false>(pb.v_cut, gpr, EFFORT_PROBES_MAX, tid, gp, nullptr, 1.f);
            else group_score<false>(vtmp, gpr, EFFORT_PROBES_MAX, tid, gp, nullptr, 1.f);  // kVSilu: materialised below
            group_cutoff<1>(gp, EFFORT_PROBES_MAX, pb.q, hdr.cut, tid, nullptr);
        }
        __syncthreads();
        cutoff = hdr.cut.result;
        if (vmode == kVSilu) {  // the staging area doubles as the ring: back to zeros (see the prologue)
            for (uint32_t a = ring_saddr + (uint32_t)lane * 16u; a < ring_saddr + (uint32_t)(D * kUnitBytes); a += 512u)
                asm volatile("st.shared.v4.u32 [%0], {%1,%1,%1,%1};" ::"r"(a), "r"(0u) : "memory");
        }
    }
    if (pb.cutoff_out && lb == 0 && tid == 0) *pb.cutoff_out = cutoff;
    V2_TRACE(6);

    // lane-constant mapping of the staging copies and of the accumulate steps
    const int seg_bytes = slice_cols * 2;         // bytes of a row slice (multiple of 16)
    const int np = seg_bytes >> 4;                // 16-byte pieces per row slice (<= 16)
    const int lpr = pb.lpr, R = pb.R;             // lanes per row / rows per step
    const int rowslot = lane / lpr, lcol = lane % lpr;
    const bool col_ok = lcol * VEC < slice_cols;  // lanes past a narrow slice (the FP16 fast path reads zeros there instead)
    const uint32_t base_lane = (tiles_saddr + (uint32_t)warp * L::kTileBytes) | (uint32_t)(lane * 4);
    const uint64_t pol = l2_policy_evict_first();
    // 16-byte units: a unit starts at bk16 + sbase[input] + rank * rstride16
    const size_t slice_off = (pb.layout == kSliceMajor) ? (size_t)pb.in * P * ((size_t)slice * pb.W) : (size_t)slice * pb.W;
    const uint4* bk16 = reinterpret_cast<const uint4*>(pb.bk + slice_off);
    const uint32_t rstride16 = (pb.layout == kInputMajor) ? (uint32_t)(C >> 3)
                               : (pb.layout == kRankMajor) ? (uint32_t)(((size_t)pb.in * C) >> 3) : (uint32_t)np;
    // piece k2 of this lane inside a unit: row prow, 16-byte column pcol
    int prow[2];
    uint32_t psrc[2], pdst[2];
#pragma unroll
    for (int k2 = 0; k2 < 2; k2++) {
        const int pidx = lane + 32 * k2;
        prow[k2] = pidx / np;
        const int pc = pidx % np;
        psrc[k2] = (uint32_t)prow[k2] * rstride16 + (uint32_t)pc;
        pdst[k2] = (uint32_t)(prow[k2] * kRowStride + pc * 16);
    }
    constexpr uint32_t kEmpty = 0xFFFFFFFFu;
    constexpr uint32_t kHdrOff = kUnitRows * kRowStride;  // unit header: [0..3] multipliers, [4] unit code

    unsigned total_sel = 0;
    // ---- passes over the inputs of this row split (one pass for every Mistral shape) ----
    for (int j0 = 0; j0 < n_in; j0 += NT) {
        const int j = j0 + tid;
        if (j0 > 0) {  // later passes: nothing was prefetched
            __syncthreads();  // previous pass completely streamed before the list is rebuilt
#pragma unroll
            for (int rho = 0; rho < 16; rho++) sel_stat[rho] = 0.f;
            my_v = 0.f;
            if (j < n_in) {
                load_stats(j, sel_stat);
                const int i = rsp + j * RS;
                my_v = pb.v[i];
                if (vmode == kVNorm) my_v = (my_v / denom) * __half2float(pb.norm_w[i]);
                else if (vmode == kVSilu) my_v = silu_mul(my_v, pb.v2[i]);
            }
        }
        // 3. selection mask of this thread's input (prepareDispatch, bucketMul.metal:66)
        unsigned mask = 0u;
#pragma unroll
        for (int rho = 0; rho < 16; rho++)
            if (rho < P && j < n_in && row_selected(cutoff, sel_stat[rho], my_v)) mask |= 1u << rho;
        if (j < n_in) {
            const int i = rsp + j * RS;
            size_t el0;  // element offset of the input's rank-0 row slice, relative to bk16
            if (pb.layout == kInputMajor) el0 = ((size_t)e_no * pb.in + i) * P * C;
            else if (pb.layout == kRankMajor) el0 = ((size_t)e_no * P * pb.in + i) * C;
            else el0 = (size_t)e_no * pb.in * P * C + (size_t)i * P * slice_cols;
            sbase[tid] = (uint32_t)(el0 >> 3);
            sval[tid] = pb.out_scale ? my_v * *pb.out_scale : my_v;  // the selection above used the unscaled input
            if constexpr (SLOTS != 16) {
#pragma unroll
                for (int rho = 0; rho < 8; rho++) sstat[tid * 8 + rho] = sel_stat[rho];
            }
        }
        // units: maximal runs of selected ranks inside each aligned group of kUnitRows ranks (a bucket row set that is
        // a prefix in rank -- the normal case, the row means fall with rank -- gives one unit per group).  The rows of
        // a unit belong to ONE input and to consecutive ranks: their weights of a column go to 4 different outputs
        // (different elements of one bucket), so the read-modify-writes of a unit never alias.
        uint32_t ucode[8];
        unsigned uvalid = 0u;
#pragma unroll
        for (int g = 0; g < 4; g++) {
            unsigned nb = (mask >> (4 * g)) & 15u;
#pragma unroll
            for (int rr = 0; rr < 2; rr++) {
                ucode[2 * g + rr] = 0u;
                if (nb) {
                    const int st = __ffs((int)nb) - 1;
                    const int len = __ffs((int)~(nb >> st)) - 1;
                    ucode[2 * g + rr] = ((uint32_t)tid << 6) | ((uint32_t)(4 * g + st) << 2) | (uint32_t)(len - 1);
                    uvalid |= 1u << (2 * g + rr);
                    nb &= ~(((1u << len) - 1u) << st);
                }
            }
        }
        const int wtot = __reduce_add_sync(0xffffffffu, __popc(uvalid));
        const int wrows = __reduce_add_sync(0xffffffffu, __popc(mask));
        if (lane == 0) { hdr.warp_cnt[warp] = wtot; hdr.warp_rows[warp] = wrows; }
        if (tid == 0) hdr.next_unit = 0;
        __syncthreads();
        int base = 0, n_units = 0, n_rows = 0;
#pragma unroll
        for (int w = 0; w < NW; w++) {
            const int wc = hdr.warp_cnt[w];
            base += (w < warp) ? wc : 0;
            n_units += wc;
            n_rows += hdr.warp_rows[w];
        }
        const unsigned lt = (1u << lane) - 1u;
#pragma unroll
        for (int sl = 0; sl < 8; sl++) {
            const unsigned b = __ballot_sync(0xffffffffu, (uvalid >> sl) & 1u);
            if ((uvalid >> sl) & 1u) list[base + __popc(b & lt)] = (uint16_t)ucode[sl];
            base += __popc(b);
        }
        total_sel += (unsigned)n_rows;
        __syncthreads();  // list, sbase, sval (and the zeroed tiles / ring) visible
        V2_TRACE(8);

        // 4. stream the units.  Every warp keeps D units in flight in its private ring and takes the next unit from a
        //    shared counter when a slot frees up (the units differ in size, a static deal would leave warps idle).
        int static_next = warp;  // batch.dynamic == 0: warp w takes units w, w + 16, ...
        const uint32_t next_unit_saddr = (uint32_t)__cvta_generic_to_shared(&hdr.next_unit);
        auto issue_next = [&](int slot_i) {
            const uint32_t slot = ring_saddr + (uint32_t)slot_i * kUnitBytes;
            int u;
            if (batch.dynamic) {
                u = 0;
                if (lane == 0) asm volatile("atom.shared.add.u32 %0, [%1], 1;" : "=r"(u) : "r"(next_unit_saddr) : "memory");
                u = __shfl_sync(0xffffffffu, u, 0);
            } else {
                u = static_next;
                static_next += NW;
            }
            uint32_t code = kEmpty;
            if (u < n_units) {
                code = list[u];
                const uint32_t jj = code >> 6, r0 = (code >> 2) & 15u;
                const int n = (int)(code & 3u) + 1;
                const uint32_t ubase = sbase[jj] + r0 * rstride16;
#pragma unroll
                for (int k2 = 0; k2 < 2; k2++)
                    if (prow[k2] < n) cp_async16(slot + pdst[k2], bk16 + (size_t)(ubase + psrc[k2]), pol);
                if constexpr (SLOTS == 16) {
                    if (lane == 0) asm volatile("st.shared.f32 [%0], %1;" ::"r"(slot + kHdrOff), "f"(sval[jj]) : "memory");
                } else {
                    if (lane < n) {
                        const float val = __fmul_rn(sval[jj], sstat[jj * 8 + r0 + lane]);  // v * avg, bucketMulQ4.metal:51
                        asm volatile("st.shared.f32 [%0], %1;" ::"r"(slot + kHdrOff + (uint32_t)lane * 4u), "f"(val) : "memory");
                    }
                }
            }
            if (lane == 0) asm volatile("st.shared.u32 [%0], %1;" ::"r"(slot + kHdrOff + 16u), "r"(code) : "memory");
            cp_async_commit();
        };
#pragma unroll
        for (int m = 0; m < D; m++) issue_next(m);
        int head = 0;
#pragma unroll 1
        for (;;) {
            const uint32_t slot = ring_saddr + (uint32_t)head * kUnitBytes;
            cp_async_wait<D - 1>();
            __syncwarp();
            uint32_t code;
            asm volatile("ld.shared.u32 %0, [%1];" : "=r"(code) : "r"(slot + kHdrOff + 16u));
            if (code == kEmpty) break;
            const int n = (int)(code & 3u) + 1;
            if constexpr (SLOTS == 16) {
                float val;
                asm volatile("ld.shared.f32 %0, [%1];" : "=f"(val) : "r"(slot + kHdrOff));
                if (R == 1) {
                    const uint32_t a0 = slot + (uint32_t)(lane * LB);
                    switch (n) {
                        case 1: accumulate_unit_fp16<VEC, 1, kRowStride>(base_lane, val, a0); break;
                        case 2: accumulate_unit_fp16<VEC, 2, kRowStride>(base_lane, val, a0); break;
                        case 3: accumulate_unit_fp16<VEC, 3, kRowStride>(base_lane, val, a0); break;
                        default: accumulate_unit_fp16<VEC, 4, kRowStride>(base_lane, val, a0); break;
                    }
                } else {  // row slices narrower than a warp: R rows per step
                    for (int st = 0; st * R < n; st++) {
                        const int r = st * R + rowslot;
                        const bool ok = (rowslot < R) && (r < n) && col_ok;
                        const int rc = ok ? r : 0;
                        uint32_t ww[2];
                        const uint32_t a = slot + (uint32_t)(rc * kRowStride + lcol * LB);
                        asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(ww[0]), "=r"(ww[1]) : "r"(a));
                        accumulate_words<SLOTS, VEC>(base_lane, ok ? val : 0.f, ww);
                    }
                }
            } else {
                float4 v4;
                asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v4.x), "=f"(v4.y), "=f"(v4.z), "=f"(v4.w) : "r"(slot + kHdrOff));
                const float vals[4] = {v4.x, v4.y, v4.z, v4.w};
                for (int st = 0; st * R < n; st++) {
                    const int r = st * R + rowslot;
                    const bool ok = (rowslot < R) && (r < n) && col_ok;  // a zero word would still add +val: mask the lane
                    const int rc = ok ? r : 0;
                    uint32_t ww[1];
                    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(ww[0]) : "r"(slot + (uint32_t)(rc * kRowStride + lcol * LB)));
                    const float val = (rc == 0) ? vals[0] : (rc == 1) ? vals[1] : (rc == 2) ? vals[2] : vals[3];
                    accumulate_words<SLOTS, VEC>(base_lane, ok ? val : 0.f, ww);
                }
            }
            __syncwarp();  // every lane is done with the slot before it is refilled
            issue_next(head);
            head = (head + 1) & (D - 1);
        }
        cp_async_wait<0>();
    }
    if (pb.sel_counts && slice == 0 && tid == 0) pb.sel_counts[rsp] = total_sel;
    __syncthreads();
    V2_TRACE(9);

    // ---- 5. CTA epilogue: sum the 16 warp tiles and add into out ----
    // thread <-> (column lane cl, slot group sg): 4 consecutive slots of one column = 4 consecutive outputs
    {
        constexpr int NG = NT / TW;        // slot groups (FP16: 4, Q4: 8)
        constexpr int SPT = SLOTS / NG;    // slots per thread = 4
        static_assert(SPT == 4, "one 16-byte reduction per thread");
        const int cl = tid % TW, sg = tid / TW;
        const int k = cl >> 5, ln = cl & 31;
        float acc[SPT] = {0.f, 0.f, 0.f, 0.f};
        const bool col_on = (ln < lpr) && (ln * VEC + k < slice_cols);
        if (col_on) {
            for (int rs2 = 0; rs2 < R; rs2++) {
                const int word0 = (sg * SPT) * TW + k * 32 + ln + rs2 * lpr;
#pragma unroll
                for (int w = 0; w < NW; w++)
#pragma unroll
                    for (int s = 0; s < SPT; s++) acc[s] += tiles[(size_t)w * TF + word0 + s * TW];
            }
        }
        if (pb.out_mode == kOutOverwrite) {  // every CTA of the slice has zeroed its share?
            if (tid == 0) {
                const unsigned* cnt = pb.sync + 2 * slice;
                const unsigned long long t0 = gtime_ns();
                while (ld_acquire_u32(cnt) < (unsigned)RS) {
                    if (gtime_ns() - t0 > 2000000000ull) {  // 2 s: a CTA of the slice never ran
                        if (pb.err_flag) atomicExch(pb.err_flag, 1u);
                        break;
                    }
                }
            }
            __syncthreads();
        }
        if (col_on) {
            const int col = slice * pb.W + ln * VEC + k;
            red_add_v4(pb.out + (size_t)col * SLOTS + sg * SPT, acc[0], acc[1], acc[2], acc[3]);
        }
        if (pb.out_mode == kOutOverwrite) {
            __syncthreads();
            if (tid == 0) {  // last CTA of the slice to leave re-arms the counters for the next launch
                unsigned* sy = pb.sync + 2 * slice;
                const unsigned old = atomicAdd(sy + 1, 1u);
                if (old == (unsigned)RS - 1u) { sy[0] = 0u; sy[1] = 0u; }
            }
        }
    }
    V2_TRACE(10);
}

}  // namespace effort
