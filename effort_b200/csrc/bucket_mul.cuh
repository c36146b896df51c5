// bucket_mul.cuh -- the gathered multiply-accumulate over the selected bucket rows.
//
// Reference kernels replaced: prepareDispatch (bucketMul.metal:47-79), roundUp/zeroRange32 (:11-31),
// bucketMul (:83-117), bucketIntegrate (:122-137); Q4: prepareDispatchQ4 / bucketMulQ4
// (bucketMulQ4.metal:25-92).
//
// Design (see DESIGN.md section 3):
//  * HBM-bound gather, no tensor cores.  A bucket row is C 16-bit words; word (row r, column c) adds
//    val_r * w into out[c*SLOTS + slot(w)] where slot is data dependent (4 position bits in the FP16
//    mantissa; sign|pos nibbles in Q4).  The reference resolves the scatter with 16 predicated adds per
//    weight (ALU bound at 50-70% of DRAM bandwidth, docs/gpu.html:183-187).  Here every WARP owns a
//    private tile of fp32 accumulators in shared memory laid out [slot][k][lane], so that the
//    read-modify-write of lane L always hits bank L: conflict free for any slot pattern, and -- because
//    a lane owns its columns exclusively -- needs no atomics.  6 instructions per weight.
//  * Decomposition: the C columns are cut into CS slices of 32*VEC columns; the grid is CS x RS CTAs.
//    CTA (slice, rs) owns one column slice and the input dims i = rs (mod RS) (round robin, so the
//    concentration of selected rows in the low ranks cannot unbalance CTAs).  All NW warps of the CTA
//    are independent row streams over the same slice: no block barrier inside the streaming loop, each
//    lane keeps U vector loads (8 or 16 bytes, L1::no_allocate) in flight.
//  * Selection is fused: the CTA tests the stats of its input dims, compacts {val,rowOffset} into a
//    shared-memory list with ballot + prefix scan (deterministic order, no global atomics, no global
//    dispatch list) and streams only those rows.
//  * Cross-CTA reduction: RS partial tiles per slice (kept in tile layout so that every write and read
//    is coalesced) + a small integrate kernel that un-permutes into `out` (deterministic order).
#pragma once
#include "common.cuh"
#include "cutoff.cuh"

namespace effort {

enum RowLayout : int {
    kInputMajor = 0,  // row(e,i,rho) = (e*in + i)*P + rho      (device repack; Q4 native order)
    kRankMajor = 1,   // row(e,i,rho) = e*P*in + rho*in + i      (reference FP16 order, convert.metal:96)
    kSliceMajor = 2,  // [e][column slice s][i][rho][W_s columns]: the rows an input selects in a slice are CONTIGUOUS
                      // (bucket_mul_v2 only); stats as kInputMajor.  W = slice width, W_s = min(W, C - s*W)
};

struct MulGeom {
    int CS;   // column slices (= tiles of 32*VEC columns)
    int RS;   // row splits; grid = CS*RS
    int R;    // rows a warp processes per step (sub-warp rows when C is small)
    int lpr;  // lanes covering one row inside the tile when R > 1 (else 32)
};

template <int VEC>
__host__ __device__ inline MulGeom make_geom(int C, int n_cta) {
    MulGeom g;
    const int TW = 32 * VEC;
    g.CS = (C + TW - 1) / TW;
    g.RS = n_cta / g.CS;
    if (g.RS < 1) g.RS = 1;
    g.R = 1;
    g.lpr = 32;
    if (g.CS == 1) {
        const int lpr = (C + VEC - 1) / VEC;
        if (lpr <= 16 && (32 % lpr) == 0) { g.R = 32 / lpr; g.lpr = lpr; }
    }
    return g;
}

struct MulProblem {
    const float* v;           // [in] fp32
    const float* v_cut;       // first n_probes entries of the full input vector (== v unless row-sharded)
    const __half* st16;       // FP16 kind: one fp16 stat per row, same row order as `bk`
    const float* st32;        // Q4 kind:   one fp32 stat (avg) per row
    const uint16_t* bk;       // bucket rows [rows][C] 16-bit words
    const __half* probes;     // [E][n_probes]
    const uint32_t* exp_no;   // device scalar or null
    const float* cutoff_in;   // precomputed cutoff (device) or null -> computed in-kernel
    float* partial;           // [RS][CS][TILE_FLOATS] in tile layout
    uint32_t* sel_counts;     // [RS] rows selected per row split (written by slice 0)
    float* cutoff_out;        // optional: CTA 0 stores the cutoff it used
    int in, C, P, n_probes, q, layout;
    int list_cap;             // capacity of the shared-memory row list (entries)
    MulGeom g;
    // optional fused rmsNorm on load (decode loop, runNetwork.swift:126-127,173-175): when norm_w != null the
    // operator's input is v_eff[i] = (v[i] / sqrt(sum(sumsq[0..n_sumsq)) / norm_dim + norm_eps)) * norm_w[i]
    // (rmsNorm32fast aux.metal:113-152 + mulVec32by16 aux.metal:269); sumsq = per-block partial sums of v[i]^2
    // written by the producer (integrate epilogue / embed kernel).
    const __half* norm_w;
    const float* sumsq;
    int n_sumsq, norm_dim;
    float norm_eps;
    unsigned long long* trace;  // optional [grid][16] phase timestamps (globaltimer ns), debugging aid
};

__device__ __forceinline__ unsigned long long gtime_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
#define EFFORT_TRACE(k)                                                                    \
    do {                                                                                   \
        if (pb.trace && threadIdx.x == 0) pb.trace[(size_t)blockIdx.x * 16 + (k)] = gtime_ns(); \
    } while (0)

// ---- shared-memory accumulate ---------------------------------------------------------------------
// A warp tile is SLOTS x (32*VEC) floats, aligned to its own size, laid out [slot][k][lane]:
//   byte address = tile_base | slot * (128*VEC) | k*128 | lane*4
// so the slot lands in its own bit field and the whole address is ONE LOP3 ((x & mask) | base_lane)
// plus an immediate; lane L always hits bank L (conflict free for any slot pattern) and owns its
// words exclusively (plain read-modify-write, no atomics).
template <int IMM>
__device__ __forceinline__ float lds_imm(uint32_t addr) {
    float x;
    asm volatile("ld.shared.f32 %0, [%1+%2];" : "=f"(x) : "r"(addr), "n"(IMM));
    return x;
}
template <int IMM>
__device__ __forceinline__ void sts_imm(uint32_t addr, float x) {
    asm volatile("st.shared.f32 [%0+%1], %2;" ::"r"(addr), "n"(IMM), "f"(x));
}

// sqrt(mean(v^2) + eps) from the producer's per-block partial sums; every warp computes it redundantly in a
// fixed order (deterministic)
__device__ __forceinline__ float rms_denom(const float* __restrict__ sumsq, int n, int dim, float eps) {
    float t = 0.f;
    for (int b = threadIdx.x & 31; b < n; b += 32) t += sumsq[b];
    t = warp_sum_f(t);
    return sqrtf(t / (float)dim + eps);
}

constexpr int kMulBatchMax = 4;
constexpr int EFFORT_PROBES_MAX = 4096;  // probesCount (bucketMul.swift:19): the fused path supports exactly this
// Several independent problems in ONE launch (q/k/v share v, runNetwork.swift:132-134; w1/w3, :178-179):
// CTAs [cta_begin[p], cta_begin[p+1]) work on problem p.
struct MulBatch {
    int n;
    int delay_ns;  // experiment knob (EFFORT_DELAY_NS): spin this long between the cutoff and the row list
    int cta_begin[kMulBatchMax + 1];
    MulProblem p[kMulBatchMax];
};

template <int VEC>
struct TileBits {
    static constexpr int kSlotShift = (VEC == 8) ? 10 : (VEC == 4) ? 9 : 8;  // log2(128*VEC)
};

// FP16 (SLOTS = 16): out[c*16 + (bits&15)] += val * float(w)       bucketMul.metal:100-106
template <int VEC, int J>
struct AccFp16 {
    static __device__ __forceinline__ void addr(const uint32_t (&words)[VEC / 2], uint32_t base_lane,
                                                uint32_t (&a)[VEC], float (&w)[VEC]) {
        constexpr int SH = TileBits<VEC>::kSlotShift;
        constexpr uint32_t MASK = 15u << SH;
        const uint32_t r = words[J];
        a[2 * J] = ((r << SH) & MASK) | base_lane;
        a[2 * J + 1] = ((r >> (16 - SH)) & MASK) | base_lane;
        const float2 f2 = __half22float2(*reinterpret_cast<const __half2*>(&r));
        w[2 * J] = f2.x;
        w[2 * J + 1] = f2.y;
        if constexpr (J + 1 < VEC / 2) AccFp16<VEC, J + 1>::addr(words, base_lane, a, w);
    }
};
template <int VEC, int K>
struct RmwFp16 {
    static __device__ __forceinline__ void load(const uint32_t (&a)[VEC], float (&acc)[VEC]) {
        acc[K] = lds_imm<K * 128>(a[K]);
        if constexpr (K + 1 < VEC) RmwFp16<VEC, K + 1>::load(a, acc);
    }
    static __device__ __forceinline__ void store(const uint32_t (&a)[VEC], const float (&acc)[VEC]) {
        sts_imm<K * 128>(a[K], acc[K]);
        if constexpr (K + 1 < VEC) RmwFp16<VEC, K + 1>::store(a, acc);
    }
};

// Q4 (SLOTS = 32): word k, nibble i (low nibble <-> i=3): out[c*32 + i*8 + (w&7)] += (w&8) ? -val : val
//                                                                   bucketMulQ4.metal:78-83
// The 4 nibbles of a word address 4 different 8-slot groups: they never alias.
template <int VEC, int K>
struct AccQ4 {
    static __device__ __forceinline__ void run(const uint32_t (&words)[(VEC + 1) / 2], uint32_t base_lane,
                                               float val) {
        constexpr int SH = TileBits<VEC>::kSlotShift;  // slot stride = 128*VEC bytes
        const uint32_t w = (words[K >> 1] >> ((K & 1) * 16)) & 0xFFFFu;
        uint32_t a[4];
        float x[4], acc[4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const uint32_t nib = (w >> (4 * (3 - i))) & 15u;
            x[i] = (nib & 8u) ? -val : val;
            a[i] = (((uint32_t)(i * 8) + (nib & 7u)) << SH) | base_lane;
        }
#pragma unroll
        for (int i = 0; i < 4; i++) acc[i] = lds_imm<K * 128>(a[i]);
#pragma unroll
        for (int i = 0; i < 4; i++) acc[i] += x[i];
#pragma unroll
        for (int i = 0; i < 4; i++) sts_imm<K * 128>(a[i], acc[i]);
        if constexpr (K + 1 < VEC) AccQ4<VEC, K + 1>::run(words, base_lane, val);
    }
};

template <int SLOTS, int VEC>
__device__ __forceinline__ void accumulate_words(uint32_t base_lane, float val,
                                                 const uint32_t (&words)[(VEC + 1) / 2]) {
    if constexpr (SLOTS == 16) {
        uint32_t a[VEC];
        float w[VEC], acc[VEC];
        AccFp16<VEC, 0>::addr(words, base_lane, a, w);
        RmwFp16<VEC, 0>::load(a, acc);
#pragma unroll
        for (int k = 0; k < VEC; k++) acc[k] = fmaf(val, w[k], acc[k]);
        RmwFp16<VEC, 0>::store(a, acc);
    } else {
        AccQ4<VEC, 0>::run(words, base_lane, val);
    }
}

template <int VEC>
__device__ __forceinline__ void load_words(const uint16_t* p, uint32_t (&words)[(VEC + 1) / 2], uint64_t pol) {
    if constexpr (VEC == 8) {
        uint4 d = ldg_stream_u4(p, pol);
        words[0] = d.x; words[1] = d.y; words[2] = d.z; words[3] = d.w;
    } else if constexpr (VEC == 4) {
        uint2 d = ldg_stream_u2(p, pol);
        words[0] = d.x; words[1] = d.y;
    } else {
        words[0] = ldg_stream_u1(p, pol);
    }
}

// ---- streaming: one warp walks its share of the row list --------------------------------------------
// list entries are {float val, uint32 rowOffset} read with one 8-byte broadcast LDS.  The loop is branch
// free (an entry past the end, or a lane past the last column, loads nothing and adds 0.0 into the lane's
// own words) and SOFTWARE PIPELINED: the U loads of batch n+1 are in flight while batch n is accumulated, so
// every lane always has U..2U vector loads outstanding (HBM latency x bandwidth needs ~40 KB per SM).
template <int SLOTS, int VEC, int U>
__device__ __forceinline__ void stream_rows(const uint2* __restrict__ list, int n_list,
                                            const uint16_t* __restrict__ bk, int C, int slice,
                                            const MulGeom g, uint32_t tile_saddr, int warp, int n_stream_warps) {
    const int lane = threadIdx.x & 31;
    const int rowslot = lane / g.lpr;
    const int col = slice * 32 * VEC + (lane % g.lpr) * VEC;
    const bool lane_on = (col < C) && (rowslot < g.R);
    const uint32_t base_lane = tile_saddr | (uint32_t)(lane * 4);
    const uint16_t* bk_col = bk + col;
    const int stride = n_stream_warps * g.R;  // list entries consumed per step by all streaming warps
    const int first = warp * g.R + rowslot;
    const int nsteps = (n_list + stride - 1) / stride;
    const uint64_t pol = l2_policy_evict_first();
    constexpr int NWD = (VEC + 1) / 2;
    uint32_t wa[U][NWD], wb[U][NWD];
    float va[U], vb[U];
    auto load_batch = [&](int n0, uint32_t (&w)[U][NWD], float (&val)[U]) {
#pragma unroll
        for (int u = 0; u < U; u++) {
            const int e = (n0 + u) * stride + first;
            const bool ok = lane_on && (e < n_list);
            val[u] = 0.f;
#pragma unroll
            for (int j = 0; j < NWD; j++) w[u][j] = 0u;
            if (ok) {
                const uint2 ent = list[e];
                val[u] = __uint_as_float(ent.x);
                load_words<VEC>(bk_col + (size_t)ent.y, w[u], pol);
            }
        }
    };
    auto process_batch = [&](const uint32_t (&w)[U][NWD], const float (&val)[U]) {
#pragma unroll
        for (int u = 0; u < U; u++) accumulate_words<SLOTS, VEC>(base_lane, val[u], w[u]);
    };
    load_batch(0, wa, va);
    for (int n0 = 0; n0 < nsteps; n0 += 2 * U) {
        load_batch(n0 + U, wb, vb);
        process_batch(wa, va);
        load_batch(n0 + 2 * U, wa, va);
        process_batch(wb, vb);
    }
}

// Same walk with the rows staged through a per-warp shared-memory ring filled by cp.async: D row slices
// (D x 32 lanes x VEC*2 bytes) are ALWAYS in flight per warp at no register cost -- the register-buffered loop
// above keeps U (8) -- which is what the long-scoreboard stalls of the streaming phase ask for (ncu: 4.7 stalled
// warps per issue on global loads).  A lane copies and later reads back only its own bytes, so the ring needs no
// barrier: cp.async.wait_group orders the lane's copies before its loads.
template <int SLOTS, int VEC, int D>
__device__ __forceinline__ void stream_rows_ring(const uint2* __restrict__ list, int n_list,
                                                 const uint16_t* __restrict__ bk, int C, int slice, const MulGeom g,
                                                 uint32_t tile_saddr, uint32_t ring_saddr, int warp, int n_stream_warps) {
    static_assert((D & (D - 1)) == 0, "ring depth must be a power of two");
    constexpr int LB = VEC * 2;       // bytes per lane per row slice
    constexpr int NWD = (VEC + 1) / 2;
    const int lane = threadIdx.x & 31;
    const int rowslot = lane / g.lpr;
    const int col = slice * 32 * VEC + (lane % g.lpr) * VEC;
    const bool lane_on = (col < C) && (rowslot < g.R);
    const uint32_t base_lane = tile_saddr | (uint32_t)(lane * 4);
    const uint16_t* bk_col = bk + col;
    const int stride = n_stream_warps * g.R;
    const int first = warp * g.R + rowslot;
    const int nsteps = (n_list + stride - 1) / stride;
    const uint64_t pol = l2_policy_evict_first();
    const uint32_t my_ring = ring_saddr + (uint32_t)lane * LB;
    auto issue = [&](int n) {
        const int e = n * stride + first;
        if (lane_on && e < n_list) cp_async_hint<LB>(my_ring + (uint32_t)(n & (D - 1)) * (32 * LB), bk_col + (size_t)list[e].y, pol);
        cp_async_commit();
    };
#pragma unroll
    for (int n = 0; n < D; n++) issue(n);
#pragma unroll 4
    for (int n = 0; n < nsteps; n++) {
        cp_async_wait<D - 1>();
        const int e = n * stride + first;
        const bool ok = lane_on && (e < n_list);
        float val = 0.f;
        uint32_t w[NWD];
#pragma unroll
        for (int j = 0; j < NWD; j++) w[j] = 0u;
        if (ok) {
            val = __uint_as_float(list[e].x);
            const uint32_t a = my_ring + (uint32_t)(n & (D - 1)) * (32 * LB);
            if constexpr (VEC == 8) asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]) : "r"(a));
            else if constexpr (VEC == 4) asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(w[0]), "=r"(w[1]) : "r"(a));
            else asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w[0]) : "r"(a));
        }
        accumulate_words<SLOTS, VEC>(base_lane, val, w);
        issue(n + D);
    }
    cp_async_wait<0>();
}

template <int NW>
struct MulSmemHeader {
    CutoffSmem cut;
    int warp_cnt[NW];
};

// dynamic smem layout (tiles first, each aligned to its own size so that slot bits can be OR-ed in):
//   [pad to TILE_BYTES][tiles: NW*TILE_BYTES][MulSmemHeader][list: cap x uint2]
template <int SLOTS, int VEC, int NW>
struct MulSmem {
    static constexpr int kTileFloats = SLOTS * 32 * VEC;
    static constexpr int kTileBytes = kTileFloats * 4;
    static constexpr size_t kHdrBytes = (sizeof(MulSmemHeader<NW>) + 15) & ~size_t(15);
    static __host__ __device__ size_t ring_bytes(int ring_depth) { return (size_t)NW * ring_depth * 32 * VEC * 2; }
    static __host__ __device__ size_t bytes(int list_cap, int ring_depth = 0) {
        return (size_t)kTileBytes /*alignment slack*/ + (size_t)NW * kTileBytes + kHdrBytes + ring_bytes(ring_depth) +
               (size_t)list_cap * 8;
    }
};

template <int NW>
struct MulSmemView {
    float* tiles;          // generic pointer to tile 0
    uint32_t tiles_saddr;  // shared-window address of tile 0 (aligned to the tile size)
    MulSmemHeader<NW>* hdr;
    uint32_t ring_saddr;   // shared-window address of the cp.async ring (warp w: + w * D * 32 * VEC * 2)
    uint2* list;
};

template <int SLOTS, int VEC, int NW>
__device__ __forceinline__ MulSmemView<NW> carve_smem(unsigned char* raw, int ring_depth = 0) {
    using L = MulSmem<SLOTS, VEC, NW>;
    const uint32_t s0 = (uint32_t)__cvta_generic_to_shared(raw);
    const uint32_t s1 = (s0 + (uint32_t)L::kTileBytes - 1u) & ~((uint32_t)L::kTileBytes - 1u);
    unsigned char* p = raw + (s1 - s0);
    MulSmemView<NW> v;
    v.tiles = reinterpret_cast<float*>(p);
    v.tiles_saddr = s1;
    p += (size_t)NW * L::kTileBytes;
    v.hdr = reinterpret_cast<MulSmemHeader<NW>*>(p);
    v.ring_saddr = s1 + (uint32_t)((size_t)NW * L::kTileBytes + L::kHdrBytes);
    v.list = reinterpret_cast<uint2*>(p + L::kHdrBytes + L::ring_bytes(ring_depth));
    return v;
}

template <int SLOTS, int VEC, int NW>
__device__ __forceinline__ void zero_my_tile(float* tiles) {
    constexpr int TF = MulSmem<SLOTS, VEC, NW>::kTileFloats;
    float4* t4 = reinterpret_cast<float4*>(tiles + (size_t)(threadIdx.x >> 5) * TF);
    for (int i = threadIdx.x & 31; i < TF / 4; i += 32) t4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
}

// ---- CTA epilogue: fold the NW warp tiles (and the R row slots) into one partial tile ----------------
// Thread t handles tile words t, t+NT, ...: consecutive lanes read consecutive banks and the global write
// is coalesced.  Lanes >= lpr of a sub-warp-row tile are folded into lane % lpr and written as 0.
template <int SLOTS, int VEC, int NW>
__device__ __forceinline__ void reduce_tiles_to_partial(const float* __restrict__ tiles, const MulGeom g,
                                                        float* __restrict__ partial) {
    constexpr int TF = MulSmem<SLOTS, VEC, NW>::kTileFloats;
    // 4 consecutive words per thread: NW independent 16-byte shared loads (conflict free), one 16-byte store
    for (int idx = threadIdx.x * 4; idx < TF; idx += NW * 32 * 4) {
        float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int w = 0; w < NW; w++) {
            const float4 a = *reinterpret_cast<const float4*>(tiles + (size_t)w * TF + idx);
            sum.x += a.x; sum.y += a.y; sum.z += a.z; sum.w += a.w;
        }
        if (g.R > 1) {  // sub-warp rows: fold the row slots into lanes < lpr (lpr is a multiple of 1, idx%32 = lane of .x)
            float s4[4] = {sum.x, sum.y, sum.z, sum.w};
#pragma unroll
            for (int e = 0; e < 4; e++) {
                const int lane = (idx + e) & 31;
                if (lane < g.lpr) {
                    for (int rs = 1; rs < g.R; rs++)
#pragma unroll
                        for (int w = 0; w < NW; w++) s4[e] += tiles[(size_t)w * TF + idx + e + rs * g.lpr];
                } else {
                    s4[e] = 0.f;
                }
            }
            sum = make_float4(s4[0], s4[1], s4[2], s4[3]);
        }
        *reinterpret_cast<float4*>(partial + idx) = sum;
    }
}

// ---- fused kernel: cutoff (optional) + selection + gather-MAC + CTA partial -------------------------
template <int SLOTS, int VEC, int U, int NW, bool NORM, int RING>
__global__ void __launch_bounds__(NW * 32, 1)
bucket_mul_fused_kernel(const __grid_constant__ MulBatch batch) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    using L = MulSmem<SLOTS, VEC, NW>;
    constexpr int NT = NW * 32;
    const MulSmemView<NW> sv = carve_smem<SLOTS, VEC, NW>(smem_raw, RING);
    MulSmemHeader<NW>& hdr = *sv.hdr;
    uint2* list = sv.list;

    int pi = 0;
#pragma unroll
    for (int k = 1; k < kMulBatchMax; k++) pi += (k < batch.n && (int)blockIdx.x >= batch.cta_begin[k]) ? 1 : 0;
    const MulProblem& pb = batch.p[pi];
    const int lb = (int)blockIdx.x - batch.cta_begin[pi];  // CTA index inside the problem

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    pdl_trigger();
    if (pb.exp_no) pdl_wait();  // the expert index may be produced by the previous kernel (MoE gate)
    const uint32_t e_no = pb.exp_no ? *pb.exp_no : 0u;
    const MulGeom g = pb.g;
    const int slice = lb % g.CS, rsp = lb / g.CS;

    EFFORT_TRACE(0);

    // 0. issue every global load the selection needs BEFORE the cutoff is known (they do not depend on
    //    it): thread <-> input dim i = rsp + j*RS, its v[i] and its P stats (32 contiguous bytes in the
    //    input-major repack).  One DRAM/L2 round trip for the whole prologue instead of one per stage.
    const int P = pb.P;
    const uint64_t keep = l2_policy_evict_last();
    const int n_in = (pb.in > rsp) ? (pb.in - 1 - rsp) / g.RS + 1 : 0;
    constexpr int KSEL = 1;  // inputs per thread held in registers; more are handled by the tail loop
    float sel_v[KSEL];
    float sel_stat[KSEL][16];
#pragma unroll
    for (int k = 0; k < KSEL; k++) {
        const int j = tid + k * NT;
        sel_v[k] = 0.f;
#pragma unroll
        for (int rho = 0; rho < 16; rho++) sel_stat[k][rho] = 0.f;
        if (j < n_in) {
            const int i = rsp + j * g.RS;
            if constexpr (SLOTS == 16) {
                if (pb.layout == kInputMajor && P == 16) {
                    const uint4* sp = reinterpret_cast<const uint4*>(pb.st16 + ((size_t)e_no * pb.in + i) * 16);
                    const uint4 s0 = ldg_keep_u4(sp, keep), s1 = ldg_keep_u4(sp + 1, keep);
                    const uint32_t ws[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
#pragma unroll
                    for (int q2 = 0; q2 < 8; q2++) {
                        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&ws[q2]));
                        sel_stat[k][2 * q2] = f.x;
                        sel_stat[k][2 * q2 + 1] = f.y;
                    }
                } else {
#pragma unroll
                    for (int rho = 0; rho < 16; rho++)
                        if (rho < P) {
                            const size_t row = (pb.layout == kInputMajor)
                                                   ? ((size_t)e_no * pb.in + i) * P + rho
                                                   : (size_t)e_no * P * pb.in + (size_t)rho * pb.in + i;
                            sel_stat[k][rho] = __half2float(pb.st16[row]);
                        }
                }
            } else {
#pragma unroll
                for (int rho = 0; rho < 16; rho++)
                    if (rho < P) sel_stat[k][rho] = pb.st32[((size_t)e_no * pb.in + i) * P + rho];
            }
        }
    }

    // the cutoff is computed by the first kCutWarps warps (cutoff.cuh, group path)
    const bool cut_thread = !pb.cutoff_in && tid < kCutThreads;
    GroupProbes prb;
    if (cut_thread) group_load_probes(pb.probes + (size_t)e_no * pb.n_probes, pb.n_probes, tid, prb, keep);
    // everything above read only constant weight metadata: under PDL it overlaps the previous kernel's tail.
    zero_my_tile<SLOTS, VEC, NW>(sv.tiles);  // while those loads are in flight
    EFFORT_TRACE(1);
    pdl_wait();
    float denom = 1.f;
    if constexpr (NORM) denom = rms_denom(pb.sumsq, pb.n_sumsq, pb.norm_dim, pb.norm_eps);
    auto v_eff = [&](int i) -> float {
        float x = pb.v[i];
        if constexpr (NORM) x = (x / denom) * __half2float(pb.norm_w[i]);
        return x;
    };
#pragma unroll
    for (int k = 0; k < KSEL; k++) {
        const int j = tid + k * NT;
        if (j < n_in) sel_v[k] = v_eff(rsp + j * g.RS);
    }
    EFFORT_TRACE(2);
    // 1. cutoff (every CTA redundantly: 24 KB of L2-resident inputs, no extra launch / global round trip)
    float cutoff;
    if (pb.cutoff_in) {
        cutoff = *pb.cutoff_in;
    } else {
        if (cut_thread) {
            GroupProducts gp;
            group_score<NORM>(pb.v_cut, prb, pb.n_probes, tid, gp, pb.norm_w, denom);
            EFFORT_TRACE(3);
            group_cutoff<1>(gp, pb.n_probes, pb.q, hdr.cut, tid, pb.trace ? pb.trace + (size_t)blockIdx.x * 16 : nullptr);
        }
        __syncthreads();
        cutoff = hdr.cut.result;
    }
    if (pb.cutoff_out && lb == 0 && tid == 0) *pb.cutoff_out = cutoff;
    EFFORT_TRACE(6);
    if (batch.delay_ns > 0) {
        const unsigned long long t0 = gtime_ns();
        while (gtime_ns() - t0 < (unsigned long long)batch.delay_ns) { }
    }

    // 2. selection + compaction.  Thread order == (input, rank) order == ascending row order, so the list
    //    is deterministic and consecutive entries are consecutive rows in HBM.
    int base = 0;
    for (int j0 = 0; j0 < n_in; j0 += NT * KSEL) {
        unsigned mask[KSEL];
        int cnt = 0;
#pragma unroll
        for (int k = 0; k < KSEL; k++) {
            mask[k] = 0u;
            const int j = j0 + tid + k * NT;
            if (j0 == 0) {
#pragma unroll
                for (int rho = 0; rho < 16; rho++)
                    if (rho < P && j < n_in && row_selected(cutoff, sel_stat[k][rho], sel_v[k])) mask[k] |= 1u << rho;
            } else if (j < n_in) {  // tail (more than NT*KSEL inputs per CTA): loads not prefetched
                const int i = rsp + j * g.RS;
                sel_v[k] = v_eff(i);
                for (int rho = 0; rho < P; rho++) {
                    const size_t row = (pb.layout == kInputMajor)
                                           ? ((size_t)e_no * pb.in + i) * P + rho
                                           : (size_t)e_no * P * pb.in + (size_t)rho * pb.in + i;
                    float st;
                    if constexpr (SLOTS == 16) st = __half2float(pb.st16[row]);
                    else st = pb.st32[row];
                    if (row_selected(cutoff, st, sel_v[k])) mask[k] |= 1u << rho;
                }
            }
            cnt += __popc(mask[k]);
        }
        EFFORT_TRACE(7);
        // block exclusive scan of cnt (order: k-major inside a thread is NOT input order, so scan per k)
#pragma unroll
        for (int k = 0; k < KSEL; k++) {
            const int c = __popc(mask[k]);
            int incl = c;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += t;
            }
            if (lane == 31) hdr.warp_cnt[warp] = incl;
            __syncthreads();
            int pre = 0, tot = 0;
#pragma unroll
            for (int w = 0; w < NW; w++) {
                const int wc = hdr.warp_cnt[w];
                pre += (w < warp) ? wc : 0;
                tot += wc;
            }
            int pos = base + pre + incl - c;
            const int j = j0 + tid + k * NT;
            if (c) {
                const int i = rsp + j * g.RS;
                unsigned m = mask[k];
                while (m) {
                    const int rho = __ffs(m) - 1;
                    m &= m - 1;
                    const size_t row = (pb.layout == kInputMajor)
                                           ? ((size_t)e_no * pb.in + i) * P + rho
                                           : (size_t)e_no * P * pb.in + (size_t)rho * pb.in + i;
                    // Q4 payload is v*avg (bucketMulQ4.metal:51)
                    float val = sel_v[k];
                    if constexpr (SLOTS != 16) {
                        float st = 0.f;
                        if (j0 == 0) {
#pragma unroll
                            for (int r2 = 0; r2 < 16; r2++) st = (r2 == rho) ? sel_stat[k][r2] : st;
                        } else {
                            st = pb.st32[row];
                        }
                        val = __fmul_rn(val, st);
                    }
                    list[pos++] = make_uint2(__float_as_uint(val), (uint32_t)(row * (size_t)pb.C));
                }
            }
            base += tot;
            __syncthreads();
        }
        (void)cnt;
    }
    const int n_list = base;
    if (pb.sel_counts && slice == 0 && tid == 0) pb.sel_counts[rsp] = (uint32_t)n_list;
    __syncthreads();  // list + zeroed tiles visible
    EFFORT_TRACE(8);

    // 3. stream the selected rows
    if constexpr (RING > 0)
        stream_rows_ring<SLOTS, VEC, RING>(list, n_list, pb.bk, pb.C, slice, g, sv.tiles_saddr + (uint32_t)warp * L::kTileBytes,
                                           sv.ring_saddr + (uint32_t)warp * (RING * 32 * VEC * 2), warp, NW);
    else
        stream_rows<SLOTS, VEC, U>(list, n_list, pb.bk, pb.C, slice, g,
                                   sv.tiles_saddr + (uint32_t)warp * L::kTileBytes, warp, NW);
    __syncthreads();
    EFFORT_TRACE(9);

    // 4. CTA partial (tile layout)
    reduce_tiles_to_partial<SLOTS, VEC, NW>(sv.tiles, g, pb.partial + (size_t)lb * L::kTileFloats);
    EFFORT_TRACE(10);
}

// ---- test-hook kernel: MAC over a reference-format dispatch list (BucketMul.mul) --------------------
// dispatch: float2 {val, float(rowOffset)} in the reference's rank-major element offsets.
template <int SLOTS, int VEC, int U, int NW>
__global__ void __launch_bounds__(NW * 32, 1)
bucket_mul_dispatch_kernel(const uint16_t* __restrict__ bk, const float2* __restrict__ dispatch,
                           const uint32_t* __restrict__ dispatch_size, int C, int list_cap, const MulGeom g,
                           float* __restrict__ partial) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    using L = MulSmem<SLOTS, VEC, NW>;
    constexpr int NT = NW * 32;
    const MulSmemView<NW> sv = carve_smem<SLOTS, VEC, NW>(smem_raw);
    uint2* list = sv.list;
    const int tid = threadIdx.x, warp = tid >> 5;
    const int slice = (int)blockIdx.x % g.CS, rsp = (int)blockIdx.x / g.CS;
    zero_my_tile<SLOTS, VEC, NW>(sv.tiles);

    // the reference splits the (padded) dispatch into 32 contiguous group slices (bucketMul.metal:94);
    // here: RS contiguous slices, walked in chunks of list_cap entries.
    const uint32_t n = *dispatch_size;
    const uint32_t per = (n + g.RS - 1) / g.RS;
    const uint32_t lo = min(n, per * (uint32_t)rsp), hi = min(n, lo + per);
    for (uint32_t c0 = lo; c0 < hi; c0 += (uint32_t)list_cap) {
        const int m = (int)min((uint32_t)list_cap, hi - c0);
        __syncthreads();
        for (int i = tid; i < m; i += NT) {
            const float2 d = dispatch[c0 + i];
            list[i] = make_uint2(__float_as_uint(d.x), (uint32_t)d.y);  // int(d[1]), bucketMul.metal:98
        }
        __syncthreads();
        stream_rows<SLOTS, VEC, U>(list, m, bk, C, slice, g, sv.tiles_saddr + (uint32_t)warp * L::kTileBytes, warp, NW);
    }
    __syncthreads();
    reduce_tiles_to_partial<SLOTS, VEC, NW>(sv.tiles, g, partial + (size_t)blockIdx.x * L::kTileFloats);
}

// ---- integrate: out[o] (=|+=) sum over the RS partial tiles   (bucketIntegrate, bucketMul.metal:122-137)
// Block = 8 warps x 32 consecutive tile words: warp w sums the partials r = w (mod 8) (coalesced 128-byte
// rows, all loads independent), shared-memory fold, then warp 0 un-permutes tile word -> output index.
// accumulate != 0 keeps the Q4 semantics (adds INTO out, bucketMulQ4.metal:89).
enum IntegrateMode : int {
    kIntStore = 0,     // out[o] = sum                     (bucketIntegrate, bucketMul.metal:122-137)
    kIntAccumulate,    // out[o] += sum                    (Q4: atomics INTO out, bucketMulQ4.metal:89)
    kIntSiluPair,      // items 0/1 = x1/x3 of one layer: out0[o] = x3 * x1 / (1 + exp(-x1))   (silu32b, matrix.metal:25-34)
    kIntResidual,      // out[o] (= h) += sum, and sumsq[block] = sum over the block's outputs of h_new^2
};
struct IntegrateItem {
    const float* partial;
    float* out;
    const uint32_t* sel_counts;
    uint32_t* n_selected;
    MulGeom g;
    int C, mode;
    float* sumsq;  // kIntResidual: [gridDim.x] per-block partial sums of squares
};
struct IntegrateBatch {
    int n;
    IntegrateItem it[kMulBatchMax];
};

// Block = 8 warps x 32 consecutive tile words: warp w sums the partials r = w (mod 8) (coalesced 128-byte rows, all
// loads independent), shared-memory fold, then warp 0 un-permutes tile word -> output index and applies the epilogue.
template <int SLOTS, int VEC>
__global__ void __launch_bounds__(256)
integrate_kernel(const __grid_constant__ IntegrateBatch ib) {
    constexpr int TW = 32 * VEC;
    constexpr int TF = SLOTS * TW;
    __shared__ float red[2][8][32];
    pdl_trigger();
    pdl_wait();
    const IntegrateItem& it = ib.it[blockIdx.y];
    const MulGeom g = it.g;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int j = blockIdx.x * 32 + lane;  // word index in [0, CS*TF)
    if (blockIdx.x * 32 >= g.CS * TF) return;  // whole block past this problem's words (block uniform)
    if (it.mode == kIntSiluPair && blockIdx.y == 1) {  // handled together with item 0
        if (it.n_selected && it.sel_counts && blockIdx.x == 0 && threadIdx.x == 0) {
            uint32_t t = 0;
            for (int r = 0; r < g.RS; r++) t += it.sel_counts[r];
            *it.n_selected = t;
        }
        return;
    }
    const int slice = j / TF, idx = j % TF;
    float s = 0.f, s2 = 0.f;
    if (slice < g.CS) {
        const size_t rstride = (size_t)g.CS * TF;
        const float* p = it.partial + (size_t)slice * TF + idx;
#pragma unroll 4
        for (int r = w; r < g.RS; r += 8) s += p[(size_t)r * rstride];
        if (it.mode == kIntSiluPair) {
            const float* p2 = ib.it[1].partial + (size_t)slice * TF + idx;
#pragma unroll 4
            for (int r = w; r < g.RS; r += 8) s2 += p2[(size_t)r * rstride];
        }
    }
    red[0][w][lane] = s;
    if (it.mode == kIntSiluPair) red[1][w][lane] = s2;
    __syncthreads();
    if (w == 0) {
        float sq = 0.f;
        if (slice < g.CS) {
            float t = 0.f, t2 = 0.f;
#pragma unroll
            for (int k = 0; k < 8; k++) t += red[0][k][lane];
            if (it.mode == kIntSiluPair) {
#pragma unroll
                for (int k = 0; k < 8; k++) t2 += red[1][k][lane];
            }
            const int slot = idx / TW, k = (idx % TW) / 32;
            if (lane < g.lpr) {
                const int col = slice * TW + lane * VEC + k;
                if (col < it.C) {
                    const int o = col * SLOTS + slot;
                    if (it.mode == kIntStore) it.out[o] = t;
                    else if (it.mode == kIntAccumulate) it.out[o] += t;
                    else if (it.mode == kIntSiluPair) it.out[o] = t2 * t / (1.f + expf(-t));
                    else {
                        const float hn = it.out[o] + t;
                        it.out[o] = hn;
                        sq = hn * hn;
                    }
                }
            }
        }
        if (it.mode == kIntResidual) {
            sq = warp_sum_f(sq);
            if (lane == 0) it.sumsq[blockIdx.x] = sq;
        }
    }
    if (it.n_selected && it.sel_counts && blockIdx.x == 0 && threadIdx.x == 0) {
        uint32_t t = 0;
        for (int r = 0; r < g.RS; r++) t += it.sel_counts[r];
        *it.n_selected = t;
    }
}

// ---- reference-format dispatch list (test hooks effort_calc_dispatch / effort_read_dispatch) --------
// prepareDispatch / prepareDispatchQ4 with a deterministic (ascending row) order: pass 1 counts the
// selected rows per chunk, pass 2 rescans and writes at the chunk's exclusive prefix.  Stats are read in
// the REFERENCE layout here (half4 .w / float2 .y) because this is the bit-for-bit hook.
constexpr int kDispChunk = 1024;

template <int KIND>
__device__ __forceinline__ bool ref_row_test(const void* stats, size_t i, const float* v, int in,
                                             float cutoff, float& payload) {
    if constexpr (KIND == 0) {
        const float s = __half2float(reinterpret_cast<const __half*>(stats)[i * 4 + 3]);
        const float val = v[i % (size_t)in];
        payload = val;
        return row_selected(cutoff, s, val);
    } else {
        const float s = reinterpret_cast<const float*>(stats)[i * 2 + 1];
        const float val = v[i / 8];  // bucketMulQ4.metal:45
        payload = __fmul_rn(val, s);
        return row_selected(cutoff, s, val);
    }
}

template <int KIND>
__global__ void __launch_bounds__(kDispChunk)
dispatch_count_kernel(const float* __restrict__ v, const void* __restrict__ stats,
                      const uint32_t* __restrict__ exp_no, const float* __restrict__ cutoff, int in,
                      int expert_size, uint32_t* __restrict__ chunk_counts) {
    __shared__ int wc[32];
    const uint32_t e_no = exp_no ? *exp_no : 0u;
    const int r = blockIdx.x * kDispChunk + threadIdx.x;
    bool sel = false;
    float payload;
    if (r < expert_size) sel = ref_row_test<KIND>(stats, (size_t)expert_size * e_no + r, v, in, *cutoff, payload);
    const unsigned m = __ballot_sync(0xffffffffu, sel);
    if ((threadIdx.x & 31) == 0) wc[threadIdx.x >> 5] = __popc(m);
    __syncthreads();
    if (threadIdx.x < 32) {
        int c = warp_sum_i(wc[threadIdx.x]);
        if (threadIdx.x == 0) chunk_counts[blockIdx.x] = (uint32_t)c;
    }
}

template <int KIND>
__global__ void __launch_bounds__(kDispChunk)
dispatch_write_kernel(const float* __restrict__ v, const void* __restrict__ stats,
                      const uint32_t* __restrict__ exp_no, const float* __restrict__ cutoff, int in, int C,
                      int expert_size, const uint32_t* __restrict__ chunk_counts, int n_chunks,
                      float2* __restrict__ dispatch, uint32_t* __restrict__ n_selected,
                      uint32_t* __restrict__ padded_size, uint32_t* __restrict__ prev_size) {
    __shared__ int wc[32];
    __shared__ uint32_t s_base, s_total;
    const uint32_t e_no = exp_no ? *exp_no : 0u;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // exclusive prefix of the chunk counts (n_chunks <= a few hundred)
    if (warp == 0) {
        uint32_t b = 0, t = 0;
        for (int k = lane; k < n_chunks; k += 32) {
            const uint32_t c = chunk_counts[k];
            t += c;
            if (k < (int)blockIdx.x) b += c;
        }
        b = (uint32_t)warp_sum_i((int)b);
        t = (uint32_t)warp_sum_i((int)t);
        if (lane == 0) { s_base = b; s_total = t; }
    }
    const int r = blockIdx.x * kDispChunk + tid;
    bool sel = false;
    float payload = 0.f;
    size_t i = (size_t)expert_size * e_no + (size_t)r;
    if (r < expert_size) sel = ref_row_test<KIND>(stats, i, v, in, *cutoff, payload);
    const unsigned m = __ballot_sync(0xffffffffu, sel);
    if (lane == 0) wc[warp] = __popc(m);
    __syncthreads();
    int pre = 0;
    for (int w = 0; w < warp; w++) pre += wc[w];
    if (sel) {
        const uint32_t pos = s_base + pre + __popc(m & ((1u << lane) - 1u));
        dispatch[pos] = make_float2(payload, (float)(uint32_t)(i * (size_t)C));  // float(i*colsCount), :71
    }
    // roundUp (bucketMul.metal:22-31) + zeroRange32 (:11-20): pad to (1 + n/2048)*2048 with {0,0}
    const uint32_t total = s_total;
    const uint32_t padded = (1u + total / 2048u) * 2048u;
    if (blockIdx.x == 0) {
        for (uint32_t p = total + tid; p < padded; p += kDispChunk) dispatch[p] = make_float2(0.f, 0.f);
        if (tid == 0) { *n_selected = total; *prev_size = total; *padded_size = padded; }
    }
}

}  // namespace effort
