// bucket_mul_v4.cuh -- the fused bucketMul for FP16 buckets in the slice-major device layout (the default path).
//
// Same operator as bucket_mul_v2_kernel (cutoff -> selection -> gather-MAC -> reductions into `out`; reference:
// BucketMul.fullMul, bucketMul.swift:34-88 and bucketMul.metal:11-247).  What the measurements of rounds 1-2 asked for
// (profiles/r02_*): the accumulate loop is ISSUE bound (every weight costs a shift, a LOP3, a convert, an LDS, an FFMA
// and an STS), so everything that is not those six instructions has to leave the accumulating warps, and the serial
// prologue has to shrink.
//
//  * 8 CONSUMER warps (0-7), each with a private 8 KB accumulator tile, do nothing but wait for a chunk, read its rows
//    and run the read-modify-writes (four rows = 16 independent updates per lane at a time);
//  * 8 PRODUCER warps (8-15), one per consumer.  Thread j of the CTA turns input j's selection mask into record j of a
//    direct-indexed list {first 16-byte piece, rows, multiplier, rows before} (slice-major layout: the ranks an input
//    selects inside this CTA's column slice are contiguous).  Each pair owns a fixed 1/8 of the pass's selected rows in
//    list order, so the same rows reach the same tile in the same order in every run.  The pair's rows fill a ring of
//    four 4 KB chunks in order, one aligned block of 16 rows of the pass per chunk; a record that crosses a chunk
//    boundary is cut there.  Each chunk has a full
//    and an empty mbarrier: the handshake is paid per 16 rows, not per input (an input selects ~4 rows at effort 0.25).
//    BULK (default): the producer stages every chunk with a free slot at once -- the whole first ring-full right after
//    the list barrier -- one lane per chunk posting the chunk's bytes (arrive.expect_tx) and every lane issuing the
//    cp.async.bulk of its record's piece.  !BULK: all lanes copy each piece with 16-byte cp.async, completion through
//    cp.async.mbarrier.arrive.noinc.  Up to 8 x 16 KB are in flight per SM.
//  * the exact-select cutoff runs on the EIGHT consumer warps (two per scheduler, 16 products per lane, a 256-thread
//    named barrier per round) while the producers zero the tiles and run the overwrite protocol.
//  * what bounds the kernel is the SM's shared-memory pipe (12 wavefronts per 128-weight row: tools/ubench), and at low
//    effort the serial prologue, which runs at one warp's dependent-issue rate (EFFORT_TRACE=2 cycle stamps): DESIGN.md 4.
#pragma once
#include "bucket_mul_v3.cuh"

namespace effort {

constexpr int kV4Pairs = 8;                    // consumer / producer warp pairs
constexpr int kV4Chunks = 4;                   // chunks per pair ring (a power of two)
constexpr int kV4ChunkRows = 16;               // rows per chunk: 16 full-width 256-byte row slices
constexpr int kV4ChunkBytes = kV4ChunkRows * 256;
constexpr int kV4RingBytes = kV4Chunks * kV4ChunkBytes;  // staging bytes per pair (16 KB)
constexpr int kV4SelWarps = 8;                                   // warps of the exact-select group (the consumers)
constexpr int kSelVals = EFFORT_PROBES_MAX / (kV4SelWarps * 32);  // probe products per thread (16)
constexpr int kSelKeys = kSelVals / 2, kSelChunks = kSelVals / 8; // packed bf16x2 registers; 8-value chunks
static_assert(kSelVals * kV4SelWarps * 32 == EFFORT_PROBES_MAX && kSelChunks >= 1, "the group holds all 4096 products");

struct V4Header {
    CutoffSmem cut;                      // bisect mode scratch
    uint2 sel_slot[2][kV4SelWarps];      // select mode: per-warp packed counts, double buffered by round parity
    float red[kV4SelWarps];
    float cutoff, denom;
    float hint;                          // the matrix's cutoff hint as thread 0 read it: one value for the whole select group
    int sel_rows;
    uint32_t warp_rows[kV2Threads / 32]; // rows selected by each warp's records (the split below)
    uint32_t start[kV4Pairs + 1];        // start[q]: the record holding pair q's first row (start[kV4Pairs] = records)
    unsigned long long full_bar[kV4Pairs][kV4Chunks];
    unsigned long long empty_bar[kV4Pairs][kV4Chunks];
};

struct V4Smem {
    static constexpr int kTileFloats = 16 * 32 * 4;
    static constexpr int kTileBytes = kTileFloats * 4;
    static constexpr size_t kHdrBytes = (sizeof(V4Header) + 127) & ~size_t(127);
    static constexpr size_t kBytes = (size_t)kTileBytes /*alignment slack*/ + (size_t)kV4Pairs * kTileBytes + kHdrBytes +
                                     (size_t)kV2MaxInputs * 16 + 128 + (size_t)kV4Pairs * kV4RingBytes +
                                     1024 /* the consumers read (and ignore) up to three rows past a unit's end */;
};

// The ring of a pair: chunk s of the pair's sequence (counted across passes and rounds) uses slot s % kV4Chunks; its
// full barrier completes phase s / kV4Chunks when its bytes have landed, its empty barrier the same phase when the
// consumer has read them.
__device__ __forceinline__ uint32_t v4_slot(uint32_t s) { return s & (kV4Chunks - 1); }
__device__ __forceinline__ uint32_t v4_phase(uint32_t s) { return (s / kV4Chunks) & 1u; }

// Lane `lane` takes record t + lane of the pass (when t + lane < r_end) and clips it to rows [c0, c1) of the pass.  Returns
// the number of leading records that end inside [.., c1): the records a cursor at t is done with once rows up to c1 are
// handled.  It is < 32 when the next record reaches past c1 (or the records run out): then rows [c0, c1) are complete.
struct V4Piece {
    uint32_t lo, hi;  // rows [lo, hi) of the pass (hi <= lo: nothing in [c0, c1))
    uint4 rec;
};
__device__ __forceinline__ uint32_t v4_pieces(const uint4* ulist, uint32_t t, uint32_t r_end, uint32_t c0, uint32_t c1, int lane,
                                              V4Piece& pc) {
    const bool have = t + (uint32_t)lane < r_end;
    pc.rec = have ? ulist[t + lane] : make_uint4(0u, 0u, 0u, 0u);
    pc.lo = max(pc.rec.w, c0);
    pc.hi = min(pc.rec.w + pc.rec.y, c1);
    const unsigned fin = __ballot_sync(0xffffffffu, have && pc.rec.w + pc.rec.y <= c1);  // a prefix: record ends never decrease
    return fin == 0xffffffffu ? 32u : (uint32_t)(__ffs((int)~fin) - 1);
}

__device__ __forceinline__ void cp_async_arrive_noinc(uint32_t bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}

// bounded mbarrier wait that lets the hardware park the warp (suspend-time hint) instead of spinning through the issue
// slots the accumulating warps need; returns false after ~1 s (a bug, never a data condition)
__device__ __forceinline__ bool mbar_wait_parked(uint32_t bar, uint32_t parity) {
    uint32_t done = 0;
    for (int tries = 0; tries < (1 << 22) && !done; tries++) {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done) : "r"(bar), "r"(parity), "r"(200u) : "memory");
    }
    return done != 0;
}

// non-blocking phase test
__device__ __forceinline__ bool mbar_test(uint32_t bar, uint32_t parity) {
    uint32_t done;
    asm volatile("{ .reg .pred p; mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    return done != 0;
}

// x / d with a shared correctly rounded reciprocal r = rn(1/d): one Newton step on the quotient (q = x*r; q += (x - q*d)*r),
// the correctly rounded quotient for every finite, normal operand pair -- 3 instructions instead of the division's subroutine
// call (the 32 normalisations of a select thread sit on the kernel's critical path)
__device__ __forceinline__ float div_by(float x, float d, float r) {
    const float q = x * r;
    return fmaf(fmaf(-q, d, x), r, q);
}

// count of keys above the threshold, kSelVals keys (kSelKeys bf16x2 registers) per thread
__device__ __forceinline__ uint32_t count_gt32(const uint32_t (&keys)[kSelKeys], uint32_t th) {
    const __nv_bfloat162 t = as_bf162(splat_bf16(th));
    __nv_bfloat162 c0 = __hgt2(as_bf162(keys[0]), t), c1 = __hgt2(as_bf162(keys[1]), t);
#pragma unroll
    for (int i = 2; i < kSelKeys; i += 2) {
        c0 = __hadd2(c0, __hgt2(as_bf162(keys[i]), t));
        c1 = __hadd2(c1, __hgt2(as_bf162(keys[i + 1]), t));
    }
    return (uint32_t)bf162_count(__hadd2(c0, c1));  // 0..kSelVals
}

// Exact select on the first kV4SelWarps warps (gt = thread index inside the group).  Q(x) = [#{keys > x} >= k+1] is true
// up to u = the key just below the (k+1)-th largest and false above; the cutoff key is u + 1 (0 when Q(0) is false).
// A quaternary search over the 15-bit key space keeps an interval (L, R) with Q(L) true (L = -1: nothing known) and
// Q(R) false and evaluates three interior thresholds per round (one pass over the keys, one 128-thread barrier).  Eight
// rounds from scratch.  With a hint -- the key of the cutoff this matrix saw on the previous call -- the first round
// brackets it (hint +- 16 keys = +- 12 % in value) and two more rounds finish when the guess holds; a miss only costs the
// bracketing round.  The result does not depend on the hint, provided every thread of the group passes the same one.
__device__ __forceinline__ float select_cutoff_group(const uint32_t (&keys)[kSelKeys], int k, V4Header& hdr, int gt, uint32_t hint_key,
                                                     int* rounds_out) {
    const int lane = gt & 31, gw = gt >> 5;
    const unsigned need = (unsigned)(k + 1);
    int L = -1, R = 0x7FFF;
    bool first = hint_key > 16u && hint_key < 0x7F00u;
    int round = 0;
#pragma unroll 1
    while (R - L > 1) {
        int p1, p2, p3;
        if (first) { p1 = (int)hint_key - 16; p2 = (int)hint_key; p3 = (int)hint_key + 16; }
        else {
            const int w = R - L;
            p1 = L + max(1, w >> 2); p2 = L + max(1, w >> 1); p3 = L + max(1, (3 * w) >> 2);
            p2 = min(p2, R - 1); p3 = min(p3, R - 1);
        }
        first = false;
        const uint32_t c1 = count_gt32(keys, (uint32_t)p1), c2 = count_gt32(keys, (uint32_t)p2), c3 = count_gt32(keys, (uint32_t)p3);
        const uint32_t a = __reduce_add_sync(0xffffffffu, c1 | (c2 << 16));
        const uint32_t bsum = __reduce_add_sync(0xffffffffu, c3);
        if (lane == 0) hdr.sel_slot[round & 1][gw] = make_uint2(a, bsum);
        asm volatile("bar.sync 2, %0;" ::"n"(kV4SelWarps * 32) : "memory");
        uint32_t A = 0, B = 0;
#pragma unroll
        for (int w = 0; w < kV4SelWarps; w++) {
            const uint2 s = hdr.sel_slot[round & 1][w];
            A += s.x;
            B += s.y;
        }
        const bool q1 = (A & 0xFFFFu) >= need, q2 = (A >> 16) >= need, q3 = B >= need;
        if (!q1) R = p1;
        else if (!q2) { L = p1; R = p2; }
        else if (!q3) { L = p2; R = p3; }
        else L = p3;
        round++;
    }
    if (rounds_out && gt == 0) *rounds_out = round;
    return __uint_as_float((uint32_t)(L + 1) << 16);
}

template <int CUT, bool BULK>
__global__ void __launch_bounds__(kV2Threads, 1)
bucket_mul_v4_kernel(const __grid_constant__ V2Batch batch) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr int SLOTS = 16, VEC = 4;
    constexpr int NT = kV2Threads, NC = kV4Pairs;
    constexpr int TF = V4Smem::kTileFloats, TW = 32 * VEC, LB = VEC * 2;
    constexpr int kRow = 32 * LB;  // 256 bytes: a full-width row slice

    int pi = 0;
#pragma unroll
    for (int k = 1; k < kMulBatchMax; k++) pi += (k < batch.n && (int)blockIdx.x >= batch.cta_begin[k]) ? 1 : 0;
    const V2Problem& pb = batch.p[pi];
    const int lb = (int)blockIdx.x - batch.cta_begin[pi];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool consumer = warp < NC;
    const int pair = warp & (NC - 1);
    const bool sel_warp = warp < kV4SelWarps;
    const int slice = lb % pb.CS, rsp = lb / pb.CS;
    const int RS = pb.RS, P = pb.P, C = pb.C;

    // ---- carve shared memory ----
    const uint32_t s0 = (uint32_t)__cvta_generic_to_shared(smem_raw);
    const uint32_t s1 = (s0 + (uint32_t)V4Smem::kTileBytes - 1u) & ~((uint32_t)V4Smem::kTileBytes - 1u);
    unsigned char* p = smem_raw + (s1 - s0);
    float* tiles = reinterpret_cast<float*>(p);
    const uint32_t tiles_saddr = s1;
    p += (size_t)NC * V4Smem::kTileBytes;
    V4Header& hdr = *reinterpret_cast<V4Header*>(p);
    p += V4Smem::kHdrBytes;
    uint4* ulist = reinterpret_cast<uint4*>(p);  // the pass's units: {first 16-byte piece, rows, multiplier bits, rows before}
    p += (size_t)kV2MaxInputs * 16;
    p = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(p) + 127) & ~uintptr_t(127));
    float* ring_f = reinterpret_cast<float*>(p);
    const uint32_t ring_saddr = (uint32_t)__cvta_generic_to_shared(p) + (uint32_t)pair * (uint32_t)kV4RingBytes;

    pdl_trigger();
    if (pb.exp_no) pdl_wait();
    const uint32_t e_no = pb.exp_no ? *pb.exp_no : 0u;
    V2_TRACE(0);
    // EFFORT_TRACE: SM-cycle stamps of the prologue phases of CTA 0, thread 0 (cheap, unlike the global timer)
    unsigned long long* cst = (pb.unit_trace && blockIdx.x == 0 && tid == 0) ? pb.unit_trace + 696 : nullptr;
    if (cst) cst[0] = (unsigned long long)clock64();

    // ---- 0. constant metadata before the dependency wait ----
    const uint64_t keep = l2_policy_evict_last();
    const int n_in = (pb.in > rsp) ? (pb.in - 1 - rsp) / RS + 1 : 0;
    float sel_stat[16];
#pragma unroll
    for (int rho = 0; rho < 16; rho++) sel_stat[rho] = 0.f;
    auto load_stats = [&](int j, float (&st)[16]) {
        const int i = rsp + j * RS;
        if (P == 16) {
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
                if (rho < P) st[rho] = __half2float(pb.st16[((size_t)e_no * pb.in + i) * P + rho]);
        }
    };
    if (tid < n_in) load_stats(tid, sel_stat);
    const int vmode = pb.norm_w ? kVNorm : (pb.v2 ? kVSilu : kVPlain);
    uint4 prb[kSelChunks], nwv[kSelChunks];
    if (CUT == kCutSelect && sel_warp) {  // kSelVals consecutive probes (and norm weights) per thread of the select group
        const uint4* pp = reinterpret_cast<const uint4*>(pb.probes + (size_t)e_no * EFFORT_PROBES_MAX) + kSelChunks * tid;
#pragma unroll
        for (int c = 0; c < kSelChunks; c++) prb[c] = ldg_keep_u4(pp + c, keep);
        if (vmode == kVNorm) {
            const uint4* np4 = reinterpret_cast<const uint4*>(pb.norm_w) + kSelChunks * tid;
#pragma unroll
            for (int c = 0; c < kSelChunks; c++) nwv[c] = np4[c];
        }
    }
    if (warp == NC) {  // first producer warp: the ring barriers
        for (int s = lane; s < NC * kV4Chunks; s += 32) {
            // LDGSTS: the 32 lanes' cp.async arrivals; bulk copy: the expect_tx arrival (bytes complete the phase)
            mbar_init((uint32_t)__cvta_generic_to_shared(&hdr.full_bar[0][0] + s), BULK ? 1 : 32);
            mbar_init((uint32_t)__cvta_generic_to_shared(&hdr.empty_bar[0][0] + s), 1);
        }
        if (lane == 0) hdr.sel_rows = 0;
        // (the __syncthreads before the first use orders the initialisation: no cluster, no async-proxy user here)
    }
    // Everything the streaming phase needs that does not depend on the input vector is set up HERE, before the dependency
    // wait: after the cutoff the CTA runs a serial tail (masks, list) at one warp's dependent-issue rate, and every
    // instruction moved out of it is worth ~4 cycles (EFFORT_TRACE=2 cycle stamps).
    const int slice_cols = min(pb.W, C - slice * pb.W);
    const int seg_bytes = slice_cols * 2;
    const bool full_width = slice_cols == TW;
    const int lpr = pb.lpr, R = pb.R;
    const uint32_t base_lane = (tiles_saddr + (uint32_t)pair * V4Smem::kTileBytes) | (uint32_t)(lane * 4);
    const uint64_t pol = l2_policy_evict_first();
    const uint4* bk16 = reinterpret_cast<const uint4*>(pb.bk + (size_t)pb.in * P * ((size_t)slice * pb.W));  // slice-major
    const uint32_t rs16 = (uint32_t)(seg_bytes >> 4);
    // first 16-byte piece of local input j's rank-0 row slice, relative to bk16
    auto src_of = [&](int j) { return (uint32_t)(((size_t)e_no * pb.in * P * C + (size_t)(rsp + j * RS) * P * slice_cols) >> 3); };
    const uint32_t my_src0 = src_of(tid);

    // debugging aid (EFFORT_TRACE): issue / arrival / release times of the first 80 chunks of pair 0 of CTA 0
    unsigned long long* utrace = (pb.unit_trace && blockIdx.x == 0 && pair == 0) ? pb.unit_trace : nullptr;
    if (utrace && tid == 0) utrace[640] = (unsigned long long)clock64();  // time base: the SM's cycle counter
    // pair state: both sides count the pair's chunks (seq) across passes and rounds
    uint32_t seq = 0;
    const uint32_t full0 = (uint32_t)__cvta_generic_to_shared(&hdr.full_bar[pair][0]);
    const uint32_t empty0 = (uint32_t)__cvta_generic_to_shared(&hdr.empty_bar[pair][0]);
    V2_TRACE(1);
    pdl_wait();
    if (cst) cst[1] = (unsigned long long)clock64();

    // ---- 1. inputs.  Select group: kSelVals entries per thread for the cutoff; everybody: the thread's own input dim ----
    float my_v = 0.f, my_x3 = 0.f, my_nw = 1.f;
    if (tid < n_in) {
        const int i = rsp + tid * RS;
        my_v = pb.v[i];
        if (vmode == kVSilu) my_x3 = pb.v2[i];
        if (vmode == kVNorm) my_nw = __half2float(pb.norm_w[i]);
    }
    const int seg_bytes0 = slice_cols * 2;
    const uint4* bk16p = reinterpret_cast<const uint4*>(pb.bk + (size_t)pb.in * P * ((size_t)slice * pb.W));
    if (batch.prefetch && pb.cutoff_hint && (CUT != kCutSelect || !sel_warp)) {
        // Speculative L2 prefetch.  The cutoff moves little from token to token, so while the select warps compute the real
        // one the other warps test their rows against the LAST cutoff this matrix saw (kVNorm: scaled by that call's
        // rmsNorm denominator, which is not known yet either) and ask the L2 for the prefix of ranks it selects: one
        // cp.async.bulk.prefetch per input.  Purely a hint: the real masks below decide what is streamed.
        const float hint = pb.cutoff_hint[e_no];
        auto spec = [&](int jj, const float (&st)[16], float vraw) {
            int n = 0;
#pragma unroll
            for (int rho = 0; rho < 16; rho++) n += (rho == n && rho < P && row_selected(hint, st[rho], vraw)) ? 1 : 0;
            if (n > 0) {
                const int i = rsp + jj * RS;
                const uint4* src = bk16p + (((size_t)e_no * pb.in * P * C + (size_t)i * P * slice_cols) >> 3);
                asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(n * seg_bytes0) : "memory");
            }
        };
        auto raw = [&](float x, float x3, float nw) { return vmode == kVSilu ? silu_mul(x, x3) : (vmode == kVNorm ? x * nw : x); };
        if (tid < n_in) spec(tid, sel_stat, raw(my_v, my_x3, my_nw));
        if (CUT == kCutSelect && tid >= kV4SelWarps * 32 && tid < 2 * kV4SelWarps * 32 && tid - kV4SelWarps * 32 < n_in) {
            const int j2 = tid - kV4SelWarps * 32;  // the select warps' inputs: covered by the other warps
            float st2[16];
#pragma unroll
            for (int rho = 0; rho < 16; rho++) st2[rho] = 0.f;
            load_stats(j2, st2);
            const int i2 = rsp + j2 * RS;
            spec(j2, st2, raw(pb.v[i2], vmode == kVSilu ? pb.v2[i2] : 0.f, vmode == kVNorm ? __half2float(pb.norm_w[i2]) : 1.f));
        }
    }
    if constexpr (CUT == kCutSelect) {
        if (sel_warp) {
            if (tid == 0 && pb.cutoff_hint) hdr.hint = pb.cutoff_hint[e_no];  // published by the barrier before the select
            const float* src = (vmode == kVPlain) ? pb.v_cut : pb.v;
            float vv[kSelVals];
#pragma unroll
            for (int c = 0; c < kSelVals / 4; c++) {
                const float4 a = *reinterpret_cast<const float4*>(src + kSelVals * tid + 4 * c);
                vv[4 * c] = a.x; vv[4 * c + 1] = a.y; vv[4 * c + 2] = a.z; vv[4 * c + 3] = a.w;
            }
            if (vmode == kVSilu) {
#pragma unroll
                for (int c = 0; c < kSelVals / 4; c++) {
                    const float4 a = *reinterpret_cast<const float4*>(pb.v2 + kSelVals * tid + 4 * c);
                    vv[4 * c] = silu_mul(vv[4 * c], a.x); vv[4 * c + 1] = silu_mul(vv[4 * c + 1], a.y);
                    vv[4 * c + 2] = silu_mul(vv[4 * c + 2], a.z); vv[4 * c + 3] = silu_mul(vv[4 * c + 3], a.w);
                }
            }
            float denom = 1.f;
            if (vmode == kVNorm) {  // rmsNorm32fast (aux.metal:113-152) over the 4096 entries the group holds
                float ss = 0.f;
#pragma unroll
                for (int m = 0; m < kSelVals; m++) ss += vv[m] * vv[m];
                ss = warp_sum_f(ss);
                if (lane == 0) hdr.red[warp] = ss;
                asm volatile("bar.sync 2, %0;" ::"n"(kV4SelWarps * 32) : "memory");
                float t = 0.f;
#pragma unroll
                for (int w = 0; w < kV4SelWarps; w++) t += hdr.red[w];
                denom = sqrtf(t / (float)pb.in + pb.norm_eps);
                if (tid == 0) hdr.denom = denom;
                const float rden = __frcp_rn(denom);
#pragma unroll
                for (int c = 0; c < kSelChunks; c++) {
                    const uint32_t nw[4] = {nwv[c].x, nwv[c].y, nwv[c].z, nwv[c].w};
#pragma unroll
                    for (int m = 0; m < 4; m++) {
                        const float2 wf = __half22float2(*reinterpret_cast<const __half2*>(&nw[m]));
                        vv[8 * c + 2 * m] = div_by(vv[8 * c + 2 * m], denom, rden) * wf.x;
                        vv[8 * c + 2 * m + 1] = div_by(vv[8 * c + 2 * m + 1], denom, rden) * wf.y;
                    }
                }
            }
            uint32_t keys[kSelKeys];
#pragma unroll
            for (int c = 0; c < kSelChunks; c++) {
                const float v8[8] = {vv[8 * c], vv[8 * c + 1], vv[8 * c + 2], vv[8 * c + 3], vv[8 * c + 4], vv[8 * c + 5], vv[8 * c + 6], vv[8 * c + 7]};
                uint32_t k4[4];
                score8(v8, prb[c], k4);
                keys[4 * c] = k4[0]; keys[4 * c + 1] = k4[1]; keys[4 * c + 2] = k4[2]; keys[4 * c + 3] = k4[3];
            }
            V2_TRACE(3);
            if (cst) cst[2] = (unsigned long long)clock64();
            uint32_t hint_key = 0u;
            if (pb.cutoff_hint) {  // last cutoff of this matrix (kVNorm: stored times that call's denominator)
                // Every select warp must start from the SAME hint.  CTA 0 of this launch overwrites it once its cutoff is
                // known, and warps that each loaded it could fall on either side of that store: they would then probe
                // different thresholds in the same round, sum counts that belong to no single threshold, and settle on a
                // wrong cutoff for this CTA (a bit-level divergence that only timing triggers, DESIGN.md section 4.7).
                // kVNorm: the denominator's barrier above already published hdr.hint.
                if (vmode != kVNorm) asm volatile("bar.sync 2, %0;" ::"n"(kV4SelWarps * 32) : "memory");
                const float hc = hdr.hint / denom;
                hint_key = (hc > 0.f && hc < 3e38f) ? (__float_as_uint(hc) >> 16) : 0u;
            }
            const float cut = select_cutoff_group(keys, EFFORT_PROBES_MAX - pb.q, hdr, tid, hint_key,
                                                  (lb == 0) ? pb.rounds_out : nullptr);
            if (tid == 0) hdr.cutoff = cut;
        }
    }
    if (!sel_warp || CUT != kCutSelect) {
        // the other warps meanwhile: zero the 8 accumulator tiles, run the overwrite protocol
        const int nz = (CUT == kCutSelect) ? (NT - kV4SelWarps * 32) : NT, z0 = (CUT == kCutSelect) ? tid - kV4SelWarps * 32 : tid;
        float4* t4 = reinterpret_cast<float4*>(tiles);
        for (int i = z0; i < NC * TF / 4; i += nz) t4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (warp == NT / 32 - 1 && pb.out_mode == kOutOverwrite) {
            // overwrite semantics: zero this CTA's share of the slice's outputs, make the zeros visible, arrive on the
            // slice counter -- inspected right before the reductions at the end of the kernel
            const int n4 = slice_cols * SLOTS / 4, per = (n4 + RS - 1) / RS;
            float4* o4 = reinterpret_cast<float4*>(pb.out + (size_t)slice * pb.W * SLOTS);
            for (int x = rsp * per + lane; x < min(n4, (rsp + 1) * per); x += 32) o4[x] = make_float4(0.f, 0.f, 0.f, 0.f);
            __syncwarp();
            if (lane == 0) {
                __threadfence();
                atomicAdd(pb.sync + 2 * slice, 1u);
            }
        }
    }
    V2_TRACE(2);
    if (cst) cst[3] = (unsigned long long)clock64();
    float denom = 1.f;
    if constexpr (CUT != kCutSelect) {
        // bit-exact replay of the reference's bisection by four warps (cutoff.cuh)
        if (vmode == kVNorm) {  // the group path scores (v / denom) * w itself: it needs the denominator first
            float ss = 0.f;
            for (int i = tid; i < pb.in; i += NT) { const float x = pb.v[i]; ss += x * x; }
            ss = warp_sum_f(ss);
            float* redf = ring_f;  // the rings are idle
            if (lane == 0) redf[warp] = ss;
            __syncthreads();
            float t = (lane < NT / 32) ? redf[lane] : 0.f;
            t = warp_sum_f(t);
            denom = sqrtf(t / (float)pb.in + pb.norm_eps);
            __syncthreads();
        }
        float* vtmp = ring_f;
        if (vmode == kVSilu) {
            for (int i = tid; i < EFFORT_PROBES_MAX; i += NT) vtmp[i] = silu_mul(pb.v[i], pb.v2[i]);
            __syncthreads();
        }
        if (tid < kCutThreads) {
            GroupProbes gpr;
            group_load_probes(pb.probes + (size_t)e_no * EFFORT_PROBES_MAX, EFFORT_PROBES_MAX, tid, gpr, keep);
            GroupProducts gp;
            if (vmode == kVNorm) group_score<true>(pb.v, gpr, EFFORT_PROBES_MAX, tid, gp, pb.norm_w, denom);
            else if (vmode == kVPlain) group_score<false>(pb.v_cut, gpr, EFFORT_PROBES_MAX, tid, gp, nullptr, 1.f);
            else group_score<false>(vtmp, gpr, EFFORT_PROBES_MAX, tid, gp, nullptr, 1.f);
            group_cutoff<1>(gp, EFFORT_PROBES_MAX, pb.q, hdr.cut, tid, nullptr);
            if (tid == 0) { hdr.cutoff = hdr.cut.result; hdr.denom = denom; }
        }
    }
    __syncthreads();  // cutoff and denominator known; tiles zeroed; barriers initialised
    if (cst) cst[4] = (unsigned long long)clock64();
    const float cutoff = hdr.cutoff;
    if (vmode == kVNorm) {
        denom = hdr.denom;
        my_v = div_by(my_v, denom, __frcp_rn(denom)) * my_nw;
    } else if (vmode == kVSilu) {
        my_v = silu_mul(my_v, my_x3);
    }
    if (cst) cst[10] = (unsigned long long)clock64();
    if (pb.cutoff_out && lb == 0 && tid == 0) *pb.cutoff_out = cutoff;
    if (pb.cutoff_hint && lb == 0 && tid == 0) pb.cutoff_hint[e_no] = cutoff * (vmode == kVNorm ? denom : 1.f);
    V2_TRACE(6);

    if (cst) cst[11] = (unsigned long long)clock64();
    bool pristine = true;  // no earlier round has used the unit list
    // ---- passes over the inputs of this row split (one pass for every Mistral shape) ----
    for (int j0 = 0; j0 < n_in; j0 += NT) {
        const int j = j0 + tid;
        if (j0 > 0) {
            __syncthreads();
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
        // 2. selection mask of this thread's input (prepareDispatch, bucketMul.metal:66)
        // The prologue is ISSUE bound (all sixteen warps run the same straight-line code: 4 warps per scheduler), so warps
        // whose 32 inputs lie past n_in skip it.  No per-row guards: statistics of ranks >= P and inputs past n_in are
        // zero, and `cutoff < 0` never holds.
        const bool warp_has_inputs = j0 + warp * 32 < n_in;
        unsigned m = 0u;
        if (cst && j0 == 0) cst[12] = (unsigned long long)clock64();
        if (warp_has_inputs) {
#pragma unroll
            for (int rho = 0; rho < 16; rho++)
                if (row_selected(cutoff, sel_stat[rho], my_v)) m |= 1u << rho;
            if (cst && j0 == 0) cst[13] = (unsigned long long)clock64();
        }
        if (cst && j0 == 0) cst[5] = (unsigned long long)clock64();
        const uint32_t my_src = (j0 == 0) ? my_src0 : src_of(j);
        const float my_val = pb.out_scale ? my_v * *pb.out_scale : my_v;  // the selection above used the unscaled input
        // ---- rounds: every input contributes its next maximal run of selected ranks as one unit.  Bucket statistics fall
        // with the rank, so a mask is a prefix of the ranks and one round is the normal case; arbitrary statistics (tests)
        // take one round per run. ----
        bool more;
        do {
            if (!pristine) __syncthreads();  // the producers are done with the previous round's list
            pristine = false;
            const uint32_t nu_pass = (uint32_t)min(NT, n_in - j0);  // records of this pass (empty ones included)
            uint32_t len = 0u;
            if (warp_has_inputs) {
                // 2b. the unit list: record j of the pass belongs to input j -- no compaction, no atomics on this serial stretch;
                // an input that selects nothing leaves an empty record (rows = 0) that the producers skip
                uint32_t st = 0u;
                if (m) {
                    st = (uint32_t)__ffs((int)m) - 1u;
                    len = (uint32_t)__ffs((int)~(m >> st)) - 1u;
                    m &= ~(((1u << len) - 1u) << st);
                }
                ulist[tid] = make_uint4(my_src + st * rs16, len, __float_as_uint(my_val), 0u);
            }
            if (cst && j0 == 0) cst[6] = (unsigned long long)clock64();
            // rows up to and including this record inside its warp; the warp totals go to the header
            uint32_t incl = len;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += y;
            }
            if (lane == 31) hdr.warp_rows[warp] = incl;
            if (tid <= NC) hdr.start[tid] = tid ? nu_pass : 0u;
            more = __syncthreads_or(m != 0u) != 0;
            // 2c. pair q accumulates rows [floor(q * total / NC), floor((q + 1) * total / NC)) of the pass in list order; a record
            // that straddles a boundary is cut between two pairs.  A static split, exact in rows, that fixes which tile
            // accumulates which row: the sums do not depend on timing.  start[q] = the record holding the pair's first row.
            uint32_t row_lo, row_hi;
            {
                uint32_t off = 0u, total = 0u;
#pragma unroll
                for (int w = 0; w < NT / 32; w++) {
                    const uint32_t x = hdr.warp_rows[w];
                    total += x;
                    if (w < warp) off += x;
                }
                row_lo = (uint32_t)pair * total / NC;
                row_hi = (uint32_t)(pair + 1) * total / NC;
                if ((uint32_t)tid < nu_pass) {
                    const uint32_t e = off + incl - len;  // rows of the records before this one
                    ulist[tid].w = e;
#pragma unroll
                    for (int q = 1; q < NC; q++) {
                        const uint32_t T = (uint32_t)q * total / NC;
                        if (e <= T && T < e + len) hdr.start[q] = (uint32_t)tid;
                    }
                }
                __syncthreads();
            }
            // the pair's rows [row_lo, row_hi) of the pass reach its ring in chunks: chunk c holds the pair's rows of
            // [(kb + c) * kV4ChunkRows, (kb + c + 1) * kV4ChunkRows), kb = row_lo / kV4ChunkRows, row r at (r % kV4ChunkRows) *
            // seg_bytes of the chunk's slot.  A record that crosses a chunk boundary is cut there, as the pair boundary cuts
            // records.  The boundaries are multiples of kV4ChunkRows in the pass's rows, not the pair's: at high effort most
            // records have 16 rows and start on such a multiple, so they stay whole -- four 4-row groups, not a cut pair of
            // partial ones.
            const uint32_t r_next = hdr.start[pair + 1];
            const uint32_t r_end = r_next < nu_pass ? r_next + 1u : nu_pass;  // (the record holding the next pair's first row)
            const uint32_t kb = row_lo / (uint32_t)kV4ChunkRows;
            const uint32_t n_chunks = row_hi > row_lo ? (row_hi - 1u) / (uint32_t)kV4ChunkRows + 1u - kb : 0u;
            auto chunk_lo = [&](uint32_t c) { return max((kb + c) * (uint32_t)kV4ChunkRows, row_lo); };
            auto chunk_hi = [&](uint32_t c) { return min((kb + c + 1u) * (uint32_t)kV4ChunkRows, row_hi); };
            auto chunk_of = [&](uint32_t r) { return r / (uint32_t)kV4ChunkRows - kb; };
            auto at = [&](uint32_t r) { return (r % (uint32_t)kV4ChunkRows) * (uint32_t)seg_bytes; };  // byte offset of row r in its slot
            const uint32_t seq0 = seq;  // chunk c of this round is chunk seq0 + c of the pair
            seq += n_chunks;
            if (cst && j0 == 0) cst[7] = (unsigned long long)clock64();
            V2_TRACE(8);

            if (!consumer) {
                // ---- 3a. producer of pair `pair`.  Every shared-memory operation of a producer queues behind the consumers'
                // read-modify-writes (the shared-memory pipe bounds the kernel), so it stages every chunk that has a free slot
                // at once -- the first ring-full right after the list barrier, then what the consumer has released -- with one
                // record per lane, 32 records per step.  BULK: one lane per chunk posts the chunk's bytes (expect_tx), every
                // lane issues the cp.async.bulk of its record's piece(s).  !BULK: all lanes copy each piece with 16-byte
                // cp.async, completion through cp.async.mbarrier.arrive.noinc. ----
                uint32_t t = hdr.start[pair];  // record cursor: the records before t are staged
#pragma unroll 1
                for (uint32_t c = 0; c < n_chunks;) {
                    // chunks c, c + 1, .. whose slots are free (chunk s reuses the slot of chunk s - kV4Chunks)
                    const uint32_t s = seq0 + c + (uint32_t)lane;
                    const bool free_slot = lane < kV4Chunks && c + (uint32_t)lane < n_chunks &&
                                           (s < (uint32_t)kV4Chunks || mbar_test(empty0 + v4_slot(s) * 8u, v4_phase(s) ^ 1u));
                    uint32_t k = (uint32_t)(__ffs((int)~__ballot_sync(0xffffffffu, free_slot)) - 1);
                    if (k == 0u) {  // all in use: wait for the oldest
                        const uint32_t so = seq0 + c;
                        if (!mbar_wait_parked(empty0 + v4_slot(so) * 8u, v4_phase(so) ^ 1u) && pb.err_flag && lane == 0)
                            atomicExch(pb.err_flag, 3u);
                        k = 1u;  // (after the ~1 s bound: give up waiting, the error flag says so)
                    }
                    if ((uint32_t)lane < k) {
                        const uint32_t cc = c + (uint32_t)lane;
                        if (BULK) mbar_expect_tx(full0 + v4_slot(seq0 + cc) * 8u, (int)((chunk_hi(cc) - chunk_lo(cc)) * (uint32_t)seg_bytes));
                        if (utrace && seq0 + cc < 80u) {
                            utrace[8 * (seq0 + cc)] = (unsigned long long)clock64();
                            utrace[8 * (seq0 + cc) + 3] = (unsigned long long)(chunk_hi(cc) - chunk_lo(cc));
                        }
                    }
                    __syncwarp();
                    const uint32_t b0 = chunk_lo(c), b1 = chunk_hi(c + k - 1u);
#pragma unroll 1
                    for (;;) {  // the record pieces of rows [b0, b1), cut at chunk boundaries (records have <= 16 rows: two pieces at most)
                        V4Piece pc;
                        const uint32_t done = v4_pieces(ulist, t, r_end, b0, b1, lane, pc);
                        if (BULK) {
                            for (uint32_t lo = pc.lo; lo < pc.hi;) {
                                const uint32_t cc = chunk_of(lo), sl = v4_slot(seq0 + cc);
                                const uint32_t hi = min(pc.hi, chunk_hi(cc));
                                bulk_g2s(ring_saddr + sl * (uint32_t)kV4ChunkBytes + at(lo),
                                         bk16 + pc.rec.x + (lo - pc.rec.w) * rs16, (int)((hi - lo) * (uint32_t)seg_bytes), full0 + sl * 8u, pol);
                                lo = hi;
                            }
                        } else {
                            unsigned todo = __ballot_sync(0xffffffffu, pc.lo < pc.hi);
                            while (todo) {
                                const int l = __ffs((int)todo) - 1;
                                todo &= todo - 1u;
                                uint32_t lo = __shfl_sync(0xffffffffu, pc.lo, l);
                                const uint32_t phi = __shfl_sync(0xffffffffu, pc.hi, l);
                                uint32_t src = __shfl_sync(0xffffffffu, pc.rec.x, l) + (lo - __shfl_sync(0xffffffffu, pc.rec.w, l)) * rs16;
                                while (lo < phi) {
                                    const uint32_t cc = chunk_of(lo);
                                    const uint32_t hi = min(phi, chunk_hi(cc));
                                    const uint32_t d0 = ring_saddr + v4_slot(seq0 + cc) * (uint32_t)kV4ChunkBytes + at(lo);
                                    const uint32_t n16 = (hi - lo) * rs16;
                                    for (uint32_t q = (uint32_t)lane; q < n16; q += 32u) cp_async16(d0 + q * 16u, bk16 + src + q, pol);
                                    src += n16;
                                    lo = hi;
                                }
                            }
                        }
                        t += done;
                        if (done < 32u) break;
                    }
                    if (!BULK)
                        for (uint32_t i = 0; i < k; i++) cp_async_arrive_noinc(full0 + v4_slot(seq0 + c + i) * 8u);  // when this lane's copies have landed
                    c += k;
                }
            } else {
                // ---- 3b. consumer: wait for the pair's next chunk, walk its record pieces, run the read-modify-writes ----
                unsigned long long rows_done = 0ull;
                uint32_t t = hdr.start[pair];  // record cursor: the records before t are accumulated
#pragma unroll 1
                for (uint32_t c = 0; c < n_chunks; c++) {
                    const uint32_t s = seq0 + c, sl = v4_slot(s);
                    const uint32_t c0 = chunk_lo(c), c1 = chunk_hi(c);
                    const bool tr = utrace && lane == 0 && s < 80u;
                    if (tr) utrace[8 * s + 1] = (unsigned long long)clock64();
                    // the chunk's first 32 records are read while its bytes may still be on their way
                    V4Piece pc;
                    uint32_t done = v4_pieces(ulist, t, r_end, c0, c1, lane, pc);
                    if (!mbar_wait(full0 + sl * 8u, v4_phase(s))) {
                        if (pb.err_flag && lane == 0) atomicExch(pb.err_flag, 2u);
                        break;
                    }
                    if (tr) utrace[8 * s + 2] = (unsigned long long)clock64();
                    if (tr) utrace[8 * s + 4] = (unsigned long long)clock64();
                    const uint32_t cbase = ring_saddr + sl * (uint32_t)kV4ChunkBytes;
                    bool first = true;
#pragma unroll 1
                    for (;;) {
                        unsigned todo = __ballot_sync(0xffffffffu, pc.lo < pc.hi);
                        while (todo) {  // the pieces in list order: each is one input's rows, as a unit was before
                            const int l = __ffs((int)todo) - 1;
                            todo &= todo - 1u;
                            const uint32_t lo = __shfl_sync(0xffffffffu, pc.lo, l);
                            const int n = (int)(__shfl_sync(0xffffffffu, pc.hi, l) - lo);
                            const float val = __uint_as_float(__shfl_sync(0xffffffffu, pc.rec.z, l));
                            const uint32_t sa = cbase + at(lo);
                            if (full_width) {
                                // 4/3/2/1-row groups inside one record: rows of one input never alias in a tile word
                                uint32_t a0 = sa + (uint32_t)(lane * LB);
                                int r = 0;
                                for (; r + 4 <= n; r += 4, a0 += 4 * kRow) accumulate_unit_fp16<VEC, 4, kRow>(base_lane, val, a0);
                                switch (n - r) {
                                    case 1: accumulate_unit_fp16<VEC, 1, kRow>(base_lane, val, a0); break;
                                    case 2: accumulate_unit_fp16<VEC, 2, kRow>(base_lane, val, a0); break;
                                    case 3: accumulate_unit_fp16<VEC, 3, kRow>(base_lane, val, a0); break;
                                    default: break;
                                }
                            } else {
                                // narrow slice: rows are seg_bytes apart, R rows per step, lanes past the slice idle.  A row's
                                // rowslot (which half-tile sums it) is its index within the pair's piece of the record, k0 + r,
                                // whether or not a chunk boundary cut the piece
                                const int rowslot = lane / lpr, lcol = lane % lpr;  // (computed here: a division the common path never pays)
                                const bool col_ok = lcol * VEC < slice_cols;
                                const int k0 = (int)(lo - max(__shfl_sync(0xffffffffu, pc.rec.w, l), row_lo));
                                for (int st = k0 / R; st * R < k0 + n; st++) {
                                    const int r = st * R + rowslot;
                                    const bool ok = (rowslot < R) && (r >= k0) && (r < k0 + n) && col_ok;
                                    uint32_t ww[2] = {0u, 0u};
                                    if (ok) asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(ww[0]), "=r"(ww[1]) : "r"(sa + (uint32_t)((r - k0) * seg_bytes + lcol * LB)));
                                    accumulate_words<SLOTS, VEC>(base_lane, ok ? val : 0.f, ww);
                                }
                            }
                            if (tr && first) utrace[8 * s + 5] = (unsigned long long)clock64();
                            first = false;
                        }
                        t += done;
                        if (done < 32u) break;
                        done = v4_pieces(ulist, t, r_end, c0, c1, lane, pc);
                    }
                    rows_done += (unsigned long long)(c1 - c0);
                    if (tr) utrace[8 * s + 6] = (unsigned long long)clock64();
                    __syncwarp();  // every lane has read the chunk's bytes
                    if (lane == 0) mbar_arrive(empty0 + sl * 8u);
                    if (tr) utrace[8 * s + 7] = (unsigned long long)clock64();
                }
                if (lane == 0 && rows_done) atomicAdd(&hdr.sel_rows, (int)rows_done);  // rows selected = rows accumulated
                if (pb.unit_trace && blockIdx.x == 0 && lane == 0) {  // when every consumer of CTA 0 ran dry, and how much it did
                    unsigned long long* fin = pb.unit_trace + 648;
                    fin[warp] = (unsigned long long)clock64();
                    fin[16 + warp] = rows_done;
                    fin[32 + warp] = (unsigned long long)seq;
                }
            }
        } while (more);
    }
    __syncthreads();
    if (pb.sel_counts && slice == 0 && tid == 0) pb.sel_counts[rsp] = (uint32_t)hdr.sel_rows;
    V2_TRACE(9);
    if (cst) cst[8] = (unsigned long long)clock64();

    // ---- 4. CTA epilogue: sum the 8 consumer tiles; the RS partial sums of the slice then meet in a fixed order ----
    {
        constexpr int NG = NT / TW, SPT = SLOTS / NG;
        static_assert(SPT == 4, "one 16-byte reduction per thread");
        const int cl = tid % TW, sg = tid / TW;
        const int k = cl >> 5, ln = cl & 31;
        float acc[SPT] = {0.f, 0.f, 0.f, 0.f};
        const bool col_on = (ln < lpr) && (ln * VEC + k < slice_cols);
        if (col_on) {
            for (int rs2 = 0; rs2 < R; rs2++) {
                const int word0 = (sg * SPT) * TW + k * 32 + ln + rs2 * lpr;
#pragma unroll
                for (int w = 0; w < NC; w++)
#pragma unroll
                    for (int s = 0; s < SPT; s++) acc[s] += tiles[(size_t)w * TF + word0 + s * TW];
            }
        }
        // this CTA's partial sum goes to scratch; once all RS CTAs of the slice have written theirs, CTA rsp adds positions
        // rsp, rsp + RS, ... of the slice, each the sum over the RS partials in row-split order: every output word gets ONE
        // addition per launch, so the result does not depend on which CTA finished first
        pb.red_part[(size_t)blockIdx.x * NT + tid] = make_float4(acc[0], acc[1], acc[2], acc[3]);
        __threadfence();
        __syncthreads();
        unsigned* rsy = pb.red_sync + 2 * slice;
        if (tid == 0) {
            atomicAdd(rsy, 1u);
            const unsigned long long t0 = gtime_ns();
            while (ld_acquire_u32(rsy) < (unsigned)RS) {
                if (gtime_ns() - t0 > 2000000000ull) {
                    if (pb.err_flag) atomicExch(pb.err_flag, 4u);
                    break;
                }
            }
            if (pb.out_mode == kOutOverwrite) {
                const unsigned* cnt = pb.sync + 2 * slice;
                while (ld_acquire_u32(cnt) < (unsigned)RS) {
                    if (gtime_ns() - t0 > 2000000000ull) {
                        if (pb.err_flag) atomicExch(pb.err_flag, 1u);
                        break;
                    }
                }
            }
        }
        __syncthreads();
        const int t = rsp + tid * RS;
        if (t < NT) {
            const int tcl = t % TW, tsg = t / TW, tk = tcl >> 5, tln = tcl & 31;
            if ((tln < lpr) && (tln * VEC + tk < slice_cols)) {
                const float4* src = pb.red_part + (size_t)(batch.cta_begin[pi] + slice) * NT + t;
                float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
                for (int r = 0; r < RS; r++) {
                    const float4 x = __ldcg(src + (size_t)r * pb.CS * NT);
                    sum.x += x.x; sum.y += x.y; sum.z += x.z; sum.w += x.w;
                }
                const int col = slice * pb.W + tln * VEC + tk;
                red_add_v4(pb.out + (size_t)col * SLOTS + tsg * SPT, sum.x, sum.y, sum.z, sum.w);
            }
        }
        __syncthreads();
        if (tid == 0) {
            const unsigned old = atomicAdd(rsy + 1, 1u);
            if (old == (unsigned)RS - 1u) { rsy[0] = 0u; rsy[1] = 0u; }
            if (pb.out_mode == kOutOverwrite) {
                unsigned* sy = pb.sync + 2 * slice;
                const unsigned o2 = atomicAdd(sy + 1, 1u);
                if (o2 == (unsigned)RS - 1u) { sy[0] = 0u; sy[1] = 0u; }
            }
        }
    }
    if (cst) cst[9] = (unsigned long long)clock64();
    V2_TRACE(10);
}

}  // namespace effort
