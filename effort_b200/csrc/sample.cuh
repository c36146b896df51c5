// sample.cuh -- next token by temperature / top-k / top-p sampling from a counter-based random stream (DESIGN.md
// section 4.6).  One CTA.  After the fp32 weights everything is integer arithmetic (uint64 weight sums, exact radix
// selects, an integer draw), so the token depends only on the bits of the logits, the parameters and the position:
// no float atomics, no order that depends on timing.  tests/sampler_model.py restates the rule.
#pragma once
#include <limits.h>

#include "../../include/effort_b200.h"
#include "common.cuh"

namespace effort {

constexpr int kSampleThreads = 1024;
constexpr int kSampleCache = 32768;  // logits staged in shared memory when n fits (128 KB); else every pass reads L2
constexpr int kSampleHistBytes = 32 * 256 * 8;  // one private 256-bin histogram per warp, in front of the staged logits

struct SampleShared {
    unsigned long long hist[256];  // radix bins merged over the warps: token counts (top-k) or weight sums (top-p)
    unsigned long long part[32];   // per-warp partials
    float fmax[32];
    int imin[32];
    unsigned long long above, bin;  // select_digit: weight of the bins above the chosen one, and the chosen bin's
    uint32_t digit;
    int idx;
};

// order-preserving key: a > b as floats <=> key(a) > key(b); -0 == +0; NaN -> 0, below -inf (0 is no float's key)
__device__ __forceinline__ uint32_t sample_key(float x) {
    if (x != x) return 0u;
    const uint32_t b = __float_as_uint(x == 0.f ? 0.f : x);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float sample_key_value(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// q = floor(expf((x - m) / T) * 2^32): IEEE subtraction and division, the scale is exact and the conversion truncates.
// The maximum weighs 2^32; NaN and weights below 2^-32 of the maximum weigh 0 and are never drawn.
__device__ __forceinline__ unsigned long long sample_weight(float x, float m, float t) {
    if (x != x) return 0ull;
    const float w = expf(__fdiv_rn(__fsub_rn(x, m), t));
    return (unsigned long long)__fmul_rn(w, 4294967296.f);
}

// word 0 of Philox4x32-10 (Salmon et al., SC'11) at counter (position, 0, 0, 0), key (seed lo, seed hi)
__device__ __forceinline__ uint32_t philox_word0(uint32_t position, unsigned long long seed) {
    uint32_t c0 = position, c1 = 0u, c2 = 0u, c3 = 0u;
    uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
    for (int r = 0; r < 10; r++) {
        if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
    }
    return c0;
}

__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long x) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    return x;
}
__device__ __forceinline__ unsigned long long warp_incl_scan_u64(unsigned long long x, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    return x;
}

__device__ __forceinline__ unsigned long long sample_block_sum(SampleShared& sh, unsigned long long v) {
    v = warp_sum_u64(v);
    if ((threadIdx.x & 31) == 0) sh.part[threadIdx.x >> 5] = v;
    __syncthreads();
    unsigned long long t = 0;
#pragma unroll 8
    for (int w = 0; w < 32; w++) t += sh.part[w];
    __syncthreads();
    return t;
}

// After the bins are filled: the digit d, scanning bins 255..0, at which the running sum reaches `target`
// (above < target <= above + hist[d]; 1 <= target <= sum of the bins).  Warp 0 scans, lane l holding bins 255-8l..248-8l.
__device__ __forceinline__ void select_digit(SampleShared& sh, unsigned long long target) {
    __syncthreads();
    if (threadIdx.x < 32) {
        const int l = threadIdx.x;
        unsigned long long s = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) s += sh.hist[255 - 8 * l - j];
        const unsigned long long incl = warp_incl_scan_u64(s, l);
        unsigned long long run = incl - s;
        if (run < target && target <= incl) {
            for (int j = 0; j < 8; j++) {
                const int b = 255 - 8 * l - j;
                if (run + sh.hist[b] >= target) { sh.digit = (uint32_t)b; sh.above = run; sh.bin = sh.hist[b]; break; }
                run += sh.hist[b];
            }
        }
    }
    __syncthreads();
}

// The smallest index i whose inclusive prefix sum of val(0..i), in index order, exceeds tgt(total).  Warp w owns one
// contiguous run of indices; the warp whose run holds the crossing walks it 32 indices at a time.
template <class Val, class Tgt>
__device__ __forceinline__ int sample_crossing(SampleShared& sh, int n, Val val, Tgt tgt) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long per = (((long long)n + 1023) / 1024) * 32;  // indices per warp, a multiple of 32
    const int i0 = (int)min((long long)n, warp * per), i1 = (int)min((long long)n, i0 + per);
    unsigned long long s = 0;
    for (int i = i0 + lane; i < i1; i += 32) s += val(i);
    s = warp_sum_u64(s);
    if (lane == 0) sh.part[warp] = s;
    __syncthreads();
    unsigned long long excl = 0, total = 0;
#pragma unroll 8
    for (int w = 0; w < 32; w++) {
        const unsigned long long p = sh.part[w];
        excl += w < warp ? p : 0ull;
        total += p;
    }
    const unsigned long long target = tgt(total);
    if (excl <= target && target < excl + s) {  // warp-uniform: exactly one warp
        unsigned long long run = excl;
        for (int b = i0; b < i1; b += 32) {
            const int i = b + lane;
            const unsigned long long incl = run + warp_incl_scan_u64(i < i1 ? val(i) : 0ull, lane);
            const unsigned hit = __ballot_sync(0xffffffffu, incl > target);
            if (hit) {
                if (lane == __ffs(hit) - 1) sh.idx = i;
                break;
            }
            run = __shfl_sync(0xffffffffu, incl, 31);
        }
    }
    __syncthreads();
    return sh.idx;
}

// h[bin] += v (COUNT: += 1) for every lane with `on`, into the warp's private histogram: lanes with equal bins are
// grouped (the logits of one vocabulary share a few top digits) and each group makes one plain add -- no atomics.
template <bool COUNT>
__device__ __forceinline__ void warp_hist_add(unsigned long long* h, bool on, uint32_t bin, unsigned long long v, int lane) {
    const unsigned peers = __match_any_sync(0xffffffffu, on ? bin : 0xffffffffu);
    const bool lead = on && __ffs(peers) - 1 == lane;
    if (COUNT) {
        if (lead) h[bin] += (unsigned long long)__popc(peers);
        return;
    }
    if (lead && __popc(peers) == 1) h[bin] += v;
    for (unsigned todo = __ballot_sync(0xffffffffu, lead && __popc(peers) > 1); todo; todo &= todo - 1) {
        const int leader = __ffs(todo) - 1;
        const uint32_t b = __shfl_sync(0xffffffffu, bin, leader);
        const unsigned long long s = warp_sum_u64(on && bin == b ? v : 0ull);
        if (lane == leader) h[b] += s;
    }
}

// Radix select over the keys of the tokens `member` admits, weighted by wt (COUNT: by 1): the key t with
// W(key > t) < target <= W(key >= t).  Returns t and above = W(key > t); sh.bin = W(key == t).  hw = [32][256] bins.
template <bool COUNT, class Member, class Wt>
__device__ __forceinline__ uint32_t sample_radix(SampleShared& sh, unsigned long long* hw, const float* src, int n,
                                                 unsigned long long target, Member member, Wt wt, unsigned long long& above) {
    const int lane = threadIdx.x & 31;
    unsigned long long* h = hw + (threadIdx.x >> 5) * 256;
    uint32_t prefix = 0u, mask = 0u;
    above = 0;
    for (int shift = 24; shift >= 0; shift -= 8) {
        for (int j = lane; j < 256; j += 32) h[j] = 0ull;
        __syncwarp();
        for (int b = threadIdx.x - lane; b < n; b += kSampleThreads) {  // warp-uniform trip count
            const int i = b + lane;
            const float x = i < n ? src[i] : 0.f;
            const uint32_t k = sample_key(x);
            const bool on = i < n && (k & mask) == prefix && member(k, i);
            warp_hist_add<COUNT>(h, on, (k >> shift) & 255u, (on && !COUNT) ? wt(x) : 0ull, lane);
        }
        __syncthreads();
        if (threadIdx.x < 256) {
            unsigned long long t = 0;
#pragma unroll 8
            for (int w = 0; w < 32; w++) t += hw[w * 256 + threadIdx.x];
            sh.hist[threadIdx.x] = t;
        }
        select_digit(sh, target - above);
        prefix |= sh.digit << shift;
        mask |= 0xffu << shift;
        above += sh.above;
    }
    return prefix;
}

// logits[0..n) -> *token.  Parameters from *prm_dev when non-null (a model's device block), else prm; position from
// *pos_dev when non-null (the model's position after the head advanced it), else `position`.
__global__ void __launch_bounds__(kSampleThreads, 1)
sample_kernel(const float* __restrict__ logits, int n, const effort_sampler_t prm, const effort_sampler_t* __restrict__ prm_dev,
              const int* __restrict__ pos_dev, uint32_t position, int32_t* __restrict__ token) {
    extern __shared__ __align__(16) unsigned char dyn[];  // [kSampleHistBytes of warp histograms][min(n, kSampleCache) logits]
    __shared__ SampleShared sh;
    unsigned long long* hw = reinterpret_cast<unsigned long long*>(dyn);
    float* cache = reinterpret_cast<float*>(dyn + kSampleHistBytes);
    pdl_trigger();
    pdl_wait();
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float T = prm_dev ? prm_dev->temperature : prm.temperature;
    const int K = prm_dev ? prm_dev->top_k : prm.top_k;
    const float P = prm_dev ? prm_dev->top_p : prm.top_p;
    const unsigned long long seed = prm_dev ? prm_dev->seed : prm.seed;
    if (pos_dev) position = (uint32_t)*pos_dev;
    const bool cached = n <= kSampleCache;

    // 1. maximum (NaN never compares greater) and the first +inf
    float mx = -INFINITY;
    int first_inf = INT_MAX;
    for (int i = tid; i < n; i += kSampleThreads) {
        const float x = logits[i];
        if (cached) cache[i] = x;
        mx = x > mx ? x : mx;
        if (x == INFINITY && i < first_inf) first_inf = i;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        first_inf = min(first_inf, __shfl_xor_sync(0xffffffffu, first_inf, o));
    }
    if (lane == 0) { sh.fmax[warp] = mx; sh.imin[warp] = first_inf; }
    __syncthreads();
    for (int w = 0; w < 32; w++) { mx = fmaxf(mx, sh.fmax[w]); first_inf = min(first_inf, sh.imin[w]); }
    if (!(mx > -INFINITY && mx < INFINITY)) {  // greedy's choice: the first +inf, or token 0 when nothing is finite
        if (tid == 0) *token = mx == INFINITY ? first_inf : 0;
        return;
    }
    const float* src = cached ? cache : logits;
    auto weight = [&](float x) { return sample_weight(x, mx, T); };
    auto count = [](float) { return 1ull; };
    auto any = [](uint32_t, int) { return true; };

    // 2. top-k: S_k = keys above tkey, plus keys equal to tkey up to index tidx (ties cut by index)
    uint32_t tkey = 0u;
    int tidx = n - 1;
    if (K > 0 && K < n) {
        unsigned long long above;
        tkey = sample_radix<true>(sh, hw, src, n, (unsigned long long)K, any, count, above);
        const unsigned long long r = (unsigned long long)K - above;  // keys equal to tkey that S_k takes
        if (r < sh.bin)
            tidx = sample_crossing(sh, n, [&](int i) { return sample_key(src[i]) == tkey ? 1ull : 0ull; },
                                   [&](unsigned long long) { return r - 1; });
    }
    auto in_k = [&](uint32_t k, int i) { return k > tkey || (k == tkey && i <= tidx); };

    // 3. top-p: S = the shortest prefix of S_k (sampling order) whose weight reaches ceil(P * Q_k)
    uint32_t pkey = 0u;
    int pidx = n - 1;
    if (P < 1.f) {
        unsigned long long qk = 0;
        for (int i = tid; i < n; i += kSampleThreads) {
            const float x = src[i];
            if (in_k(sample_key(x), i)) qk += weight(x);
        }
        qk = sample_block_sum(sh, qk);
        const unsigned long long need = (unsigned long long)ceil((double)P * (double)qk);
        unsigned long long above;
        pkey = sample_radix<false>(sh, hw, src, n, need, in_k, weight, above);
        const unsigned long long qp = weight(sample_key_value(pkey));  // every token with key pkey weighs qp > 0
        const unsigned long long r = (need - above + qp - 1) / qp;
        if (r < sh.bin / qp)
            pidx = sample_crossing(sh, n, [&](int i) { const uint32_t k = sample_key(src[i]); return k == pkey && in_k(k, i) ? 1ull : 0ull; },
                                   [&](unsigned long long) { return r - 1; });
    }

    // 4. draw: target = (x * Q) >> 32; the token is the first index of S whose inclusive weight prefix exceeds it
    const uint32_t x = philox_word0(position, seed);
    const int t = sample_crossing(
        sh, n,
        [&](int i) {
            const float v = src[i];
            const uint32_t k = sample_key(v);
            return in_k(k, i) && (k > pkey || (k == pkey && i <= pidx)) ? weight(v) : 0ull;
        },
        [&](unsigned long long q) { return __umul64hi(q, (unsigned long long)x << 32); });
    if (tid == 0) *token = t;
}

}  // namespace effort
