// score.cuh -- one record {argmax, rank, logprob} of a target token against a logits vector (DESIGN.md section 4.7).
// One CTA per record, two passes over the logits (L2-resident after the head): the greedy maximum and argmax, then the
// fp32 sum of expf(l_i - m) and the exact rank count.  Every sum has a fixed order (per-thread strided sums, a shuffle
// tree, then the warps in index order) and there are no atomics, so the record depends only on the logits' bits and the
// target.  tests/score_model.py restates the rule.
#pragma once
#include <limits.h>

#include "../../include/effort_b200.h"
#include "common.cuh"
#include "sample.cuh"  // sample_key: the sampler's order-preserving keys, which define the rank

namespace effort {

constexpr int kScoreThreads = 1024;

// record r = blockIdx.x, or *pos_dev - gridDim.x + blockIdx.x when pos_dev is non-null (the model's position after the
// head advanced it: pos - 1 for a step, the chunk's positions for a prefill chunk); records outside [0, n_rec) are not
// written.  The target is targets[r]; outside [0, n) it means "no target".  Block b reads the logits row
// logits + b * ld (ld = 0: every record scores the same vector).
__global__ void __launch_bounds__(kScoreThreads, 1)
score_kernel(const float* __restrict__ logits, int n, const int32_t* __restrict__ targets, int n_rec,
             const int* __restrict__ pos_dev, effort_score_t* __restrict__ out, int ld) {
    __shared__ float bv[32], ws[32];
    __shared__ int bi[32], wc[32];
    pdl_trigger();
    pdl_wait();
    const int r = pos_dev ? *pos_dev - (int)gridDim.x + (int)blockIdx.x : (int)blockIdx.x;
    if (r < 0 || r >= n_rec) return;
    logits += (size_t)blockIdx.x * ld;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int t = targets[r];
    const bool has_t = t >= 0 && t < n;

    // 1. maximum and argmax, argmax_advance_kernel's rule: lowest index of the maximum, NaN never wins
    float best = -INFINITY;
    int idx = INT_MAX;
    for (int i = tid; i < n; i += kScoreThreads) {
        const float x = logits[i];
        if (x > best || (x == best && i < idx)) { best = x; idx = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
        if (ob > best || (ob == best && oi < idx)) { best = ob; idx = oi; }
    }
    if (lane == 0) { bv[warp] = best; bi[warp] = idx; }
    __syncthreads();
    for (int w = 0; w < 32; w++)
        if (bv[w] > best || (bv[w] == best && bi[w] < idx)) { best = bv[w]; idx = bi[w]; }
    const float m = best;  // the maximum over the non-NaN logits; -inf when there are none
    const bool finite = m > -INFINITY && m < INFINITY;

    // 2. S = sum of expf(l_i - m) over the non-NaN logits; rank = #{key_i > key_t} + #{i < t : key_i == key_t}
    const float lt = has_t ? logits[t] : 0.f;
    const uint32_t kt = sample_key(lt);
    float s = 0.f;
    int c = 0;
    for (int i = tid; i < n; i += kScoreThreads) {
        const float x = logits[i];
        if (finite && x == x) s = __fadd_rn(s, expf(__fsub_rn(x, m)));  // __fadd_rn: no contraction into expf's tail
        const uint32_t k = sample_key(x);
        c += (k > kt || (k == kt && i < t)) ? 1 : 0;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
    c = __reduce_add_sync(0xffffffffu, c);
    if (lane == 0) { ws[warp] = s; wc[warp] = c; }
    __syncthreads();
    if (tid != 0) return;
    float S = 0.f;
    int rank = 0;
    for (int w = 0; w < 32; w++) { S = __fadd_rn(S, ws[w]); rank += wc[w]; }
    const float qnan = __int_as_float(0x7fc00000);
    float lp = qnan;
    if (has_t && finite) lp = (lt != lt || lt == -INFINITY) ? -INFINITY : __fsub_rn(__fsub_rn(lt, m), logf(S));
    effort_score_t rec;
    rec.argmax = idx < n ? idx : 0;
    rec.rank = has_t ? rank : -1;
    rec.logprob = lp;
    out[r] = rec;
}

}  // namespace effort
