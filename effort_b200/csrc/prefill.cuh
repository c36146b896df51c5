// prefill.cuh -- reading a prompt up to kPrefillMax tokens per pass (DESIGN.md section 4.8): the multi-token effort GEMV
// (per-token cutoff, per-token row test, one weight read per selected row shared by the chunk), the chunk's causal
// attention and its glue.  The decode chain (decode.cuh, bucket_mul_v4.cuh) is untouched.
#pragma once
#include "common.cuh"

namespace effort {

constexpr int kPrefillMax = 16;        // tokens per pass: one warp per token in the GEMV
constexpr int kPrefillProbes = 4096;   // EFFORT_PROBES_COUNT
constexpr int kPrefillMaxProblems = 3; // q/k/v share one input

// one weight matrix of a launch group; every problem of a group reads the same input V [T][in]
struct PrefillProblem {
    const uint16_t* bk;      // slice-major rows [slice][in][P][Ws]
    const __half* st16;      // one stat per row, row = i * P + rank
    const __half* probes;    // [4096]
    int in, C, P, W, CS, RS; // W = full slice width in words (min(C, 128)), CS slices, RS input splits
    int k;                   // select rank: n_probes - q (>= 4096: cutoff 0)
    float* cut;              // [T] per-token cutoff
    float* part;             // [RS][T][out] per-split partial sums
    uint32_t* cnt_part;      // [RS][T] per-split selected-row counts
    float* out;              // [T][out]
    uint32_t* count;         // [T] selected rows per token, may be null
    int accumulate;          // out += sum (residual) instead of out = sum
};
struct PrefillGroup {
    PrefillProblem p[kPrefillMaxProblems];
    int n, T;
    const float* V;
};

// The select rule of EFFORT_CUTOFF_SELECT for token blockIdx.x and problem blockIdx.y: the probe products
// bf16(|1e5 * v[i] * bf16(probe[i])|) are non-negative bf16 values, so their top 16 bits order them; a two-digit radix
// select finds the one at descending rank k, exactly oracle_select_cutoff.  Integer histograms only.
__global__ void __launch_bounds__(1024)
prefill_cutoff_kernel(const PrefillGroup g) {
    __shared__ int hist[256];
    __shared__ int sel_hi, sel_rem;
    pdl_trigger();
    pdl_wait();
    const PrefillProblem& P = g.p[blockIdx.y];
    const int t = blockIdx.x, tid = threadIdx.x;
    if (P.k >= kPrefillProbes) {
        if (tid == 0) P.cut[t] = 0.f;
        return;
    }
    uint32_t key[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int i = tid + 1024 * j;
        const float pr = bf16_round(__half2float(P.probes[i]));
        const float x = __fmul_rn(__fmul_rn(kCutoffScale, g.V[(size_t)t * P.in + i]), pr);
        key[j] = __float_as_uint(bf16_round(fabsf(x))) >> 16;
    }
    int rem = P.k, hi = 0;
#pragma unroll
    for (int digit = 0; digit < 2; digit++) {
        if (tid < 256) hist[tid] = 0;
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 4; j++)
            if (digit == 0 || (key[j] >> 8) == (uint32_t)hi) atomicAdd(&hist[digit == 0 ? key[j] >> 8 : key[j] & 255], 1);
        __syncthreads();
        if (tid == 0) {
            int b = 255, cum = 0;
            while (b > 0 && cum + hist[b] <= rem) { cum += hist[b]; b--; }
            sel_hi = b;
            sel_rem = rem - cum;
        }
        __syncthreads();
        if (digit == 0) hi = sel_hi;
        rem = sel_rem;
        __syncthreads();
    }
    if (tid == 0) P.cut[t] = __uint_as_float((((uint32_t)hi << 8) | (uint32_t)sel_hi) << 16);
}

// out[t] (+)= W(V[t]) for the rows token t selects.  CTA = (problem, column slice, input split); warp t = token t; lane
// owns 4 words of the slice's rows.  Each warp walks its split's inputs in order and, per input, the ranks its token
// selects in order, accumulating into its own 8 KB fp32 tile [position][word][lane] (conflict-free).  Each warp loads
// its own rows: the warps of a CTA walk the same inputs, so a row several tokens select may be served from L1/L2 after
// its first read, but nothing makes it so and the HBM traffic has not been measured.  A token's sum depends only on its
// own input and cutoff: the partition is a function of the matrix alone, each split's rows are summed in a fixed order
// and the splits are added in split order by prefill_reduce_kernel.
__global__ void __launch_bounds__(32 * kPrefillMax, 1)
prefill_mul_kernel(const PrefillGroup g) {
    extern __shared__ float tile_all[];
    int b = blockIdx.x, pi = 0;
    while (pi + 1 < g.n && b >= g.p[pi].CS * g.p[pi].RS) { b -= g.p[pi].CS * g.p[pi].RS; pi++; }
    const PrefillProblem& P = g.p[pi];
    const int sl = b / P.RS, rs = b % P.RS;
    const int t = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* tile = tile_all + t * (16 * 4 * 32);
    for (int j = lane; j < 16 * 4 * 32; j += 32) tile[j] = 0.f;
    pdl_trigger();
    pdl_wait();
    const int i0 = (int)((long long)rs * P.in / P.RS), i1 = (int)((long long)(rs + 1) * P.in / P.RS);
    const int Ws = min(P.W, P.C - sl * P.W);
    const bool active = lane * 4 < Ws;
    const uint16_t* slice = P.bk + (size_t)P.in * P.P * sl * P.W + lane * 4;
    const float cut = P.cut[t];
    const float* v = g.V + (size_t)t * P.in;
    uint32_t count = 0;
    for (int base = i0; base < i1; base += 32) {
        const int i = base + lane;
        float x = 0.f;
        uint32_t mask = 0;
        if (i < i1) {
            x = v[i];
            const __half* st = P.st16 + (size_t)i * P.P;
            for (int r = 0; r < P.P; r++)
                if (row_selected(cut, __half2float(st[r]), x)) mask |= 1u << r;
        }
        count += __popc(mask);
        const int nb = min(32, i1 - base);
        for (int j = 0; j < nb; j++) {
            uint32_t m = __shfl_sync(0xffffffffu, mask, j);
            const float xv = __shfl_sync(0xffffffffu, x, j);
            const uint16_t* rows = slice + (size_t)(base + j) * P.P * Ws;
            while (m) {  // up to four of the input's rows in flight, then accumulated in rank order
                int r[4];
                uint2 d[4];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    r[u] = m ? __ffs(m) - 1 : -1;
                    if (m) m &= m - 1;
                    d[u] = make_uint2(0u, 0u);
                    if (r[u] >= 0 && active) d[u] = __ldg(reinterpret_cast<const uint2*>(rows + (size_t)r[u] * Ws));
                }
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    if (r[u] < 0 || !active) continue;
                    const uint32_t ws[2] = {d[u].x, d[u].y};
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        const uint16_t bits = (uint16_t)(ws[k >> 1] >> (16 * (k & 1)));
                        float& a = tile[((bits & 15) * 4 + k) * 32 + lane];
                        a = fmaf(xv, half_bits_to_float(bits), a);
                    }
                }
            }
        }
    }
    count = __reduce_add_sync(0xffffffffu, count);
    if (lane == 0 && sl == 0) P.cnt_part[rs * g.T + t] = count;  // every slice of a split sees the same selection
    __syncwarp();
    if (!active) return;
    const int out_n = P.C * 16;
    float* dst = P.part + ((size_t)rs * g.T + t) * out_n + (size_t)(sl * P.W + lane * 4) * 16;
#pragma unroll
    for (int k = 0; k < 4; k++)
#pragma unroll
        for (int q = 0; q < 16; q += 4)
            *reinterpret_cast<float4*>(dst + k * 16 + q) =
                make_float4(tile[(q * 4 + k) * 32 + lane], tile[((q + 1) * 4 + k) * 32 + lane],
                            tile[((q + 2) * 4 + k) * 32 + lane], tile[((q + 3) * 4 + k) * 32 + lane]);
}

// out[t][o] (+)= sum over the splits, in split order; block 0 of each problem also sums the counts
__global__ void __launch_bounds__(256)
prefill_reduce_kernel(const PrefillGroup g) {
    pdl_trigger();
    pdl_wait();
    for (int pi = 0; pi < g.n; pi++) {
        const PrefillProblem& P = g.p[pi];
        const int out_n = P.C * 16;
        const size_t n4 = (size_t)g.T * out_n / 4;
        for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n4; e += (size_t)gridDim.x * blockDim.x) {
            const size_t t = e * 4 / out_n, o = e * 4 % out_n;
            float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int r = 0; r < P.RS; r++) {
                const float4 p = *reinterpret_cast<const float4*>(P.part + ((size_t)r * g.T + t) * out_n + o);
                s.x += p.x; s.y += p.y; s.z += p.z; s.w += p.w;
            }
            float4* dst = reinterpret_cast<float4*>(P.out + t * out_n + o);
            if (P.accumulate) { const float4 a = *dst; s.x = a.x + s.x; s.y = a.y + s.y; s.z = a.z + s.z; s.w = a.w + s.w; }
            *dst = s;
        }
        if (blockIdx.x == 0 && P.count && threadIdx.x < (unsigned)g.T) {
            uint32_t c = 0;
            for (int r = 0; r < P.RS; r++) c += P.cnt_part[r * g.T + threadIdx.x];
            P.count[threadIdx.x] = c;
        }
    }
}

// x[t] = float(tok_embeddings[token[t]]) for the chunk; out-of-range tokens read row 0, as embed_kernel does
__global__ void __launch_bounds__(256)
prefill_embed_kernel(const int* __restrict__ tokens, const __half* __restrict__ emb, int dim, int vocab, float* __restrict__ x) {
    pdl_trigger();
    pdl_wait();
    int tok = tokens[blockIdx.x];
    tok = (tok < 0 || tok >= vocab) ? 0 : tok;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) x[(size_t)blockIdx.x * dim + i] = __half2float(emb[(size_t)tok * dim + i]);
}

// out[t] = rmsNorm(h[t]) * w, one CTA per token (add_rmsnorm_kernel's arithmetic)
__global__ void __launch_bounds__(1024)
prefill_rmsnorm_kernel(const float* __restrict__ h, const __half* __restrict__ w, int dim, float eps, float* __restrict__ out) {
    __shared__ float red[32];
    __shared__ float total;
    pdl_trigger();
    pdl_wait();
    h += (size_t)blockIdx.x * dim;
    out += (size_t)blockIdx.x * dim;
    float ss = 0.f;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) { const float x = h[i]; ss += x * x; }
    ss = warp_sum_f(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    if (threadIdx.x < 32) {
        float t = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.f;
        t = warp_sum_f(t);
        if (threadIdx.x == 0) total = t;
    }
    __syncthreads();
    const float denom = sqrtf(total / (float)dim + eps);
    for (int i = threadIdx.x; i < dim; i += blockDim.x) out[i] = (h[i] / denom) * __half2float(w[i]);
}

// Causal attention for the chunk's T queries at positions p0 .. p0+T-1 (p0 = the device position).  One CTA per KV
// head: it first appends the chunk's T roped keys and values to the cache (attention_kernel's rope), then every
// (query head of the group, token) pair attends to positions <= p0 + t, reading each 32-position K/V tile of the group
// once from the cache into shared memory (a group with more than kChunkAttnPairs pairs is split over grid.y; every
// CTA of the group writes the same cache rows).  Softmax without max subtraction, scale 1/sqrt(128), as attention_kernel.
// Warp w takes pairs w, w + nwarps, ...; lane <-> 4 head dims.
constexpr int kChunkAttnThreads = 512;
constexpr int kChunkAttnTile = 32;
constexpr int kChunkAttnPairs = 128;  // (query head, token) pairs per CTA; larger groups take more CTAs (grid.y)
__global__ void __launch_bounds__(kChunkAttnThreads)
chunk_attention_kernel(const float* __restrict__ xq, const float* __restrict__ xk, const float* __restrict__ xv, int T,
                       float* __restrict__ kcache, float* __restrict__ vcache, const int* __restrict__ pos_dev, int n_heads,
                       int n_kv, float theta, int max_seq, float* __restrict__ attn_out) {
    constexpr int HD = 128;
    extern __shared__ __align__(16) float sm[];
    float* ks = sm;                                // [tile][128]
    float* vs = ks + kChunkAttnTile * HD;          // [tile][128]
    float* qs = vs + kChunkAttnTile * HD;          // [group * T][128] roped queries
    const int kvh = blockIdx.x, G = n_heads / n_kv;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    pdl_trigger();
    pdl_wait();
    int p0 = *pos_dev;
    p0 = p0 < 0 ? 0 : (p0 + T > max_seq ? max_seq - T : p0);  // backstop: the host refuses chunks past max_seq
    const int kvd = n_kv * HD;
    for (int e = tid; e < T * HD; e += blockDim.x) {  // append the chunk's keys (roped) and values
        const int t = e / HD, d = e % HD, j = d & 63;
        const float freq = powf(1e-6f * (1e6f / theta), (float)j / 64.f);
        const float ang = (float)(p0 + t) * freq;
        const float c = cosf(ang), s = sinf(ang);
        const float* kh = xk + (size_t)t * kvd + (size_t)kvh * HD;
        const float ka = kh[d], kb = (d < 64) ? kh[d + 64] : kh[d - 64];
        kcache[((size_t)(p0 + t) * n_kv + kvh) * HD + d] = (d < 64) ? ka * c - kb * s : ka * c + kb * s;
        vcache[((size_t)(p0 + t) * n_kv + kvh) * HD + d] = xv[(size_t)t * kvd + (size_t)kvh * HD + d];
    }
    const int pair0 = blockIdx.y * kChunkAttnPairs, n_pairs = min(kChunkAttnPairs, G * T - pair0);
    for (int e = tid; e < n_pairs * HD; e += blockDim.x) {  // pair = g * T + t
        const int pr = e / HD, d = e % HD, j = d & 63, g = (pair0 + pr) / T, t = (pair0 + pr) % T;
        const float freq = powf(1e-6f * (1e6f / theta), (float)j / 64.f);
        const float ang = (float)(p0 + t) * freq;
        const float c = cosf(ang), s = sinf(ang);
        const float* qh = xq + (size_t)t * n_heads * HD + (size_t)(kvh * G + g) * HD;
        const float qa = qh[d], qb = (d < 64) ? qh[d + 64] : qh[d - 64];
        qs[(size_t)pr * HD + d] = (d < 64) ? qa * c - qb * s : qa * c + qb * s;
    }
    __syncthreads();
    const float scale = rsqrtf((float)HD);
    constexpr int kMaxPairsPerWarp = kChunkAttnPairs / (kChunkAttnThreads / 32);
    float4 acc[kMaxPairsPerWarp];
    float sum[kMaxPairsPerWarp];
#pragma unroll
    for (int u = 0; u < kMaxPairsPerWarp; u++) { acc[u] = make_float4(0.f, 0.f, 0.f, 0.f); sum[u] = 0.f; }
    const int last = p0 + T - 1;
    for (int tb = 0; tb <= last; tb += kChunkAttnTile) {
        __syncthreads();
        for (int e = tid; e < kChunkAttnTile * HD / 4; e += blockDim.x) {
            const int r = e / (HD / 4), c4 = e % (HD / 4), p = tb + r;
            float4 kk = make_float4(0.f, 0.f, 0.f, 0.f), vv = kk;
            if (p <= last) {
                kk = *reinterpret_cast<const float4*>(kcache + ((size_t)p * n_kv + kvh) * HD + c4 * 4);
                vv = *reinterpret_cast<const float4*>(vcache + ((size_t)p * n_kv + kvh) * HD + c4 * 4);
            }
            reinterpret_cast<float4*>(ks)[e] = kk;
            reinterpret_cast<float4*>(vs)[e] = vv;
        }
        __syncthreads();
#pragma unroll
        for (int u = 0; u < kMaxPairsPerWarp; u++) {
            const int pr = warp + u * nw;
            if (pr >= n_pairs) continue;
            const int qpos = p0 + (pair0 + pr) % T;
            const float4 q4 = *reinterpret_cast<const float4*>(qs + (size_t)pr * HD + lane * 4);
            const int pend = min(tb + kChunkAttnTile - 1, qpos);
            for (int p = tb; p <= pend; p++) {
                const float4 k4 = *reinterpret_cast<const float4*>(ks + (p - tb) * HD + lane * 4);
                const float4 v4 = *reinterpret_cast<const float4*>(vs + (p - tb) * HD + lane * 4);
                float d = q4.x * k4.x + q4.y * k4.y + q4.z * k4.z + q4.w * k4.w;
                d = warp_sum_f(d);
                const float pe = expf(d * scale);
                sum[u] += pe;
                acc[u].x += pe * v4.x; acc[u].y += pe * v4.y; acc[u].z += pe * v4.z; acc[u].w += pe * v4.w;
            }
        }
    }
#pragma unroll
    for (int u = 0; u < kMaxPairsPerWarp; u++) {
        const int pr = warp + u * nw;
        if (pr >= n_pairs) continue;
        const int g = (pair0 + pr) / T, t = (pair0 + pr) % T;
        const float inv = sum[u];
        float4 o = make_float4(acc[u].x / inv, acc[u].y / inv, acc[u].z / inv, acc[u].w / inv);
        *reinterpret_cast<float4*>(attn_out + (size_t)t * n_heads * HD + (size_t)(kvh * G + g) * HD + lane * 4) = o;
    }
}

// the dense lm_head for T vectors (basicMul: v cast to fp16 first, fp32 accumulate), one warp per vocabulary row, the row
// read once for the chunk; row T - 1 is also written to `last` (the model's logits)
__global__ void __launch_bounds__(256)
prefill_head_kernel(const float* __restrict__ x, int T, const __half* __restrict__ W, int out, int in,
                    float* __restrict__ logits, float* __restrict__ last) {
    extern __shared__ __half xs[];  // [T][in]
    pdl_trigger();
    pdl_wait();
    for (int e = threadIdx.x; e < T * in; e += blockDim.x) xs[e] = __float2half_rn(x[e]);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int o = blockIdx.x * 8 + warp; o < out; o += gridDim.x * 8) {
        const __half* row = W + (size_t)o * in;
        float acc[kPrefillMax];
#pragma unroll
        for (int t = 0; t < kPrefillMax; t++) acc[t] = 0.f;
        for (int c = lane * 8; c < in; c += 256) {
            const uint4 d = ldg_stream_u4(row + c);
            const uint32_t ws[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&ws[j]));
#pragma unroll
                for (int t = 0; t < kPrefillMax; t++) {
                    if (t >= T) break;
                    const float2 xv = __half22float2(*reinterpret_cast<const __half2*>(xs + (size_t)t * in + c + 2 * j));
                    acc[t] = fmaf(xv.x, f.x, acc[t]);
                    acc[t] = fmaf(xv.y, f.y, acc[t]);
                }
            }
        }
#pragma unroll
        for (int t = 0; t < kPrefillMax; t++) {
            if (t >= T) break;
            const float a = warp_sum_f(acc[t]);
            if (lane == 0) {
                logits[(size_t)t * out + o] = a;
                if (t == T - 1) last[o] = a;
            }
        }
    }
}

// pos += by: the chunk's first T - 1 positions (the head that follows advances the last one, as in a step)
__global__ void prefill_advance_kernel(int* __restrict__ pos_dev, int by) {
    pdl_trigger();
    pdl_wait();
    *pos_dev = *pos_dev + by;
}

}  // namespace effort
