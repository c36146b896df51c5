// convert.cuh -- one-time weight conversion (reference: convert.swift:209-260 + convert.metal:14-119)
// and the load-time device repack.
//
// GPU-first restructuring of bucketize: the reference sorts every transposed weight row by |w|
// (in x log^2(out) bitonic launches, convert.swift:227-229) only to walk it and deal the weights into
// their 16-wide buckets in arrival order.  The rank a weight gets inside its bucket depends only on
// the 16 weights of that bucket, so one thread ranks one (input, bucket) group by counting -- a single
// launch, no sort -- and the result is byte-identical to the row-sort formulation (tests/test_convert*).
#pragma once
#include "common.cuh"

namespace effort {

// probes: getProbes, convert.metal:14-22.  rep = out>=n ? 1 : n/out; probes[id*rep+j] = w[id + j + id*in]
__global__ void get_probes_kernel(const uint16_t* __restrict__ w, int in, int rep, int n_probes,
                                  uint16_t* __restrict__ probes) {
    const int id = blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= n_probes / rep) return;
    for (int j = 0; j < rep; j++) probes[id * rep + j] = w[(size_t)id + j + (size_t)id * in];
}

// bucketize: block = 32 inputs x 32 buckets.  Thread (gl = tid/32, il = tid%32) loads the 16 weights
// W[(g*16+j), i] (coalesced over i), ranks them by (|w| desc, index asc), stages the 16 rank rows in
// shared memory and the block writes 64-byte row segments buckets[(rank*in + i)*C + g0 .. g0+31].
__global__ void __launch_bounds__(1024)
bucketize_kernel(const uint16_t* __restrict__ w, int out, int in, uint16_t* __restrict__ buckets) {
    __shared__ uint16_t tile[16][32][34];  // [rank][i_local][g_local], padded
    const int C = out / 16;
    const int il = threadIdx.x & 31, gl = threadIdx.x >> 5;
    const int i = blockIdx.x * 32 + il, g = blockIdx.y * 32 + gl;
    if (i < in && g < C) {
        uint16_t b[16];
#pragma unroll
        for (int j = 0; j < 16; j++) b[j] = w[(size_t)(g * 16 + j) * in + i];
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const uint16_t aj = b[j] & 0x7FFFu;
            int rank = 0;
#pragma unroll
            for (int k = 0; k < 16; k++) {
                const uint16_t ak = b[k] & 0x7FFFu;
                rank += (ak > aj || (ak == aj && k < j)) ? 1 : 0;
            }
            tile[rank][il][gl] = (uint16_t)((b[j] & 0xFFF0u) | (uint16_t)j);  // convert.metal:64-70
        }
    }
    __syncthreads();
    // write: thread (row = tid/32 -> (rank, i_local) pairs, lane -> g_local)
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
    const int gg = blockIdx.y * 32 + lane;
    for (int p = wrp; p < 16 * 32; p += 32) {
        const int rank = p / 32, ii = p % 32;
        const int gi = blockIdx.x * 32 + ii;
        if (gi < in && gg < C) buckets[((size_t)rank * in + gi) * C + gg] = tile[rank][ii][lane];
    }
}

// makeStats, convert.metal:105-119: mean |w| of a bucket row, fp32 SEQUENTIAL sum (same order as the
// reference's loop so the fp16 result is reproducible), replicated into the 4 lanes of a half4.
__global__ void make_stats_kernel(const uint16_t* __restrict__ buckets, size_t rows, int C,
                                  __half* __restrict__ stats4) {
    const size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    const uint16_t* row = buckets + r * C;
    float sum = 0.f;
    for (int c = 0; c < C; c++) sum = __fadd_rn(sum, fabsf(half_bits_to_float(row[c])));
    const __half h = __float2half_rn(__fdiv_rn(sum, (float)C));
    stats4[r * 4 + 0] = h; stats4[r * 4 + 1] = h; stats4[r * 4 + 2] = h; stats4[r * 4 + 3] = h;
}

// ---- load-time repack (effort_weights_create) -------------------------------------------------------
// stats: reference half4 (all lanes equal, .w is the one read, bucketMul.metal:64-66) -> one fp16/row;
// Q4: float2 (avg,avg), .y read (bucketMulQ4.metal:44-46) -> one fp32/row.  8 B/row -> 2 or 4 B/row.
// to_input_major != 0 also reorders rows rank-major -> input-major.
__global__ void repack_stats_fp16_kernel(const __half* __restrict__ stats4, int n_experts, int in, int P,
                                         int to_input_major, __half* __restrict__ st16) {
    const size_t n = (size_t)n_experts * in * P;
    const size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // destination row
    if (r >= n) return;
    size_t src = r;
    if (to_input_major) {
        const size_t e = r / ((size_t)in * P), rem = r % ((size_t)in * P);
        const size_t i = rem / P, rho = rem % P;
        src = e * (size_t)in * P + rho * in + i;
    }
    st16[r] = stats4[src * 4 + 3];
}
__global__ void repack_stats_q4_kernel(const float* __restrict__ stats2, size_t n, float* __restrict__ st32) {
    const size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n) st32[r] = stats2[r * 2 + 1];
}
// bucket rows rank-major -> input-major; one warp per destination row, 16-byte copies when possible.
__global__ void repack_rows_kernel(const uint16_t* __restrict__ src, int n_experts, int in, int P, int C,
                                   uint16_t* __restrict__ dst) {
    const size_t n = (size_t)n_experts * in * P;
    const size_t r = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= n) return;
    const size_t e = r / ((size_t)in * P), rem = r % ((size_t)in * P);
    const size_t i = rem / P, rho = rem % P;
    const size_t s = e * (size_t)in * P + rho * in + i;
    if ((C & 7) == 0) {
        const uint4* a = reinterpret_cast<const uint4*>(src + s * C);
        uint4* b = reinterpret_cast<uint4*>(dst + r * C);
        for (int c = lane; c < C / 8; c += 32) b[c] = a[c];
    } else {
        for (int c = lane; c < C; c += 32) dst[r * C + c] = src[s * C + c];
    }
}

// bucket rows -> slice-major [e][slice][i][rho][W_s]; src is rank-major (src_rank_major) or input-major.  One thread per
// 16-byte piece (C % 8 == 0, W % 8 == 0).
__global__ void repack_slices_kernel(const uint16_t* __restrict__ src, int n_experts, int in, int P, int C, int W,
                                     int src_rank_major, uint16_t* __restrict__ dst) {
    const size_t pieces_per_row = (size_t)C / 8;
    const size_t n = (size_t)n_experts * in * P * pieces_per_row;
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const size_t r = t / pieces_per_row;            // destination-independent logical row (e, i, rho)
    const int c0 = (int)(t % pieces_per_row) * 8;   // first column of the piece
    const size_t e = r / ((size_t)in * P), rem = r % ((size_t)in * P);
    const size_t i = rem / P, rho = rem % P;
    const size_t srow = src_rank_major ? e * (size_t)in * P + rho * in + i : r;
    const int sl = c0 / W, cw = c0 % W;
    const int Ws = (C - sl * W) < W ? (C - sl * W) : W;
    const size_t d = e * (size_t)in * P * C + (size_t)in * P * ((size_t)sl * W) + (i * P + rho) * (size_t)Ws + cw;
    *reinterpret_cast<uint4*>(dst + d) = *reinterpret_cast<const uint4*>(src + srow * C + c0);
}

// ---- dense comparator: basicMul (helpers/mps.swift:14-47, matrix.metal:150-162) ----------------------
// v is cast to fp16 first (mps.swift:19); fp16 x fp16 products accumulated in fp32.  One warp per output
// row, 16-byte weight loads, v staged once per CTA in shared memory as fp16-rounded floats.
__global__ void __launch_bounds__(256)
basic_mul_kernel(const float* __restrict__ v, const __half* __restrict__ W, int out, int in,
                 float* __restrict__ outv) {
    extern __shared__ float vs[];
    pdl_trigger();
    pdl_wait();
    for (int i = threadIdx.x; i < in; i += blockDim.x) vs[i] = __half2float(__float2half_rn(v[i]));
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int wpb = blockDim.x >> 5;
    for (int o = blockIdx.x * wpb + (threadIdx.x >> 5); o < out; o += gridDim.x * wpb) {
        const __half* row = W + (size_t)o * in;
        float acc = 0.f;
        if ((in & 7) == 0) {
            for (int c = lane * 8; c < in; c += 256) {
                const uint4 d = ldg_stream_u4(row + c);
                const uint32_t ws[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&ws[j]));
                    acc = fmaf(vs[c + 2 * j], f.x, acc);
                    acc = fmaf(vs[c + 2 * j + 1], f.y, acc);
                }
            }
        } else {
            for (int c = lane; c < in; c += 32) acc = fmaf(vs[c], __half2float(row[c]), acc);
        }
        acc = warp_sum_f(acc);
        if (lane == 0) outv[o] = acc;
    }
}

// calcOutliers, bucketMulQ4.metal:13-21: out[o.z] += v[o.y] * o.x (atomic: several outliers may share
// an output).  Order of the fp32 adds is non-deterministic exactly as in the reference.
__global__ void calc_outliers_kernel(const float* __restrict__ v, const float4* __restrict__ outliers, int n,
                                     float* __restrict__ out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const float4 o = outliers[k];
    atomicAdd(&out[(uint32_t)o.z], __fmul_rn(v[(uint32_t)o.y], o.x));
}

}  // namespace effort
