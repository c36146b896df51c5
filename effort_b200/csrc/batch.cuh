// batch.cuh -- decoding up to kPrefillMax sequences per step, each with its own KV cache and position (DESIGN.md section
// 4.9).  The GEMVs and the glue are prefill's per-row kernels (prefill.cuh); the one kernel a batch adds is its attention.
#pragma once
#include "common.cuh"

namespace effort {

// attention_kernel's arithmetic for slot blockIdx.y of a batch: the slot's q / k / v rows, its own cache (slot b's cache is
// kcache + b * slot_stride, [max_seq][n_kv][128]) and its own position pos_dev[b].  Rope of q and k, append k / v at the
// position, 8 warps striding over the positions four at a time, the warps combined in index order, softmax without max
// subtraction.  A slot's output depends on its own inputs only: not on the batch size or the other slots.
__global__ void __launch_bounds__(256)
batch_attention_kernel(const float* __restrict__ xq, const float* __restrict__ xk, const float* __restrict__ xv,
                       float* __restrict__ kcache, float* __restrict__ vcache, size_t slot_stride,
                       const int* __restrict__ pos_dev, int n_heads, int n_kv, float theta, int max_seq,
                       float* __restrict__ attn_out) {
    constexpr int HD = 128;
    __shared__ __align__(16) float q[HD];
    __shared__ __align__(16) float kcur[HD];
    __shared__ float acc_s[8][HD];
    __shared__ float sum_s[8];
    const int h = blockIdx.x, b = blockIdx.y, kvh = h / (n_heads / n_kv);
    xq += (size_t)b * n_heads * HD;
    xk += (size_t)b * n_kv * HD;
    xv += (size_t)b * n_kv * HD;
    kcache += (size_t)b * slot_stride;
    vcache += (size_t)b * slot_stride;
    attn_out += (size_t)b * n_heads * HD;
    pdl_trigger();
    pdl_wait();
    int pos = pos_dev[b];
    pos = pos < 0 ? 0 : (pos >= max_seq ? max_seq - 1 : pos);  // backstop: the host refuses steps past max_seq
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < HD) {
        const int j = tid & 63;
        const float freq = powf(1e-6f * (1e6f / theta), (float)j / 64.f);
        const float ang = (float)pos * freq;
        const float c = cosf(ang), s = sinf(ang);
        const float* qh = xq + (size_t)h * HD;
        const float* kh = xk + (size_t)kvh * HD;
        const float qa = qh[tid], qb = (tid < 64) ? qh[tid + 64] : qh[tid - 64];
        const float ka = kh[tid], kb = (tid < 64) ? kh[tid + 64] : kh[tid - 64];
        q[tid] = (tid < 64) ? qa * c - qb * s : qa * c + qb * s;
        const float kr = (tid < 64) ? ka * c - kb * s : ka * c + kb * s;
        kcur[tid] = kr;
        if (h % (n_heads / n_kv) == 0) {
            kcache[((size_t)pos * n_kv + kvh) * HD + tid] = kr;
            vcache[((size_t)pos * n_kv + kvh) * HD + tid] = xv[(size_t)kvh * HD + tid];
        }
    }
    __syncthreads();
    const float4 q4 = *reinterpret_cast<const float4*>(&q[lane * 4]);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    float sum = 0.f;
    const float scale = rsqrtf((float)HD);
    for (int tb = warp; tb <= pos; tb += 32) {
        float4 k4[4], v4[4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int t = tb + 8 * i;
            k4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            v4[i] = k4[i];
            if (t < pos) {
                k4[i] = *reinterpret_cast<const float4*>(kcache + ((size_t)t * n_kv + kvh) * HD + lane * 4);
                v4[i] = *reinterpret_cast<const float4*>(vcache + ((size_t)t * n_kv + kvh) * HD + lane * 4);
            } else if (t == pos) {
                k4[i] = *reinterpret_cast<const float4*>(&kcur[lane * 4]);
                v4[i] = *reinterpret_cast<const float4*>(xv + (size_t)kvh * HD + lane * 4);
            }
        }
#pragma unroll
        for (int i = 0; i < 4; i++) {
            if (tb + 8 * i <= pos) {
                float d = q4.x * k4[i].x + q4.y * k4[i].y + q4.z * k4[i].z + q4.w * k4[i].w;
                d = warp_sum_f(d);
                const float p = expf(d * scale);
                sum += p;
                acc.x += p * v4[i].x; acc.y += p * v4[i].y; acc.z += p * v4[i].z; acc.w += p * v4[i].w;
            }
        }
    }
    *reinterpret_cast<float4*>(&acc_s[warp][lane * 4]) = acc;
    if (lane == 0) sum_s[warp] = sum;
    __syncthreads();
    if (tid < HD) {
        float a = 0.f, s = 0.f;
#pragma unroll
        for (int w = 0; w < 8; w++) { a += acc_s[w][tid]; s += sum_s[w]; }
        attn_out[(size_t)h * HD + tid] = a / s;
    }
}

}  // namespace effort
