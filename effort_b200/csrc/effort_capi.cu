// effort_capi.cu -- the C-ABI shim (include/effort_b200.h) over the sm_90a kernels.
// Host orchestration here mirrors bucketMul.swift:34-88 / bucketMulQ4.swift:35-85 / expertMul.swift:20-38.
#include "../../include/effort_b200.h"

#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <new>
#include <string>
#include <utility>
#include <vector>

#include "bucket_mul.cuh"
#include "bucket_mul_v2.cuh"
#include "bucket_mul_v3.cuh"
#include "bucket_mul_v4.cuh"
#include "comm.cuh"
#include "convert.cuh"
#include "cutoff.cuh"
#include "q4.cuh"
#include "sample.cuh"
#include "score.cuh"
#include "prefill.cuh"
#include "batch.cuh"

using namespace effort;

static std::atomic<uint64_t> g_launches{0};
static thread_local std::string g_cuda_err;

#define CK(expr)                                                                         \
    do {                                                                                 \
        cudaError_t _e = (expr);                                                         \
        if (_e != cudaSuccess) {                                                         \
            g_cuda_err = std::string(#expr) + ": " + cudaGetErrorString(_e);             \
            return EFFORT_ECUDA;                                                         \
        }                                                                                \
    } while (0)
#define LAUNCHED()                     \
    do {                               \
        g_launches.fetch_add(1);       \
        CK(cudaGetLastError());        \
    } while (0)

struct effort_weights {
    int in = 0, out = 0, n_experts = 1, P = 16, kind = EFFORT_KIND_FP16;
    int n_probes = EFFORT_PROBES_COUNT;
    int C = 0;  // 16-bit words per bucket row
    unsigned flags = 0;
    // caller-owned, reference layout
    const uint16_t* buckets = nullptr;
    const void* stats = nullptr;
    const __half* probes = nullptr;
    const float4* outliers = nullptr;
    int n_outliers = 0;
    const __half* core = nullptr;
    // owned device copies
    uint16_t* bk_own = nullptr;  // input-major rows (FP16 kind, unless NO_REPACK)
    __half* probes_own = nullptr;  // copy of the caller's probes (8 KB per expert)
    __half* st16 = nullptr;      // FP16: one stat per row (row order == fast-path bucket order)
    float* st32 = nullptr;       // Q4
    float* hint = nullptr;       // [n_experts] last cutoff seen (bucket_mul_v4's L2 prefetch hint); +inf = none yet
    size_t owned = 0;
    int layout = kInputMajor;
    int device = 0;
    const uint16_t* fast_bk() const { return bk_own ? bk_own : buckets; }
};

struct effort_ctx {
    int device = 0;
    int n_sms = 0;               // multiProcessorCount of `device`
    // scratch
    float* cutoff = nullptr;     // [kMaxBatch]
    int* loops = nullptr;        // [1]
    uint32_t* sizes = nullptr;   // [0]=n_selected [1]=padded [2]=prev  [3]=fused n_selected (+kMaxBatch)
    float2* dispatch = nullptr;  // maxDispatchSize entries
    size_t dispatch_cap = 0;
    uint32_t* chunk_counts = nullptr;
    size_t chunk_cap = 0;
    float* partial = nullptr;
    size_t partial_cap = 0;  // floats
    uint32_t* sel_counts = nullptr;
    size_t sel_cap = 0;
    bool have_dispatch = false;
    int dispatch_kind = 0;
    unsigned long long* trace = nullptr;  // [n_sms][16] when EFFORT_TRACE=1
    // round-2 fused kernel (bucket_mul_v2.cuh)
    unsigned* v2_sync = nullptr;          // [kMaxBatch][kV2MaxSlices][2] arrive/depart counters (overwrite protocol)
    unsigned* v2_err = nullptr;           // [1] set by a kernel whose overwrite barrier timed out
    float4* v4_part = nullptr;            // [n_sms][kV2Threads] bucket_mul_v4 epilogue partial sums
    unsigned* v4_sync = nullptr;          // [kMaxBatch][kV2MaxSlices][2] bucket_mul_v4 partial-sum exchange counters
    int cutoff_mode = 0;                  // EFFORT_CUTOFF_SELECT / EFFORT_CUTOFF_BISECT
    int stage_mode = 4;                   // 4 = consumer/producer warp pairs fed by bulk copies (slice-major FP16 weights; default), 3 = the pairs with 16-byte cp.async
                                          // 2 = one TMA producer warp + byte ring (slice-major FP16 weights; measured slower)
                                          // 0 = per-warp cp.async rings, units of <= 4 rows (any layout, Q4)
    int engine = 2;                       // 2 = bucket_mul_v2_kernel, 1 = round-1 fused kernel + integrate
    int prefetch = 0;                     // bucket_mul_v4: speculative L2 prefetch of the rows the previous cutoff selects
                                          // (measured: no gain at effort 0.25, -13 % at 1.0: the gather is not DRAM-latency bound)
    int use_hint = 1;                     // bucket_mul_v4: the select starts from the matrix's previous cutoff
    int dynamic = 0;                      // v2 per-warp rings: units from a shared counter (1) or static round robin (0, measured faster)
    int last_rs[8] = {0};                 // row splits of the last v2 launch per batch slot (effort_last_selected)
    int last_slots = 0;                   // batch slots 0 .. last_slots-1 hold results of the last v2 launch group
    bool last_was_v2 = false;
    void* comm = nullptr;                  // ncclComm_t
    int comm_rank = 0, comm_world = 1;
    unsigned char* p2p_local = nullptr;    // this rank's symmetric buffer
    void* p2p_peer[16] = {nullptr};        // mapped peers (own entry = p2p_local)
    bool p2p_ready = false;
    // multi-token GEMV hook (effort_bucket_mul_multi); the model owns its own prefill scratch
    float* pf_part = nullptr;
    size_t pf_part_cap = 0;
    uint32_t* pf_cnt = nullptr;
    size_t pf_cnt_cap = 0;
    float* pf_cut = nullptr;              // [kPrefillMax]
};

static constexpr int kMaxBatch = 8;
static constexpr int kV2MaxSlices = 64;

static bool default_slice_major();

extern "C" int effort_version(void) { return EFFORT_B200_VERSION; }
extern "C" const char* effort_last_cuda_error(void) { return g_cuda_err.c_str(); }
extern "C" uint64_t effort_launch_count(void) { return g_launches.load(); }

extern "C" const char* effort_strerror(int code) {
    switch (code) {
        case EFFORT_OK: return "ok";
        case EFFORT_EINVAL: return "invalid argument / reference precondition failed";
        case EFFORT_ECUDA: return "CUDA runtime error";
        case EFFORT_ENOMEM: return "out of memory";
        case EFFORT_ESHAPE: return "shape not supported by the kernels";
        case EFFORT_ESTATE: return "call sequence error";
        case EFFORT_ENOTLOADED: return "buckets not loaded and no dense core";
        default: return "unknown error";
    }
}

// ---------------------------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------------------------
extern "C" int effort_ctx_create(int device, effort_ctx_t** ctx_out) {
    if (!ctx_out) return EFFORT_EINVAL;
    *ctx_out = nullptr;
    int dev = device;
    if (dev < 0) CK(cudaGetDevice(&dev));
    else CK(cudaSetDevice(dev));
    effort_ctx* c = new (std::nothrow) effort_ctx();
    if (!c) return EFFORT_ENOMEM;
    c->device = dev;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, dev));
    c->n_sms = prop.multiProcessorCount;
    CK(cudaMalloc(&c->cutoff, sizeof(float) * kMaxBatch));
    CK(cudaMalloc(&c->loops, sizeof(int)));
    CK(cudaMalloc(&c->sizes, sizeof(uint32_t) * (4 + kMaxBatch)));
    CK(cudaMemset(c->sizes, 0, sizeof(uint32_t) * (4 + kMaxBatch)));
    CK(cudaMemset(c->cutoff, 0, sizeof(float) * kMaxBatch));
    CK(cudaMemset(c->loops, 0, sizeof(int)));
    CK(cudaMalloc(&c->v2_sync, sizeof(unsigned) * kMaxBatch * kV2MaxSlices * 2));
    CK(cudaMemset(c->v2_sync, 0, sizeof(unsigned) * kMaxBatch * kV2MaxSlices * 2));
    CK(cudaMalloc(&c->v4_part, sizeof(float4) * kV2Threads * c->n_sms));
    CK(cudaMalloc(&c->v4_sync, sizeof(unsigned) * kMaxBatch * kV2MaxSlices * 2));
    CK(cudaMemset(c->v4_sync, 0, sizeof(unsigned) * kMaxBatch * kV2MaxSlices * 2));
    CK(cudaMalloc(&c->v2_err, sizeof(unsigned)));
    CK(cudaMemset(c->v2_err, 0, sizeof(unsigned)));
    CK(cudaMalloc(&c->sel_counts, sizeof(uint32_t) * kMaxBatch * c->n_sms));  // fixed size: graphs keep the pointer
    CK(cudaMemset(c->sel_counts, 0, sizeof(uint32_t) * kMaxBatch * c->n_sms));
    c->sel_cap = (size_t)kMaxBatch * c->n_sms;
    { const char* e = getenv("EFFORT_CUTOFF"); if (e && !strcmp(e, "bisect")) c->cutoff_mode = 1; }
    { const char* e = getenv("EFFORT_STAGE"); if (e) c->stage_mode = !strcmp(e, "ldgsts") ? 0 : !strcmp(e, "tma") ? 2 : !strcmp(e, "pairs-ldgsts") ? 3 : 4; }
    { const char* e = getenv("EFFORT_ENGINE"); if (e && atoi(e) == 1) c->engine = 1; }
    { const char* e = getenv("EFFORT_DYN"); if (e) c->dynamic = atoi(e) ? 1 : 0; }
    { const char* e = getenv("EFFORT_PREFETCH"); if (e) c->prefetch = atoi(e) ? 1 : 0; }
    { const char* e = getenv("EFFORT_HINT"); if (e) c->use_hint = atoi(e) ? 1 : 0; }
    if (getenv("EFFORT_TRACE")) {
        CK(cudaMalloc(&c->trace, sizeof(unsigned long long) * (16 * c->n_sms + 648 + 48 + 16)));
        CK(cudaMemset(c->trace, 0, sizeof(unsigned long long) * (16 * c->n_sms + 648 + 48 + 16)));
    }
    *ctx_out = c;
    return EFFORT_OK;
}

extern "C" int effort_ctx_set_cutoff_mode(effort_ctx_t* c, int mode) {
    if (!c || (mode != EFFORT_CUTOFF_SELECT && mode != EFFORT_CUTOFF_BISECT)) return EFFORT_EINVAL;
    c->cutoff_mode = mode;
    return EFFORT_OK;
}

extern "C" int effort_ctx_set_option(effort_ctx_t* c, const char* name, int value) {
    if (!c || !name) return EFFORT_EINVAL;
    if (!strcmp(name, "engine")) { if (value != 1 && value != 2) return EFFORT_EINVAL; c->engine = value; return EFFORT_OK; }
    if (!strcmp(name, "stage")) { if (value != 0 && value != 2 && value != 3 && value != 4) return EFFORT_EINVAL; c->stage_mode = value; return EFFORT_OK; }
    if (!strcmp(name, "hint")) { if (value != 0 && value != 1) return EFFORT_EINVAL; c->use_hint = value; return EFFORT_OK; }
    if (!strcmp(name, "prefetch")) { if (value != 0 && value != 1) return EFFORT_EINVAL; c->prefetch = value; return EFFORT_OK; }
    if (!strcmp(name, "dynamic")) { if (value != 0 && value != 1) return EFFORT_EINVAL; c->dynamic = value; return EFFORT_OK; }
    return EFFORT_EINVAL;
}

extern "C" int effort_ctx_error_flag(effort_ctx_t* c, unsigned* flag_out, void* stream) {
    if (!c || !flag_out) return EFFORT_EINVAL;
    CK(cudaStreamSynchronize((cudaStream_t)stream));
    CK(cudaMemcpy(flag_out, c->v2_err, sizeof(unsigned), cudaMemcpyDeviceToHost));
    return EFFORT_OK;
}

// debugging aid (not part of the public header): copies the [n_sms][8] phase timestamps of the last fused
// launch; returns the number of CTAs rows or <0.
extern "C" int effort_debug_read_unit_trace(effort_ctx_t* c, unsigned long long* host648) {
    if (!c || !c->trace || !host648) return EFFORT_EINVAL;
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(host648, c->trace + 16 * c->n_sms, sizeof(unsigned long long) * (648 + 48 + 16), cudaMemcpyDeviceToHost));
    CK(cudaMemset(c->trace + 16 * c->n_sms, 0, sizeof(unsigned long long) * (648 + 48 + 16)));
    return EFFORT_OK;
}

extern "C" int effort_debug_read_trace(effort_ctx_t* c, unsigned long long* host, int max_rows) {
    if (!c || !c->trace || !host) return EFFORT_EINVAL;
    CK(cudaDeviceSynchronize());
    int n = c->n_sms < max_rows ? c->n_sms : max_rows;
    CK(cudaMemcpy(host, c->trace, sizeof(unsigned long long) * 16 * n, cudaMemcpyDeviceToHost));
    return n;
}

extern "C" int effort_ctx_destroy(effort_ctx_t* c) {
    if (!c) return EFFORT_OK;
    cudaFree(c->cutoff); cudaFree(c->loops); cudaFree(c->sizes); cudaFree(c->dispatch);
    cudaFree(c->chunk_counts); cudaFree(c->partial); cudaFree(c->sel_counts);
    cudaFree(c->trace); cudaFree(c->v2_sync); cudaFree(c->v2_err); cudaFree(c->v4_part); cudaFree(c->v4_sync);
    cudaFree(c->pf_part); cudaFree(c->pf_cnt); cudaFree(c->pf_cut);
    for (int p = 0; p < 16; p++)
        if (c->p2p_peer[p] && c->p2p_peer[p] != (void*)c->p2p_local) cudaIpcCloseMemHandle(c->p2p_peer[p]);
    cudaFree(c->p2p_local);
    effort_comm_destroy(c);
    delete c;
    return EFFORT_OK;
}

// Launch with the programmatic-dependent-launch attribute (all kernels of the decode chain call pdl_wait()
// before touching dependent data).  EFFORT_PDL=0 disables it (plain stream order).
static bool pdl_enabled() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("EFFORT_PDL"); v = (e && atoi(e) == 0) ? 0 : 1; }
    return v == 1;
}
extern "C" int effort_pdl_enabled(void) { return pdl_enabled() ? 1 : 0; }
template <typename... KArgs, typename... Args>
static cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                              Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    cfg.attrs = at; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

template <typename T>
static int ensure(T*& p, size_t& cap, size_t need) {
    if (need <= cap) return EFFORT_OK;
    if (p) CK(cudaFree(p));
    p = nullptr; cap = 0;
    CK(cudaMalloc(&p, need * sizeof(T)));
    cap = need;
    return EFFORT_OK;
}

// ---------------------------------------------------------------------------------------------------
// weights
// ---------------------------------------------------------------------------------------------------
extern "C" int effort_weights_create(const void* buckets_dev, const void* stats_dev, const void* probes_dev,
                                     const void* outliers_dev, int n_outliers, const void* core_dev,
                                     int in_dim, int out_dim, int n_experts, int percent_load, int kind,
                                     unsigned flags, void* stream_, effort_weights_t** w_out) {
    if (!w_out) return EFFORT_EINVAL;
    *w_out = nullptr;
    cudaStream_t stream = (cudaStream_t)stream_;
    if (in_dim <= 0 || out_dim <= 0 || n_experts <= 0) return EFFORT_EINVAL;
    if (kind != EFFORT_KIND_FP16 && kind != EFFORT_KIND_Q4) return EFFORT_EINVAL;
    const int bsize = kind == EFFORT_KIND_FP16 ? 16 : 8;
    if (percent_load <= 0 || percent_load > bsize) return EFFORT_EINVAL;
    if (!buckets_dev && !core_dev) return EFFORT_ENOTLOADED;
    if (buckets_dev && (!stats_dev || !probes_dev)) return EFFORT_EINVAL;
    const int words_div = kind == EFFORT_KIND_FP16 ? 16 : 32;
    if (out_dim % words_div) return EFFORT_ESHAPE;
    effort_weights* w = new (std::nothrow) effort_weights();
    if (!w) return EFFORT_ENOMEM;
    CK(cudaGetDevice(&w->device));
    w->in = in_dim; w->out = out_dim; w->n_experts = n_experts; w->P = percent_load; w->kind = kind;
    w->flags = flags; w->C = out_dim / words_div;
    w->buckets = (const uint16_t*)buckets_dev; w->stats = stats_dev; w->probes = (const __half*)probes_dev;
    w->outliers = (const float4*)outliers_dev; w->n_outliers = outliers_dev ? n_outliers : 0;
    w->core = (const __half*)core_dev;
    if (buckets_dev) {
        // numBuckets % 4 == 0 is asserted by the reference (bucketMul.swift:76); the kernels need the
        // row to be a whole number of 8-byte (FP16) / 4-byte (Q4) vectors.
        if (kind == EFFORT_KIND_FP16 && (w->C % 4)) { delete w; return EFFORT_ESHAPE; }
        if (kind == EFFORT_KIND_Q4 && (w->C % 2)) { delete w; return EFFORT_ESHAPE; }
        const size_t rows = (size_t)n_experts * in_dim * percent_load;
        if (rows * (size_t)w->C >= (size_t)1 << 32) { delete w; return EFFORT_ESHAPE; }
        const int TB = 256;
        CK(cudaMalloc(&w->probes_own, (size_t)n_experts * EFFORT_PROBES_COUNT * sizeof(__half)));
        CK(cudaMemcpyAsync(w->probes_own, probes_dev, (size_t)n_experts * EFFORT_PROBES_COUNT * sizeof(__half),
                           cudaMemcpyDeviceToDevice, stream));
        w->probes = w->probes_own;
        w->owned += (size_t)n_experts * EFFORT_PROBES_COUNT * sizeof(__half);
        {
            std::vector<float> inf((size_t)n_experts, __builtin_inff());
            CK(cudaMalloc(&w->hint, sizeof(float) * n_experts));
            CK(cudaMemcpyAsync(w->hint, inf.data(), sizeof(float) * n_experts, cudaMemcpyHostToDevice, stream));
            CK(cudaStreamSynchronize(stream));  // `inf` leaves scope
        }
        if (kind == EFFORT_KIND_FP16) {
            const bool repack = !(flags & EFFORT_WEIGHTS_NO_REPACK);
            const bool slice_major = repack && !(flags & EFFORT_WEIGHTS_INPUT_MAJOR) &&
                                     ((flags & EFFORT_WEIGHTS_SLICE_MAJOR) || default_slice_major()) && (w->C % 8) == 0;
            w->layout = repack ? (slice_major ? kSliceMajor : kInputMajor) : kRankMajor;
            CK(cudaMalloc(&w->st16, rows * sizeof(__half)));
            w->owned += rows * sizeof(__half);
            repack_stats_fp16_kernel<<<(unsigned)((rows + TB - 1) / TB), TB, 0, stream>>>(
                (const __half*)stats_dev, n_experts, in_dim, percent_load, repack ? 1 : 0, w->st16);
            LAUNCHED();
            if (repack) {
                CK(cudaMalloc(&w->bk_own, rows * (size_t)w->C * 2));
                w->owned += rows * (size_t)w->C * 2;
                if (slice_major) {
                    const size_t pieces = rows * (size_t)(w->C / 8);
                    const int W = w->C < 128 ? w->C : 128;
                    repack_slices_kernel<<<(unsigned)((pieces + TB - 1) / TB), TB, 0, stream>>>(
                        w->buckets, n_experts, in_dim, percent_load, w->C, W, 1, w->bk_own);
                } else {
                    repack_rows_kernel<<<(unsigned)((rows * 32 + TB - 1) / TB), TB, 0, stream>>>(
                        w->buckets, n_experts, in_dim, percent_load, w->C, w->bk_own);
                }
                LAUNCHED();
            }
        } else {
            w->layout = kInputMajor;  // Q4 rows are already inIdx*8 + rank (q4_draft.py:150-168)
            CK(cudaMalloc(&w->st32, rows * sizeof(float)));
            w->owned += rows * sizeof(float);
            repack_stats_q4_kernel<<<(unsigned)((rows + TB - 1) / TB), TB, 0, stream>>>(
                (const float*)stats_dev, rows, w->st32);
            LAUNCHED();
        }
    }
    *w_out = w;
    return EFFORT_OK;
}

extern "C" int effort_weights_destroy(effort_weights_t* w) {
    if (!w) return EFFORT_OK;
    cudaFree(w->bk_own); cudaFree(w->st16); cudaFree(w->st32); cudaFree(w->probes_own); cudaFree(w->hint);
    delete w;
    return EFFORT_OK;
}
extern "C" size_t effort_weights_owned_bytes(const effort_weights_t* w) { return w ? w->owned : 0; }
extern "C" float* effort_weights_hint(const effort_weights_t* w) { return w ? w->hint : nullptr; }

// ---------------------------------------------------------------------------------------------------
// helpers
// ---------------------------------------------------------------------------------------------------
static inline int effort_q(double effort, int n_probes) {
    // let q = Int(Double(probesCount-1)*(1-effort))   bucketMul.swift:39
    double x = (double)(n_probes - 1) * (1.0 - effort);
    return (int)x;
}

static bool default_slice_major() {  // the device copy is slice-major unless EFFORT_LAYOUT=input (round-1 engine: input-major only)
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("EFFORT_LAYOUT");
        const char* g = getenv("EFFORT_ENGINE");
        v = ((e && !strcmp(e, "input")) || (g && atoi(g) == 1)) ? 0 : 1;
    }
    return v == 1;
}

static int check_mul_args(const effort_ctx* ctx, const float* v, const effort_weights* w, const float* out,
                          double effort) {
    if (!ctx || !v || !w || !out) return EFFORT_EINVAL;
    if (!(effort >= 0.0 && effort <= 1.0)) return EFFORT_EINVAL;
    return EFFORT_OK;
}

static constexpr size_t kMaxSmem = 227 * 1024;
static bool ring_enabled() {  // EFFORT_RING=1: cp.async ring instead of the register-buffered streaming loop (measured slower)
    static int v = -1;
    if (v < 0) { const char* e = getenv("EFFORT_RING"); v = (e && atoi(e) == 1) ? 1 : 0; }
    return v == 1;
}


struct MulCall {  // one problem of a launch group, host side
    MulProblem pb;
    float* out;
    int mode;       // IntegrateMode of the group's integrate launch
    float* sumsq;   // kIntResidual: per-block partial sums of squares of the updated residual stream
    uint32_t* n_selected_dev;
};

// One launch group: [fused select+MAC kernel over all problems] -> [integrate over all problems].
// CTAs are dealt to the problems in proportion to their bucket bytes.
template <int SLOTS, int VEC, int U, int NW>
static int launch_fused_batch(MulCall* calls, int n, int n_cta, cudaStream_t stream) {
    if (n < 1 || n > kMulBatchMax) return EFFORT_EINVAL;
    MulBatch batch{};
    IntegrateBatch ib{};
    batch.n = n; ib.n = n;
    { static int d = -1; if (d < 0) { const char* e = getenv("EFFORT_DELAY_NS"); d = e ? atoi(e) : 0; } batch.delay_ns = d; }
    double total_bytes = 0;
    int cs_sum = 0;
    for (int k = 0; k < n; k++) {
        total_bytes += (double)calls[k].pb.in * calls[k].pb.C;
        cs_sum += make_geom<VEC>(calls[k].pb.C, n_cta).CS;
    }
    if (cs_sum > n_cta) return EFFORT_ESHAPE;
    int list_cap = 0, cta = 0, max_words = 0;
    constexpr int TF = SLOTS * 32 * VEC;
    for (int k = 0; k < n; k++) {
        MulProblem& pb = calls[k].pb;
        MulGeom g = make_geom<VEC>(pb.C, n_cta);
        const double share = (double)pb.in * pb.C / total_bytes;
        int rs = (int)((n_cta - (cs_sum - g.CS)) * share / g.CS);  // leave at least one row split to the others
        if (n == 1) rs = n_cta / g.CS;
        if (rs < 1) rs = 1;
        g.RS = rs;
        pb.g = g;
        const int per_cta = (pb.in + g.RS - 1) / g.RS;
        const int cap = ((per_cta < NW * 32 ? per_cta : NW * 32) * pb.P + 3) & ~3;  // entries added per scan round
        const int full = ((per_cta * pb.P) + 3) & ~3;
        list_cap = full > list_cap ? full : list_cap;
        (void)cap;
        batch.cta_begin[k] = cta;
        cta += g.CS * g.RS;
        batch.p[k] = pb;
        ib.it[k] = IntegrateItem{pb.partial, calls[k].out, pb.sel_counts, calls[k].n_selected_dev, g, pb.C,
                                 calls[k].mode, calls[k].sumsq};
        max_words = g.CS * TF > max_words ? g.CS * TF : max_words;
    }
    if (cta > n_cta) return EFFORT_ESHAPE;
    batch.cta_begin[n] = cta;
    for (int k = 0; k < n; k++) batch.p[k].list_cap = list_cap;
    const size_t smem = MulSmem<SLOTS, VEC, NW>::bytes(list_cap);
    if (smem > kMaxSmem) return EFFORT_ESHAPE;
    static size_t configured = 0;
    {
        bool norm = batch.p[0].norm_w != nullptr;
        for (int k = 1; k < n; k++)
            if ((batch.p[k].norm_w != nullptr) != norm) return EFFORT_EINVAL;  // a group is all-norm or all-plain
        // cp.async ring (16 row slices in flight per warp) when the selection list leaves room for it
        constexpr int kRing = 16;
        const size_t smem_ring = MulSmem<SLOTS, VEC, NW>::bytes(list_cap, kRing);
        const bool ring = ring_enabled() && smem_ring <= kMaxSmem;
        static size_t configured_ring = 0;
        if (ring) {
            if (smem_ring > configured_ring) {
                CK(cudaFuncSetAttribute(bucket_mul_fused_kernel<SLOTS, VEC, U, NW, false, kRing>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_ring));
                CK(cudaFuncSetAttribute(bucket_mul_fused_kernel<SLOTS, VEC, U, NW, true, kRing>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_ring));
                configured_ring = smem_ring;
            }
            if (norm) CK(launch_pdl(bucket_mul_fused_kernel<SLOTS, VEC, U, NW, true, kRing>, dim3(cta), dim3(NW * 32), smem_ring, stream, batch));
            else CK(launch_pdl(bucket_mul_fused_kernel<SLOTS, VEC, U, NW, false, kRing>, dim3(cta), dim3(NW * 32), smem_ring, stream, batch));
        } else {
            if (smem > configured) {
                CK(cudaFuncSetAttribute(bucket_mul_fused_kernel<SLOTS, VEC, U, NW, false, 0>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                CK(cudaFuncSetAttribute(bucket_mul_fused_kernel<SLOTS, VEC, U, NW, true, 0>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                configured = smem;
            }
            if (norm) CK(launch_pdl(bucket_mul_fused_kernel<SLOTS, VEC, U, NW, true, 0>, dim3(cta), dim3(NW * 32), smem, stream, batch));
            else CK(launch_pdl(bucket_mul_fused_kernel<SLOTS, VEC, U, NW, false, 0>, dim3(cta), dim3(NW * 32), smem, stream, batch));
        }
    }
    LAUNCHED();
    CK(launch_pdl(integrate_kernel<SLOTS, VEC>, dim3((max_words + 31) / 32, n), dim3(256), 0, stream, ib));
    LAUNCHED();
    return EFFORT_OK;
}


// ---------------------------------------------------------------------------------------------------
// round-2 engine: bucket_mul_v2_kernel (one launch per group, no integrate)
// ---------------------------------------------------------------------------------------------------
struct V2Call {  // one problem of a launch group, host side
    const float* v = nullptr;       // input / residual stream (norm_w != null) / x1 (v2 != null)
    const float* v2 = nullptr;      // x3 -> input = silu(x1) * x3
    const float* v_cut = nullptr;   // row shards: first 4096 entries of the full input
    const __half* norm_w = nullptr; // input = rmsNorm(v) * norm_w
    float norm_eps = 1e-5f;
    const effort_weights* w = nullptr;
    const uint32_t* exp_no = nullptr;
    const float* out_scale = nullptr;  // device scalar: out (+)= scale * (W v)
    float* out = nullptr;
    double effort = 0.25;
    int out_mode = kOutOverwrite;
};

static bool v2_supported(const effort_weights* w) {
    if (!w->buckets && !w->bk_own) return false;
    if (w->layout == kSliceMajor && w->kind != EFFORT_KIND_FP16) return false;
    if (w->n_probes != EFFORT_PROBES_MAX) return false;
    if (w->kind == EFFORT_KIND_FP16) return (w->C % 8) == 0 && w->P <= 16;
    return (w->C % 8) == 0 && w->P <= 8;
}

template <int SLOTS, int VEC>
static int launch_v2_batch(effort_ctx* ctx, const V2Call* calls, int n, int slot0, cudaStream_t stream) {
    if (n < 1 || n > kMulBatchMax) return EFFORT_EINVAL;
    constexpr int D = 4;
    // at most one CTA per SM (every variant needs most of the SM's shared memory), so all CTAs of a launch are resident
    // at once: the in-kernel waits between the CTAs of a column slice rely on it (overwrite zeroing; bucket_mul_v4's
    // partial-sum exchange)
    const int n_cta = ctx->n_sms;
    V2Batch batch{};
    batch.n = n;
    double total_bytes = 0;
    int cs_sum = 0;
    for (int k = 0; k < n; k++) {
        const effort_weights* w = calls[k].w;
        total_bytes += (double)w->in * w->C;
        cs_sum += make_geom<VEC>(w->C, n_cta).CS;
    }
    if (cs_sum > n_cta) return EFFORT_ESHAPE;
    int cta = 0, list_cap = 0;
    for (int k = 0; k < n; k++) {
        const V2Call& c = calls[k];
        const effort_weights* w = c.w;
        MulGeom g = make_geom<VEC>(w->C, n_cta);
        if (g.CS > kV2MaxSlices) return EFFORT_ESHAPE;
        const double share = (double)w->in * w->C / total_bytes;
        int rs = (int)((n_cta - (cs_sum - g.CS)) * share / g.CS);
        if (n == 1) rs = n_cta / g.CS;
        if (rs < 1) rs = 1;
        if (rs > w->in) rs = w->in;
        V2Problem& pb = batch.p[k];
        const bool norm = c.norm_w != nullptr, silu = c.v2 != nullptr;
        if (norm && silu) return EFFORT_EINVAL;
        if ((norm || silu) && c.v_cut) return EFFORT_EINVAL;        // glue-on-load needs the whole input locally
        if (norm && w->in != 8 * kV2Threads) return EFFORT_ESHAPE;   // the fused rmsNorm sums exactly 4096 entries
        if (!c.v_cut && w->in < EFFORT_PROBES_MAX) return EFFORT_ESHAPE;
        pb.v = c.v; pb.v2 = c.v2; pb.v_cut = c.v_cut ? c.v_cut : c.v; pb.norm_w = c.norm_w; pb.norm_eps = c.norm_eps;
        pb.st16 = w->st16; pb.st32 = w->st32; pb.bk = w->fast_bk(); pb.probes = w->probes; pb.exp_no = c.exp_no;
        pb.out = c.out; pb.out_scale = c.out_scale;
        pb.sync = ctx->v2_sync + (size_t)(slot0 + k) * kV2MaxSlices * 2;
        pb.red_sync = ctx->v4_sync + (size_t)(slot0 + k) * kV2MaxSlices * 2;
        pb.red_part = ctx->v4_part;
        pb.sel_counts = ctx->sel_counts + (size_t)(slot0 + k) * ctx->n_sms;
        pb.cutoff_out = ctx->cutoff + slot0 + k;
        pb.cutoff_hint = ctx->use_hint ? w->hint : nullptr;
        pb.rounds_out = (slot0 + k == 0) ? ctx->loops : nullptr;
        pb.err_flag = ctx->v2_err;
        pb.trace = ctx->trace;
        pb.unit_trace = ctx->trace ? ctx->trace + 16 * ctx->n_sms : nullptr;
        pb.in = w->in; pb.C = w->C; pb.P = w->P; pb.q = effort_q(c.effort, w->n_probes); pb.layout = w->layout;
        pb.out_mode = c.out_mode;
        pb.CS = g.CS; pb.RS = rs; pb.W = (g.CS == 1) ? w->C : 32 * VEC; pb.R = g.R; pb.lpr = g.lpr;
        const int per_cta = (w->in + rs - 1) / rs;
        const int cap = (per_cta < kV2MaxInputs ? per_cta : kV2MaxInputs) * V2Smem<SLOTS, VEC>::kUnitsPerInput;
        list_cap = cap > list_cap ? cap : list_cap;
        batch.cta_begin[k] = cta;
        cta += g.CS * rs;
        ctx->last_rs[slot0 + k] = rs;
    }
    if (cta > n_cta) return EFFORT_ESHAPE;
    batch.cta_begin[n] = cta;
    batch.list_cap = (list_cap + 63) & ~63;
    using L = V2Smem<SLOTS, VEC>;
    batch.dynamic = ctx->dynamic;
    batch.prefetch = ctx->prefetch;
    { static const int tc = [] { const char* e = getenv("EFFORT_TRACE"); return e && atoi(e) == 2 ? 1 : 0; }(); batch.trace_cycles = tc; }
    const size_t smem = L::bytes(batch.list_cap, D);
    if (smem > kMaxSmem) return EFFORT_ESHAPE;
    // every kernel needs its own opt-in to > 48 KB of dynamic shared memory (per device): keyed by the function pointer
    // (all instantiations share ONE pointer type, so a static inside a generic lambda would be shared between them)
    auto go = [&](void (*kernel)(const V2Batch), int threads, size_t smem_bytes) -> int {
        static std::map<std::pair<int, const void*>, bool> configured;
        const auto key = std::make_pair(ctx->device, (const void*)kernel);
        if (!configured.count(key)) {
            cudaFuncAttributes fa{};
            CK(cudaFuncGetAttributes(&fa, kernel));  // static shared memory counts against the same 227 KB
            CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kMaxSmem - fa.sharedSizeBytes)));
            configured[key] = true;
        }
        CK(launch_pdl(kernel, dim3(cta), dim3(threads), smem_bytes, stream, batch));
        return EFFORT_OK;
    };
    int rc;
    const bool bisect = ctx->cutoff_mode == 1;
    bool all_slice = true;
    for (int k = 0; k < n; k++) all_slice = all_slice && calls[k].w->layout == kSliceMajor;
    if (SLOTS == 16 && all_slice && ctx->stage_mode == 3) {
        // consumer / producer warp pairs with private rings (bucket_mul_v4.cuh), 16-byte cp.async per lane: the default path
        rc = bisect ? go(bucket_mul_v4_kernel<kCutBisect, false>, kV2Threads, V4Smem::kBytes)
                    : go(bucket_mul_v4_kernel<kCutSelect, false>, kV2Threads, V4Smem::kBytes);
    } else if (SLOTS == 16 && all_slice && ctx->stage_mode == 4) {
        // the same pairs, one bulk copy (TMA) per unit
        rc = bisect ? go(bucket_mul_v4_kernel<kCutBisect, true>, kV2Threads, V4Smem::kBytes)
                    : go(bucket_mul_v4_kernel<kCutSelect, true>, kV2Threads, V4Smem::kBytes);
    } else if (SLOTS == 16 && all_slice && ctx->stage_mode == 2) {
        // TMA pipeline: producer warp + byte ring (bucket_mul_v3.cuh)
        batch.ring_bytes = (int)((kMaxSmem - V3Smem::kFixed) & ~(size_t)255);
        if (batch.ring_bytes < 2 * (kV3BatchBytes + 4096)) return EFFORT_ESHAPE;
        const size_t smem3 = V3Smem::kFixed + (size_t)batch.ring_bytes;
        rc = bisect ? go(bucket_mul_v3_kernel<kCutBisect>, kV3Threads, smem3) : go(bucket_mul_v3_kernel<kCutSelect>, kV3Threads, smem3);
    } else if (bisect) {
        rc = go(bucket_mul_v2_kernel<SLOTS, VEC, kCutBisect, D>, kV2Threads, smem);
    } else {
        rc = go(bucket_mul_v2_kernel<SLOTS, VEC, kCutSelect, D>, kV2Threads, smem);
    }
    if (rc) return rc;
    LAUNCHED();
    ctx->last_was_v2 = true;
    ctx->last_slots = slot0 + n;
    return EFFORT_OK;
}

static int launch_v2(effort_ctx* ctx, const V2Call* calls, int n, int slot0, cudaStream_t stream) {
    const int kind = calls[0].w->kind;
    for (int k = 1; k < n; k++)
        if (calls[k].w->kind != kind) return EFFORT_EINVAL;
    if (kind == EFFORT_KIND_FP16) return launch_v2_batch<16, 4>(ctx, calls, n, slot0, stream);
    return launch_v2_batch<32, 2>(ctx, calls, n, slot0, stream);
}

// floats of partial scratch one problem needs (upper bound over variants)
static size_t partial_floats(const effort_ctx* ctx, const effort_weights* w) {
    const int slots = w->kind == EFFORT_KIND_FP16 ? 16 : 32;
    return (size_t)ctx->n_sms * slots * 32 * 8;
}

static MulCall make_call(effort_ctx* ctx, const float* v, const effort_weights* w, const uint32_t* exp_no,
                         float* out, double effort, int accumulate, int slot, size_t partial_off,
                         const float* v_cut = nullptr) {
    MulCall c{};
    MulProblem& pb = c.pb;
    pb.v = v; pb.v_cut = v_cut ? v_cut : v; pb.st16 = w->st16; pb.st32 = w->st32; pb.bk = w->fast_bk(); pb.probes = w->probes;
    pb.exp_no = exp_no; pb.cutoff_in = nullptr;
    pb.partial = ctx->partial + partial_off;
    pb.sel_counts = ctx->sel_counts + (size_t)slot * ctx->n_sms;
    pb.cutoff_out = ctx->cutoff + slot;
    pb.in = w->in; pb.C = w->C; pb.P = w->P; pb.n_probes = w->n_probes;
    pb.q = effort_q(effort, w->n_probes);
    pb.layout = w->layout;
    pb.trace = ctx->trace;
    c.out = out; c.mode = accumulate ? kIntAccumulate : kIntStore; c.sumsq = nullptr;
    c.n_selected_dev = ctx->sizes + 3 + slot;
    return c;
}

static int launch_calls(effort_ctx* ctx, MulCall* calls, int n, int kind, bool all_c8, cudaStream_t stream) {
    (void)all_c8;  // a 16-byte-load variant (C % 8 == 0) was measured no faster than 8-byte loads and removed
    if (kind == EFFORT_KIND_FP16) return launch_fused_batch<16, 4, 8, 16>(calls, n, ctx->n_sms, stream);
    return launch_fused_batch<32, 2, 8, 16>(calls, n, ctx->n_sms, stream);
}

// Round-1 engine scratch (partial tiles): allocated ONCE at its maximum (kMaxBatch problems of the larger kind) so that
// captured CUDA graphs never see the pointer change (a later, larger call used to cudaFree it under them).
static int ensure_mul_scratch(effort_ctx* ctx, size_t, int) {
    if (ctx->partial) return EFFORT_OK;
    const size_t need = (size_t)kMaxBatch * ctx->n_sms * 32 * 32 * 8;
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    (void)st;
    return ensure(ctx->partial, ctx->partial_cap, need);
}

// One fused bucketMul.  slot = scratch slot inside a batch.
static int enqueue_bucket_mul(effort_ctx* ctx, const float* v, const effort_weights* w, const uint32_t* exp_no,
                              float* out, double effort, int accumulate, int slot, size_t partial_off,
                              cudaStream_t stream) {
    if (ctx->engine == 2 && v2_supported(w)) {
        V2Call c;
        c.v = v; c.w = w; c.exp_no = exp_no; c.out = out; c.effort = effort;
        c.out_mode = accumulate ? kOutAccumulate : kOutOverwrite;
        return launch_v2(ctx, &c, 1, slot, stream);
    }
    ctx->last_was_v2 = false;
    if (w->layout == kSliceMajor) return EFFORT_ESHAPE;  // the round-1 kernels read input-major / rank-major rows only
    int rc = ensure_mul_scratch(ctx, 0, kMaxBatch);
    if (rc) return rc;
    MulCall c = make_call(ctx, v, w, exp_no, out, effort, accumulate, slot, partial_off);
    return launch_calls(ctx, &c, 1, w->kind, (w->C % 8) == 0, stream);
}


// ---------------------------------------------------------------------------------------------------
// operator entry points
// ---------------------------------------------------------------------------------------------------
extern "C" int effort_bucket_mul(effort_ctx_t* ctx, const float* v_dev, const effort_weights_t* w,
                                 const uint32_t* exp_no_dev, float* out_dev, double effort, void* stream_) {
    int rc = check_mul_args(ctx, v_dev, w, out_dev, effort);
    if (rc) return rc;
    if (w->kind != EFFORT_KIND_FP16) return EFFORT_EINVAL;  // assert(!goQ8...) bucketMul.swift:72
    if (!w->buckets) return EFFORT_ENOTLOADED;
    return enqueue_bucket_mul(ctx, v_dev, w, exp_no_dev, out_dev, effort, 0, 0, 0, (cudaStream_t)stream_);
}

static int enqueue_outliers(const float* v, const effort_weights* w, float* out, cudaStream_t stream) {
    if (w->outliers && w->n_outliers > 0) {
        calc_outliers_kernel<<<(w->n_outliers + 255) / 256, 256, 0, stream>>>(v, w->outliers, w->n_outliers, out);
        LAUNCHED();
    }
    return EFFORT_OK;
}

extern "C" int effort_bucket_mul_q4(effort_ctx_t* ctx, const float* v_dev, const effort_weights_t* w,
                                    const uint32_t* exp_no_dev, float* out_dev, double effort, void* stream_) {
    int rc = check_mul_args(ctx, v_dev, w, out_dev, effort);
    if (rc) return rc;
    if (w->kind != EFFORT_KIND_Q4) return EFFORT_EINVAL;
    if (!w->buckets) return EFFORT_ENOTLOADED;
    // bucketMulQ4 accumulates into out (atomics, bucketMulQ4.metal:89), then calcOutliers (:61)
    rc = enqueue_bucket_mul(ctx, v_dev, w, exp_no_dev, out_dev, effort, 1, 0, 0, (cudaStream_t)stream_);
    if (rc) return rc;
    return enqueue_outliers(v_dev, w, out_dev, (cudaStream_t)stream_);
}

static int enqueue_basic_mul(const float* v, const __half* core, int out_dim, int in_dim, float* out,
                             int n_sms, cudaStream_t stream) {
    if (in_dim % 16) return EFFORT_EINVAL;  // assert(weights.cols % 16 == 0) mps.swift:18
    const size_t smem = (size_t)in_dim * sizeof(float);
    static size_t configured = 0;
    if (smem > 48 * 1024 && smem > configured) {
        CK(cudaFuncSetAttribute(basic_mul_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured = smem;
    }
    int grid = (out_dim + 7) / 8;
    const int max_grid = n_sms * 8;
    if (grid > max_grid) grid = max_grid;
    CK(launch_pdl(basic_mul_kernel, dim3(grid), dim3(256), smem, stream, v, core, out_dim, in_dim, out));
    LAUNCHED();
    return EFFORT_OK;
}

extern "C" int effort_basic_mul(effort_ctx_t* ctx, const float* v_dev, const void* core_dev, int out_dim,
                                int in_dim, float* out_dev, void* stream_) {
    if (!ctx || !v_dev || !core_dev || !out_dev || out_dim <= 0 || in_dim <= 0) return EFFORT_EINVAL;
    if ((size_t)in_dim * sizeof(float) > 200 * 1024) return EFFORT_ESHAPE;
    return enqueue_basic_mul(v_dev, (const __half*)core_dev, out_dim, in_dim, out_dev, ctx->n_sms,
                             (cudaStream_t)stream_);
}

static int expert_mul_one(effort_ctx* ctx, const effort_mul_args_t& a, int slot, size_t partial_off,
                          cudaStream_t stream) {
    const effort_weights* w = a.w;
    if (w->kind == EFFORT_KIND_Q4) {  // expertMul.swift:25-31
        if (w->buckets) {
            const bool v2 = ctx->engine == 2 && v2_supported(w);  // the v2 kernel zeroes `out` itself (overwrite mode)
            if (!v2) CK(cudaMemsetAsync(a.out_dev, 0, sizeof(float) * w->out, stream));  // out.zero()
            int rc = enqueue_bucket_mul(ctx, a.v_dev, w, a.exp_no_dev, a.out_dev, a.effort, v2 ? 0 : 1, slot, partial_off, stream);
            if (rc) return rc;
            return enqueue_outliers(a.v_dev, w, a.out_dev, stream);
        }
        if (!w->core) return EFFORT_ENOTLOADED;
        return enqueue_basic_mul(a.v_dev, w->core, w->out, w->in, a.out_dev, ctx->n_sms, stream);
    }
    if (!w->buckets) return EFFORT_ENOTLOADED;
    return enqueue_bucket_mul(ctx, a.v_dev, w, a.exp_no_dev, a.out_dev, a.effort, 0, slot, partial_off, stream);
}

extern "C" int effort_expert_mul_batch(effort_ctx_t* ctx, const effort_mul_args_t* args, int n, void* stream_) {
    if (!ctx || !args || n <= 0 || n > kMaxBatch) return EFFORT_EINVAL;
    cudaStream_t stream = (cudaStream_t)stream_;
    size_t total = 0;
    for (int k = 0; k < n; k++) {
        int rc = check_mul_args(ctx, args[k].v_dev, args[k].w, args[k].out_dev, args[k].effort);
        if (rc) return rc;
        total += partial_floats(ctx, args[k].w);
    }
    int rc = 0;
    if (ctx->engine == 2) {
        // FP16 problems with buckets loaded go into ONE launch of the v2 kernel (up to kMulBatchMax); everything else
        // (Q4: overwrite + outliers; dense fallback; shapes the v2 kernel does not take) is enqueued one by one in order.
        V2Call group[kMulBatchMax];
        int ng = 0, slot0 = 0;
        auto flush = [&]() -> int {
            if (!ng) return EFFORT_OK;
            int r = launch_v2(ctx, group, ng, slot0, stream);
            ng = 0;
            return r;
        };
        for (int k = 0; k < n; k++) {
            const effort_weights* w = args[k].w;
            if (w->kind == EFFORT_KIND_FP16 && w->buckets && v2_supported(w)) {
                if (ng == kMulBatchMax && (rc = flush())) return rc;
                if (ng == 0) slot0 = k;
                V2Call& c = group[ng++];
                c = V2Call{};
                c.v = args[k].v_dev; c.v_cut = args[k].v_cutoff_dev; c.w = w; c.exp_no = args[k].exp_no_dev;
                c.out = args[k].out_dev; c.effort = args[k].effort; c.out_mode = kOutOverwrite;
            } else {
                if ((rc = flush())) return rc;
                if ((rc = expert_mul_one(ctx, args[k], k, 0, stream))) return rc;
            }
        }
        return flush();
    }
    ctx->last_was_v2 = false;
    rc = ensure_mul_scratch(ctx, total, kMaxBatch);
    if (rc) return rc;
    // round-1 engine: FP16 problems with buckets loaded go into ONE launch group (up to kMulBatchMax); everything else
    // (Q4: out.zero() + outliers; dense fallback) is enqueued one by one in order.
    MulCall group[kMulBatchMax];
    int ng = 0;
    bool c8 = true;
    size_t off = 0;
    auto flush = [&]() -> int {
        if (!ng) return EFFORT_OK;
        int r = launch_calls(ctx, group, ng, EFFORT_KIND_FP16, c8, stream);
        ng = 0; c8 = true;
        return r;
    };
    for (int k = 0; k < n; k++) {
        const effort_weights* w = args[k].w;
        if (w->kind == EFFORT_KIND_FP16 && w->buckets) {
            if (w->layout == kSliceMajor) return EFFORT_ESHAPE;
            if (ng == kMulBatchMax && (rc = flush())) return rc;
            group[ng++] = make_call(ctx, args[k].v_dev, w, args[k].exp_no_dev, args[k].out_dev, args[k].effort, 0, k, off,
                                    args[k].v_cutoff_dev);
            c8 = c8 && (w->C % 8) == 0;
        } else {
            if ((rc = flush())) return rc;
            if ((rc = expert_mul_one(ctx, args[k], k, off, stream))) return rc;
        }
        off += partial_floats(ctx, w);
    }
    return flush();
}

extern "C" int effort_expert_mul(effort_ctx_t* ctx, const float* v_dev, const effort_weights_t* w,
                                 const uint32_t* exp_no_dev, float* out_dev, double effort, void* stream_) {
    effort_mul_args_t a{v_dev, w, exp_no_dev, out_dev, effort, nullptr};
    return effort_expert_mul_batch(ctx, &a, 1, stream_);
}

// ---------------------------------------------------------------------------------------------------
// test hooks
// ---------------------------------------------------------------------------------------------------
extern "C" int effort_find_cutoff(effort_ctx_t* ctx, const float* v_dev, const effort_weights_t* w,
                                  const uint32_t* exp_no_dev, double effort, void* stream_) {
    if (!ctx || !v_dev || !w || !w->probes) return EFFORT_EINVAL;
    if (!(effort >= 0.0 && effort <= 1.0)) return EFFORT_EINVAL;
    if (w->n_probes > kCutoffThreads * kCutoffMaxPerThread) return EFFORT_ESHAPE;
    find_cutoff_kernel<<<1, kCutoffThreads, 0, (cudaStream_t)stream_>>>(
        v_dev, w->probes, exp_no_dev, w->n_probes, effort_q(effort, w->n_probes), ctx->cutoff, ctx->loops);
    LAUNCHED();
    return EFFORT_OK;
}

extern "C" int effort_calc_dispatch(effort_ctx_t* ctx, const float* v_dev, const effort_weights_t* w,
                                    const uint32_t* exp_no_dev, double effort, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!ctx || !v_dev || !w) return EFFORT_EINVAL;
    if (!w->buckets) return EFFORT_ENOTLOADED;
    int rc = effort_find_cutoff(ctx, v_dev, w, exp_no_dev, effort, stream_);
    if (rc) return rc;
    const int expert_size = w->P * w->in;  // loader.swift:50
    // assert(dispatch.rows >= ew.buckets.rows*2) bucketMul.swift:35 -> grow instead
    rc = ensure(ctx->dispatch, ctx->dispatch_cap, (size_t)expert_size + 2048);
    if (rc) return rc;
    const int n_chunks = (expert_size + kDispChunk - 1) / kDispChunk;
    rc = ensure(ctx->chunk_counts, ctx->chunk_cap, (size_t)n_chunks);
    if (rc) return rc;
    if (w->kind == EFFORT_KIND_FP16) {
        dispatch_count_kernel<0><<<n_chunks, kDispChunk, 0, stream>>>(v_dev, w->stats, exp_no_dev, ctx->cutoff,
                                                                      w->in, expert_size, ctx->chunk_counts);
        LAUNCHED();
        dispatch_write_kernel<0><<<n_chunks, kDispChunk, 0, stream>>>(
            v_dev, w->stats, exp_no_dev, ctx->cutoff, w->in, w->C, expert_size, ctx->chunk_counts, n_chunks,
            ctx->dispatch, ctx->sizes + 0, ctx->sizes + 1, ctx->sizes + 2);
        LAUNCHED();
    } else {
        dispatch_count_kernel<1><<<n_chunks, kDispChunk, 0, stream>>>(v_dev, w->stats, exp_no_dev, ctx->cutoff,
                                                                      w->in, expert_size, ctx->chunk_counts);
        LAUNCHED();
        dispatch_write_kernel<1><<<n_chunks, kDispChunk, 0, stream>>>(
            v_dev, w->stats, exp_no_dev, ctx->cutoff, w->in, w->C, expert_size, ctx->chunk_counts, n_chunks,
            ctx->dispatch, ctx->sizes + 0, ctx->sizes + 1, ctx->sizes + 2);
        LAUNCHED();
    }
    ctx->have_dispatch = true;
    ctx->dispatch_kind = w->kind;
    return EFFORT_OK;
}

template <int SLOTS, int VEC, int U, int NW>
static int launch_dispatch_mac(effort_ctx* ctx, const effort_weights* w, float* out, cudaStream_t stream) {
    const MulGeom g = make_geom<VEC>(w->C, ctx->n_sms);
    const int list_cap = 2048;
    const size_t smem = MulSmem<SLOTS, VEC, NW>::bytes(list_cap);
    static size_t configured = 0;
    if (smem > configured) {
        CK(cudaFuncSetAttribute(bucket_mul_dispatch_kernel<SLOTS, VEC, U, NW>,
                                cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured = smem;
    }
    bucket_mul_dispatch_kernel<SLOTS, VEC, U, NW><<<g.CS * g.RS, NW * 32, smem, stream>>>(
        w->buckets, ctx->dispatch, ctx->sizes + 1, w->C, list_cap, g, ctx->partial);
    LAUNCHED();
    constexpr int TF = SLOTS * 32 * VEC;
    IntegrateBatch ib{};
    ib.n = 1;
    ib.it[0] = IntegrateItem{ctx->partial, out, nullptr, nullptr, g, w->C,
                             w->kind == EFFORT_KIND_Q4 ? kIntAccumulate : kIntStore, nullptr};
    integrate_kernel<SLOTS, VEC><<<dim3((g.CS * TF + 31) / 32, 1), 256, 0, stream>>>(ib);
    LAUNCHED();
    return EFFORT_OK;
}

extern "C" int effort_mul(effort_ctx_t* ctx, const effort_weights_t* w, float* out_dev, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!ctx || !w || !out_dev) return EFFORT_EINVAL;
    if (!ctx->have_dispatch || ctx->dispatch_kind != w->kind) return EFFORT_ESTATE;
    if (!w->buckets) return EFFORT_ENOTLOADED;
    int rc = ensure_mul_scratch(ctx, partial_floats(ctx, w), kMaxBatch);
    if (rc) return rc;
    if (w->kind == EFFORT_KIND_FP16) return launch_dispatch_mac<16, 4, 8, 16>(ctx, w, out_dev, stream);
    return launch_dispatch_mac<32, 2, 8, 16>(ctx, w, out_dev, stream);
}

extern "C" int effort_read_dispatch(effort_ctx_t* ctx, float* dispatch_host, size_t capacity,
                                    uint32_t* n_selected, uint32_t* padded_size, float* cutoff,
                                    int* cutoff_loops, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!ctx) return EFFORT_EINVAL;
    CK(cudaStreamSynchronize(stream));
    uint32_t sizes[3] = {0, 0, 0};
    CK(cudaMemcpy(sizes, ctx->sizes, sizeof(sizes), cudaMemcpyDeviceToHost));
    if (n_selected) *n_selected = sizes[0];
    if (padded_size) *padded_size = sizes[1];
    if (cutoff) CK(cudaMemcpy(cutoff, ctx->cutoff, sizeof(float), cudaMemcpyDeviceToHost));
    if (cutoff_loops) CK(cudaMemcpy(cutoff_loops, ctx->loops, sizeof(int), cudaMemcpyDeviceToHost));
    if (dispatch_host && ctx->have_dispatch) {
        size_t n = sizes[1] < capacity ? sizes[1] : capacity;
        if (n) CK(cudaMemcpy(dispatch_host, ctx->dispatch, n * sizeof(float2), cudaMemcpyDeviceToHost));
    }
    return EFFORT_OK;
}

extern "C" int effort_last_selected(effort_ctx_t* ctx, uint32_t* n_selected, void* stream_) {
    if (!ctx || !n_selected) return EFFORT_EINVAL;
    CK(cudaStreamSynchronize((cudaStream_t)stream_));
    if (ctx->last_was_v2) {  // v2 kernel: one count per row split of batch slot 0
        std::vector<uint32_t> c((size_t)ctx->last_rs[0]);
        CK(cudaMemcpy(c.data(), ctx->sel_counts, sizeof(uint32_t) * c.size(), cudaMemcpyDeviceToHost));
        uint32_t t = 0;
        for (uint32_t x : c) t += x;
        *n_selected = t;
        return EFFORT_OK;
    }
    CK(cudaMemcpy(n_selected, ctx->sizes + 3, sizeof(uint32_t), cudaMemcpyDeviceToHost));
    return EFFORT_OK;
}

extern "C" int effort_fused_mul_batch(effort_ctx_t* ctx, const effort_fused_args_t* a, int n, void* stream) {
    if (!ctx || !a || n < 1 || n > kMulBatchMax || ctx->engine != 2) return EFFORT_EINVAL;
    V2Call calls[kMulBatchMax];
    for (int k = 0; k < n; k++) {
        const effort_fused_args_t& x = a[k];
        int rc = check_mul_args(ctx, x.v_dev, x.w, x.out_dev, x.effort);
        if (rc) return rc;
        if (x.norm_w_dev && x.x3_dev) return EFFORT_EINVAL;
        if (x.w->kind != EFFORT_KIND_FP16 || !x.w->buckets || !v2_supported(x.w)) return EFFORT_ESHAPE;
        if (x.norm_w_dev && x.w->in != 8 * kV2Threads) return EFFORT_ESHAPE;
        V2Call& c = calls[k];
        c.v = x.v_dev; c.v2 = x.x3_dev; c.norm_w = (const __half*)x.norm_w_dev; c.norm_eps = x.norm_eps; c.w = x.w;
        c.exp_no = x.exp_no_dev; c.out_scale = x.out_scale_dev; c.out = x.out_dev; c.effort = x.effort;
        c.out_mode = x.accumulate ? kOutAccumulate : kOutOverwrite;
    }
    return launch_v2(ctx, calls, n, 0, (cudaStream_t)stream);
}

extern "C" int effort_last_problem(effort_ctx_t* ctx, int slot, float* cutoff, uint32_t* n_selected, void* stream) {
    if (!ctx || slot < 0 || slot >= kMaxBatch) return EFFORT_EINVAL;
    if (!ctx->last_was_v2 || slot >= ctx->last_slots) return EFFORT_ESTATE;
    CK(cudaStreamSynchronize((cudaStream_t)stream));
    if (cutoff) CK(cudaMemcpy(cutoff, ctx->cutoff + slot, sizeof(float), cudaMemcpyDeviceToHost));
    if (n_selected) {
        std::vector<uint32_t> c((size_t)ctx->last_rs[slot]);
        CK(cudaMemcpy(c.data(), ctx->sel_counts + (size_t)slot * ctx->n_sms, sizeof(uint32_t) * c.size(),
                      cudaMemcpyDeviceToHost));
        uint32_t t = 0;
        for (uint32_t x : c) t += x;
        *n_selected = t;
    }
    return EFFORT_OK;
}

// ---------------------------------------------------------------------------------------------------
// multi-token GEMV (csrc/prefill.cuh): out[t] = W(v[t]) for up to kPrefillMax inputs, each with its own cutoff
// ---------------------------------------------------------------------------------------------------
static bool prefill_supported(const effort_weights* w) {
    return w && w->kind == EFFORT_KIND_FP16 && w->layout == kSliceMajor && w->bk_own && w->st16 && w->n_experts == 1 &&
           w->n_probes == kPrefillProbes && w->in >= kPrefillProbes && w->P <= 16;
}

// the geometry is a function of the matrix and the device only, so a token's result does not depend on the chunk
static PrefillProblem prefill_problem(const effort_ctx* ctx, const effort_weights* w, double effort, float* out, int accumulate) {
    PrefillProblem p{};
    p.bk = w->bk_own; p.st16 = w->st16; p.probes = w->probes;
    p.in = w->in; p.C = w->C; p.P = w->P;
    p.W = w->C < 128 ? w->C : 128;
    p.CS = (w->C + p.W - 1) / p.W;
    p.RS = ctx->n_sms / p.CS < 1 ? 1 : ctx->n_sms / p.CS;
    p.k = w->n_probes - effort_q(effort, w->n_probes);
    p.out = out; p.accumulate = accumulate;
    return p;
}

// scratch of a group at T = kPrefillMax: partial-sum floats and count words
static void prefill_scratch_need(const PrefillGroup& g, size_t* floats, size_t* counts) {
    *floats = 0; *counts = 0;
    for (int k = 0; k < g.n; k++) {
        *floats += (size_t)g.p[k].RS * kPrefillMax * g.p[k].C * 16;
        *counts += (size_t)g.p[k].RS * kPrefillMax;
    }
}

// point each problem of the group at its share of the scratch and enqueue cutoff, GEMV and split reduction
static int enqueue_prefill_group(effort_ctx* ctx, PrefillGroup& g, float* part, uint32_t* cnt, float* cut, cudaStream_t s) {
    static bool configured[64] = {false};
    if (!configured[ctx->device & 63]) {
        CK(cudaFuncSetAttribute(prefill_mul_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPrefillMax * 16 * 4 * 32 * 4));
        configured[ctx->device & 63] = true;
    }
    int ctas = 0;
    for (int k = 0; k < g.n; k++) {
        PrefillProblem& p = g.p[k];
        p.part = part; p.cnt_part = cnt;
        if (!p.cut) p.cut = cut + k * kPrefillMax;
        part += (size_t)p.RS * g.T * p.C * 16;
        cnt += (size_t)p.RS * g.T;
        ctas += p.CS * p.RS;
    }
    CK(launch_pdl(prefill_cutoff_kernel, dim3(g.T, g.n), dim3(1024), 0, s, (const PrefillGroup)g));
    LAUNCHED();
    CK(launch_pdl(prefill_mul_kernel, dim3(ctas), dim3(32 * g.T), (size_t)g.T * 16 * 4 * 32 * 4, s, (const PrefillGroup)g));
    LAUNCHED();
    CK(launch_pdl(prefill_reduce_kernel, dim3(2 * ctx->n_sms), dim3(256), 0, s, (const PrefillGroup)g));
    LAUNCHED();
    return EFFORT_OK;
}

extern "C" int effort_bucket_mul_multi(effort_ctx_t* ctx, const float* v_dev, int n, const effort_weights_t* w, float* out_dev,
                                       double effort, float* cutoff_dev, uint32_t* count_dev, void* stream) {
    if (!ctx || !v_dev || !w || !out_dev || n < 1 || n > kPrefillMax || !(effort >= 0.0 && effort <= 1.0)) return EFFORT_EINVAL;
    if (!prefill_supported(w)) return EFFORT_ESHAPE;
    PrefillGroup g{};
    g.n = 1; g.T = n; g.V = v_dev;
    g.p[0] = prefill_problem(ctx, w, effort, out_dev, 0);
    g.p[0].cut = cutoff_dev;
    g.p[0].count = count_dev;
    size_t nf, nc;
    prefill_scratch_need(g, &nf, &nc);
    int rc;
    if ((rc = ensure(ctx->pf_part, ctx->pf_part_cap, nf)) || (rc = ensure(ctx->pf_cnt, ctx->pf_cnt_cap, nc))) return rc;
    if (!ctx->pf_cut) CK(cudaMalloc(&ctx->pf_cut, sizeof(float) * kPrefillMax * kPrefillMaxProblems));
    return enqueue_prefill_group(ctx, g, ctx->pf_part, ctx->pf_cnt, ctx->pf_cut, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------------
// convert
// ---------------------------------------------------------------------------------------------------
extern "C" int effort_bucketize(const void* w_dev, int out_dim, int in_dim, void* buckets_dev, void* stats_dev,
                                void* probes_dev, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!w_dev || !buckets_dev || !stats_dev || !probes_dev) return EFFORT_EINVAL;
    const int NP = EFFORT_PROBES_COUNT;
    // preconditions, convert.swift:210-215
    if (!(out_dim >= NP || (out_dim > 0 && NP % out_dim == 0))) return EFFORT_EINVAL;
    if (in_dim < NP) return EFFORT_EINVAL;
    if (out_dim > 32000 || in_dim > 32000) return EFFORT_EINVAL;
    if (out_dim % 16) return EFFORT_EINVAL;  // assert(outDim % bSize == 0) :239
    const int rep = out_dim >= NP ? 1 : NP / out_dim;
    get_probes_kernel<<<(NP / rep + 255) / 256, 256, 0, stream>>>((const uint16_t*)w_dev, in_dim, rep, NP,
                                                                 (uint16_t*)probes_dev);
    LAUNCHED();
    const int C = out_dim / 16;
    dim3 grid((in_dim + 31) / 32, (C + 31) / 32);
    bucketize_kernel<<<grid, 1024, 0, stream>>>((const uint16_t*)w_dev, out_dim, in_dim, (uint16_t*)buckets_dev);
    LAUNCHED();
    const size_t rows = (size_t)in_dim * 16;
    make_stats_kernel<<<(unsigned)((rows + 127) / 128), 128, 0, stream>>>((const uint16_t*)buckets_dev, rows, C,
                                                                          (__half*)stats_dev);
    LAUNCHED();
    return EFFORT_OK;
}

extern "C" int effort_q4_bucketize(const void* wT_dev, int in_dim, int out_dim, void* buckets_dev, void* stats_dev,
                                   void* probes_dev, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!wT_dev || !buckets_dev || !stats_dev || !probes_dev || in_dim <= 0 || out_dim <= 0) return EFFORT_EINVAL;
    if (out_dim % 32) return EFFORT_EINVAL;  // 4 nibbles per word, q4_draft.py:305-312 asserts whole words
    const size_t rows = (size_t)in_dim * 8;
    const int n = out_dim / 8;
    __half* absvals = nullptr;
    CK(cudaMallocAsync(&absvals, rows * n * sizeof(__half), stream));
    const size_t threads = (size_t)in_dim * (out_dim / 32);
    q4_bucketize_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(
        (const uint16_t*)wT_dev, in_dim, out_dim, (uint16_t*)buckets_dev, (uint16_t*)absvals);
    LAUNCHED();
    q4_stats_kernel<<<(unsigned)((rows + 127) / 128), 128, 0, stream>>>(absvals, rows, n, (float*)stats_dev);
    LAUNCHED();
    const int np = in_dim < out_dim ? in_dim : out_dim;
    q4_probes_kernel<<<(np + 255) / 256, 256, 0, stream>>>((const uint16_t*)wT_dev, out_dim, np, (uint16_t*)probes_dev);
    LAUNCHED();
    CK(cudaFreeAsync(absvals, stream));
    return EFFORT_OK;
}

// ---------------------------------------------------------------------------------------------------
// tensor-parallel plumbing: NCCL resolved at run time
// ---------------------------------------------------------------------------------------------------
#include <dlfcn.h>

namespace {
struct NcclUniqueId { char internal[128]; };
typedef int (*nccl_get_unique_id_t)(NcclUniqueId*);
typedef int (*nccl_comm_init_rank_t)(void**, int, NcclUniqueId, int);
typedef int (*nccl_comm_destroy_t)(void*);
typedef int (*nccl_all_reduce_t)(const void*, void*, size_t, int, int, void*, cudaStream_t);
typedef int (*nccl_all_gather_t)(const void*, void*, size_t, int, void*, cudaStream_t);
typedef const char* (*nccl_get_error_string_t)(int);
struct NcclApi {
    nccl_get_unique_id_t get_unique_id = nullptr;
    nccl_comm_init_rank_t comm_init_rank = nullptr;
    nccl_comm_destroy_t comm_destroy = nullptr;
    nccl_all_reduce_t all_reduce = nullptr;
    nccl_all_gather_t all_gather = nullptr;
    nccl_get_error_string_t get_error_string = nullptr;
    bool ok = false;
};
constexpr int kNcclFloat = 7, kNcclSum = 0;

NcclApi& nccl() {
    static NcclApi api;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* h = RTLD_DEFAULT;
        if (!dlsym(h, "ncclAllReduce")) {
            h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
            if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        }
        if (h) {
            api.get_unique_id = (nccl_get_unique_id_t)dlsym(h, "ncclGetUniqueId");
            api.comm_init_rank = (nccl_comm_init_rank_t)dlsym(h, "ncclCommInitRank");
            api.comm_destroy = (nccl_comm_destroy_t)dlsym(h, "ncclCommDestroy");
            api.all_reduce = (nccl_all_reduce_t)dlsym(h, "ncclAllReduce");
            api.all_gather = (nccl_all_gather_t)dlsym(h, "ncclAllGather");
            api.get_error_string = (nccl_get_error_string_t)dlsym(h, "ncclGetErrorString");
            api.ok = api.get_unique_id && api.comm_init_rank && api.comm_destroy && api.all_reduce && api.all_gather;
        }
    }
    return api;
}
}  // namespace

#define NK(expr)                                                                                  \
    do {                                                                                          \
        int _r = (expr);                                                                          \
        if (_r != 0) {                                                                            \
            g_cuda_err = std::string(#expr) + ": nccl error " + std::to_string(_r) +              \
                         (nccl().get_error_string ? std::string(" ") + nccl().get_error_string(_r) : ""); \
            return EFFORT_ECUDA;                                                                  \
        }                                                                                         \
    } while (0)

extern "C" int effort_comm_unique_id(void* id128_out) {
    if (!id128_out) return EFFORT_EINVAL;
    if (!nccl().ok) { g_cuda_err = "libnccl not available"; return EFFORT_ECUDA; }
    NcclUniqueId id;
    NK(nccl().get_unique_id(&id));
    memcpy(id128_out, &id, sizeof(id));
    return EFFORT_OK;
}

extern "C" int effort_comm_init(effort_ctx_t* ctx, const void* id128, int rank, int world) {
    if (!ctx || !id128 || world < 1 || rank < 0 || rank >= world) return EFFORT_EINVAL;
    if (!nccl().ok) { g_cuda_err = "libnccl not available"; return EFFORT_ECUDA; }
    if (ctx->comm) return EFFORT_ESTATE;
    NcclUniqueId id;
    memcpy(&id, id128, sizeof(id));
    CK(cudaSetDevice(ctx->device));
    NK(nccl().comm_init_rank(&ctx->comm, world, id, rank));
    ctx->comm_rank = rank; ctx->comm_world = world;
    return EFFORT_OK;
}

extern "C" int effort_comm_destroy(effort_ctx_t* ctx) {
    if (!ctx) return EFFORT_EINVAL;
    if (ctx->comm) { nccl().comm_destroy(ctx->comm); ctx->comm = nullptr; }
    ctx->comm_world = 1; ctx->comm_rank = 0;
    return EFFORT_OK;
}

// ---- one-shot NVLink collectives over CUDA-IPC mapped peer memory (comm.cuh) ----
static bool p2p_enabled() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("EFFORT_P2P"); v = (e && atoi(e) == 0) ? 0 : 1; }
    return v == 1;
}

extern "C" int effort_comm_p2p_local_handle(effort_ctx_t* ctx, void* handle64_out) {
    if (!ctx || !handle64_out) return EFFORT_EINVAL;
    if (!ctx->p2p_local) {
        CK(cudaMalloc(&ctx->p2p_local, P2PLayout::total));
        CK(cudaMemset(ctx->p2p_local, 0, P2PLayout::total));
        CK(cudaDeviceSynchronize());
    }
    cudaIpcMemHandle_t h;
    CK(cudaIpcGetMemHandle(&h, ctx->p2p_local));
    static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
    memcpy(handle64_out, &h, 64);
    return EFFORT_OK;
}

extern "C" int effort_comm_p2p_connect(effort_ctx_t* ctx, const void* handles, int rank, int world) {
    if (!ctx || !handles || !ctx->p2p_local || world < 1 || world > kP2PMaxRanks || rank < 0 || rank >= world)
        return EFFORT_EINVAL;
    for (int p = 0; p < world; p++) {
        if (p == rank) { ctx->p2p_peer[p] = ctx->p2p_local; continue; }
        cudaIpcMemHandle_t h;
        memcpy(&h, (const char*)handles + 64 * p, 64);
        CK(cudaIpcOpenMemHandle(&ctx->p2p_peer[p], h, cudaIpcMemLazyEnablePeerAccess));
    }
    ctx->comm_rank = rank; ctx->comm_world = world;
    ctx->p2p_ready = true;
    return EFFORT_OK;
}

extern "C" int effort_comm_p2p_disable(effort_ctx_t* ctx) {
    if (!ctx) return EFFORT_EINVAL;
    ctx->p2p_ready = false;  // the mappings stay until the context is destroyed; the token loop takes the NCCL path
    return EFFORT_OK;
}

template <int MODE>
static int p2p_launch(effort_ctx* ctx, int site, const float* send, float* out, size_t count, cudaStream_t s) {
    if (site < 0 || site >= kP2PSites || count * 8 * (size_t)ctx->comm_world > kP2PSiteBytes)  // 8-byte {value, seq} packets
        return EFFORT_ESHAPE;
    P2PArgs a{};
    for (int p = 0; p < ctx->comm_world; p++) a.peer[p] = (unsigned char*)ctx->p2p_peer[p];
    a.rank = ctx->comm_rank; a.world = ctx->comm_world; a.site = site; a.err = ctx->v2_err;
    CK(launch_pdl(p2p_collective_kernel<MODE>, dim3(kP2PBlocks), dim3(kP2PThreads), 0, s, a, send, out, (int)count));
    LAUNCHED();
    return EFFORT_OK;
}

// site-aware internal entry points: P2P when connected, else NCCL
static int comm_all_reduce_site(effort_ctx* ctx, int site, float* buf, size_t count, cudaStream_t s) {
    if (ctx->comm_world == 1) return EFFORT_OK;
    if (ctx->p2p_ready && p2p_enabled()) return p2p_launch<1>(ctx, site, buf, buf, count, s);
    return effort_comm_all_reduce(ctx, buf, count, s);
}
static int comm_all_gather_site(effort_ctx* ctx, int site, const float* send, float* recv, size_t count, cudaStream_t s) {
    if (ctx->comm_world > 1 && ctx->p2p_ready && p2p_enabled()) return p2p_launch<0>(ctx, site, send, recv, count, s);
    return effort_comm_all_gather(ctx, send, recv, count, s);
}

extern "C" int effort_comm_p2p_collective(effort_ctx_t* ctx, int mode, int site, const float* send_dev, float* out_dev,
                                          size_t count, void* stream) {
    if (!ctx || !send_dev || !out_dev || (mode != 0 && mode != 1)) return EFFORT_EINVAL;
    if (!ctx->p2p_ready || ctx->comm_world < 2) return EFFORT_ESTATE;
    return mode == 0 ? p2p_launch<0>(ctx, site, send_dev, out_dev, count, (cudaStream_t)stream)
                     : p2p_launch<1>(ctx, site, send_dev, out_dev, count, (cudaStream_t)stream);
}

extern "C" int effort_comm_all_reduce(effort_ctx_t* ctx, float* buf_dev, size_t count, void* stream) {
    if (!ctx || !buf_dev) return EFFORT_EINVAL;
    if (ctx->comm_world == 1) return EFFORT_OK;
    if (!ctx->comm) return EFFORT_ESTATE;
    NK(nccl().all_reduce(buf_dev, buf_dev, count, kNcclFloat, kNcclSum, ctx->comm, (cudaStream_t)stream));
    return EFFORT_OK;
}

extern "C" int effort_comm_all_gather(effort_ctx_t* ctx, const float* send_dev, float* recv_dev, size_t send_count,
                                      void* stream) {
    if (!ctx || !send_dev || !recv_dev) return EFFORT_EINVAL;
    if (ctx->comm_world == 1) {
        if (send_dev != recv_dev)
            CK(cudaMemcpyAsync(recv_dev, send_dev, send_count * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
        return EFFORT_OK;
    }
    if (!ctx->comm) return EFFORT_ESTATE;
    NK(nccl().all_gather(send_dev, recv_dev, send_count, kNcclFloat, ctx->comm, (cudaStream_t)stream));
    return EFFORT_OK;
}

// ---------------------------------------------------------------------------------------------------
// decode loop (runNetwork.swift:68-316 mirror)
// ---------------------------------------------------------------------------------------------------
#include <map>

#include "decode.cuh"

struct effort_model {
    effort_ctx* ctx = nullptr;
    effort_model_config_t cfg{};
    struct Layer {
        const effort_weights *wq = nullptr, *wk = nullptr, *wv = nullptr, *wo = nullptr, *w1 = nullptr, *w2 = nullptr,
                             *w3 = nullptr;
        const __half *attn_norm = nullptr, *ffn_norm = nullptr;
        float *kc = nullptr, *vc = nullptr;
        const __half* gate = nullptr;  // MoE: [n_experts, dim] fp16 (layers.N.feed_forward.gate, loader.swift:208-212)
        int n_experts = 1;
    };
    std::vector<Layer> layers;
    const __half *norm = nullptr, *out_core = nullptr, *emb = nullptr;
    float *attn_full = nullptr, *x2_full = nullptr, *logits_local = nullptr;  // tensor-parallel gather buffers
    float *sumsq_a = nullptr, *sumsq_b = nullptr;  // per-block sum(h^2) partials for the fused rmsNorm-on-load
    bool fuse_glue = false;  // rmsNorm-on-load / residual+silu in the integrate epilogue: 9 launches per layer, but measured
                             // slower than the 12-launch chain since the cutoff moved to four warps (the norm divides sit on them)
    float *h = nullptr, *h_norm = nullptr, *xq = nullptr, *xk = nullptr, *xv = nullptr, *attn = nullptr,
          *attn_ffn_out = nullptr, *fxn = nullptr, *x1 = nullptr, *x3 = nullptr, *x2 = nullptr, *ffn_out = nullptr,
          *out_normed = nullptr, *logits = nullptr;
    int *pos = nullptr, *token = nullptr, *next = nullptr;
    // round-2 chain: the GEMV outputs are ACCUMULATED (reductions) into double-buffered vectors that an earlier kernel of
    // the chain has cleared (layer parity picks the buffer)
    float *xq2[2] = {nullptr, nullptr}, *xk2[2] = {nullptr, nullptr}, *xv2[2] = {nullptr, nullptr};
    float *x1_2[2] = {nullptr, nullptr}, *x3_2[2] = {nullptr, nullptr};
    uint32_t* gate_idx = nullptr;  // MoE: the two routed experts of the current layer (device, read as expNo)
    float* gate_val = nullptr;     // MoE: their softmax weights
    float* h_keep = nullptr;       // MoE: the hidden state both routed experts normalise (h itself takes the first one's output)
    float2* head_cand = nullptr;   // per-CTA argmax candidates of head_kernel
    unsigned* head_ticket = nullptr;
    int host_pos = 0;              // tokens decoded since the last reset (bounds the KV cache, ADVICE r1)
    int chain = 2;                 // 2 = fused v2 chain (5 launches per layer), 1 = one kernel per reference op
    int *h_token = nullptr, *h_next = nullptr;  // pinned
    float* h_logits = nullptr;                  // pinned
    std::map<int, cudaGraphExec_t> graphs;      // keyed by q = Int(4095*(1-effort))
    // the token path of the last enqueued or replayed step (effort_model_buffer): 0 = none yet, 1 = one of the
    // chain-1 paths (generic, fused glue, tensor parallel), 2 = the fused chain; and the path each graph captured
    int path = 0;
    std::map<int, int> graph_path;
    uint64_t launches_per_token = 0;
    bool use_graphs = true;
    bool warmed = false;
    // sampler (effort_model_set_sampler): the step's sample kernel reads `sampler_dev`, refreshed from the pinned
    // `sampler_host` on the step's stream when it changed, so a graph replay sees new parameters without recapture
    bool sampling = false, sampler_dirty = false;
    effort_sampler_t* sampler_dev = nullptr;
    effort_sampler_t* sampler_host = nullptr;   // pinned
    cudaEvent_t sampler_copied = nullptr;       // the last copy out of sampler_host has run
    // scoring (effort_model_set_scoring): the step's score kernel reads target row entry pos - 1 and writes that record
    bool scoring = false;
    int32_t* score_targets = nullptr;          // [max_seq], -1 = no target
    effort_score_t* scores = nullptr;          // [max_seq]
    // prefill (effort_model_prefill): chunk buffers [kPrefillMax][...] and the multi-token GEMV scratch, allocated once at
    // their maximum size by the first prefill; graphs live in `graphs` under prefill_graph_key
    bool pf_ready = false, pf_warmed = false, pf_scored = false;
    float *pf_h = nullptr, *pf_xn = nullptr, *pf_q = nullptr, *pf_k = nullptr, *pf_v = nullptr, *pf_attn = nullptr,
          *pf_x1 = nullptr, *pf_x3 = nullptr, *pf_x2 = nullptr, *pf_logits = nullptr, *pf_part = nullptr, *pf_cut = nullptr;
    uint32_t* pf_cnt = nullptr;
    int* pf_tok = nullptr;
    int* pf_lens = nullptr;                    // {0, 1, .., kPrefillMax}: EFFORT_BUF_CHUNK_LEN points at entry T
    int pf_len = 0;                            // length of the last chunk
    std::map<int, uint64_t> pf_launches;       // kernels one replay of a prefill graph launches
    std::vector<void*> owned;
};

template <typename T>
static int model_alloc(effort_model* m, T*& p, size_t n) {
    CK(cudaMalloc(&p, n * sizeof(T)));
    CK(cudaMemset(p, 0, n * sizeof(T)));
    m->owned.push_back(p);
    return EFFORT_OK;
}

static int model_create_buffers(effort_model* m, effort_ctx* ctx, const effort_model_config_t* cfg, int G);
extern "C" int effort_model_destroy(effort_model_t* m);

extern "C" int effort_model_create(effort_ctx_t* ctx, const effort_model_config_t* cfg, effort_model_t** m_out) {
    if (!ctx || !cfg || !m_out) return EFFORT_EINVAL;
    *m_out = nullptr;
    if (cfg->head_dim != 128 || cfg->n_heads * cfg->head_dim != cfg->dim) return EFFORT_ESHAPE;
    if (cfg->n_kv_heads <= 0 || cfg->n_heads % cfg->n_kv_heads) return EFFORT_EINVAL;
    if (cfg->n_layers <= 0 || cfg->max_seq <= 0 || cfg->vocab <= 0) return EFFORT_EINVAL;
    const int G = cfg->tp_size < 1 ? 1 : cfg->tp_size;
    if (G > 1) {
        if ((!ctx->comm && !ctx->p2p_ready) || ctx->comm_world != G || ctx->comm_rank != cfg->tp_rank) return EFFORT_ESTATE;
        if (cfg->n_kv_heads % G || cfg->hidden_dim % G || cfg->vocab % G || (cfg->hidden_dim / G) % 16) return EFFORT_ESHAPE;
    }
    effort_model* m = new (std::nothrow) effort_model();
    if (!m) return EFFORT_ENOMEM;
    m->ctx = ctx; m->cfg = *cfg;
    m->layers.resize(cfg->n_layers);
    m->cfg.tp_size = G;
    const int rc_alloc = model_create_buffers(m, ctx, cfg, G);
    if (rc_alloc) {  // every failure path releases what was allocated so far
        effort_model_destroy(m);
        return rc_alloc;
    }
    *m_out = m;
    return EFFORT_OK;
}

static int model_create_buffers(effort_model* m, effort_ctx* ctx, const effort_model_config_t* cfg, int G) {
    const size_t kv = (size_t)cfg->max_seq * (cfg->n_kv_heads / G) * cfg->head_dim;
    int rc = 0;
    for (auto& l : m->layers) {
        if ((rc = model_alloc(m, l.kc, kv))) return rc;
        if ((rc = model_alloc(m, l.vc, kv))) return rc;
    }
    const int kvd = cfg->n_kv_heads * cfg->head_dim;
    if ((rc = model_alloc(m, m->h, cfg->dim)) || (rc = model_alloc(m, m->h_norm, cfg->dim)) ||
        (rc = model_alloc(m, m->xq, cfg->dim)) || (rc = model_alloc(m, m->xk, kvd)) ||
        (rc = model_alloc(m, m->xv, kvd)) || (rc = model_alloc(m, m->attn, cfg->dim)) ||
        (rc = model_alloc(m, m->attn_ffn_out, cfg->dim)) || (rc = model_alloc(m, m->fxn, cfg->dim)) ||
        (rc = model_alloc(m, m->x1, cfg->hidden_dim)) || (rc = model_alloc(m, m->x3, cfg->hidden_dim)) ||
        (rc = model_alloc(m, m->x2, cfg->hidden_dim)) || (rc = model_alloc(m, m->ffn_out, cfg->dim)) ||
        (rc = model_alloc(m, m->out_normed, cfg->dim)) || (rc = model_alloc(m, m->logits, cfg->vocab)) ||
        (rc = model_alloc(m, m->pos, 1)) || (rc = model_alloc(m, m->token, 1)) || (rc = model_alloc(m, m->next, 1)) ||
        (rc = model_alloc(m, m->attn_full, cfg->dim)) || (rc = model_alloc(m, m->x2_full, cfg->hidden_dim)) ||
        (rc = model_alloc(m, m->logits_local, cfg->vocab)) || (rc = model_alloc(m, m->sumsq_a, 1024)) ||
        (rc = model_alloc(m, m->sumsq_b, 1024)))
        return rc;
    { const char* e = getenv("EFFORT_FUSE_GLUE"); m->fuse_glue = e && atoi(e) == 1; }
    { const char* e = getenv("EFFORT_CHAIN"); if (e && atoi(e) == 1) m->chain = 1; }
    for (int b = 0; b < 2; b++) {
        if ((rc = model_alloc(m, m->xq2[b], cfg->dim)) || (rc = model_alloc(m, m->xk2[b], kvd)) ||
            (rc = model_alloc(m, m->xv2[b], kvd)) || (rc = model_alloc(m, m->x1_2[b], cfg->hidden_dim)) ||
            (rc = model_alloc(m, m->x3_2[b], cfg->hidden_dim)))
            return rc;
    }
    if ((rc = model_alloc(m, m->head_cand, (size_t)ctx->n_sms * 8)) || (rc = model_alloc(m, m->head_ticket, 1)) ||
        (rc = model_alloc(m, m->gate_idx, 2)) || (rc = model_alloc(m, m->gate_val, 2)) ||
        (rc = model_alloc(m, m->h_keep, (size_t)cfg->dim)) || (rc = model_alloc(m, m->score_targets, cfg->max_seq)) ||
        (rc = model_alloc(m, m->scores, cfg->max_seq)))
        return rc;
    CK(cudaMemset(m->score_targets, 0xff, sizeof(int32_t) * cfg->max_seq));  // all -1: no target
    CK(cudaMallocHost(&m->h_token, sizeof(int)));
    CK(cudaMallocHost(&m->h_next, sizeof(int)));
    CK(cudaMallocHost(&m->h_logits, sizeof(float) * cfg->vocab));
    return EFFORT_OK;
}

extern "C" int effort_model_destroy(effort_model_t* m) {
    if (!m) return EFFORT_OK;
    for (auto& g : m->graphs) cudaGraphExecDestroy(g.second);
    for (void* p : m->owned) cudaFree(p);
    cudaFreeHost(m->h_token); cudaFreeHost(m->h_next); cudaFreeHost(m->h_logits); cudaFreeHost(m->sampler_host);
    if (m->sampler_copied) cudaEventDestroy(m->sampler_copied);
    delete m;
    return EFFORT_OK;
}

extern "C" int effort_model_set_layer(effort_model_t* m, int layer, const effort_weights_t* wq,
                                      const effort_weights_t* wk, const effort_weights_t* wv,
                                      const effort_weights_t* wo, const effort_weights_t* w1,
                                      const effort_weights_t* w2, const effort_weights_t* w3,
                                      const void* attn_norm_dev, const void* ffn_norm_dev) {
    if (!m || layer < 0 || layer >= m->cfg.n_layers) return EFFORT_EINVAL;
    if (!wq || !wk || !wv || !wo || !w1 || !w2 || !w3 || !attn_norm_dev || !ffn_norm_dev) return EFFORT_EINVAL;
    const auto& c = m->cfg;
    const int G = c.tp_size;
    const int kvd = c.n_kv_heads * c.head_dim;
    auto ok = [](const effort_weights* w, int in, int out) { return w->in == in && w->out == out; };
    if (!ok(wq, c.dim, c.dim / G) || !ok(wk, c.dim, kvd / G) || !ok(wv, c.dim, kvd / G) || !ok(wo, c.dim / G, c.dim) ||
        !ok(w1, c.dim, c.hidden_dim / G) || !ok(w3, c.dim, c.hidden_dim / G) || !ok(w2, c.hidden_dim / G, c.dim))
        return EFFORT_ESHAPE;
    auto& l = m->layers[layer];
    l.wq = wq; l.wk = wk; l.wv = wv; l.wo = wo; l.w1 = w1; l.w2 = w2; l.w3 = w3;
    l.attn_norm = (const __half*)attn_norm_dev; l.ffn_norm = (const __half*)ffn_norm_dev;
    for (auto& g : m->graphs) cudaGraphExecDestroy(g.second);
    m->graphs.clear();
    return EFFORT_OK;
}

extern "C" int effort_model_set_moe(effort_model_t* m, int layer, const void* gate_dev, int n_experts) {
    if (!m || layer < 0 || layer >= m->cfg.n_layers || !gate_dev || n_experts < 2 || n_experts > 64) return EFFORT_EINVAL;
    auto& l = m->layers[layer];
    if (!l.w1 || l.w1->n_experts != n_experts || l.w2->n_experts != n_experts || l.w3->n_experts != n_experts) return EFFORT_ESHAPE;
    l.gate = (const __half*)gate_dev;
    l.n_experts = n_experts;
    for (auto& g : m->graphs) cudaGraphExecDestroy(g.second);
    m->graphs.clear();
    return EFFORT_OK;
}

extern "C" int effort_model_set_head(effort_model_t* m, const void* norm_dev, const void* output_core_dev,
                                     const void* tok_embeddings_dev) {
    if (!m || !norm_dev || !output_core_dev || !tok_embeddings_dev) return EFFORT_EINVAL;
    m->norm = (const __half*)norm_dev; m->out_core = (const __half*)output_core_dev;
    m->emb = (const __half*)tok_embeddings_dev;
    for (auto& g : m->graphs) cudaGraphExecDestroy(g.second);  // captured graphs hold the old pointers
    m->graphs.clear();
    return EFFORT_OK;
}

extern "C" int effort_model_reset(effort_model_t* m, void* stream) {
    if (!m) return EFFORT_EINVAL;
    CK(cudaMemsetAsync(m->pos, 0, sizeof(int), (cudaStream_t)stream));
    m->host_pos = 0;
    return EFFORT_OK;
}

extern "C" int effort_model_rewind(effort_model_t* m, int pos, void* stream) {
    if (!m || pos < 0 || pos >= m->cfg.max_seq) return EFFORT_EINVAL;
    // pageable source: the copy has taken the value once the call returns
    CK(cudaMemcpyAsync(m->pos, &pos, sizeof(int), cudaMemcpyHostToDevice, (cudaStream_t)stream));
    m->host_pos = pos;
    return EFFORT_OK;
}

extern "C" int effort_model_set_graphs(effort_model_t* m, int enable) {
    if (!m) return EFFORT_EINVAL;
    m->use_graphs = enable != 0;
    return EFFORT_OK;
}

extern "C" int effort_model_set_fused_glue(effort_model_t* m, int enable) {
    if (!m) return EFFORT_EINVAL;
    if (m->fuse_glue != (enable != 0)) {
        for (auto& g : m->graphs) cudaGraphExecDestroy(g.second);
        m->graphs.clear();
    }
    m->fuse_glue = enable != 0;
    return EFFORT_OK;
}

extern "C" int effort_model_set_chain(effort_model_t* m, int chain) {
    if (!m || (chain != 1 && chain != 2)) return EFFORT_EINVAL;
    if (m->chain != chain) {
        for (auto& g : m->graphs) cudaGraphExecDestroy(g.second);
        m->graphs.clear();
    }
    m->chain = chain;
    return EFFORT_OK;
}

static bool sampler_valid(const effort_sampler_t* s) {
    return s->temperature > 0.f && s->temperature <= 3.402823466e38f && s->top_k >= 0 && s->top_p > 0.f && s->top_p <= 1.f;
}

static int enqueue_sample(effort_ctx* ctx, const float* logits, int n, const effort_sampler_t& prm,
                          const effort_sampler_t* prm_dev, const int* pos_dev, uint32_t position, int32_t* token,
                          cudaStream_t s) {
    static bool configured[64] = {false};
    if (!configured[ctx->device & 63]) {
        CK(cudaFuncSetAttribute(sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                kSampleHistBytes + (int)(kSampleCache * sizeof(float))));
        configured[ctx->device & 63] = true;
    }
    const size_t smem = kSampleHistBytes + (size_t)(n < kSampleCache ? n : kSampleCache) * sizeof(float);
    CK(launch_pdl(sample_kernel, dim3(1), dim3(kSampleThreads), smem, s, logits, n, prm, prm_dev, pos_dev, position, token));
    LAUNCHED();
    return EFFORT_OK;
}

extern "C" int effort_sample(effort_ctx_t* ctx, const float* logits_dev, int n, const effort_sampler_t* s, uint32_t position,
                             int32_t* token_dev, void* stream) {
    if (!ctx || !logits_dev || !s || !token_dev || n <= 0 || !sampler_valid(s)) return EFFORT_EINVAL;
    return enqueue_sample(ctx, logits_dev, n, *s, nullptr, nullptr, position, token_dev, (cudaStream_t)stream);
}

extern "C" int effort_model_set_sampler(effort_model_t* m, const effort_sampler_t* s) {
    if (!m || (s && !sampler_valid(s))) return EFFORT_EINVAL;
    if (m->sampling != (s != nullptr)) {  // the step's launch sequence changes
        for (auto& g : m->graphs) cudaGraphExecDestroy(g.second);
        m->graphs.clear();
    }
    m->sampling = s != nullptr;
    if (!s) return EFFORT_OK;
    if (!m->sampler_dev) {
        int rc = model_alloc(m, m->sampler_dev, 1);
        if (rc) return rc;
        CK(cudaMallocHost(&m->sampler_host, sizeof(effort_sampler_t)));
        CK(cudaEventCreateWithFlags(&m->sampler_copied, cudaEventDisableTiming));
    }
    CK(cudaEventSynchronize(m->sampler_copied));  // a copy still queued reads the pinned block
    *m->sampler_host = *s;
    m->sampler_dirty = true;
    return EFFORT_OK;
}

// the sampler's kernel after the head / argmax that advanced pos: overwrites `next` with the draw
static int model_enqueue_sample(effort_model* m, cudaStream_t s) {
    if (!m->sampling) return EFFORT_OK;
    return enqueue_sample(m->ctx, m->logits, m->cfg.vocab, *m->sampler_host, m->sampler_dev, m->pos, 0u, m->next, s);
}

static int enqueue_score(const float* logits, int n, const int32_t* targets, int n_rec, const int* pos_dev, int grid,
                         effort_score_t* out, cudaStream_t s, int ld = 0) {
    CK(launch_pdl(score_kernel, dim3(grid), dim3(kScoreThreads), 0, s, logits, n, targets, n_rec, pos_dev, out, ld));
    LAUNCHED();
    return EFFORT_OK;
}

extern "C" int effort_score(effort_ctx_t* ctx, const float* logits_dev, int n, const int32_t* targets_dev, int n_targets,
                            effort_score_t* out_dev, void* stream) {
    if (!ctx || !logits_dev || !targets_dev || !out_dev || n <= 0 || n_targets <= 0) return EFFORT_EINVAL;
    return enqueue_score(logits_dev, n, targets_dev, n_targets, nullptr, n_targets, out_dev, (cudaStream_t)stream);
}

extern "C" int effort_model_set_scoring(effort_model_t* m, int enable) {
    if (!m) return EFFORT_EINVAL;
    if (m->scoring != (enable != 0)) {  // the step's launch sequence changes
        for (auto& g : m->graphs) cudaGraphExecDestroy(g.second);
        m->graphs.clear();
    }
    m->scoring = enable != 0;
    return EFFORT_OK;
}

extern "C" int effort_model_set_score_targets(effort_model_t* m, const int32_t* targets_dev, int n, void* stream) {
    if (!m || n < 0 || n > m->cfg.max_seq || (!targets_dev && n > 0)) return EFFORT_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;
    if (n > 0) CK(cudaMemcpyAsync(m->score_targets, targets_dev, sizeof(int32_t) * n, cudaMemcpyDeviceToDevice, s));
    if (n < m->cfg.max_seq) CK(cudaMemsetAsync(m->score_targets + n, 0xff, sizeof(int32_t) * (m->cfg.max_seq - n), s));
    return EFFORT_OK;
}

extern "C" const effort_score_t* effort_model_scores(const effort_model_t* m) { return m ? m->scores : nullptr; }

// the scorer's kernel last in the step (after the sampler's, if any): record pos - 1 from the step's logits
static int model_enqueue_score(effort_model* m, cudaStream_t s) {
    if (!m->scoring) return EFFORT_OK;
    return enqueue_score(m->logits, m->cfg.vocab, m->score_targets, m->cfg.max_seq, m->pos, 1, m->scores, s);
}

// what every token path enqueues after the head / argmax that advanced pos
static int model_enqueue_tail(effort_model* m, cudaStream_t s) {
    int rc = model_enqueue_sample(m, s);
    return rc ? rc : model_enqueue_score(m, s);
}

extern "C" const float* effort_model_logits(const effort_model_t* m) { return m ? m->logits : nullptr; }
extern "C" const int32_t* effort_model_next_token(const effort_model_t* m) { return m ? m->next : nullptr; }

extern "C" const void* effort_model_buffer(const effort_model_t* m, int which, int layer, size_t* count) {
    if (count) *count = 0;
    if (!m || m->path == 0) return nullptr;
    const auto& c = m->cfg;
    if (m->path == 3 || (which >= EFFORT_BUF_CHUNK_Q && which <= EFFORT_BUF_CHUNK_LEN)) {  // the last prefill chunk
        if (m->path != 3) return nullptr;
        const size_t T = m->pf_len, kv = (size_t)c.n_kv_heads * c.head_dim;
        const void* p = nullptr;
        size_t n = 0;
        switch (which) {
            case EFFORT_BUF_KCACHE:
            case EFFORT_BUF_VCACHE:
                if (layer < 0 || layer >= c.n_layers) return nullptr;
                p = which == EFFORT_BUF_KCACHE ? m->layers[layer].kc : m->layers[layer].vc;
                n = (size_t)c.max_seq * kv;
                break;
            case EFFORT_BUF_POS: p = m->pos; n = 1; break;
            case EFFORT_BUF_CHUNK_Q: p = m->pf_q; n = T * c.dim; break;
            case EFFORT_BUF_CHUNK_K: p = m->pf_k; n = T * kv; break;
            case EFFORT_BUF_CHUNK_V: p = m->pf_v; n = T * kv; break;
            case EFFORT_BUF_CHUNK_ATTN: p = m->pf_attn; n = T * c.dim; break;
            case EFFORT_BUF_CHUNK_LOGITS: if (m->pf_scored) { p = m->pf_logits; n = T * c.vocab; } break;
            case EFFORT_BUF_CHUNK_LEN: p = m->pf_lens + T; n = 1; break;
            default: return nullptr;
        }
        if (p && count) *count = n;
        return p;
    }
    const int G = c.tp_size;
    const bool chain2 = m->path == 2;
    const int b = (c.n_layers - 1) & 1;  // the fused chain's parity buffers of the last layer
    const size_t q = (size_t)(c.n_heads / G) * c.head_dim, kv = (size_t)(c.n_kv_heads / G) * c.head_dim;
    bool moe = false;
    for (const auto& l : m->layers) moe = moe || l.gate != nullptr;
    const void* p = nullptr;
    size_t n = 0;
    switch (which) {
        case EFFORT_BUF_Q: p = chain2 ? m->xq2[b] : m->xq; n = q; break;
        case EFFORT_BUF_K: p = chain2 ? m->xk2[b] : m->xk; n = kv; break;
        case EFFORT_BUF_V: p = chain2 ? m->xv2[b] : m->xv; n = kv; break;
        case EFFORT_BUF_ATTN: p = m->attn; n = q; break;
        case EFFORT_BUF_KCACHE:
        case EFFORT_BUF_VCACHE:
            if (layer < 0 || layer >= c.n_layers) return nullptr;
            p = which == EFFORT_BUF_KCACHE ? m->layers[layer].kc : m->layers[layer].vc;
            n = (size_t)c.max_seq * kv;
            break;
        case EFFORT_BUF_HIDDEN: p = m->h; n = c.dim; break;
        case EFFORT_BUF_NORMED: if (!chain2) { p = m->out_normed; n = c.dim; } break;
        case EFFORT_BUF_GATE_IN: if (chain2 && moe) { p = m->h_keep; n = c.dim; } break;
        case EFFORT_BUF_GATE_IDX: if (chain2 && moe) { p = m->gate_idx; n = 2; } break;
        case EFFORT_BUF_GATE_VAL: if (chain2 && moe) { p = m->gate_val; n = 2; } break;
        case EFFORT_BUF_POS: p = m->pos; n = 1; break;
        default: return nullptr;
    }
    if (p && count) *count = n;
    return p;
}
extern "C" size_t effort_model_bucket_bytes(const effort_model_t* m) {
    if (!m) return 0;
    size_t b = 0;
    for (const auto& l : m->layers)
        for (const effort_weights* w : {l.wq, l.wk, l.wv, l.wo, l.w1, l.w2, l.w3})
            if (w) b += (w->kind == EFFORT_KIND_FP16) ? (size_t)w->in * w->out * 2 : (size_t)w->in * w->out / 2;
    return b;
}


// ---- round-2 decode chain (single GPU, FP16 buckets): 5 launches per layer ------------------------------------------
//   [q,k,v]  one v2 launch, rmsNorm(h)*attn_norm applied on load, results accumulated into the parity buffers
//   attention (+ clears the buffers of the next layer)
//   wo       v2, plain input, accumulates straight into the residual stream h        (h.add(by:), runNetwork.swift:172)
//   [w1,w3]  one v2 launch, rmsNorm(h)*ffn_norm on load
//   w2       v2, input = silu(x1)*x3 computed on load, accumulates into h             (runNetwork.swift:181-183)
// then head_kernel: final norm on load + lm_head + argmax + position advance.
static bool model_all_fp16_v2(const effort_model* m) {
    for (const auto& l : m->layers)
        for (const effort_weights* w : {l.wq, l.wk, l.wv, l.wo, l.w1, l.w2, l.w3})
            if (!w || w->kind != EFFORT_KIND_FP16 || !w->buckets || !v2_supported(w)) return false;
    return m->cfg.dim == 8 * kV2Threads;
}

static int enqueue_head(effort_model* m, const float* h, const __half* norm_w, const __half* core, int rows, int row0,
                        float* logits, bool do_argmax, cudaStream_t s) {
    const auto& c = m->cfg;
    const size_t smem = (size_t)c.dim * sizeof(float);
    static bool configured[64] = {false};
    if (smem > 48 * 1024 && !configured[m->ctx->device & 63]) {
        CK(cudaFuncSetAttribute(head_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured[m->ctx->device & 63] = true;
    }
    int grid = (rows + 7) / 8;
    const int max_grid = m->ctx->n_sms * 8;
    if (grid > max_grid) grid = max_grid;
    CK(launch_pdl(head_kernel, dim3(grid), dim3(256), smem, s, h, norm_w, c.norm_eps, core, rows, c.dim, row0, logits,
                  m->head_cand, m->head_ticket, m->next, m->pos, do_argmax ? 1 : 0));
    LAUNCHED();
    return EFFORT_OK;
}

static int model_enqueue_token_v2(effort_model* m, double effort, cudaStream_t s) {
    const auto& c = m->cfg;
    effort_ctx* ctx = m->ctx;
    const int kvd = c.n_kv_heads * c.head_dim;
    int rc;
    {   // the first layer accumulates into parity-0 buffers: cleared here (whatever the layer count's parity)
        ZeroList z{};
        z.p[0] = m->xq2[0]; z.n[0] = c.dim; z.p[1] = m->xk2[0]; z.n[1] = kvd; z.p[2] = m->xv2[0]; z.n[2] = kvd;
        z.p[3] = m->x1_2[0]; z.n[3] = c.hidden_dim; z.p[4] = m->x3_2[0]; z.n[4] = c.hidden_dim;
        CK(launch_pdl(embed_kernel, dim3(4), dim3(1024), 0, s, (const int*)m->token, m->emb, c.dim, c.vocab, m->h,
                      (float*)nullptr, z));
        LAUNCHED();
    }
    for (int li = 0; li < c.n_layers; li++) {
        auto& l = m->layers[li];
        const int b = li & 1, nb = b ^ 1;
        V2Call qkv[3];
        const effort_weights* wqkv[3] = {l.wq, l.wk, l.wv};
        float* oqkv[3] = {m->xq2[b], m->xk2[b], m->xv2[b]};
        for (int k = 0; k < 3; k++) {
            qkv[k].v = m->h; qkv[k].norm_w = l.attn_norm; qkv[k].norm_eps = c.norm_eps; qkv[k].w = wqkv[k];
            qkv[k].out = oqkv[k]; qkv[k].effort = effort; qkv[k].out_mode = kOutAccumulate;
        }
        if ((rc = launch_v2(ctx, qkv, 3, 0, s))) return rc;
        ZeroList z{};
        z.p[0] = m->xq2[nb]; z.n[0] = c.dim; z.p[1] = m->xk2[nb]; z.n[1] = kvd; z.p[2] = m->xv2[nb]; z.n[2] = kvd;
        z.p[3] = m->x1_2[nb]; z.n[3] = c.hidden_dim; z.p[4] = m->x3_2[nb]; z.n[4] = c.hidden_dim;
        CK(launch_pdl(attention_kernel, dim3(c.n_heads), dim3(256), 0, s, (const float*)m->xq2[b], (const float*)m->xk2[b],
                      (const float*)m->xv2[b], l.kc, l.vc, (const int*)m->pos, c.n_heads, c.n_kv_heads, c.rope_theta, c.max_seq,
                      m->attn, z));
        LAUNCHED();
        V2Call wo;
        wo.v = m->attn; wo.w = l.wo; wo.out = m->h; wo.effort = effort; wo.out_mode = kOutAccumulate;
        if ((rc = launch_v2(ctx, &wo, 1, 0, s))) return rc;
        const int n_routed = l.gate ? 2 : 1;  // MoE: the two experts the gate picks (runNetwork.swift:185-200)
        if (l.gate) {
            CK(launch_pdl(moe_gate_kernel, dim3(1), dim3(256), 0, s, (const float*)m->h, l.ffn_norm, c.norm_eps, l.gate, l.n_experts,
                          c.dim, m->gate_idx, m->gate_val, m->h_keep));
            LAUNCHED();
        }
        for (int r = 0; r < n_routed; r++) {
            V2Call w13[2];
            const effort_weights* ww[2] = {l.w1, l.w3};
            float* o13[2] = {m->x1_2[b], m->x3_2[b]};
            for (int k = 0; k < 2; k++) {
                w13[k].v = l.gate ? m->h_keep : m->h; w13[k].norm_w = l.ffn_norm; w13[k].norm_eps = c.norm_eps; w13[k].w = ww[k];
                w13[k].out = o13[k]; w13[k].effort = effort;
                // dense layers accumulate into buffers an earlier kernel cleared; a routed expert overwrites (the second
                // expert reuses the buffers of the first)
                w13[k].out_mode = l.gate ? kOutOverwrite : kOutAccumulate;
                w13[k].exp_no = l.gate ? m->gate_idx + r : nullptr;
            }
            if ((rc = launch_v2(ctx, w13, 2, 0, s))) return rc;
            V2Call w2;
            w2.v = m->x1_2[b]; w2.v2 = m->x3_2[b]; w2.w = l.w2; w2.out = m->h; w2.effort = effort; w2.out_mode = kOutAccumulate;
            if (l.gate) { w2.exp_no = m->gate_idx + r; w2.out_scale = m->gate_val + r; }  // h += gateVal * ffnOut (:196-199)
            if ((rc = launch_v2(ctx, &w2, 1, 0, s))) return rc;
        }
    }
    if ((rc = enqueue_head(m, m->h, m->norm, m->out_core, c.vocab, 0, m->logits, true, s))) return rc;
    return model_enqueue_tail(m, s);
}

// enqueue one token (no graph logic).  token lives in m->token (device).  With tp_size = G > 1 this rank holds
// heads [rank*32/G, ...) and hidden columns [rank*14336/G, ...): q/k/v/w1/w3 are column shards (no exchange),
// wo/w2 are row shards: all-gather the first 4096 dims of their input (cutoff parity), all-reduce the output.
static int model_enqueue_token(effort_model* m, double effort, cudaStream_t s) {
    const auto& c = m->cfg;
    effort_ctx* ctx = m->ctx;
    const int G = c.tp_size;
    const int dim_l = c.dim / G, hid_l = c.hidden_dim / G, heads_l = c.n_heads / G, kv_l = c.n_kv_heads / G;
    if (!m->norm) return EFFORT_ESTATE;
    int rc;
    const bool v2_chain = G == 1 && m->chain == 2 && ctx->engine == 2 && model_all_fp16_v2(m);
    m->path = v2_chain ? 2 : 1;
    if (v2_chain) return model_enqueue_token_v2(m, effort, s);
    for (const auto& l : m->layers)
        if (l.gate) return EFFORT_ESTATE;  // expert routing lives in the fused chain only
    CK(launch_pdl(embed_kernel, dim3(4), dim3(1024), 0, s, (const int*)m->token, m->emb, c.dim, c.vocab, m->h, m->sumsq_a,
                  ZeroList{}));
    LAUNCHED();
    if (G == 1 && m->fuse_glue && m->layers[0].wq && m->layers[0].wq->kind == EFFORT_KIND_FP16 &&
        m->layers[0].wq->buckets) {
        // Fused glue (single GPU, FP16): rmsNorm*w is applied on load inside the bucketMul kernels from per-block
        // sum(h^2) partials, the residual add and silu*mul ride in the integrate epilogues: 9 launches per layer.
        const size_t pf = partial_floats(ctx, m->layers[0].wq);
        if ((rc = ensure_mul_scratch(ctx, 3 * pf, kMaxBatch))) return rc;
        int n_sumsq = 4;  // embed_kernel grid
        auto with_norm = [&](MulCall& mc, const __half* w, const float* sumsq, int n) {
            mc.pb.norm_w = w; mc.pb.sumsq = sumsq; mc.pb.n_sumsq = n; mc.pb.norm_dim = c.dim; mc.pb.norm_eps = c.norm_eps;
        };
        auto blocks_of = [&](const effort_weights* w) { return make_geom<4>(w->C, ctx->n_sms).CS * (16 * 128) / 32; };  // integrate grid.x
        for (int li = 0; li < c.n_layers; li++) {
            auto& l = m->layers[li];
            if (!l.wq) return EFFORT_ESTATE;
            MulCall qkv[3] = {make_call(ctx, m->h, l.wq, nullptr, m->xq, effort, 0, 0, 0),
                              make_call(ctx, m->h, l.wk, nullptr, m->xk, effort, 0, 1, pf),
                              make_call(ctx, m->h, l.wv, nullptr, m->xv, effort, 0, 2, 2 * pf)};
            for (auto& mc : qkv) with_norm(mc, l.attn_norm, m->sumsq_a, n_sumsq);
            if ((rc = launch_calls(ctx, qkv, 3, EFFORT_KIND_FP16, false, s))) return rc;
            CK(launch_pdl(attention_kernel, dim3(heads_l), dim3(256), 0, s, (const float*)m->xq, (const float*)m->xk,
                          (const float*)m->xv, l.kc, l.vc, (const int*)m->pos, heads_l, kv_l, c.rope_theta, c.max_seq, m->attn, ZeroList{}));
            LAUNCHED();
            MulCall wo = make_call(ctx, m->attn, l.wo, nullptr, m->h, effort, 0, 0, 0);
            wo.mode = kIntResidual; wo.sumsq = m->sumsq_b;  // h += wo(attn); sumsq_b = partial sum(h^2)
            if ((rc = launch_calls(ctx, &wo, 1, EFFORT_KIND_FP16, false, s))) return rc;
            MulCall w13[2] = {make_call(ctx, m->h, l.w1, nullptr, m->x2, effort, 0, 0, 0),
                              make_call(ctx, m->h, l.w3, nullptr, m->x3, effort, 0, 1, pf)};
            for (auto& mc : w13) { with_norm(mc, l.ffn_norm, m->sumsq_b, blocks_of(l.wo)); mc.mode = kIntSiluPair; }
            if ((rc = launch_calls(ctx, w13, 2, EFFORT_KIND_FP16, false, s))) return rc;
            MulCall w2 = make_call(ctx, m->x2, l.w2, nullptr, m->h, effort, 0, 0, 0);
            w2.mode = kIntResidual; w2.sumsq = m->sumsq_a;  // h += w2(x2)
            if ((rc = launch_calls(ctx, &w2, 1, EFFORT_KIND_FP16, false, s))) return rc;
            n_sumsq = blocks_of(l.w2);
        }
        CK(launch_pdl(add_rmsnorm_kernel, dim3(1), dim3(1024), 0, s, m->h, (const float*)nullptr, m->norm, c.dim,
                      c.norm_eps, m->out_normed));
        LAUNCHED();
        if ((rc = enqueue_basic_mul(m->out_normed, m->out_core, c.vocab, c.dim, m->logits, ctx->n_sms, s))) return rc;
        CK(launch_pdl(argmax_advance_kernel, dim3(1), dim3(1024), 0, s, (const float*)m->logits, c.vocab, m->next, m->pos));
        LAUNCHED();
        return model_enqueue_tail(m, s);
    }
    // tensor parallel with the one-shot NVLink collectives: the all-reduce of each row-parallel GEMV is fused with
    // the residual add and the following rmsNorm*w, the x2 all-gather with silu*mul (csrc/comm.cuh)
    const bool p2p = G > 1 && ctx->p2p_ready && p2p_enabled() && c.dim <= 4 * kP2PThreads && (size_t)c.hidden_dim * 8 <= kP2PSiteBytes;
    auto p2p_args = [&](int site) {
        P2PArgs a{};
        for (int p = 0; p < G; p++) a.peer[p] = (unsigned char*)ctx->p2p_peer[p];
        a.rank = ctx->comm_rank; a.world = G; a.site = site; a.err = ctx->v2_err;
        return a;
    };
    for (int li = 0; li < c.n_layers; li++) {
        auto& l = m->layers[li];
        if (!l.wq) return EFFORT_ESTATE;
        if (!p2p || li == 0) {
            CK(launch_pdl(add_rmsnorm_kernel, dim3(1), dim3(1024), 0, s, m->h, (const float*)((li && !p2p) ? m->ffn_out : nullptr),
                          l.attn_norm, c.dim, c.norm_eps, m->h_norm));
            LAUNCHED();
        }  // else: h_norm was produced by the previous layer's fused all-reduce
        effort_mul_args_t qkv[3] = {{m->h_norm, l.wq, nullptr, m->xq, effort, nullptr},
                                    {m->h_norm, l.wk, nullptr, m->xk, effort, nullptr},
                                    {m->h_norm, l.wv, nullptr, m->xv, effort, nullptr}};
        if ((rc = effort_expert_mul_batch(ctx, qkv, 3, s))) return rc;
        CK(launch_pdl(attention_kernel, dim3(heads_l), dim3(256), 0, s, (const float*)m->xq, (const float*)m->xk,
                      (const float*)m->xv, l.kc, l.vc, (const int*)m->pos, heads_l, kv_l, c.rope_theta, c.max_seq, m->attn, ZeroList{}));
        LAUNCHED();
        const float* wo_cut = nullptr;
        if (G > 1) {
            if ((rc = comm_all_gather_site(ctx, 0, m->attn, m->attn_full, dim_l, s))) return rc;
            wo_cut = m->attn_full;
        }
        effort_mul_args_t wo = {m->attn, l.wo, nullptr, m->attn_ffn_out, effort, wo_cut};
        if ((rc = effort_expert_mul_batch(ctx, &wo, 1, s))) return rc;
        if (p2p) {
            CK(launch_pdl(p2p_allreduce_residual_rmsnorm_kernel, dim3(1), dim3(kP2PThreads), 0, s, p2p_args(1),
                          (const float*)m->attn_ffn_out, m->h, l.ffn_norm, c.dim, c.norm_eps, m->fxn));
            LAUNCHED();
        } else {
            if (G > 1 && (rc = comm_all_reduce_site(ctx, 1, m->attn_ffn_out, c.dim, s))) return rc;
            CK(launch_pdl(add_rmsnorm_kernel, dim3(1), dim3(1024), 0, s, m->h, (const float*)m->attn_ffn_out, l.ffn_norm,
                          c.dim, c.norm_eps, m->fxn));
            LAUNCHED();
        }
        effort_mul_args_t w13[2] = {{m->fxn, l.w1, nullptr, m->x1, effort, nullptr}, {m->fxn, l.w3, nullptr, m->x3, effort, nullptr}};
        if ((rc = effort_expert_mul_batch(ctx, w13, 2, s))) return rc;
        const float* w2_cut = nullptr;
        if (p2p) {
            CK(launch_pdl(p2p_silu_allgather_kernel, dim3(1), dim3(kP2PThreads), 0, s, p2p_args(2), (const float*)m->x1,
                          (const float*)m->x3, hid_l, m->x2, m->x2_full));
            LAUNCHED();
            w2_cut = m->x2_full;
        } else {
            CK(launch_pdl(silu_mul_kernel, dim3((hid_l + 255) / 256), dim3(256), 0, s, (const float*)m->x1,
                          (const float*)m->x3, hid_l, m->x2));
            LAUNCHED();
            if (G > 1) {
                if ((rc = comm_all_gather_site(ctx, 2, m->x2, m->x2_full, hid_l, s))) return rc;
                w2_cut = m->x2_full;
            }
        }
        effort_mul_args_t w2 = {m->x2, l.w2, nullptr, m->ffn_out, effort, w2_cut};
        if ((rc = effort_expert_mul_batch(ctx, &w2, 1, s))) return rc;
        if (p2p) {  // h += all-reduce(ffn_out); the norm that follows is the next layer's attention norm or the final norm
            const bool last = li + 1 == c.n_layers;
            CK(launch_pdl(p2p_allreduce_residual_rmsnorm_kernel, dim3(1), dim3(kP2PThreads), 0, s, p2p_args(3),
                          (const float*)m->ffn_out, m->h, last ? m->norm : m->layers[li + 1].attn_norm, c.dim, c.norm_eps,
                          last ? m->out_normed : m->h_norm));
            LAUNCHED();
        } else if (G > 1 && (rc = comm_all_reduce_site(ctx, 3, m->ffn_out, c.dim, s))) return rc;
    }
    if (!p2p) {
        CK(launch_pdl(add_rmsnorm_kernel, dim3(1), dim3(1024), 0, s, m->h, (const float*)m->ffn_out, m->norm, c.dim,
                      c.norm_eps, m->out_normed));
        LAUNCHED();
    }
    if (G > 1) {  // vocab-sharded lm_head + all-gather of the logits
        if ((rc = enqueue_basic_mul(m->out_normed, m->out_core, c.vocab / G, c.dim, m->logits_local, ctx->n_sms, s))) return rc;
        if ((rc = comm_all_gather_site(ctx, 4, m->logits_local, m->logits, c.vocab / G, s))) return rc;
    } else {
        if ((rc = enqueue_basic_mul(m->out_normed, m->out_core, c.vocab, c.dim, m->logits, ctx->n_sms, s))) return rc;
    }
    CK(launch_pdl(argmax_advance_kernel, dim3(1), dim3(1024), 0, s, (const float*)m->logits, c.vocab, m->next, m->pos));
    LAUNCHED();
    return model_enqueue_tail(m, s);
}

extern "C" int effort_model_step(effort_model_t* m, const int32_t* token_dev, double effort, void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    if (!m) return EFFORT_EINVAL;
    if (!(effort >= 0.0 && effort <= 1.0)) return EFFORT_EINVAL;
    if (m->host_pos >= m->cfg.max_seq) return EFFORT_ESTATE;  // KV cache full (the reference bounds the loop by maxSeqLen)
    m->host_pos++;
    CK(cudaMemcpyAsync(m->token, token_dev ? (const void*)token_dev : (const void*)m->next, sizeof(int),
                       cudaMemcpyDeviceToDevice, s));
    if (m->sampling && m->sampler_dirty) {
        CK(cudaMemcpyAsync(m->sampler_dev, m->sampler_host, sizeof(effort_sampler_t), cudaMemcpyHostToDevice, s));
        CK(cudaEventRecord(m->sampler_copied, s));
        m->sampler_dirty = false;
    }
    const int key = effort_q(effort, EFFORT_PROBES_COUNT);
    if (!m->use_graphs || s == nullptr) return model_enqueue_token(m, effort, s);  // legacy stream cannot capture
    auto it = m->graphs.find(key);
    if (it == m->graphs.end()) {
        if (!m->warmed) {  // first token: eager (allocates scratch, sets kernel attributes)
            m->warmed = true;
            return model_enqueue_token(m, effort, s);
        }
        cudaGraph_t g = nullptr;
        const uint64_t l0 = g_launches.load();
        CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
        int rc = model_enqueue_token(m, effort, s);
        cudaError_t e = cudaStreamEndCapture(s, &g);
        if (rc) { if (g) cudaGraphDestroy(g); return rc; }
        CK(e);
        cudaGraphExec_t ge = nullptr;
        CK(cudaGraphInstantiate(&ge, g, 0));
        CK(cudaGraphDestroy(g));
        m->graphs[key] = ge;
        m->graph_path[key] = m->path;
        it = m->graphs.find(key);
        m->launches_per_token = g_launches.load() - l0;
        g_launches.store(l0);  // captured, not launched: the replay below counts them
    }
    CK(cudaGraphLaunch(it->second, s));
    m->path = m->graph_path[key];
    g_launches.fetch_add(m->launches_per_token);  // kernels one replay launches
    return EFFORT_OK;
}

extern "C" int effort_model_step_host(effort_model_t* m, const int32_t* token_host, double effort,
                                      int32_t* next_token_host, float* logits_host, void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    if (!m) return EFFORT_EINVAL;
    const int32_t* tok_dev = nullptr;
    if (token_host) {
        *m->h_token = *token_host;
        CK(cudaMemcpyAsync(m->next, m->h_token, sizeof(int), cudaMemcpyHostToDevice, s));  // staged through `next`
    }
    int rc = effort_model_step(m, tok_dev, effort, stream_);
    if (rc) return rc;
    CK(cudaMemcpyAsync(m->h_next, m->next, sizeof(int), cudaMemcpyDeviceToHost, s));
    if (logits_host) CK(cudaMemcpyAsync(m->h_logits, m->logits, sizeof(float) * m->cfg.vocab, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    if (next_token_host) *next_token_host = *m->h_next;
    if (logits_host) memcpy(logits_host, m->h_logits, sizeof(float) * m->cfg.vocab);
    return EFFORT_OK;
}

// ---- prefill: up to kPrefillMax tokens per pass (DESIGN.md section 4.8) ---------------------------------------------
// Per layer: rmsNorm*w (T vectors) -> [q,k,v] multi-token GEMV -> chunk attention (appends T cache rows) -> wo accumulated
// into the residual rows -> rmsNorm*w -> [w1,w3] -> silu*mul -> w2 accumulated into the residual rows.  Then the head on
// the last row (or, with scoring, the dense lm_head for every row), the sampler and the scorer, as a step ends.
static bool model_prefill_fused(const effort_model* m) {
    if (m->cfg.tp_size != 1 || m->chain != 2 || m->ctx->engine != 2 || m->ctx->cutoff_mode != EFFORT_CUTOFF_SELECT ||
        !m->norm || !model_all_fp16_v2(m))
        return false;
    for (const auto& l : m->layers) {
        if (l.gate) return false;
        for (const effort_weights* w : {l.wq, l.wk, l.wv, l.wo, l.w1, l.w2, l.w3})
            if (!prefill_supported(w)) return false;
    }
    return true;
}

// the row buffers [T][...] one layer of multi-token groups reads and writes (a model's prefill chunk, or a batch step)
struct RowBuffers {
    float *h, *xn, *q, *k, *v, *attn, *x1, *x3, *x2;
};

static int row_groups(const effort_ctx* ctx, const effort_model::Layer& l, double effort, const RowBuffers& r, PrefillGroup g[4]) {
    for (int k = 0; k < 4; k++) g[k] = PrefillGroup{};
    g[0].n = 3; g[0].V = r.xn;
    g[0].p[0] = prefill_problem(ctx, l.wq, effort, r.q, 0);
    g[0].p[1] = prefill_problem(ctx, l.wk, effort, r.k, 0);
    g[0].p[2] = prefill_problem(ctx, l.wv, effort, r.v, 0);
    g[1].n = 1; g[1].V = r.attn;
    g[1].p[0] = prefill_problem(ctx, l.wo, effort, r.h, 1);
    g[2].n = 2; g[2].V = r.xn;
    g[2].p[0] = prefill_problem(ctx, l.w1, effort, r.x1, 0);
    g[2].p[1] = prefill_problem(ctx, l.w3, effort, r.x3, 0);
    g[3].n = 1; g[3].V = r.x2;
    g[3].p[0] = prefill_problem(ctx, l.w2, effort, r.h, 1);
    return EFFORT_OK;
}

// partial-sum floats and count words the largest group of a layer needs at T = kPrefillMax (every layer has the same shapes)
static void row_scratch_need(const effort_model* m, size_t* nf, size_t* nc) {
    *nf = 0; *nc = 0;
    PrefillGroup g[4];
    row_groups(m->ctx, m->layers[0], 1.0, RowBuffers{}, g);
    for (auto& gr : g) {
        size_t f, k;
        prefill_scratch_need(gr, &f, &k);
        *nf = f > *nf ? f : *nf;
        *nc = k > *nc ? k : *nc;
    }
}

static int prefill_groups(effort_model* m, const effort_model::Layer& l, double effort, PrefillGroup g[4]) {
    return row_groups(m->ctx, l, effort,
                      RowBuffers{m->pf_h, m->pf_xn, m->pf_q, m->pf_k, m->pf_v, m->pf_attn, m->pf_x1, m->pf_x3, m->pf_x2}, g);
}

static int model_prefill_buffers(effort_model* m) {
    if (m->pf_ready) return EFFORT_OK;
    const auto& c = m->cfg;
    const size_t T = kPrefillMax, kvd = (size_t)c.n_kv_heads * c.head_dim;
    size_t nf, nc;
    row_scratch_need(m, &nf, &nc);
    int rc;
    if ((rc = model_alloc(m, m->pf_h, T * c.dim)) || (rc = model_alloc(m, m->pf_xn, T * c.dim)) ||
        (rc = model_alloc(m, m->pf_q, T * c.dim)) || (rc = model_alloc(m, m->pf_k, T * kvd)) ||
        (rc = model_alloc(m, m->pf_v, T * kvd)) || (rc = model_alloc(m, m->pf_attn, T * c.dim)) ||
        (rc = model_alloc(m, m->pf_x1, T * c.hidden_dim)) || (rc = model_alloc(m, m->pf_x3, T * c.hidden_dim)) ||
        (rc = model_alloc(m, m->pf_x2, T * c.hidden_dim)) || (rc = model_alloc(m, m->pf_logits, T * c.vocab)) ||
        (rc = model_alloc(m, m->pf_part, nf)) || (rc = model_alloc(m, m->pf_cnt, nc)) ||
        (rc = model_alloc(m, m->pf_cut, (size_t)kPrefillMax * kPrefillMaxProblems)) || (rc = model_alloc(m, m->pf_tok, T)) ||
        (rc = model_alloc(m, m->pf_lens, T + 1)))
        return rc;
    int lens[kPrefillMax + 1];
    for (int i = 0; i <= kPrefillMax; i++) lens[i] = i;
    CK(cudaMemcpy(m->pf_lens, lens, sizeof(lens), cudaMemcpyHostToDevice));
    // kernel attributes before any capture
    CK(cudaFuncSetAttribute(chunk_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (2 * kChunkAttnTile + kChunkAttnPairs) * 128 * (int)sizeof(float)));
    CK(cudaFuncSetAttribute(prefill_head_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)(T * c.dim * sizeof(__half))));
    m->pf_ready = true;
    return EFFORT_OK;
}

// one chunk of T tokens already in pf_tok, at the device position (no graph logic)
static int model_enqueue_chunk(effort_model* m, double effort, int T, cudaStream_t s) {
    const auto& c = m->cfg;
    effort_ctx* ctx = m->ctx;
    int rc;
    CK(launch_pdl(prefill_embed_kernel, dim3(T), dim3(256), 0, s, (const int*)m->pf_tok, m->emb, c.dim, c.vocab, m->pf_h));
    LAUNCHED();
    const int G = c.n_heads / c.n_kv_heads;
    const dim3 attn_grid(c.n_kv_heads, (G * T + kChunkAttnPairs - 1) / kChunkAttnPairs);
    const size_t attn_smem = (size_t)(2 * kChunkAttnTile + kChunkAttnPairs) * 128 * sizeof(float);
    for (int li = 0; li < c.n_layers; li++) {
        const auto& l = m->layers[li];
        PrefillGroup g[4];
        prefill_groups(m, l, effort, g);
        for (auto& gr : g) gr.T = T;
        CK(launch_pdl(prefill_rmsnorm_kernel, dim3(T), dim3(1024), 0, s, (const float*)m->pf_h, l.attn_norm, c.dim, c.norm_eps, m->pf_xn));
        LAUNCHED();
        if ((rc = enqueue_prefill_group(ctx, g[0], m->pf_part, m->pf_cnt, m->pf_cut, s))) return rc;
        CK(launch_pdl(chunk_attention_kernel, attn_grid, dim3(kChunkAttnThreads), attn_smem, s, (const float*)m->pf_q,
                      (const float*)m->pf_k, (const float*)m->pf_v, T, l.kc, l.vc, (const int*)m->pos, c.n_heads, c.n_kv_heads,
                      c.rope_theta, c.max_seq, m->pf_attn));
        LAUNCHED();
        if ((rc = enqueue_prefill_group(ctx, g[1], m->pf_part, m->pf_cnt, m->pf_cut, s))) return rc;
        CK(launch_pdl(prefill_rmsnorm_kernel, dim3(T), dim3(1024), 0, s, (const float*)m->pf_h, l.ffn_norm, c.dim, c.norm_eps, m->pf_xn));
        LAUNCHED();
        if ((rc = enqueue_prefill_group(ctx, g[2], m->pf_part, m->pf_cnt, m->pf_cut, s))) return rc;
        const int nx = T * c.hidden_dim;
        CK(launch_pdl(silu_mul_kernel, dim3((nx + 255) / 256), dim3(256), 0, s, (const float*)m->pf_x1, (const float*)m->pf_x3, nx,
                      m->pf_x2));
        LAUNCHED();
        if ((rc = enqueue_prefill_group(ctx, g[3], m->pf_part, m->pf_cnt, m->pf_cut, s))) return rc;
    }
    CK(launch_pdl(prefill_advance_kernel, dim3(1), dim3(1), 0, s, m->pos, T - 1));
    LAUNCHED();
    m->pf_scored = m->scoring;
    if (m->scoring) {  // logits for every row: the dense lm_head on rmsNorm(h[t]) * norm, then greedy on the last row
        CK(launch_pdl(prefill_rmsnorm_kernel, dim3(T), dim3(1024), 0, s, (const float*)m->pf_h, m->norm, c.dim, c.norm_eps, m->pf_xn));
        LAUNCHED();
        int grid = (c.vocab + 7) / 8;
        if (grid > ctx->n_sms * 2) grid = ctx->n_sms * 2;
        CK(launch_pdl(prefill_head_kernel, dim3(grid), dim3(256), (size_t)T * c.dim * sizeof(__half), s, (const float*)m->pf_xn, T,
                      m->out_core, c.vocab, c.dim, m->pf_logits, m->logits));
        LAUNCHED();
        CK(launch_pdl(argmax_advance_kernel, dim3(1), dim3(1024), 0, s, (const float*)m->logits, c.vocab, m->next, m->pos));
        LAUNCHED();
        if ((rc = model_enqueue_sample(m, s))) return rc;
        // records p0 .. p0+T-1 from the chunk's rows (score_kernel: record pos - T + block)
        return enqueue_score(m->pf_logits, c.vocab, m->score_targets, c.max_seq, m->pos, T, m->scores, s, c.vocab);
    }
    if ((rc = enqueue_head(m, m->pf_h + (size_t)(T - 1) * c.dim, m->norm, m->out_core, c.vocab, 0, m->logits, true, s))) return rc;
    return model_enqueue_sample(m, s);
}

static int prefill_graph_key(double effort, int T) { return (T << 12) | effort_q(effort, EFFORT_PROBES_COUNT); }

static int model_prefill_chunk(effort_model* m, double effort, int T, cudaStream_t s) {
    if (!m->use_graphs || s == nullptr || !m->pf_warmed) {  // the first chunk runs eagerly, as the first step does
        m->pf_warmed = m->pf_warmed || (m->use_graphs && s != nullptr);
        m->path = 3; m->pf_len = T;
        return model_enqueue_chunk(m, effort, T, s);
    }
    const int key = prefill_graph_key(effort, T);
    auto it = m->graphs.find(key);
    if (it == m->graphs.end()) {
        cudaGraph_t g = nullptr;
        const uint64_t l0 = g_launches.load();
        CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
        int rc = model_enqueue_chunk(m, effort, T, s);
        cudaError_t e = cudaStreamEndCapture(s, &g);
        if (rc) { if (g) cudaGraphDestroy(g); return rc; }
        CK(e);
        cudaGraphExec_t ge = nullptr;
        CK(cudaGraphInstantiate(&ge, g, 0));
        CK(cudaGraphDestroy(g));
        m->graphs[key] = ge;
        m->graph_path[key] = 3;
        m->pf_launches[key] = g_launches.load() - l0;
        g_launches.store(l0);
        it = m->graphs.find(key);
    }
    CK(cudaGraphLaunch(it->second, s));
    m->path = 3; m->pf_len = T; m->pf_scored = m->scoring;
    g_launches.fetch_add(m->pf_launches[key]);
    return EFFORT_OK;
}

extern "C" int effort_model_prefill(effort_model_t* m, const int32_t* tokens_dev, int n, double effort, void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    if (!m || !tokens_dev || n < 1 || !(effort >= 0.0 && effort <= 1.0)) return EFFORT_EINVAL;
    if (n > m->cfg.max_seq - m->host_pos) return EFFORT_ESTATE;  // the KV cache would overflow
    int rc;
    if (!model_prefill_fused(m)) {  // every other configuration steps: the same launches and bits as n steps
        for (int i = 0; i < n; i++)
            if ((rc = effort_model_step(m, tokens_dev + i, effort, stream_))) return rc;
        return EFFORT_OK;
    }
    if ((rc = model_prefill_buffers(m))) return rc;
    if (m->sampling && m->sampler_dirty) {
        CK(cudaMemcpyAsync(m->sampler_dev, m->sampler_host, sizeof(effort_sampler_t), cudaMemcpyHostToDevice, s));
        CK(cudaEventRecord(m->sampler_copied, s));
        m->sampler_dirty = false;
    }
    for (int c0 = 0; c0 < n; c0 += kPrefillMax) {
        const int T = n - c0 < kPrefillMax ? n - c0 : kPrefillMax;
        CK(cudaMemcpyAsync(m->pf_tok, tokens_dev + c0, sizeof(int32_t) * T, cudaMemcpyDeviceToDevice, s));
        m->host_pos += T;
        if ((rc = model_prefill_chunk(m, effort, T, s))) return rc;
    }
    return EFFORT_OK;
}

// ---- batch decode: up to kPrefillMax sequences per step, each with its own state (DESIGN.md section 4.9) -------------
// A step is prefill's per-row path with one row per slot: embed, per layer rmsNorm*w rows -> [q,k,v] -> batch attention
// (each slot on its own cache at its own position) -> wo into the residual rows -> rmsNorm*w -> [w1,w3] -> silu*mul -> w2
// into the residual rows, then the final norm, the lm_head for every row, and each slot's tail as a model step ends it.
struct effort_batch {
    effort_model* m = nullptr;
    int n = 0;                                 // slots
    size_t slot_kv = 0;                        // floats of one slot's cache of one layer: max_seq * n_kv * 128
    std::vector<float*> kc, vc;                // per layer: [n][max_seq][n_kv][128]
    RowBuffers r{};                            // [n][...]
    float* logits = nullptr;                   // [n + 1][vocab]: one row per slot, and a sink for the head's "last row" copy
    float *part = nullptr, *cut = nullptr;     // multi-token GEMV scratch, owned: a batch never shares the model's
    uint32_t* cnt = nullptr;
    int *pos = nullptr, *tok = nullptr, *next = nullptr;  // [n]
    std::vector<int> host_pos;                 // mirrors pos: bounds every slot's cache
    std::vector<char> sampling;                // per slot: a sampler is set
    bool sampler_dirty = false;
    effort_sampler_t* sampler_dev = nullptr;   // [n], refreshed from the pinned sampler_host on the stream when it changed
    effort_sampler_t* sampler_host = nullptr;
    cudaEvent_t sampler_copied = nullptr;      // the last copy out of sampler_host has run
    bool scoring = false;
    int32_t* score_targets = nullptr;          // [n][max_seq], -1 = no target
    effort_score_t* scores = nullptr;          // [n][max_seq]
    bool warmed = false, stepped = false;
    std::map<int, cudaGraphExec_t> graphs;     // keyed by q = Int(4095*(1-effort))
    std::map<int, uint64_t> graph_launches;    // kernels one replay launches
    std::vector<void*> owned;
};

template <typename T>
static int batch_alloc(effort_batch* b, T*& p, size_t n) {
    const cudaError_t e = cudaMalloc(&p, n * sizeof(T));
    if (e == cudaErrorMemoryAllocation) { cudaGetLastError(); p = nullptr; return EFFORT_ENOMEM; }
    CK(e);
    b->owned.push_back(p);
    CK(cudaMemset(p, 0, n * sizeof(T)));
    return EFFORT_OK;
}

static void batch_drop_graphs(effort_batch* b) {
    for (auto& g : b->graphs) cudaGraphExecDestroy(g.second);
    b->graphs.clear();
}

static int batch_create_buffers(effort_batch* b) {
    const auto& c = b->m->cfg;
    const size_t N = b->n, kvd = (size_t)c.n_kv_heads * c.head_dim;
    b->slot_kv = (size_t)c.max_seq * kvd;
    b->kc.assign(c.n_layers, nullptr);
    b->vc.assign(c.n_layers, nullptr);
    int rc;
    for (int li = 0; li < c.n_layers; li++)
        if ((rc = batch_alloc(b, b->kc[li], N * b->slot_kv)) || (rc = batch_alloc(b, b->vc[li], N * b->slot_kv))) return rc;
    size_t nf, nc;
    row_scratch_need(b->m, &nf, &nc);
    RowBuffers& r = b->r;
    if ((rc = batch_alloc(b, r.h, N * c.dim)) || (rc = batch_alloc(b, r.xn, N * c.dim)) || (rc = batch_alloc(b, r.q, N * c.dim)) ||
        (rc = batch_alloc(b, r.k, N * kvd)) || (rc = batch_alloc(b, r.v, N * kvd)) || (rc = batch_alloc(b, r.attn, N * c.dim)) ||
        (rc = batch_alloc(b, r.x1, N * c.hidden_dim)) || (rc = batch_alloc(b, r.x3, N * c.hidden_dim)) ||
        (rc = batch_alloc(b, r.x2, N * c.hidden_dim)) || (rc = batch_alloc(b, b->logits, (N + 1) * c.vocab)) ||
        (rc = batch_alloc(b, b->part, nf)) || (rc = batch_alloc(b, b->cnt, nc)) ||
        (rc = batch_alloc(b, b->cut, (size_t)kPrefillMax * kPrefillMaxProblems)) || (rc = batch_alloc(b, b->pos, N)) ||
        (rc = batch_alloc(b, b->tok, N)) || (rc = batch_alloc(b, b->next, N)) || (rc = batch_alloc(b, b->sampler_dev, N)) ||
        (rc = batch_alloc(b, b->score_targets, N * c.max_seq)) || (rc = batch_alloc(b, b->scores, N * c.max_seq)))
        return rc;
    CK(cudaMemset(b->score_targets, 0xff, sizeof(int32_t) * N * c.max_seq));  // all -1: no target
    if (cudaMallocHost(&b->sampler_host, sizeof(effort_sampler_t) * N) != cudaSuccess) {
        cudaGetLastError();
        b->sampler_host = nullptr;
        return EFFORT_ENOMEM;
    }
    CK(cudaEventCreateWithFlags(&b->sampler_copied, cudaEventDisableTiming));
    b->host_pos.assign(N, 0);
    b->sampling.assign(N, 0);
    // kernel attributes before any capture
    CK(cudaFuncSetAttribute(prefill_head_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)(kPrefillMax * c.dim * sizeof(__half))));
    return EFFORT_OK;
}

extern "C" int effort_batch_create(effort_model_t* m, int n_seq, effort_batch_t** out) {
    if (!m || !out || n_seq < 1 || n_seq > kPrefillMax) return EFFORT_EINVAL;
    *out = nullptr;
    if (!model_prefill_fused(m)) return EFFORT_ESHAPE;
    effort_batch* b = new (std::nothrow) effort_batch();
    if (!b) return EFFORT_ENOMEM;
    b->m = m;
    b->n = n_seq;
    const int rc = batch_create_buffers(b);
    if (rc) {  // release what was allocated so far
        effort_batch_destroy(b);
        return rc;
    }
    *out = b;
    return EFFORT_OK;
}

extern "C" int effort_batch_destroy(effort_batch_t* b) {
    if (!b) return EFFORT_EINVAL;
    batch_drop_graphs(b);
    for (void* p : b->owned) cudaFree(p);
    cudaFreeHost(b->sampler_host);
    if (b->sampler_copied) cudaEventDestroy(b->sampler_copied);
    delete b;
    return EFFORT_OK;
}

// seq = -1: every slot
static bool batch_slots(const effort_batch* b, int seq, int* s0, int* s1) {
    if (seq < -1 || seq >= b->n) return false;
    *s0 = seq < 0 ? 0 : seq;
    *s1 = seq < 0 ? b->n : seq + 1;
    return true;
}

extern "C" int effort_batch_reset(effort_batch_t* b, int seq, void* stream) {
    int s0, s1;
    if (!b || !batch_slots(b, seq, &s0, &s1)) return EFFORT_EINVAL;
    CK(cudaMemsetAsync(b->pos + s0, 0, sizeof(int) * (s1 - s0), (cudaStream_t)stream));
    for (int i = s0; i < s1; i++) b->host_pos[i] = 0;
    return EFFORT_OK;
}

extern "C" int effort_batch_set_sampler(effort_batch_t* b, int seq, const effort_sampler_t* sp) {
    int s0, s1;
    if (!b || !batch_slots(b, seq, &s0, &s1) || (sp && !sampler_valid(sp))) return EFFORT_EINVAL;
    CK(cudaEventSynchronize(b->sampler_copied));  // a copy still queued reads the pinned block
    for (int i = s0; i < s1; i++) {
        if (b->sampling[i] != (sp != nullptr)) batch_drop_graphs(b);  // the step's launch sequence changes
        b->sampling[i] = sp != nullptr;
        if (sp) {
            b->sampler_host[i] = *sp;
            b->sampler_dirty = true;
        }
    }
    return EFFORT_OK;
}

extern "C" int effort_batch_set_scoring(effort_batch_t* b, int enable) {
    if (!b) return EFFORT_EINVAL;
    if (b->scoring != (enable != 0)) batch_drop_graphs(b);
    b->scoring = enable != 0;
    return EFFORT_OK;
}

extern "C" int effort_batch_set_score_targets(effort_batch_t* b, int seq, const int32_t* targets_dev, int n, void* stream) {
    int s0, s1;
    if (!b || !batch_slots(b, seq, &s0, &s1)) return EFFORT_EINVAL;
    const int max_seq = b->m->cfg.max_seq;
    if (n < 0 || n > max_seq || (!targets_dev && n > 0)) return EFFORT_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;
    for (int i = s0; i < s1; i++) {
        int32_t* row = b->score_targets + (size_t)i * max_seq;
        if (n > 0) CK(cudaMemcpyAsync(row, targets_dev, sizeof(int32_t) * n, cudaMemcpyDeviceToDevice, s));
        if (n < max_seq) CK(cudaMemsetAsync(row + n, 0xff, sizeof(int32_t) * (max_seq - n), s));
    }
    return EFFORT_OK;
}

extern "C" const float* effort_batch_logits(const effort_batch_t* b) { return b ? b->logits : nullptr; }
extern "C" const int32_t* effort_batch_next_tokens(const effort_batch_t* b) { return b ? b->next : nullptr; }
extern "C" const effort_score_t* effort_batch_scores(const effort_batch_t* b) { return b ? b->scores : nullptr; }

extern "C" const void* effort_batch_buffer(const effort_batch_t* b, int which, int layer, int seq, size_t* count) {
    if (count) *count = 0;
    if (!b) return nullptr;
    const auto& c = b->m->cfg;
    const size_t N = b->n, kvd = (size_t)c.n_kv_heads * c.head_dim;
    const void* p = nullptr;
    size_t n = 0;
    switch (which) {
        case EFFORT_BUF_Q: if (b->stepped) { p = b->r.q; n = N * c.dim; } break;
        case EFFORT_BUF_K: if (b->stepped) { p = b->r.k; n = N * kvd; } break;
        case EFFORT_BUF_V: if (b->stepped) { p = b->r.v; n = N * kvd; } break;
        case EFFORT_BUF_ATTN: if (b->stepped) { p = b->r.attn; n = N * c.dim; } break;
        case EFFORT_BUF_KCACHE:
        case EFFORT_BUF_VCACHE:
            if (layer < 0 || layer >= c.n_layers || seq < 0 || seq >= b->n) return nullptr;
            p = (which == EFFORT_BUF_KCACHE ? b->kc[layer] : b->vc[layer]) + (size_t)seq * b->slot_kv;
            n = b->slot_kv;
            break;
        case EFFORT_BUF_POS: p = b->pos; n = N; break;
        default: return nullptr;
    }
    if (p && count) *count = n;
    return p;
}

static int batch_flush_sampler(effort_batch* b, cudaStream_t s) {
    if (!b->sampler_dirty) return EFFORT_OK;
    CK(cudaMemcpyAsync(b->sampler_dev, b->sampler_host, sizeof(effort_sampler_t) * b->n, cudaMemcpyHostToDevice, s));
    CK(cudaEventRecord(b->sampler_copied, s));
    b->sampler_dirty = false;
    return EFFORT_OK;
}

// what a model step ends with, for slot i on its logits row: the greedy argmax that advances the slot's position, the
// slot's draw at that position, and with scoring on, record pos - 1 from the slot's target row
static int batch_enqueue_tail(effort_batch* b, int i, cudaStream_t s) {
    const auto& c = b->m->cfg;
    const float* row = b->logits + (size_t)i * c.vocab;
    CK(launch_pdl(argmax_advance_kernel, dim3(1), dim3(1024), 0, s, row, c.vocab, b->next + i, b->pos + i));
    LAUNCHED();
    int rc;
    if (b->sampling[i] &&
        (rc = enqueue_sample(b->m->ctx, row, c.vocab, b->sampler_host[i], b->sampler_dev + i, b->pos + i, 0u, b->next + i, s)))
        return rc;
    if (!b->scoring) return EFFORT_OK;
    return enqueue_score(row, c.vocab, b->score_targets + (size_t)i * c.max_seq, c.max_seq, b->pos + i, 1,
                         b->scores + (size_t)i * c.max_seq, s);
}

// one step of every slot, the tokens already in `tok` (no graph logic)
static int batch_enqueue_step(effort_batch* b, double effort, cudaStream_t s) {
    effort_model* m = b->m;
    const auto& c = m->cfg;
    effort_ctx* ctx = m->ctx;
    const int T = b->n;
    const RowBuffers& r = b->r;
    int rc;
    CK(launch_pdl(prefill_embed_kernel, dim3(T), dim3(256), 0, s, (const int*)b->tok, m->emb, c.dim, c.vocab, r.h));
    LAUNCHED();
    for (int li = 0; li < c.n_layers; li++) {
        const auto& l = m->layers[li];
        PrefillGroup g[4];
        row_groups(ctx, l, effort, r, g);
        for (auto& gr : g) gr.T = T;
        CK(launch_pdl(prefill_rmsnorm_kernel, dim3(T), dim3(1024), 0, s, (const float*)r.h, l.attn_norm, c.dim, c.norm_eps, r.xn));
        LAUNCHED();
        if ((rc = enqueue_prefill_group(ctx, g[0], b->part, b->cnt, b->cut, s))) return rc;
        CK(launch_pdl(batch_attention_kernel, dim3(c.n_heads, T), dim3(256), 0, s, (const float*)r.q, (const float*)r.k,
                      (const float*)r.v, b->kc[li], b->vc[li], b->slot_kv, (const int*)b->pos, c.n_heads, c.n_kv_heads,
                      c.rope_theta, c.max_seq, r.attn));
        LAUNCHED();
        if ((rc = enqueue_prefill_group(ctx, g[1], b->part, b->cnt, b->cut, s))) return rc;
        CK(launch_pdl(prefill_rmsnorm_kernel, dim3(T), dim3(1024), 0, s, (const float*)r.h, l.ffn_norm, c.dim, c.norm_eps, r.xn));
        LAUNCHED();
        if ((rc = enqueue_prefill_group(ctx, g[2], b->part, b->cnt, b->cut, s))) return rc;
        const int nx = T * c.hidden_dim;
        CK(launch_pdl(silu_mul_kernel, dim3((nx + 255) / 256), dim3(256), 0, s, (const float*)r.x1, (const float*)r.x3, nx, r.x2));
        LAUNCHED();
        if ((rc = enqueue_prefill_group(ctx, g[3], b->part, b->cnt, b->cut, s))) return rc;
    }
    CK(launch_pdl(prefill_rmsnorm_kernel, dim3(T), dim3(1024), 0, s, (const float*)r.h, m->norm, c.dim, c.norm_eps, r.xn));
    LAUNCHED();
    int grid = (c.vocab + 7) / 8;
    if (grid > ctx->n_sms * 2) grid = ctx->n_sms * 2;
    CK(launch_pdl(prefill_head_kernel, dim3(grid), dim3(256), (size_t)T * c.dim * sizeof(__half), s, (const float*)r.xn, T,
                  m->out_core, c.vocab, c.dim, b->logits, b->logits + (size_t)T * c.vocab));
    LAUNCHED();
    for (int i = 0; i < T; i++)
        if ((rc = batch_enqueue_tail(b, i, s))) return rc;
    return EFFORT_OK;
}

extern "C" int effort_batch_step(effort_batch_t* b, const int32_t* tokens_dev, double effort, void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    if (!b || !(effort >= 0.0 && effort <= 1.0)) return EFFORT_EINVAL;
    effort_model* m = b->m;
    if (!model_prefill_fused(m)) return EFFORT_ESHAPE;  // the chain or the context's options may have changed since create
    for (int i = 0; i < b->n; i++)
        if (b->host_pos[i] >= m->cfg.max_seq) return EFFORT_ESTATE;  // that slot's cache is full
    CK(cudaMemcpyAsync(b->tok, tokens_dev ? (const void*)tokens_dev : (const void*)b->next, sizeof(int32_t) * b->n,
                       cudaMemcpyDeviceToDevice, s));
    for (int& p : b->host_pos) p++;
    int rc;
    if ((rc = batch_flush_sampler(b, s))) return rc;
    b->stepped = true;
    if (!m->use_graphs || s == nullptr) return batch_enqueue_step(b, effort, s);  // legacy stream cannot capture
    const int key = effort_q(effort, EFFORT_PROBES_COUNT);
    auto it = b->graphs.find(key);
    if (it == b->graphs.end()) {
        if (!b->warmed) {  // first step: eager (sets kernel attributes), as the model's first step
            b->warmed = true;
            return batch_enqueue_step(b, effort, s);
        }
        cudaGraph_t g = nullptr;
        const uint64_t l0 = g_launches.load();
        CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
        rc = batch_enqueue_step(b, effort, s);
        cudaError_t e = cudaStreamEndCapture(s, &g);
        if (rc) { if (g) cudaGraphDestroy(g); return rc; }
        CK(e);
        cudaGraphExec_t ge = nullptr;
        CK(cudaGraphInstantiate(&ge, g, 0));
        CK(cudaGraphDestroy(g));
        b->graphs[key] = ge;
        b->graph_launches[key] = g_launches.load() - l0;
        g_launches.store(l0);  // captured, not launched: the replay below counts them
        it = b->graphs.find(key);
    }
    CK(cudaGraphLaunch(it->second, s));
    g_launches.fetch_add(b->graph_launches[key]);
    return EFFORT_OK;
}

extern "C" int effort_batch_fork(effort_batch_t* b, int seq, void* stream_) {
    cudaStream_t s = (cudaStream_t)stream_;
    int s0, s1;
    if (!b || !batch_slots(b, seq, &s0, &s1)) return EFFORT_EINVAL;
    effort_model* m = b->m;
    if (!model_prefill_fused(m)) return EFFORT_ESHAPE;
    const int p = m->host_pos;
    if (p == 0) return EFFORT_ESTATE;  // nothing to fork: no logits, no cache rows
    const auto& c = m->cfg;
    const size_t rows = (size_t)p * c.n_kv_heads * c.head_dim;
    int rc;
    if ((rc = batch_flush_sampler(b, s))) return rc;
    for (int i = s0; i < s1; i++) {
        for (int li = 0; li < c.n_layers; li++) {
            CK(cudaMemcpyAsync(b->kc[li] + (size_t)i * b->slot_kv, m->layers[li].kc, sizeof(float) * rows, cudaMemcpyDeviceToDevice, s));
            CK(cudaMemcpyAsync(b->vc[li] + (size_t)i * b->slot_kv, m->layers[li].vc, sizeof(float) * rows, cudaMemcpyDeviceToDevice, s));
        }
        CK(cudaMemcpyAsync(b->logits + (size_t)i * c.vocab, m->logits, sizeof(float) * c.vocab, cudaMemcpyDeviceToDevice, s));
        CK(cudaMemcpyAsync(b->pos + i, m->pos, sizeof(int), cudaMemcpyDeviceToDevice, s));
        // the tail's argmax advances the position, as the head of the step that produced the logits did: start one back
        CK(launch_pdl(prefill_advance_kernel, dim3(1), dim3(1), 0, s, b->pos + i, -1));
        LAUNCHED();
        if ((rc = batch_enqueue_tail(b, i, s))) return rc;
        b->host_pos[i] = p;
    }
    return EFFORT_OK;
}
