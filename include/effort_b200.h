/*
 * effort_b200.h -- C-ABI of the H100-native (sm_90a) bucketMul hot path.
 *
 * Drop-in boundary for kolinko/effort's approximate GEMV.  The reference has no
 * FFI layer today: its boundary is a handful of Swift free functions plus the
 * deliberately non-private BucketMul.shared test hooks.  Each entry point below
 * names the reference interface (file:line under the reference checkout) that
 * it replaces.  All pointers named *_dev are CUDA device pointers; `stream` is
 * a cudaStream_t passed as void* (0 = legacy default stream).  Every call that
 * takes a stream only ENQUEUES work on it (the reference's gpu.deploy is
 * enqueue-only, helpers/gpu.swift:135-196; completion = gpu.eval(), :109-119).
 * All functions return 0 or a negative EFFORT_E* code; nothing aborts (the
 * reference asserts, bucketMul.swift:35-36).
 *
 * No torch / C++ types cross this boundary.  The library fails at load time if
 * the CUDA runtime is missing; there is no CPU fallback.
 */
#ifndef EFFORT_B200_H
#define EFFORT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EFFORT_B200_VERSION 200

/* error codes */
#define EFFORT_OK 0
#define EFFORT_EINVAL (-1)    /* bad argument / failed reference precondition  */
#define EFFORT_ECUDA (-2)     /* CUDA runtime error (see effort_last_cuda_error) */
#define EFFORT_ENOMEM (-3)
#define EFFORT_ESHAPE (-4)    /* shape outside what the kernels support          */
#define EFFORT_ESTATE (-5)    /* e.g. effort_mul without a prior calc_dispatch    */
#define EFFORT_ENOTLOADED (-6)/* buckets not loaded and no dense core to fall back on */

/* weight kinds: main.swift:49-51 globals goQ4 / goQ8 (Q8 asserts false, expertMul.swift:33-36) */
#define EFFORT_KIND_FP16 0
#define EFFORT_KIND_Q4 1

/* effort_weights_create flags */
#define EFFORT_WEIGHTS_DEFAULT 0u
/* keep using the caller's rank-major buffers for the fast path too (no input-major device repack;
 * slower gathers, zero extra memory).  Without it the library builds its own repacked copy and the
 * caller's buckets/stats are only needed again by the effort_calc_dispatch/effort_mul test hooks. */
#define EFFORT_WEIGHTS_NO_REPACK 1u
/* device copy in the slice-major layout [column slice of 128][input][rank]: the rank rows an input selects inside a
 * column slice are contiguous, so a streaming unit is one cp.async.bulk (TMA) copy.  Round-2 engine only; the default
 * for FP16 weights (EFFORT_LAYOUT=input or EFFORT_ENGINE=1 in the environment makes input-major the default). */
#define EFFORT_WEIGHTS_SLICE_MAJOR 2u
/* device copy input-major ([input][rank][all columns]) even when slice-major is the default: what the round-1 engine reads */
#define EFFORT_WEIGHTS_INPUT_MAJOR 4u

#define EFFORT_PROBES_COUNT 4096 /* bucketMul.swift:19, loader.swift:66 */

typedef struct effort_ctx effort_ctx_t;         /* replaces the BucketMul.shared / BucketMulQ4.shared singletons
                                                   (bucketMul.swift:18-32): per-context scratch, one stream at a time */
typedef struct effort_weights effort_weights_t; /* replaces class ExpertWeights (loader.swift:46-167) */

/* ---- library ---------------------------------------------------------- */
int effort_version(void);
const char* effort_strerror(int code);
/* text of the last CUDA error seen by this thread's calls ("" if none) */
const char* effort_last_cuda_error(void);

/* ---- context ---------------------------------------------------------- */
/* Scratch: dispatch list (maxDispatchSize = 229376*2 float2 entries, bucketMul.swift:20-29),
 * cutoff scalar, partial-sum buffer (tmpMulVec [32,16384], bucketMul.swift:52 -> here [nCTA, out]).
 * `device` = CUDA device ordinal (-1 = current). */
int effort_ctx_create(int device, effort_ctx_t** ctx_out);
int effort_ctx_destroy(effort_ctx_t* ctx);
/*
 * How calcDispatch's cutoff (findCutoff32, bucketMul.metal:141-247) is computed by the fused operator:
 *   EFFORT_CUTOFF_SELECT (default)  the exact order statistic the reference's bisection approximates: the (k+1)-th
 *                                   largest of the 4096 bf16 probe products, k = 4096 - Int(4095*(1-effort)), so exactly
 *                                   k products lie above it (0 when k = 4096) -- a radix select, ~1 us;
 *   EFFORT_CUTOFF_BISECT            the reference's loop replayed bit for bit (same fp32 result and loop count).
 * Both satisfy the reference's own acceptance rule (count within 2 of k, bucketMul.metal:236).  effort_find_cutoff and
 * effort_calc_dispatch (the test hooks) always run the bisection.  Environment default: EFFORT_CUTOFF=bisect.
 */
#define EFFORT_CUTOFF_SELECT 0
#define EFFORT_CUTOFF_BISECT 1
int effort_ctx_set_cutoff_mode(effort_ctx_t* ctx, int mode);
/* Tuning / A-B knobs of the fused operator (tests and tools; every value computes the same operator):
 *   "engine"   2 (default) round-2 kernel: one launch per group, staged streaming, reductions into `out`;
 *              1 round-1 kernel + integrate launch (deterministic fp32 order)
 *   "stage"    4 (default) eight consumer warps accumulate, eight producer warps stage each pair's rows into a ring of
 *              four 16-row chunks with bulk async copies (cp.async.bulk, one per record piece) and hand the chunks over
 *              through mbarriers (slice-major FP16 weights; other weights take stage 0); 3 the same pairs and chunks fed by
 *              16-byte cp.async; 2 one TMA producer warp, a shared byte ring and 16 consumers (measured
 *              slower: the single producer's serial issue is the limit); 0 sixteen self-serving warps with private cp.async
 *              rings, units of at most 4 rows
 *   "dynamic"  per-warp rings (stage 0/1) only: 0 (default) static round robin of the units, 1 units from a shared counter
 *   "hint"     1 (default) stages 3-4: the exact select starts its search at the cutoff the same matrix produced on the
 *              previous call (3 rounds instead of 8 when it moved by less than 12 %; the result never depends on it)
 *   "prefetch" 0 (default) / 1 stages 3-4: while the cutoff is being computed, rows that the matrix's previous cutoff
 *              would select are prefetched into L2 (measured: no gain -- the gather is not DRAM-latency bound)
 * Returns EFFORT_EINVAL for an unknown name or value.  Environment defaults: EFFORT_ENGINE, EFFORT_STAGE (ldgsts|tma|pairs-ldgsts),
 * EFFORT_DYN, EFFORT_PREFETCH, EFFORT_HINT. */
int effort_ctx_set_option(effort_ctx_t* ctx, const char* name, int value);
/* Non-zero once a kernel of this context gave up a bounded wait: its output is invalid.  1 = the overwrite protocol
 * of a fused GEMV (co-resident CTAs never arrived), 2 / 3 = a consumer / producer warp of bucket_mul_v4 waited ~1 s on
 * its ring, 4 = a tensor-parallel exchange waited 2 s for a peer's packets (peer died or launched in another order).
 * Synchronises `stream`. */
int effort_ctx_error_flag(effort_ctx_t* ctx, unsigned* flag_out, void* stream);

/* ---- weights ---------------------------------------------------------- */
/*
 * ExpertWeights (loader.swift:46-167).  Shapes as the reference stores them:
 *   FP16: buckets [n_experts, in*percent_load, out/16] f16    stats [n_experts, in*percent_load, 4] f16
 *   Q4:   buckets [n_experts, in*8, out/32] u16 (viewed f16)  stats [n_experts, in*8, 2] f32
 *   probes [n_experts, 4096] f16;  outliers [n_outliers, 4] f32 or NULL (Q4);
 *   core [out, in] f16 or NULL (dense fallback, expertMul.swift:29-31).
 * percent_load = number of rank rows kept per input dim (16 = all, loader.swift:50,157-159); Q4 uses 8.
 * buckets_dev may be NULL only when core_dev is given ("buckets not loaded", loader.swift:105-108).
 * The handle never owns the caller's buffers.
 */
int effort_weights_create(const void* buckets_dev, const void* stats_dev, const void* probes_dev,
                          const void* outliers_dev, int n_outliers, const void* core_dev,
                          int in_dim, int out_dim, int n_experts, int percent_load, int kind,
                          unsigned flags, void* stream, effort_weights_t** w_out);
int effort_weights_destroy(effort_weights_t* w);
/* bytes of device memory the handle owns (the repacked copy) */
size_t effort_weights_owned_bytes(const effort_weights_t* w);
/* Test hooks.  The matrix's cutoff hints, device float [n_experts] (the last cutoff each expert's select found, times
 * the rmsNorm denominator on norm-on-load launches; +inf before the first; NULL for weights the default kernel does not
 * run), which a caller may overwrite between launches: the select's result does not depend on them.  And whether
 * kernels are launched with programmatic dependent launch (EFFORT_PDL, read once per process). */
float* effort_weights_hint(const effort_weights_t* w);
int effort_pdl_enabled(void);

/* ---- the operator ------------------------------------------------------ */
/*
 * bucketMul(v:by:expNo:out:effort:)  bucketMul.swift:11  (FP16; overwrites out, bucketMul.metal:133)
 *   v_dev [in] f32, out_dev [out] f32, exp_no_dev: device uint32 (NULL = expert 0,
 *   expertMul.swift:18), effort in [0,1] (default 0.25 in the reference).
 */
int effort_bucket_mul(effort_ctx_t* ctx, const float* v_dev, const effort_weights_t* w,
                      const uint32_t* exp_no_dev, float* out_dev, double effort, void* stream);
/* bucketMulQ4(v:by:expNo:out:effort:)  bucketMulQ4.swift:11  (accumulates INTO out, then calcOutliers) */
int effort_bucket_mul_q4(effort_ctx_t* ctx, const float* v_dev, const effort_weights_t* w,
                         const uint32_t* exp_no_dev, float* out_dev, double effort, void* stream);
/* expertMul(v:by:expNo:out:effort:)  expertMul.swift:24-38: Q4 -> out.zero(); bucketMulQ4 if buckets
 * loaded else basicMul(core); FP16 -> bucketMul. */
int effort_expert_mul(effort_ctx_t* ctx, const float* v_dev, const effort_weights_t* w,
                      const uint32_t* exp_no_dev, float* out_dev, double effort, void* stream);
/* basicMul(v:by:out:)  helpers/mps.swift:14-47: dense fp16 [out,in] x fp16(v) -> fp32 out */
int effort_basic_mul(effort_ctx_t* ctx, const float* v_dev, const void* core_dev, int out_dim, int in_dim,
                     float* out_dev, void* stream);

/*
 * Several bucketMuls that do not depend on each other (q/k/v share v, runNetwork.swift:132-134;
 * w1/w3, :178-179) enqueued as ONE launch group.  Semantically identical to n calls of
 * effort_expert_mul in order.
 */
typedef struct {
    const float* v_dev;
    const effort_weights_t* w;
    const uint32_t* exp_no_dev;
    float* out_dev;
    double effort;
    /* Tensor-parallel row shards only (DESIGN.md section 6): the first 4096 entries of the FULL input vector,
     * which findCutoff32 probes (bucketMul.metal:158-163), when v_dev is a rank-local slice.  NULL = v_dev. */
    const float* v_cutoff_dev;
} effort_mul_args_t;
int effort_expert_mul_batch(effort_ctx_t* ctx, const effort_mul_args_t* args, int n, void* stream);

/* ---- test hooks (kept callable "for testing", bucketMul.swift:17) ------- */
/* BucketMul.calcDispatch  bucketMul.swift:34-48: findCutoff32 + prepareDispatch into ctx scratch
 * (reference dispatch format: float2 {v, float(rowOffset)}; here in ascending row order), then the
 * roundUp/zeroRange32 padding of fullMul (bucketMul.swift:57-58). Works for both kinds. */
int effort_calc_dispatch(effort_ctx_t* ctx, const float* v_dev, const effort_weights_t* w,
                         const uint32_t* exp_no_dev, double effort, void* stream);
/* BucketMul.mul  bucketMul.swift:69-88: MAC over the ctx dispatch list + integrate (FP16: overwrites
 * out; Q4: accumulates into out). */
int effort_mul(effort_ctx_t* ctx, const effort_weights_t* w, float* out_dev, void* stream);
/* findCutoff32 only (bucketMul.metal:141-247); result stays in ctx scratch */
int effort_find_cutoff(effort_ctx_t* ctx, const float* v_dev, const effort_weights_t* w,
                       const uint32_t* exp_no_dev, double effort, void* stream);
/* Synchronising reads of ctx scratch (host pointers).  n_selected = rows selected before padding,
 * padded_size = dispatch.size after roundUp. dispatch_host may be NULL; else it must hold
 * 2*capacity floats and receives min(padded_size, capacity) entries. */
int effort_read_dispatch(effort_ctx_t* ctx, float* dispatch_host, size_t capacity, uint32_t* n_selected,
                         uint32_t* padded_size, float* cutoff, int* cutoff_loops, void* stream);

/* ---- convert ------------------------------------------------------------ */
/*
 * bucketize(_:outTensorsPref:tensors:)  convert.swift:209-260 (goQ8 = false): w_dev [out,in] f16 ->
 * buckets [in*16, out/16] f16, stats [in*16, 4] f16, probes [4096] f16, byte-identical to the
 * reference layout.  Preconditions of convert.swift:210-215 are returned as EFFORT_EINVAL.
 */
int effort_bucketize(const void* w_dev, int out_dim, int in_dim, void* buckets_dev, void* stats_dev,
                     void* probes_dev, void* stream);
/*
 * Q4 convert(core2)  q4_draft.py:70-322 after outlier extraction: wT_dev is W^T [in,out] f16 with the
 * outliers already zeroed (outlier selection is a global top-2% sort done once on the host side, see
 * effort_b200/convert.py) -> buckets [in*8, out/32] u16, stats [in*8, 2] f32, probes [min(in,out)] f16.
 */
int effort_q4_bucketize(const void* wT_dev, int in_dim, int out_dim, void* buckets_dev, void* stats_dev,
                        void* probes_dev, void* stream);

/* ---- tensor-parallel plumbing (DESIGN.md section 6) ------------------------------------------------- */
/*
 * One process per GPU.  The collectives of the sharded decode loop (all-gather of the row-parallel GEMV's
 * cutoff input, all-reduce of its partial output) are NCCL calls enqueued on the caller's stream from inside
 * the library (so they can live in the token's CUDA graph).  libnccl is resolved at run time (the copy already
 * loaded by the host process, else dlopen("libnccl.so.2")).  Rank 0 creates the 128-byte id and hands it to the
 * other ranks through whatever transport the host has (a process-group broadcast in effort_b200/model.py).
 */
int effort_comm_unique_id(void* id128_out);
int effort_comm_init(effort_ctx_t* ctx, const void* id128, int rank, int world);
int effort_comm_destroy(effort_ctx_t* ctx);
/* One-shot NVLink collectives (csrc/comm.cuh): every rank maps every peer's symmetric buffer through CUDA IPC and a
 * collective is one kernel per rank (peer stores + release flag + acquire spin), CUDA-graph replayable.  Used by the
 * sharded decode loop when connected (EFFORT_P2P=0 forces NCCL).  local_handle: allocates this rank's buffer and
 * returns its 64-byte cudaIpcMemHandle_t; connect: takes all ranks' handles (world x 64 bytes, rank order). */
int effort_comm_p2p_local_handle(effort_ctx_t* ctx, void* handle64_out);
int effort_comm_p2p_connect(effort_ctx_t* ctx, const void* handles, int rank, int world);
/* Test hook for the one-shot NVLink collectives themselves (the decode loop calls them internally): mode 0 = all-gather
 * (send: count floats, out: world*count floats in rank order), mode 1 = all-reduce (out: count floats, summed in rank
 * order); `site` (0..15) names the call position -- every rank must use the same sequence of sites, and a site may be
 * reused only after a later site's collective.  EFFORT_ESTATE unless effort_comm_p2p_connect succeeded. */
int effort_comm_p2p_collective(effort_ctx_t* ctx, int mode, int site, const float* send_dev, float* out_dev, size_t count,
                               void* stream);
/* back to NCCL for the exchanges (call on EVERY rank when any rank failed to connect: the choice must be collective) */
int effort_comm_p2p_disable(effort_ctx_t* ctx);
/* in-place sum all-reduce / all-gather of fp32 device buffers over the ctx communicator (test + building block) */
int effort_comm_all_reduce(effort_ctx_t* ctx, float* buf_dev, size_t count, void* stream);
int effort_comm_all_gather(effort_ctx_t* ctx, const float* send_dev, float* recv_dev, size_t send_count, void* stream);

/* ---- decode loop (host orchestration of the callers either side of the path) ----------------------- */
/*
 * runNetwork(tokens:effort:)  runNetwork.swift:68-316, one token per call: per layer rmsNormFast*attnNorm,
 * expertMul x3 (wq,wk,wv), rope_mx + calcScores + softmax + sumScores, expertMul wo, residual, rmsNormFast*
 * ffnNorm, expertMul w1,w3, silu, expertMul w2, residual (:124-183); final rmsNorm*norm and the dense
 * lm_head basicMul (:206-209); greedy next token = top-1 (:235-257), or a seeded draw once a sampler is set
 * (effort_model_set_sampler); per-position predictions and log-probabilities of given tokens (returnPredictions,
 * :228-232) once scoring is on (effort_model_set_scoring).  north_star keeps this orchestration in
 * Swift; there is no Swift toolchain here, so the mirror lives behind the same C-ABI and a Swift build would
 * call the per-operator entry points above instead.  Dims follow main.swift:45-46,56,72-77.
 */
typedef struct effort_model effort_model_t;
typedef struct {
    int dim;         /* stateDim 4096 */
    int hidden_dim;  /* hiddenDim 14336 */
    int n_layers;    /* numLayers 32 */
    int n_heads;     /* numHeads 32 */
    int n_kv_heads;  /* 8 (kvRepeats = 4) */
    int head_dim;    /* headDim 128 (the attention kernel requires 128) */
    int vocab;       /* 32000 */
    int max_seq;     /* maxSeqLen 2048 */
    float rope_theta;/* 1e6: freqs = 1e-6^(j/64), model.swift:701 */
    float norm_eps;  /* 1e-5, aux.metal:151 */
    int tp_rank, tp_size; /* tensor-parallel shard of this process (tp_size 1 = unsharded).  With tp_size = G > 1 the
                             ctx must have a communicator (effort_comm_init) and the weights passed to
                             effort_model_set_layer / set_head are this rank's shards: wq [dim -> dim/G],
                             wk/wv [dim -> kv_dim/G], wo [dim/G -> dim] (row shard), w1/w3 [dim -> hidden/G],
                             w2 [hidden/G -> dim] (row shard), output.core [vocab/G, dim]. */
} effort_model_config_t;

int effort_model_create(effort_ctx_t* ctx, const effort_model_config_t* cfg, effort_model_t** m_out);
int effort_model_destroy(effort_model_t* m);
/* Layer weights (loader.swift:201-225).  The handles and norm vectors (fp16 [dim]) stay owned by the caller. */
int effort_model_set_layer(effort_model_t* m, int layer, const effort_weights_t* wq, const effort_weights_t* wk,
                           const effort_weights_t* wv, const effort_weights_t* wo, const effort_weights_t* w1,
                           const effort_weights_t* w2, const effort_weights_t* w3, const void* attn_norm_dev,
                           const void* ffn_norm_dev);
/* Mixture of experts (runNetwork.swift:185-200, loader.swift:208-212): `gate_dev` = layers.N.feed_forward.gate [n_experts,
 * dim] f16; the layer's w1 / w2 / w3 handles must hold n_experts experts.  Per token: gate logits = basicMul(rmsNorm(h) *
 * ffn_norm, gate), the two largest (device indices, read by the expert GEMVs as expNo -- no host sync), softmax over
 * the two, h += gateVal_i * w2_e(silu(w1_e x) * w3_e x) for both.  Fused chain only (effort_model_set_chain 2). */
int effort_model_set_moe(effort_model_t* m, int layer, const void* gate_dev, int n_experts);
/* model.norm [dim] f16, output.core [vocab,dim] f16, tok_embeddings.core [vocab,dim] f16 (loader.swift:254-272) */
int effort_model_set_head(effort_model_t* m, const void* norm_dev, const void* output_core_dev,
                          const void* tok_embeddings_dev);
/* position <- 0 (the KV cache is logically emptied) */
int effort_model_reset(effort_model_t* m, void* stream);
/* position <- pos, 0 <= pos < max_seq (a test hook): the cache rows stay, as after a reset, so the next step repeats
 * step pos on the rows the earlier steps left.  EINVAL for a NULL model or pos out of range. */
int effort_model_rewind(effort_model_t* m, int pos, void* stream);
/*
 * One decode step at the current position, enqueue-only.  token_dev: device int32 (NULL = the token the
 * previous step predicted).  After it: logits in effort_model_logits(), next token in effort_model_next_token().
 * The first call for a given effort value runs eagerly and captures a CUDA graph; later calls replay it.
 */
int effort_model_step(effort_model_t* m, const int32_t* token_dev, double effort, void* stream);
/* Feed n known tokens (tokens_dev [n], device) at the current position, as n effort_model_step calls would: afterwards
 * the position has advanced by n, the KV caches hold all n rows, effort_model_logits() holds the last position's logits
 * and effort_model_next_token() greedy's choice (or the sampler's draw at position start + n); with scoring on, records
 * start .. start+n-1 are written from the target row.  Enqueue-only.  Single-GPU FP16 models on the fused chain (chain 2,
 * round-2 engine, select cutoff mode, slice-major weights, no MoE layer) run chunks of up to 16 tokens through the
 * multi-token GEMV and a chunk attention (DESIGN.md section 4.8): the logits agree with stepping to the decode's bars,
 * not bit for bit.  Every other configuration runs n effort_model_step calls.  CUDA graphs follow
 * effort_model_set_graphs, one per (effort, chunk length).  EFFORT_EINVAL for n < 1, EFFORT_ESTATE when start + n >
 * max_seq; nothing is enqueued in either case.  Out-of-range tokens are read as token 0, as a step reads them. */
int effort_model_prefill(effort_model_t* m, const int32_t* tokens_dev, int n, double effort, void* stream);
/* Same step driven with HOST buffers (the end-to-end call): token_host (NULL = previous prediction) is copied
 * H2D from pinned memory, the step runs, next token (and logits if logits_host != NULL) are copied D2H and the
 * stream is synchronised. */
int effort_model_step_host(effort_model_t* m, const int32_t* token_host, double effort, int32_t* next_token_host,
                           float* logits_host, void* stream);
const float* effort_model_logits(const effort_model_t* m);        /* device [vocab] f32 */
const int32_t* effort_model_next_token(const effort_model_t* m);  /* device int32 */
/* bytes of bucket weights one token streams at effort 1.0 (sum of in*out*2 over the 7x n_layers matrices) */
size_t effort_model_bucket_bytes(const effort_model_t* m);
/* use CUDA graphs for effort_model_step (default 1) */
int effort_model_set_graphs(effort_model_t* m, int enable);
/* round-1 engine only (default 0): apply rmsNorm*w on load inside the round-1 bucketMul kernels and fold the residual
 * add and silu*mul into the integrate epilogues (9 launches per layer instead of 12) */
int effort_model_set_fused_glue(effort_model_t* m, int enable);
/* Token chain: 2 (default; single GPU, FP16 buckets, round-2 engine) = 5 launches per layer -- [q,k,v] with
 * rmsNorm*w applied on load, attention, wo accumulating into the residual stream, [w1,w3] with rmsNorm*w on load, w2
 * with silu(x1)*x3 on load accumulating into the residual stream -- then one head kernel (final norm + lm_head +
 * argmax); 1 = one kernel per reference op (runNetwork.swift:124-183 order).  Other configurations (tensor parallel,
 * Q4, round-1 engine) always use chain 1.  Environment default: EFFORT_CHAIN. */
int effort_model_set_chain(effort_model_t* m, int chain);

/*
 * Sampling on the device (DESIGN.md section 4.6).  Greedy (the argmax above) stays the default.  With a sampler set,
 * every step ends with one more kernel that overwrites the next token with a draw from the step's logits l[0..V):
 *   1. order: a before b if l_a > l_b, or l_a == l_b (+0 == -0) and a < b; NaN is never drawn.  No finite maximum:
 *      the first +inf if there is one (greedy's choice), else token 0.
 *   2. top-k: S_k = the first K tokens of that order (ties cut by index, |S_k| = K); all V when K = 0 or K >= V.
 *   3. m = max l; for i in S_k: w_i = expf((l_i - m) / T) in fp32 (IEEE subtraction and division),
 *      q_i = floor(w_i * 2^32) as uint64 (the maximum weighs 2^32; q_i = 0, a relative probability below 2^-32, is
 *      never drawn).
 *   4. top-p: Q_k = sum of q over S_k; need = ceil((double)P * (double)Q_k); S = the shortest prefix of S_k, in the
 *      order of 1, whose sum of q reaches need.
 *   5. x = word 0 of Philox4x32-10 with counter (position, 0, 0, 0) and key (seed & 0xffffffff, seed >> 32);
 *      Q = sum of q over S; target = (x * Q) >> 32; the token is the smallest index in S whose inclusive prefix sum of
 *      q over S, in INDEX order, exceeds target.
 * Everything after the expf is integer arithmetic, so the draw depends only on the input bits.  In the model the
 * position is the position after the step: the n-th step after effort_model_reset draws with position n.
 */
typedef struct {
    float temperature;  /* T > 0, finite */
    int top_k;          /* K >= 0; 0 = no limit */
    float top_p;        /* P in (0, 1]; 1 = no limit */
    uint64_t seed;
} effort_sampler_t;
/* NULL = greedy (the default).  Parameters are copied; a change of parameters takes effect at the next step without
 * recapturing the step's CUDA graph; switching between greedy and sampling drops the captured graphs.  EFFORT_EINVAL
 * for a NaN, infinite or non-positive temperature, top_k < 0, or top_p outside (0, 1]. */
int effort_model_set_sampler(effort_model_t* m, const effort_sampler_t* s);
/* Test hook: one draw from logits_dev[0..n) with `position` as the Philox counter into token_dev (device int32).
 * Enqueue-only; the same kernel the model runs.  EFFORT_EINVAL for n <= 0 and the parameter errors above. */
int effort_sample(effort_ctx_t* ctx, const float* logits_dev, int n, const effort_sampler_t* s, uint32_t position,
                  int32_t* token_dev, void* stream);

/*
 * Scoring on the device (DESIGN.md section 4.7): one record per target token t against logits l[0..V) (fp32).
 *   1. argmax: the greedy token, the lowest index of the maximum (NaN never wins; all NaN gives 0).
 *   2. rank: with key = the sampler's order-preserving key (-0 == +0, NaN below -inf),
 *      rank = #{i : key_i > key_t} + #{i < t : key_i == key_t}, exact.  Rank 0 means greedy would pick t.
 *   3. logprob: m = max over the non-NaN logits.  When m is finite, S = sum over non-NaN i of expf(l_i - m), summed in
 *      fp32 in a fixed order (per-thread strided sums over 1024 threads, a shuffle tree, then the 32 warps in index
 *      order), and logprob = (l_t - m) - logf(S) with IEEE subtraction; a NaN or -inf target gives -inf.  When m is not
 *      finite (all NaN, all -inf, or some +inf) logprob is NaN.
 *   4. t outside [0, V) (-1 = no target): rank = -1, logprob = NaN; argmax is still written.
 * A record depends only on the logits' bits and t, so scoring keeps the decode bit-reproducible.
 */
typedef struct {
    int32_t argmax;
    int32_t rank;
    float logprob;
} effort_score_t;
/* Test hook and operator: score targets_dev[0..n_targets) (device int32) against logits_dev[0..n) into
 * out_dev[0..n_targets), one CTA per target, with the kernel the model runs.  Enqueue-only.  EFFORT_EINVAL for a NULL
 * pointer, n <= 0 or n_targets <= 0. */
int effort_score(effort_ctx_t* ctx, const float* logits_dev, int n, const int32_t* targets_dev, int n_targets,
                 effort_score_t* out_dev, void* stream);
/* Off by default.  When on, every step ends with one more launch (after the sampler's, when one is set) that writes
 * record p = (position after the step) - 1 of effort_model_scores() from target row entry p: step p after
 * effort_model_reset scores the token the caller says follows its input.  Switching on or off drops the captured graphs. */
int effort_model_set_scoring(effort_model_t* m, int enable);
/* Enqueue a copy of targets_dev[0..n) (device int32) into the model's target row [max_seq] and set the rest to -1 (no
 * target).  The row starts as all -1.  New targets need no graph recapture.  EFFORT_EINVAL for n < 0, n > max_seq, or
 * a NULL targets_dev with n > 0. */
int effort_model_set_score_targets(effort_model_t* m, const int32_t* targets_dev, int n, void* stream);
/* Device records [max_seq]: record p is the one the last step at position p wrote; zero until then.  Reset does not
 * clear them. */
const effort_score_t* effort_model_scores(const effort_model_t* m);

/* Test hook: read-only device pointer to one of the model's working buffers as the last step left it, so that each
 * kernel of the step can be checked on the inputs it actually consumed.  `count` (may be NULL) receives the element
 * count.  NULL (count 0) when the buffer does not exist on the path the model last enqueued or replayed, or for a bad
 * `which` / `layer`.  The caller synchronises the step's stream first; the pointer stays valid until the model is
 * destroyed, and its contents until the next step. */
#define EFFORT_BUF_Q 0        /* f32 [n_heads*128]: the last layer's q GEMV output before rope, as the attention read it */
#define EFFORT_BUF_K 1        /* f32 [n_kv*128]: the same for k */
#define EFFORT_BUF_V 2        /* f32 [n_kv*128]: the same for v */
#define EFFORT_BUF_ATTN 3     /* f32 [n_heads][128]: the last layer's attention output */
#define EFFORT_BUF_KCACHE 4   /* f32 [max_seq][n_kv][128]: `layer`'s roped key cache */
#define EFFORT_BUF_VCACHE 5   /* f32 [max_seq][n_kv][128]: `layer`'s value cache */
#define EFFORT_BUF_HIDDEN 6   /* f32 [dim]: the residual stream after the last layer (the final norm's input) */
#define EFFORT_BUF_NORMED 7   /* f32 [dim]: rmsNorm(h) * norm, the lm_head's input; NULL on chain 2 (its head norms on load) */
#define EFFORT_BUF_GATE_IN 8  /* f32 [dim]: the hidden state the last MoE layer's gate normalised; NULL without MoE */
#define EFFORT_BUF_GATE_IDX 9 /* u32 [2]: that layer's two routed experts, the first one first */
#define EFFORT_BUF_GATE_VAL 10/* f32 [2]: their softmax weights */
#define EFFORT_BUF_POS 11     /* i32 [1]: the device position (tokens decoded since the last reset) */
/* The last effort_model_prefill chunk of T tokens (NULL unless the model's last call was a multi-token prefill; then
 * EFFORT_BUF_KCACHE / _VCACHE / _POS are available too and the single-token ids above are NULL): */
#define EFFORT_BUF_CHUNK_Q 12      /* f32 [T][n_heads*128]: the last layer's q GEMV outputs before rope */
#define EFFORT_BUF_CHUNK_K 13      /* f32 [T][n_kv*128]: the same for k */
#define EFFORT_BUF_CHUNK_V 14      /* f32 [T][n_kv*128]: the same for v */
#define EFFORT_BUF_CHUNK_ATTN 15   /* f32 [T][n_heads*128]: the last layer's attention outputs */
#define EFFORT_BUF_CHUNK_LOGITS 16 /* f32 [T][vocab]: every row's logits; only with scoring on */
#define EFFORT_BUF_CHUNK_LEN 17    /* i32 [1]: T */
const void* effort_model_buffer(const effort_model_t* m, int which, int layer, size_t* count);

/* Test hook: one launch group of the fused chain (effort_model_set_chain 2), with the glue it applies on load.  Entry k
 * computes, with x its input,
 *     x = v                                 (plain: wo)
 *     x = rmsNorm(v) * norm_w               (norm_w_dev != NULL: [q,k,v] and [w1,w3]; v is the residual stream h)
 *     x = silu(v) * x3 = x3 * v / (1 + expf(-v))   (x3_dev != NULL: w2; v is x1)
 *     out = s * W_e(x)  or  out += s * W_e(x)       (accumulate 0 / 1)
 * where W_e is expert *exp_no_dev of w (expert 0 when NULL), s = *out_scale_dev (1 when NULL; the MoE gate value), and
 * the rows are selected, and the cutoff taken, on the unscaled x.  rmsNorm(v) = v / sqrtf(sum(v^2) / 4096 + norm_eps).
 * All n entries go into ONE launch with the chain's geometry and batch slots 0..n-1: the same kernel, mode, stage and
 * row splits as the model's step on the same weights.  Enqueue-only.  EFFORT_EINVAL for n outside 1..4, a NULL pointer,
 * effort outside [0, 1], norm and silu in one entry, or the round-1 engine; EFFORT_ESHAPE when the fused chain could not
 * run the weights (not FP16 buckets the round-2 kernel takes, or norm with in != 4096). */
typedef struct {
    const float* v_dev;          /* input; with norm_w_dev: the residual h; with x3_dev: x1 */
    const float* x3_dev;         /* non-NULL: input = silu(v) * x3 */
    const void* norm_w_dev;      /* non-NULL: input = rmsNorm(v) * norm_w, fp16 [in], in == 4096 */
    float norm_eps;
    const effort_weights_t* w;
    const uint32_t* exp_no_dev;  /* device expert index, NULL = 0 */
    const float* out_scale_dev;  /* non-NULL: out (+)= scale * W(input); rows selected on the unscaled input */
    float* out_dev;
    double effort;
    int accumulate;              /* 1: out += ..., 0: out = ... */
} effort_fused_args_t;
int effort_fused_mul_batch(effort_ctx_t* ctx, const effort_fused_args_t* a, int n, void* stream);
/* The cutoff and the selected-row count of batch slot `slot` (0..7) of the last round-2 launch group on this ctx
 * (effort_last_selected reads slot 0 only).  Synchronises `stream`.  EFFORT_ESTATE when the last launch was not one, or
 * had no such slot. */
int effort_last_problem(effort_ctx_t* ctx, int slot, float* cutoff, uint32_t* n_selected, void* stream);

/* Multi-token effort GEMV (the model's prefill kernel and geometry): out[t] = W(v[t]) for t < n <= 16 inputs
 * (v_dev [n][in], out_dev [n][out], device).  Token t's cutoff is the EFFORT_CUTOFF_SELECT rule on its own probe
 * products and its rows are those with cutoff[t] < (1e5 * stat) * |v[t][i]|, whatever the context's cutoff mode; out[t]
 * is the fp32 sum of exactly those rows, in an order fixed by the matrix, so it repeats bit for bit and does not depend
 * on the other inputs.  cutoff_dev [n] and count_dev [n] (may be NULL) receive each token's cutoff and selected-row
 * count.  Enqueue-only.  EFFORT_EINVAL for n outside 1..16, a NULL pointer or effort outside [0, 1]; EFFORT_ESHAPE for
 * weights other than single-expert FP16 buckets in the default slice-major layout with in >= 4096. */
int effort_bucket_mul_multi(effort_ctx_t* ctx, const float* v_dev, int n, const effort_weights_t* w, float* out_dev,
                            double effort, float* cutoff_dev, uint32_t* count_dev, void* stream);

/*
 * Batch decode (DESIGN.md section 4.9): n_seq (1..16) slots decoded together on one model, each with its own KV caches
 * ([max_seq][n_kv][128] per layer), device position, logits row, next token, sampler (greedy by default) and score target
 * and record rows ([max_seq] each).  A step feeds every slot one token and is prefill's per-row path with T = n_seq: the
 * multi-token GEMV groups, an attention in which each slot reads its own cache at its own position, and one lm_head pass
 * for all rows; each slot then ends as a model step does (greedy argmax advancing its position, its draw, its record
 * pos - 1).  A slot's logits, next token, cache rows and records depend only on its own tokens, state, sampler
 * parameters and the effort: not on n_seq, its index or the other slots.  The model's weights are read; the model's
 * buffers are read only by fork.  Graphs follow effort_model_set_graphs: the first step runs eagerly, then one graph per
 * effort is captured and replayed.  The batch's graphs hold the model's weight pointers: set the model's layers and head
 * before creating a batch, and destroy the batch before its model.
 */
typedef struct effort_batch effort_batch_t;
/* Allocates everything a step needs (caches, row buffers, GEMV scratch), so a captured graph never sees a reallocation.
 * EFFORT_EINVAL for n_seq outside 1..16 or a NULL pointer; EFFORT_ESHAPE unless the model takes the multi-token prefill
 * path (single GPU, chain 2, FP16 slice-major buckets, select cutoffs, no MoE); EFFORT_ENOMEM when the device is full. */
int effort_batch_create(effort_model_t* m, int n_seq, effort_batch_t** out);
int effort_batch_destroy(effort_batch_t* b);
/* Every function below takes seq -1 for all slots where it takes a slot.  Reset: the slot's position becomes 0. */
int effort_batch_reset(effort_batch_t* b, int seq, void* stream);
/* Copies the model's current state into the slot (cache rows [0, pos) of every layer, the position and the last logits),
 * then runs the slot's tail on those logits: greedy argmax, or a draw at position pos with the slot's sampler, and with
 * scoring on, record pos - 1.  The slot is then where a model step would have left it.  Enqueue-only.  EFFORT_ESTATE
 * (nothing enqueued) when the model is at position 0; EFFORT_ESHAPE as for create. */
int effort_batch_fork(effort_batch_t* b, int seq, void* stream);
/* One step of every slot: slot b takes tokens_dev[b] (device int32 [n_seq]), or its own previous next token when
 * tokens_dev is NULL.  Enqueue-only.  EFFORT_EINVAL for effort outside [0, 1]; EFFORT_ESTATE (nothing enqueued) while any
 * slot sits at max_seq; EFFORT_ESHAPE as for create. */
int effort_batch_step(effort_batch_t* b, const int32_t* tokens_dev, double effort, void* stream);
/* The slot's sampler, as effort_model_set_sampler: NULL = greedy.  Parameters are copied on the stream of the next step
 * or fork, without recapture; switching a slot between greedy and sampling drops the batch's graphs. */
int effort_batch_set_sampler(effort_batch_t* b, int seq, const effort_sampler_t* s);
/* Off by default; switching drops the batch's graphs.  As effort_model_set_scoring, per slot. */
int effort_batch_set_scoring(effort_batch_t* b, int enable);
/* As effort_model_set_score_targets, into the slot's target row. */
int effort_batch_set_score_targets(effort_batch_t* b, int seq, const int32_t* targets_dev, int n, void* stream);
const float* effort_batch_logits(const effort_batch_t* b);          /* device [n_seq][vocab] */
const int32_t* effort_batch_next_tokens(const effort_batch_t* b);   /* device [n_seq] */
const effort_score_t* effort_batch_scores(const effort_batch_t* b); /* device [n_seq][max_seq] */
/* Test hook, as effort_model_buffer: EFFORT_BUF_Q / K / V / ATTN give the last layer's values of the last step as
 * [n_seq][...] (NULL before the first step); KCACHE / VCACHE give `layer`'s cache of slot `seq`; POS gives [n_seq]; every
 * other id gives NULL. */
const void* effort_batch_buffer(const effort_batch_t* b, int which, int layer, int seq, size_t* count);

/* ---- introspection used by bench / tests -------------------------------- */
/* number of kernels this library has launched since load (process-wide) */
uint64_t effort_launch_count(void);
/* rows selected by the last fused bucket_mul on this ctx (synchronises `stream`) */
int effort_last_selected(effort_ctx_t* ctx, uint32_t* n_selected, void* stream);

/* ---- bucketed-safetensors model directory (host side, no CUDA) --------------------------------------------
 * Replaces TensorLoader (helpers/safetensors.swift:87-216): `<model>.safetensors.index.json` maps tensor names to
 * the per-layer files written by TensorSaver.save (:38-85); a name missing from the index is retried as
 * name + ".weight" (:141-146); only BF16 / F16 / F32 tensors are accepted (:176); data_offsets must span
 * prod(shape) * sizeof(dtype) bytes (:182).  Files are mapped read-only and stay mapped until effort_loader_close,
 * so `data` can be passed to cudaMemcpy (or wrapped without a copy).  ExpertWeights (loader.swift:113-166) keeps
 * only the first percentLoad * inDim rows of `buckets` / `bucket.stats`: rows are the leading dimension, so that
 * truncation is a prefix of `data` (see effort_b200/weights_io.py, NativeTensorLoader.expert_weights). */
#define EFFORT_ST_F16 0
#define EFFORT_ST_BF16 1
#define EFFORT_ST_F32 2
#define EFFORT_ST_MAX_DIMS 8
typedef struct effort_loader effort_loader_t;
typedef struct {
    int dtype;                         /* EFFORT_ST_* */
    int ndim;
    int64_t shape[EFFORT_ST_MAX_DIMS];
    const void* data;                  /* inside the read-only mapping */
    size_t nbytes;
} effort_tensor_info_t;
int effort_loader_open(const char* dir, const char* model, effort_loader_t** out);   /* TensorLoader(path:model:) :105-110 */
void effort_loader_close(effort_loader_t* loader);
int effort_loader_count(const effort_loader_t* loader);
const char* effort_loader_name(const effort_loader_t* loader, int i);                /* index order */
int effort_loader_has(const effort_loader_t* loader, const char* name);              /* hasTensor :132-134 */
int effort_loader_tensor(effort_loader_t* loader, const char* name, effort_tensor_info_t* info);  /* fetchTensor :136-216 */
/* convertBF16 (the reference converts BF16 tensors to fp16 after loading, safetensors.swift:207-210) */
int effort_bf16_to_f16(const uint16_t* src, uint16_t* dst, size_t n);

/* Replaces TensorSaver (helpers/safetensors.swift:38-85) + saveSafetensors (:222-280): tensors are collected per output
 * file (the reference writes one file per layer, convert.swift:68,121) and effort_saver_save writes
 * "<model>-%05d-of-%05d.safetensors" files (u64 LE header size, JSON header with dtype / shape / data_offsets per tensor and
 * "__metadata__": {"description"}, tensor bytes in header order) plus "<model>.safetensors.index.json"
 * {"weight_map": {name: file}}.  Only F16 / F32 (and BF16 pass-through) tensors, as in the reference (:231-247).  The saver
 * does not copy: `data_host` must stay valid until effort_saver_save returns.  A name may be added once (EFFORT_ESTATE). */
typedef struct effort_saver effort_saver_t;
int effort_saver_open(const char* dir, const char* model, const char* description /* NULL = the reference's text */,
                      effort_saver_t** out);
int effort_saver_add(effort_saver_t* saver, int file_index, const char* name, int dtype, int ndim, const int64_t* shape,
                     const void* data_host, size_t nbytes);
int effort_saver_save(effort_saver_t* saver);
void effort_saver_close(effort_saver_t* saver);

#ifdef __cplusplus
}
#endif
#endif /* EFFORT_B200_H */
