"""Host-side mirror of the reference's model containers for the decode loop.

    Model / Layer            loader.swift:201-272   (ExpertWeights per projection, norms, output, embeddings)
    runNetwork(tokens:effort:)  runNetwork.swift:68  -> DecodeModel.step / step_host (one token per call)

The orchestration itself (layer loop, graph capture) is native code behind the C-ABI (effort_model_* in
include/effort_b200.h); this module only owns device memory and builds weights.  `random_init` creates a
random-initialised model of the Mistral-7B architecture (main.swift:45-46,56,72-77) directly on the GPU and
converts it with the library's own bucketize -- there is no network access for real checkpoints.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional

import torch

from . import _lib, ops, sharding
from ._lib import ModelConfig, check


def init_comm(ctx: "ops.Context", rank: int, world: int) -> None:
    """Create the library's NCCL communicator for this process (one process per GPU).  The 128-byte id is made
    by rank 0 and broadcast through the caller's torch.distributed group (plumbing only)."""
    import torch.distributed as dist
    L = _lib.load()
    buf = (C.c_char * 128)()
    if rank == 0:
        check(L.effort_comm_unique_id(buf), "effort_comm_unique_id")
    t = torch.frombuffer(bytearray(bytes(buf)), dtype=torch.uint8).cuda()
    dist.broadcast(t, src=0)
    raw = bytes(t.cpu().numpy().tobytes())
    check(L.effort_comm_init(ctx._h, raw, rank, world), "effort_comm_init")
    # one-shot NVLink collectives: exchange the CUDA-IPC handles of the symmetric buffers
    import os
    if os.environ.get("EFFORT_P2P", "1") != "0":
        hb = (C.c_char * 64)()
        check(L.effort_comm_p2p_local_handle(ctx._h, hb), "effort_comm_p2p_local_handle")
        mine = torch.frombuffer(bytearray(bytes(hb)), dtype=torch.uint8).cuda()
        allh = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(allh, mine)
        blob = b"".join(bytes(x.cpu().numpy().tobytes()) for x in allh)
        ok = 1 if L.effort_comm_p2p_connect(ctx._h, blob, rank, world) == 0 else 0
        # peer mapping can be refused (no CUDA IPC between the devices / in the container): the decision to use the
        # peer-memory kernels must be the same on every rank, so agree on it and fall back to NCCL together
        flag = torch.tensor([ok], dtype=torch.int32, device="cuda")
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        if int(flag.item()) == 0:
            check(L.effort_comm_p2p_disable(ctx._h), "effort_comm_p2p_disable")
            if rank == 0:
                import warnings
                warnings.warn("effort_b200: CUDA-IPC peer mapping unavailable, tensor-parallel exchanges use NCCL")
        dist.barrier()


@dataclass
class MistralConfig:
    dim: int = 4096          # stateDim, main.swift:45
    hidden_dim: int = 14336  # hiddenDim, main.swift:46
    n_layers: int = 32       # numLayers, main.swift:56
    n_heads: int = 32        # numHeads, main.swift:72
    n_kv_heads: int = 8      # kvRepeats = 4, main.swift:73-74
    head_dim: int = 128
    vocab: int = 32000
    max_seq: int = 2048      # maxSeqLen, main.swift:76
    rope_theta: float = 1e6  # freqs = 1e-6^(j/64), model.swift:701
    norm_eps: float = 1e-5   # aux.metal:151


def _rand_w(out_dim, in_dim, gen, scale=0.02):
    return (torch.randn((out_dim, in_dim), generator=gen, device="cuda", dtype=torch.float32) * scale).half()


class DecodeModel:
    def __init__(self, cfg: MistralConfig, ctx: Optional[ops.Context] = None, tp_rank: int = 0, tp_size: int = 1):
        self.cfg = cfg
        self.ctx = ctx or ops.default_context()
        self.tp_rank, self.tp_size = tp_rank, tp_size
        self._L = _lib.load()
        c = ModelConfig(cfg.dim, cfg.hidden_dim, cfg.n_layers, cfg.n_heads, cfg.n_kv_heads, cfg.head_dim, cfg.vocab,
                        cfg.max_seq, cfg.rope_theta, cfg.norm_eps, tp_rank, tp_size)
        h = C.c_void_p()
        check(self._L.effort_model_create(self.ctx._h, C.byref(c), C.byref(h)), "effort_model_create")
        self._h = h
        self.layers = []      # keeps ExpertWeights + norm tensors alive
        self.head = None
        self._next = C.c_int32(0)
        self._scoring = False

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self._L.effort_model_destroy(self._h)
                self._h = None
        except Exception:
            pass

    # -- weights ------------------------------------------------------------------------------------------
    def set_layer(self, i: int, wq, wk, wv, wo, w1, w2, w3, attn_norm: torch.Tensor, ffn_norm: torch.Tensor):
        check(self._L.effort_model_set_layer(self._h, i, wq._h, wk._h, wv._h, wo._h, w1._h, w2._h, w3._h,
                                             attn_norm.data_ptr(), ffn_norm.data_ptr()), "effort_model_set_layer")
        while len(self.layers) <= i:
            self.layers.append(None)
        self.layers[i] = (wq, wk, wv, wo, w1, w2, w3, attn_norm, ffn_norm)

    def set_moe(self, i: int, gate: torch.Tensor):
        """layers.i.feed_forward.gate [n_experts, dim] f16 (loader.swift:208-212); the layer's w1/w2/w3 hold n_experts experts."""
        check(self._L.effort_model_set_moe(self._h, i, gate.data_ptr(), gate.shape[0]), "effort_model_set_moe")
        self.layers[i] = self.layers[i] + (gate,)

    def set_head(self, norm: torch.Tensor, output_core: torch.Tensor, tok_embeddings: torch.Tensor):
        check(self._L.effort_model_set_head(self._h, norm.data_ptr(), output_core.data_ptr(),
                                            tok_embeddings.data_ptr()), "effort_model_set_head")
        self.head = (norm, output_core, tok_embeddings)

    @classmethod
    def random_init(cls, cfg: MistralConfig = MistralConfig(), seed: int = 1234, keep_reference_layout: bool = False,
                    ctx: Optional[ops.Context] = None, norm_jitter: float = 0.1, tp_rank: int = 0,
                    tp_size: int = 1, weight_flags: int = 0, weight_fn=None, keep_dense: bool = False) -> "DecodeModel":
        """Random-init weights ~ N(0, 0.02^2) (SURVEY.md section 8d), converted on the GPU (effort_bucketize).
        With tp_size > 1 every rank draws the SAME full matrices (same seed), converts them and keeps its shard
        (effort_b200/sharding.py): the sharded model computes what the unsharded one does."""
        m = cls(cfg, ctx, tp_rank, tp_size)
        gen = torch.Generator(device="cuda").manual_seed(seed)
        kvd = cfg.n_kv_heads * cfg.head_dim
        m.dense = [] if keep_dense else None    # keep_dense: the dense fp16 [out,in] matrices per layer (quality baseline)
        cur = []

        def make(out_dim, in_dim, mode="column"):
            w = (weight_fn or _rand_w)(out_dim, in_dim, gen)
            if keep_dense:
                cur.append(w)
            t = ops.bucketize(w)
            if tp_size > 1:
                fn = sharding.shard_columns if mode == "column" else sharding.shard_rows
                t = fn(t, in_dim, out_dim, tp_rank, tp_size)
                in_dim, out_dim = t["in"], t["out"]
            ew = ops.ExpertWeights(t["buckets"], t["bucket.stats"], t["probes"], inDim=in_dim, outDim=out_dim, flags=weight_flags)
            if not keep_reference_layout:
                ew.release_reference_layout()
            return ew

        def norm_vec():
            return (1.0 + norm_jitter * torch.randn(cfg.dim, generator=gen, device="cuda")).half()

        for i in range(cfg.n_layers):
            m.set_layer(i, make(cfg.dim, cfg.dim), make(kvd, cfg.dim), make(kvd, cfg.dim), make(cfg.dim, cfg.dim, "row"),
                        make(cfg.hidden_dim, cfg.dim), make(cfg.dim, cfg.hidden_dim, "row"),
                        make(cfg.hidden_dim, cfg.dim), norm_vec(), norm_vec())
            if keep_dense:
                m.dense.append(list(cur))
                cur.clear()
        out_core = _rand_w(cfg.vocab, cfg.dim, gen)
        if tp_size > 1:
            v0, v1 = cfg.vocab * tp_rank // tp_size, cfg.vocab * (tp_rank + 1) // tp_size
            out_core = out_core[v0:v1].contiguous()
        m.set_head(norm_vec(), out_core, _rand_w(cfg.vocab, cfg.dim, gen, scale=1.0))
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        return m

    @classmethod
    def random_init_moe(cls, cfg: MistralConfig = MistralConfig(), n_experts: int = 4, seed: int = 1234,
                        ctx: Optional[ops.Context] = None, norm_jitter: float = 0.1) -> "DecodeModel":
        """A Mixtral-shaped random model (runNetwork.swift:185-200): attention as random_init, every layer's MLP with
        `n_experts` experts (buckets / stats / probes concatenated along the expert dimension, loader.swift:113-166) and a
        dense gate.  The reference layout tensors stay on the ExpertWeights objects for the CPU restatement."""
        m = cls(cfg, ctx)
        gen = torch.Generator(device="cuda").manual_seed(seed)
        kvd = cfg.n_kv_heads * cfg.head_dim

        def one(out_dim, in_dim):
            return ops.bucketize(_rand_w(out_dim, in_dim, gen))

        def make(out_dim, in_dim, e=1):
            ts = [one(out_dim, in_dim) for _ in range(e)]
            t = {k: torch.cat([x[k] for x in ts]) for k in ts[0]}
            return ops.ExpertWeights(t["buckets"], t["bucket.stats"], t["probes"], inDim=in_dim, outDim=out_dim, numExperts=e)

        def norm_vec():
            return (1.0 + norm_jitter * torch.randn(cfg.dim, generator=gen, device="cuda")).half()

        for i in range(cfg.n_layers):
            m.set_layer(i, make(cfg.dim, cfg.dim), make(kvd, cfg.dim), make(kvd, cfg.dim), make(cfg.dim, cfg.dim),
                        make(cfg.hidden_dim, cfg.dim, n_experts), make(cfg.dim, cfg.hidden_dim, n_experts),
                        make(cfg.hidden_dim, cfg.dim, n_experts), norm_vec(), norm_vec())
            m.set_moe(i, _rand_w(n_experts, cfg.dim, gen, scale=0.02))   # logits ~ N(0, 1.3^2): exp() stays finite
        m.set_head(norm_vec(), _rand_w(cfg.vocab, cfg.dim, gen), _rand_w(cfg.vocab, cfg.dim, gen, scale=1.0))
        torch.cuda.synchronize()
        return m

    @classmethod
    def random_init_q4(cls, cfg: MistralConfig = MistralConfig(), seed: int = 1234, ctx: Optional[ops.Context] = None,
                       norm_jitter: float = 0.1, bucketed=("wq", "w1", "w2", "w3"), keep_tensors: bool = False) -> "DecodeModel":
        """BASELINE configs[2]: a Q4 model.  The reference's converter bucketizes only wq / w1 / w2 / w3
        (q4_convert.py:53,59: 2 % outliers kept as fp32 records, the rest as sign|position nibbles in size-8 buckets,
        q4_draft.py:70-322); wk / wv / wo stay dense fp16 `core` tensors and expertMul routes them to basicMul
        (expertMul.swift:26-31).  keep_tensors=True leaves the converted tensors on the ExpertWeights objects
        (`q4_tensors`, `dense`) for the CPU restatement in tests."""
        from . import convert
        m = cls(cfg, ctx)
        gen = torch.Generator(device="cuda").manual_seed(seed)
        kvd = cfg.n_kv_heads * cfg.head_dim

        def make(name, out_dim, in_dim):
            w = _rand_w(out_dim, in_dim, gen)
            if name in bucketed:
                t = convert.q4_convert(w.t().contiguous())          # W^T [in, out], as q4_convert.py:53 passes it
                ew = ops.ExpertWeights(t["buckets"], t["bucket.stats"], t["probes"], t["outliers"], None, inDim=in_dim,
                                       outDim=out_dim, kind=ops.KIND_Q4)
                if keep_tensors:
                    ew.q4_tensors = t
            else:
                ew = ops.ExpertWeights(core=w, inDim=in_dim, outDim=out_dim, kind=ops.KIND_Q4)
            if keep_tensors:
                ew.dense = w
            return ew

        def norm_vec():
            return (1.0 + norm_jitter * torch.randn(cfg.dim, generator=gen, device="cuda")).half()

        for i in range(cfg.n_layers):
            m.set_layer(i, make("wq", cfg.dim, cfg.dim), make("wk", kvd, cfg.dim), make("wv", kvd, cfg.dim),
                        make("wo", cfg.dim, cfg.dim), make("w1", cfg.hidden_dim, cfg.dim), make("w2", cfg.dim, cfg.hidden_dim),
                        make("w3", cfg.hidden_dim, cfg.dim), norm_vec(), norm_vec())
        m.set_head(norm_vec(), _rand_w(cfg.vocab, cfg.dim, gen), _rand_w(cfg.vocab, cfg.dim, gen, scale=1.0))
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        return m

    # -- model directory (the reference's on-disk contract, weights_io.py) ------------------------------------
    @staticmethod
    def random_hf_source(cfg: MistralConfig = MistralConfig(), seed: int = 1234, norm_jitter: float = 0.1):
        """A random-init Mistral checkpoint under the HF tensor names convertMistral reads (convert.swift:59-106), one
        layer at a time.  Draws the SAME random sequence as random_init (same seed => same model), so a converted +
        loaded model can be compared with the in-memory one."""
        from . import weights_io
        gen = torch.Generator(device="cuda").manual_seed(seed)
        kvd = cfg.n_kv_heads * cfg.head_dim
        cache = {}
        state = {"layer": -1}

        def norm_vec():
            return (1.0 + norm_jitter * torch.randn(cfg.dim, generator=gen, device="cuda")).half()

        def gen_layer(i):   # random_init's order: wq wk wv wo w1 w2 w3, attention_norm, ffn_norm
            assert i == state["layer"] + 1, "layers must be requested in order"
            cache.clear()
            p = f"model.layers.{i}."
            for key, (o, n) in (("wq", (cfg.dim, cfg.dim)), ("wk", (kvd, cfg.dim)), ("wv", (kvd, cfg.dim)), ("wo", (cfg.dim, cfg.dim))):
                cache[p + weights_io.HF_ATTN[key]] = _rand_w(o, n, gen)
            for key, (o, n) in (("w1", (cfg.hidden_dim, cfg.dim)), ("w2", (cfg.dim, cfg.hidden_dim)), ("w3", (cfg.hidden_dim, cfg.dim))):
                cache[p + weights_io.HF_MLP[key]] = _rand_w(o, n, gen)
            cache[p + "input_layernorm.weight"] = norm_vec()
            cache[p + "post_attention_layernorm.weight"] = norm_vec()
            state["layer"] = i

        head = {}

        def source(name: str):
            if name in weights_io.HF_HEAD.values():
                if not head:   # drawn after the last layer in random_init: generate every layer's draws first
                    raise KeyError("head tensors are produced by finish()")
                return head[name].cpu().numpy()
            i = int(name.split(".")[2])
            if i != state["layer"]:
                gen_layer(i)
            return cache[name].cpu().numpy()

        def finish():
            out_core = _rand_w(cfg.vocab, cfg.dim, gen)
            head["model.norm.weight"] = norm_vec()
            head["lm_head.weight"] = out_core
            head["model.embed_tokens.weight"] = _rand_w(cfg.vocab, cfg.dim, gen, scale=1.0)

        source.finish = finish
        return source

    @staticmethod
    def convert_random_to_directory(path: str, cfg: MistralConfig = MistralConfig(), seed: int = 1234,
                                    norm_jitter: float = 0.1, native: bool = True) -> str:
        """convertMistral (convert.swift:59-127) on a random-init HF-named checkpoint: bucketize every projection on the
        GPU and write one bucketed-safetensors file per layer + the index (through the C-ABI saver, or the Python
        safetensors package with native=False)."""
        from . import weights_io
        src = DecodeModel.random_hf_source(cfg, seed, norm_jitter)
        # the head tensors live in layer 0's file but are drawn last: materialise all layers' tensors lazily through a
        # two-pass source (layer tensors cached per layer on the host)
        layers = {}
        for i in range(cfg.n_layers):
            names = [f"model.layers.{i}." + n for n in list(weights_io.HF_ATTN.values()) + list(weights_io.HF_MLP.values()) +
                     list(weights_io.HF_NORMS.values())]
            layers[i] = {n: src(n) for n in names}
        src.finish()

        def source(name):
            if name in weights_io.HF_HEAD.values():
                return src(name)
            return layers[int(name.split(".")[2])][name]

        def bucketize(w):
            t = ops.bucketize(torch.from_numpy(w).cuda())
            torch.cuda.synchronize()
            return {k: v.cpu().numpy() for k, v in t.items()}

        return weights_io.convert_mistral(source, path, cfg.n_layers, bucketize, native=native)

    @classmethod
    def from_directory(cls, path: str, cfg: MistralConfig = MistralConfig(), percent_load: int = 16, native: bool = True,
                       model: str = "buckets-FP16", ctx: Optional[ops.Context] = None) -> "DecodeModel":
        """Model.init(from: TensorLoader) (model.swift:40-112) over a bucketed-safetensors directory.  native=True
        reads through the library's C-ABI loader (effort_loader_*), else through the Python safetensors package."""
        from . import weights_io
        tl = (weights_io.NativeTensorLoader if native else weights_io.TensorLoader)(path, model)
        m = cls(cfg, ctx)
        kvd = cfg.n_kv_heads * cfg.head_dim
        dims = {"wq": (cfg.dim, cfg.dim), "wk": (cfg.dim, kvd), "wv": (cfg.dim, kvd), "wo": (cfg.dim, cfg.dim),
                "w1": (cfg.dim, cfg.hidden_dim), "w2": (cfg.hidden_dim, cfg.dim), "w3": (cfg.dim, cfg.hidden_dim)}  # (in, out)

        def dev(a):
            return torch.from_numpy(a).cuda()

        for i in range(cfg.n_layers):
            names = weights_io.layer_tensor_names(i)
            ews = []
            for key in ("wq", "wk", "wv", "wo", "w1", "w2", "w3"):
                in_dim, out_dim = dims[key]
                t = tl.expert_weights(names[key], in_dim, out_dim, percent_load)
                ew = ops.ExpertWeights(dev(t["buckets"]), dev(t["bucket.stats"]), dev(t["probes"]), inDim=in_dim, outDim=out_dim,
                                       percentLoad=percent_load)
                ew.release_reference_layout()
                ews.append(ew)
            m.set_layer(i, *ews, dev(tl[f"layers.{i}.attention_norm"]), dev(tl[f"layers.{i}.ffn_norm"]))
        m.set_head(dev(tl["model.norm"]), dev(tl["output.core"]), dev(tl["tok_embeddings.core"]))
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        return m

    # -- run ----------------------------------------------------------------------------------------------
    def reset(self):
        check(self._L.effort_model_reset(self._h, ops._stream_ptr()), "effort_model_reset")

    def rewind(self, pos: int):
        """Set the position to `pos` (0 <= pos < max_seq), keeping the cache rows: the next step repeats step `pos` on
        the rows the earlier steps left (a test hook for repeating one step from a fixed state)."""
        check(self._L.effort_model_rewind(self._h, int(pos), ops._stream_ptr()), "effort_model_rewind")

    def set_graphs(self, enable: bool):
        check(self._L.effort_model_set_graphs(self._h, 1 if enable else 0), "effort_model_set_graphs")

    def set_fused_glue(self, enable: bool):
        check(self._L.effort_model_set_fused_glue(self._h, 1 if enable else 0), "effort_model_set_fused_glue")

    def set_chain(self, chain: int):
        """2 = fused round-2 chain (5 launches per layer, default), 1 = one kernel per reference op."""
        check(self._L.effort_model_set_chain(self._h, int(chain)), "effort_model_set_chain")

    def set_sampler(self, temperature: Optional[float] = None, top_k: int = 0, top_p: float = 1.0, seed: int = 0):
        """Draw each step's next token on the device (DESIGN.md section 4.6) instead of taking the argmax; None = greedy,
        the default.  New parameters take effect at the next step without recapturing its CUDA graph."""
        prm = None if temperature is None else _lib.Sampler(float(temperature), int(top_k), float(top_p), int(seed))
        check(self._L.effort_model_set_sampler(self._h, None if prm is None else C.byref(prm)), "effort_model_set_sampler")

    def set_scoring(self, enable: bool):
        """Score every step on the device (DESIGN.md section 4.7): step p after reset writes record p of scores() from
        target p of set_score_targets.  Off by default."""
        check(self._L.effort_model_set_scoring(self._h, 1 if enable else 0), "effort_model_set_scoring")
        self._scoring = bool(enable)

    def set_score_targets(self, targets: Optional[torch.Tensor]):
        """Targets (device int32 [n <= max_seq]; None = none) for scoring: entry p is the token that should follow the
        input of step p.  The rest of the row becomes -1 (no target).  Ordered on the current stream; no recapture."""
        n = 0 if targets is None else targets.numel()
        if targets is not None:
            ops._need(targets, torch.int32, "targets")
        check(self._L.effort_model_set_score_targets(self._h, None if targets is None else targets.data_ptr(), n,
                                                     ops._stream_ptr()), "effort_model_set_score_targets")

    def scores(self) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """A device copy of the records [max_seq] as (argmax, rank, logprob) columns; record p is the one the last step
        at position p wrote."""
        ptr = self._L.effort_model_scores(self._h)
        rec = _tensor_from_ptr(ptr, 3 * self.cfg.max_seq, torch.int32).clone().view(self.cfg.max_seq, 3)
        return ops.score_columns(rec)

    def score(self, tokens: list[int], effort: float = 0.25) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Teacher-force `tokens` from a reset and score each next one (runNetwork's returnPredictions, plus the
        log-likelihood).  Returns host tensors: the greedy prediction after every token [n] (int32), the log-probability
        [n - 1] (float32) and the rank [n - 1] (int32) of tokens[1:].  The host synchronises once, at the end; the scoring
        state is restored."""
        n = len(tokens)
        if n < 1 or n > self.cfg.max_seq:
            raise ValueError(f"score needs 1 <= len(tokens) <= max_seq ({self.cfg.max_seq}), got {n}")
        was = self._scoring
        toks = torch.tensor(tokens, dtype=torch.int32, device="cuda")
        try:
            self.set_scoring(True)
            self.set_score_targets(toks[1:])
            self.reset()
            for i in range(n):
                self.step(toks[i:i + 1], effort)
            ptr = self._L.effort_model_scores(self._h)
            rec = _tensor_from_ptr(ptr, 3 * n, torch.int32).view(n, 3).cpu()
        finally:
            self.set_scoring(was)
        argmax, rank, logprob = ops.score_columns(rec)
        return argmax.clone(), logprob[:n - 1].clone(), rank[:n - 1].clone()

    def choose(self, prompt: list[int], candidates: list[int], effort: float = 0.25, top: int = 16) -> Optional[int]:
        """runNetwork's limitLogits rule: feed `prompt` from a reset and rank the candidates against the last logits
        (effort_score).  Returns the index of the lowest-ranked candidate (the first one on equal ranks) when its rank is
        below `top`, else None (the reference's 99)."""
        if not prompt or not candidates:
            raise ValueError("choose needs a non-empty prompt and candidate list")
        if len(prompt) > self.cfg.max_seq:
            raise ValueError(f"prompt ({len(prompt)}) exceeds max_seq ({self.cfg.max_seq})")
        toks = torch.tensor(prompt, dtype=torch.int32, device="cuda")
        self.reset()
        for i in range(len(prompt)):
            self.step(toks[i:i + 1], effort)
        logits = _tensor_from_ptr(self._L.effort_model_logits(self._h), self.cfg.vocab)
        _, rank, _ = ops.score(logits, torch.tensor(candidates, dtype=torch.int32, device="cuda"), self.ctx)
        r = rank.cpu()
        best = int(torch.argmin(torch.where(r < 0, torch.iinfo(torch.int32).max, r)))   # no target (out of range) never wins
        return best if 0 <= int(r[best]) < top else None

    def step(self, token: Optional[torch.Tensor] = None, effort: float = 0.25):
        """Enqueue one decode step (token: device int32[1]; None = previous prediction)."""
        check(self._L.effort_model_step(self._h, None if token is None else token.data_ptr(), float(effort),
                                        ops._stream_ptr()), "effort_model_step")

    def prefill(self, tokens, effort: float = 0.25):
        """Enqueue `tokens` (a list of ints or a device int32 tensor) at the current position, as len(tokens) steps would:
        up to 16 tokens per pass through the multi-token GEMV where the model runs the fused chain (effort_model_prefill),
        plain steps otherwise.  No host synchronisation."""
        if isinstance(tokens, torch.Tensor):
            toks = tokens.to(device="cuda", dtype=torch.int32).contiguous()
        else:
            toks = torch.tensor(list(tokens), dtype=torch.int32, device="cuda")
        check(self._L.effort_model_prefill(self._h, toks.data_ptr(), int(toks.numel()), float(effort), ops._stream_ptr()),
              "effort_model_prefill")

    def step_host(self, token: Optional[int] = None, effort: float = 0.25, logits=None) -> int:
        """End-to-end step with host buffers: H2D token, decode, D2H next token (+ logits into a numpy array)."""
        tok = None
        if token is not None:
            tok = C.c_int32(int(token))
        nxt = C.c_int32(0)
        check(self._L.effort_model_step_host(self._h, None if tok is None else C.byref(tok), float(effort),
                                             C.byref(nxt), None if logits is None else logits.ctypes.data,
                                             ops._stream_ptr()), "effort_model_step_host")
        return int(nxt.value)

    def generate(self, prompt: list[int], n_new: int, effort: float = 0.25) -> list[int]:
        """Reset, feed `prompt`, then n_new - 1 further steps on the previous prediction; returns the n_new predicted
        tokens (greedy, or drawn by the sampler).  Each step's token is copied into a device buffer on the current
        stream; the host synchronises once, at the end."""
        n_steps = len(prompt) + n_new - 1
        if not prompt or n_new < 1:
            raise ValueError("generate needs a non-empty prompt and n_new >= 1")
        if n_steps > self.cfg.max_seq:
            raise ValueError(f"prompt ({len(prompt)}) + n_new ({n_new}) - 1 steps exceed max_seq ({self.cfg.max_seq})")
        toks = torch.tensor(prompt, dtype=torch.int32, device="cuda")
        out = torch.empty(n_new, dtype=torch.int32, device="cuda")
        nxt = _tensor_from_ptr(self._L.effort_model_next_token(self._h), 1, torch.int32)
        self.reset()
        for i in range(len(prompt)):
            self.step(toks[i:i + 1], effort)
        out[0:1].copy_(nxt)
        for j in range(1, n_new):
            self.step(None, effort)
            out[j:j + 1].copy_(nxt)
        torch.cuda.current_stream().synchronize()
        return out.tolist()

    def generate_batch(self, prompts: list[list[int]], n_new: int, effort: float = 0.25,
                       samplers: Optional[list[Optional[dict]]] = None) -> list[list[int]]:
        """Continue up to 16 prompts side by side (DESIGN.md section 4.9).  Each distinct prompt is prefilled into this model
        once and forked into every slot that asks for it; then n_new - 1 batch steps on each slot's previous prediction.
        samplers[b] is None (greedy) or set_sampler's keyword arguments for slot b.  Returns the n_new predicted tokens per
        prompt.  The model is left at the last prompt; the host synchronises once, at the end."""
        n = len(prompts)
        if n < 1 or n_new < 1 or any(not p for p in prompts):
            raise ValueError("generate_batch needs non-empty prompts and n_new >= 1")
        longest = max(len(p) for p in prompts)
        if longest + n_new - 1 > self.cfg.max_seq:
            raise ValueError(f"prompt ({longest}) + n_new ({n_new}) - 1 positions exceed max_seq ({self.cfg.max_seq})")
        batch = DecodeBatch(self, n)
        for b, s in enumerate(samplers or []):
            if s is not None:
                batch.set_sampler(b, **s)
        slots: dict[tuple, list[int]] = {}
        for b, p in enumerate(prompts):
            slots.setdefault(tuple(p), []).append(b)
        for p, bs in slots.items():
            self.reset()
            self.prefill(list(p), effort)
            for b in bs:
                batch.fork(b)
        out = torch.empty(n_new, n, dtype=torch.int32, device="cuda")
        nxt = batch.next_tokens_view()
        out[0].copy_(nxt)
        for j in range(1, n_new):
            batch.step(None, effort)
            out[j].copy_(nxt)
        rows = out.t().cpu()
        return rows.tolist()

    def score_continuations(self, context: list[int], continuations: list[list[int]],
                            effort: float = 0.25) -> list[tuple[float, bool]]:
        """Score up to 16 continuations of one context in lock step, HellaSwag style (DESIGN.md section 4.9): the context
        is prefilled once and forked into one slot per continuation, whose tokens are teacher-forced; shorter continuations
        are padded and their extra targets are -1.  Returns, per continuation, the summed log-probability of its tokens
        and whether every one of them had rank 0 (was greedy's choice).  The host synchronises once."""
        n, c = len(continuations), len(context)
        if not context or n < 1 or any(not t for t in continuations):
            raise ValueError("score_continuations needs a non-empty context and non-empty continuations")
        L = max(len(t) for t in continuations)
        if c + L - 1 > self.cfg.max_seq:
            raise ValueError(f"context ({c}) + longest continuation ({L}) - 1 positions exceed max_seq ({self.cfg.max_seq})")
        batch = DecodeBatch(self, n)
        batch.set_scoring(True)
        for b, t in enumerate(continuations):   # record c - 1 + j scores token j of the continuation
            row = [-1] * (c - 1) + list(t) + [-1] * (L - len(t))
            batch.set_score_targets(b, torch.tensor(row, dtype=torch.int32, device="cuda"))
        feed = torch.tensor([[t[j] if j < len(t) else 0 for t in continuations] for j in range(L - 1)],
                            dtype=torch.int32, device="cuda").view(max(L - 1, 0), n)
        self.reset()
        self.prefill(context, effort)
        batch.fork()
        for j in range(L - 1):
            batch.step(feed[j], effort)
        rank, logprob = batch.scores_view()[1:]
        rank, logprob = rank.view(n, -1)[:, c - 1:c - 1 + L].cpu(), logprob.view(n, -1)[:, c - 1:c - 1 + L].cpu()
        out = []
        for b, t in enumerate(continuations):
            k = len(t)
            out.append((float(logprob[b, :k].double().sum()), bool((rank[b, :k] == 0).all())))
        return out

    def logits(self) -> torch.Tensor:
        """Device logits of the last step as a torch view (copy)."""
        import numpy as np
        n = self.cfg.vocab
        out = torch.empty(n, dtype=torch.float32, device="cuda")
        ptr = self._L.effort_model_logits(self._h)
        from ctypes import c_void_p
        # device-to-device copy through torch: wrap the raw pointer
        src = _tensor_from_ptr(ptr, n)
        out.copy_(src)
        return out

    def next_token(self) -> int:
        ptr = self._L.effort_model_next_token(self._h)
        return int(_tensor_from_ptr(ptr, 1, torch.int32).cpu()[0])

    BUFFERS = {"Q": 0, "K": 1, "V": 2, "ATTN": 3, "KCACHE": 4, "VCACHE": 5, "HIDDEN": 6, "NORMED": 7, "GATE_IN": 8,
               "GATE_IDX": 9, "GATE_VAL": 10, "POS": 11, "CHUNK_Q": 12, "CHUNK_K": 13, "CHUNK_V": 14, "CHUNK_ATTN": 15,
               "CHUNK_LOGITS": 16, "CHUNK_LEN": 17}

    def buffer_view(self, name: str, layer: int = -1) -> Optional[torch.Tensor]:
        """A flat device view of one working buffer as the last step left it (effort_model_buffer; the names are its
        EFFORT_BUF_* without the prefix), or None where the path that step took has no such buffer.  `layer` picks the
        KCACHE / VCACHE layer (negative counts from the end).  The view is ordered on the current stream, and its
        contents change with the next step: copy what must outlive it."""
        if layer < 0:
            layer += self.cfg.n_layers
        n = C.c_size_t(0)
        ptr = self._L.effort_model_buffer(self._h, self.BUFFERS[name], int(layer), C.byref(n))
        if not ptr:
            return None
        return _tensor_from_ptr(ptr, n.value, torch.float32 if name not in ("GATE_IDX", "POS", "CHUNK_LEN") else torch.int32)

    def buffer(self, name: str, layer: int = -1) -> Optional[torch.Tensor]:
        """A device copy of buffer_view(name, layer).  GATE_IDX comes back as int32 (the experts are < 64)."""
        v = self.buffer_view(name, layer)
        return None if v is None else v.clone()

    @property
    def bucket_bytes(self) -> int:
        return int(self._L.effort_model_bucket_bytes(self._h))


class DecodeBatch:
    """Up to 16 sequences decoded together on one DecodeModel (effort_batch_*, DESIGN.md section 4.9).  Every slot has its
    own KV caches, position, logits row, next token, sampler and score rows; a step feeds every slot one token.  A slot's
    results do not depend on the batch size, its index or the other slots.  Keep the batch no longer than its model."""

    def __init__(self, model: DecodeModel, n_seq: int):
        self.model, self.cfg, self.n_seq = model, model.cfg, int(n_seq)
        self._L = model._L
        h = C.c_void_p()
        check(self._L.effort_batch_create(model._h, self.n_seq, C.byref(h)), "effort_batch_create")
        self._h = h

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self._L.effort_batch_destroy(self._h)
                self._h = None
        except Exception:
            pass

    @staticmethod
    def _seq(seq: Optional[int]) -> int:
        return -1 if seq is None else int(seq)

    def reset(self, seq: Optional[int] = None):
        """Position 0 for slot `seq` (None = every slot)."""
        check(self._L.effort_batch_reset(self._h, self._seq(seq), ops._stream_ptr()), "effort_batch_reset")

    def fork(self, seq: Optional[int] = None):
        """Copy the model's current state (cache rows, position, last logits) into slot `seq` (None = every slot) and end
        it as a model step would: its greedy or sampled next token and, with scoring on, record pos - 1."""
        check(self._L.effort_batch_fork(self._h, self._seq(seq), ops._stream_ptr()), "effort_batch_fork")

    def step(self, tokens: Optional[torch.Tensor] = None, effort: float = 0.25):
        """Enqueue one step of every slot (tokens: device int32 [n_seq]; None = each slot's previous prediction)."""
        if tokens is not None:
            ops._need(tokens, torch.int32, "tokens")
            if tokens.numel() != self.n_seq:
                raise ValueError(f"tokens must hold {self.n_seq} entries, got {tokens.numel()}")
        check(self._L.effort_batch_step(self._h, None if tokens is None else tokens.data_ptr(), float(effort),
                                        ops._stream_ptr()), "effort_batch_step")

    def set_sampler(self, seq: Optional[int], temperature: Optional[float] = None, top_k: int = 0, top_p: float = 1.0,
                    seed: int = 0):
        """Slot `seq`'s sampler (None = every slot), as DecodeModel.set_sampler; temperature None = greedy."""
        prm = None if temperature is None else _lib.Sampler(float(temperature), int(top_k), float(top_p), int(seed))
        check(self._L.effort_batch_set_sampler(self._h, self._seq(seq), None if prm is None else C.byref(prm)),
              "effort_batch_set_sampler")

    def set_scoring(self, enable: bool):
        check(self._L.effort_batch_set_scoring(self._h, 1 if enable else 0), "effort_batch_set_scoring")

    def set_score_targets(self, seq: Optional[int], targets: Optional[torch.Tensor]):
        """Slot `seq`'s targets (None = every slot), as DecodeModel.set_score_targets."""
        n = 0 if targets is None else targets.numel()
        if targets is not None:
            ops._need(targets, torch.int32, "targets")
        check(self._L.effort_batch_set_score_targets(self._h, self._seq(seq), None if targets is None else targets.data_ptr(),
                                                     n, ops._stream_ptr()), "effort_batch_set_score_targets")

    def scores_view(self) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """(argmax, rank, logprob) views of every slot's records, flat [n_seq * max_seq]"""
        n = self.n_seq * self.cfg.max_seq
        return ops.score_columns(_tensor_from_ptr(self._L.effort_batch_scores(self._h), 3 * n, torch.int32).view(n, 3))

    def scores(self, seq: int) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """A device copy of slot `seq`'s records [max_seq] as (argmax, rank, logprob) columns."""
        m = self.cfg.max_seq
        return tuple(col[seq * m:(seq + 1) * m].clone() for col in self.scores_view())

    def logits(self) -> torch.Tensor:
        """A device copy of every slot's logits [n_seq][vocab]."""
        return _tensor_from_ptr(self._L.effort_batch_logits(self._h), self.n_seq * self.cfg.vocab).view(self.n_seq, -1).clone()

    def next_tokens_view(self) -> torch.Tensor:
        return _tensor_from_ptr(self._L.effort_batch_next_tokens(self._h), self.n_seq, torch.int32)

    def next_tokens(self) -> list[int]:
        return self.next_tokens_view().cpu().tolist()

    def buffer_view(self, name: str, layer: int = -1, seq: int = 0) -> Optional[torch.Tensor]:
        """A flat device view of one of the batch's buffers (effort_batch_buffer): Q, K, V, ATTN as [n_seq][...] of the last
        layer, KCACHE / VCACHE of `layer` (negative counts from the end) and slot `seq`, POS [n_seq]; None otherwise."""
        if layer < 0:
            layer += self.cfg.n_layers
        n = C.c_size_t(0)
        ptr = self._L.effort_batch_buffer(self._h, DecodeModel.BUFFERS[name], int(layer), int(seq), C.byref(n))
        if not ptr:
            return None
        return _tensor_from_ptr(ptr, n.value, torch.int32 if name == "POS" else torch.float32)

    def buffer(self, name: str, layer: int = -1, seq: int = 0) -> Optional[torch.Tensor]:
        v = self.buffer_view(name, layer, seq)
        return None if v is None else v.clone()


class _CudaArray:
    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (int(ptr), False), "version": 2}


def _tensor_from_ptr(ptr, n, dtype=torch.float32) -> torch.Tensor:
    typestr = "<f4" if dtype == torch.float32 else "<i4"
    return torch.as_tensor(_CudaArray(ptr, n, typestr), device="cuda")
