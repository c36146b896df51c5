"""Bit-reproducibility of long fused-chain decodes (DESIGN.md section 4.7): teacher-force one sequence once as the
reference, then repeat single steps from the reference state and count the repeats whose bits differ.

Each repeat rewinds the model (effort_model_rewind) and runs `--steps` steps ending at position p: 1 repeats step p
alone (its matrices' cutoff hints then equal the cutoffs the step computes), 2 runs step p - 1 first, so that each
step starts from the hints the step before it left, as in a decode.  A repeat is bad when a step's logits, next token,
K/V rows or score record differ from the reference in any bit; the rows it wrote are restored from the reference
afterwards, so one bad repeat does not spoil the next.  All comparisons stay on the device: one sync per position.

Everything runs on a side stream: the model captures and replays CUDA graphs only there (--graphs 0: eager steps).

    python tools/chain_repro.py --repeats 4096 --positions 1200,1500,1750,2047 [--hint 0] [--stage 3] [--prefetch 1]
                                [--graphs 0] [--layers 1] [--steps 1] [--scoring 0]
    EFFORT_PDL=0 python tools/chain_repro.py ...   (plain stream order: read once per process)

Prints one JSON line: per position the number of bad repeats and the first bad one (-1: none)."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from effort_b200 import ops  # noqa: E402
from effort_b200.model import DecodeModel, MistralConfig, _tensor_from_ptr  # noqa: E402

EFFORT = 0.25


def make_model(n_layers=2, vocab=32000, max_seq=2048, seed=11):
    return DecodeModel.random_init(MistralConfig(n_layers=n_layers, vocab=vocab, max_seq=max_seq), seed=seed)


def sequence(m, seed=5):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, m.cfg.vocab, (m.cfg.max_seq,), generator=g, dtype=torch.int32).cuda()


class Views:
    """live device views of the model's logits, next token, score records and K/V caches"""

    def __init__(self, m):
        L, h, c = m._L, m._h, m.cfg
        self.logits = _tensor_from_ptr(L.effort_model_logits(h), c.vocab).view(torch.int32)
        self.next = _tensor_from_ptr(L.effort_model_next_token(h), 1, torch.int32)
        self.rec = _tensor_from_ptr(L.effort_model_scores(h), 3 * c.max_seq, torch.int32).view(c.max_seq, 3)
        self.kvd = c.n_kv_heads * c.head_dim
        self.kv = None  # the caches have a buffer view only once a step has run

    def caches(self, m):
        if self.kv is None:
            self.kv = [m.buffer_view(n, l).view(m.cfg.max_seq, self.kvd) for l in range(m.cfg.n_layers) for n in ("KCACHE", "VCACHE")]
        return self.kv


class Reference:
    """one teacher-forced decode with scoring and sampling off: every step's logits and next token, the final K/V caches
    and the records effort_score gives on each step's logits"""

    def __init__(self, m, toks, effort=EFFORT):
        S, V = m.cfg.max_seq, m.cfg.vocab
        m.set_scoring(False)
        m.set_sampler(None)
        self.views = Views(m)
        self.logits = torch.empty((S, V), dtype=torch.int32, device="cuda")
        self.next = torch.empty(S, dtype=torch.int32, device="cuda")
        m.reset()
        for p in range(S):
            m.step(toks[p:p + 1], effort)
            self.logits[p].copy_(self.views.logits)
            self.next[p:p + 1].copy_(self.views.next)
        self.kv = [t.clone() for t in self.views.caches(m)]
        targets = torch.cat([toks[1:], torch.tensor([-1], dtype=torch.int32, device="cuda")])
        self.rec = torch.empty((S, 3), dtype=torch.int32, device="cuda")
        for p in range(S):
            a, r, lp = ops.score(self.logits[p].view(torch.float32), targets[p:p + 1])
            self.rec[p, 0], self.rec[p, 1], self.rec[p, 2] = a[0], r[0], lp.view(torch.int32)[0]
        self.targets = targets
        torch.cuda.synchronize()


def side_stream():
    """a non-default stream: the model captures and replays CUDA graphs only there (the legacy stream cannot capture)"""
    return torch.cuda.stream(torch.cuda.Stream())


def _step_bad(ref, views, p, scoring, greedy=True):
    """device bool: step p's logits (and greedy token, record) differ from the reference"""
    bad = (views.logits != ref.logits[p]).any()
    if greedy:
        bad = bad | (views.next[0] != ref.next[p])
    if scoring:
        bad = bad | (views.rec[p] != ref.rec[p]).any()
    return bad


def repeat_steps(m, ref, toks, p, repeats, steps=2, scoring=True, effort=EFFORT):
    """(bad repeats, first bad repeat or -1, error flag) of `repeats` repeats of steps p - steps + 1 .. p from the reference state"""
    assert torch.cuda.current_stream().cuda_stream != 0, "on the legacy stream the model never replays its graphs"
    views = ref.views
    kv = views.caches(m)
    p0 = p - steps + 1
    assert p0 >= 0
    for t, r in zip(kv, ref.kv):  # whatever an earlier run left in the caches
        t.copy_(r)
    if scoring:
        m.set_score_targets(ref.targets)
    bad_count = torch.zeros((), dtype=torch.int32, device="cuda")
    first = torch.full((), -1, dtype=torch.int32, device="cuda")
    for i in range(repeats):
        m.rewind(p0)
        if scoring:
            views.rec[p0:p + 1].fill_(0x5A5A5A5A)  # a scorer that wrote nothing cannot match
        bad = torch.zeros((), dtype=torch.bool, device="cuda")
        for q in range(p0, p + 1):
            m.step(toks[q:q + 1], effort)
            bad = bad | _step_bad(ref, views, q, scoring)
        for t, r in zip(kv, ref.kv):
            bad = bad | (t[p0:p + 1] != r[p0:p + 1]).any()
            t[p0:p + 1].copy_(r[p0:p + 1])
        bad_count += bad.to(torch.int32)
        first = torch.where((first < 0) & bad, torch.tensor(i, dtype=torch.int32, device="cuda"), first)
    torch.cuda.synchronize()
    return int(bad_count), int(first), ops.default_context().errorFlag()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=4096)
    ap.add_argument("--positions", default="1200,1500,1750,2047")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--layers", type=int, default=2)
    ap.add_argument("--stage", type=int, default=4)
    ap.add_argument("--hint", type=int, default=1)
    ap.add_argument("--prefetch", type=int, default=0)
    ap.add_argument("--graphs", type=int, default=1)
    ap.add_argument("--scoring", type=int, default=1)
    a = ap.parse_args()
    ctx = ops.default_context()
    ctx.setCutoffMode("select")
    ctx.setOption("stage", a.stage)
    ctx.setOption("hint", a.hint)
    ctx.setOption("prefetch", a.prefetch)
    out = {"knobs": {k: v for k, v in vars(a).items() if k != "positions"}, "pdl": ops.pdl_enabled(), "positions": {}}
    with side_stream():
        m = make_model(n_layers=a.layers)
        m.set_graphs(bool(a.graphs))
        toks = sequence(m)
        ref = Reference(m, toks)
        m.set_scoring(bool(a.scoring))
        for p in [int(x) for x in a.positions.split(",")]:
            n, first, flag = repeat_steps(m, ref, toks, p, a.repeats, a.steps, bool(a.scoring))
            out["positions"][p] = {"bad": n, "first": first, "err_flag": flag}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
