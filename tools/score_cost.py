"""Per-token cost of the device scorer (DESIGN.md section 4.7) on one GPU, in one process:

  * the card's name and power limit;
  * the Mistral-7B random model's greedy device-resident decode at one effort with scoring off and on (every step scores
    the next token of the sequence), alternated `--rounds` times, CUDA events around `--steps` graph-replayed steps after
    `--warmup`;
  * the scorer alone at V = 32000: `--calls` hook calls (one target each) captured in one CUDA graph, CUDA events around
    its replay.

Prints one JSON line.  bench.py measures greedy decoding without scoring."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--effort", type=float, default=0.25)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--vocab", type=int, default=32000)
    ap.add_argument("--calls", type=int, default=1000)
    args = ap.parse_args()

    import torch
    from effort_b200 import _lib, ops
    from effort_b200.model import DecodeModel, MistralConfig
    from tools.clocks import ClockSampler

    card = ClockSampler(index=torch.cuda.current_device())
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        cfg = MistralConfig(n_layers=args.layers, vocab=args.vocab, max_seq=max(2048, args.steps + args.warmup + 8))
        model = DecodeModel.random_init(cfg, seed=1234)
        seq = torch.randint(0, cfg.vocab, (args.warmup + args.steps,), generator=torch.Generator().manual_seed(4242),
                            dtype=torch.int32).cuda()
        toks = [seq[i:i + 1] for i in range(len(seq))]
        model.set_score_targets(seq[1:])

        def decode(scoring):
            model.set_scoring(scoring)
            model.reset()
            for t in toks[:args.warmup]:
                model.step(t, args.effort)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for t in toks[args.warmup:]:
                model.step(t, args.effort)
            e1.record(stream)
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) * 1e3 / args.steps   # us per token

        runs = {"greedy": [], "scoring": []}
        for _ in range(args.rounds):
            runs["greedy"].append(decode(False))
            runs["scoring"].append(decode(True))
        model.set_scoring(False)

        ctx = ops.default_context()
        lg = torch.randn(32000, generator=torch.Generator(device="cuda").manual_seed(5), device="cuda") * 2
        tgt = torch.tensor([17], dtype=torch.int32, device="cuda")
        out = torch.empty(3, dtype=torch.int32, device="cuda")

        def calls():
            s = torch.cuda.current_stream().cuda_stream
            for _ in range(args.calls):
                _lib.check(ctx._L.effort_score(ctx._h, lg.data_ptr(), lg.numel(), tgt.data_ptr(), 1, out.data_ptr(), s),
                           "effort_score")

        calls()                                               # warm-up (module load)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            calls()
        g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        g.replay()
        e1.record(stream)
        torch.cuda.synchronize()
        hook_us = e0.elapsed_time(e1) * 1e3 / args.calls

    med = {k: sorted(v)[len(v) // 2] for k, v in runs.items()}
    print(json.dumps({
        "gpu": card.name, "power_limit_w": card.power_limit_w, "effort": args.effort, "layers": args.layers,
        "vocab": args.vocab, "steps": args.steps,
        "us_per_token": {k: [round(x, 1) for x in v] for k, v in runs.items()},
        "median_cost_us_per_token": round(med["scoring"] - med["greedy"], 1),
        "median_cost_pct": round(100.0 * (med["scoring"] - med["greedy"]) / med["greedy"], 2),
        "hook_us_per_call_v32000": round(hook_us, 2),
    }))


if __name__ == "__main__":
    main()
