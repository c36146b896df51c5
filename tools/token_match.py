"""Token match against effort 1.0 (the reference's goBenchmarkSimilarity, benchmarks/benchmark.swift:128-156) on one GPU:

  1. a seeded prompt, then `--tokens` tokens generated greedily at effort 1.0;
  2. the whole sequence teacher-forced at effort 1.0 with scoring on (DecodeModel.score): the control predictions;
  3. for each effort of the reference's makeScale (1, .9 ... .35, then .30 down to .00 in steps of .02): the % of positions
     whose prediction equals the control's, the mean log-probability of the generated continuation, and the share of
     its tokens at rank 0.

Runs on the random-init Mistral-7B by default, or on a bucketed directory (`--model-dir`, DecodeModel.from_directory),
which is what the reference's chart is for: on random weights the low-effort regime is chaotic (DESIGN.md section 2)
and the numbers say little about a trained model.  Prints one JSON line with the card's name and power limit."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def make_scale():
    """benchmark.swift:34-45"""
    return [1.0, 0.9, 0.8, 0.7, 0.6, 0.5, 0.4, 0.35] + [round(0.3 - i * 0.02, 2) for i in range(16)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model-dir", default=None, help="bucketed-safetensors directory (default: random-init model)")
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--vocab", type=int, default=32000)
    ap.add_argument("--tokens", type=int, default=500, help="tokens generated at effort 1.0")
    ap.add_argument("--prompt-len", type=int, default=16)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--efforts", default=None, help="comma-separated efforts (default: the reference's makeScale)")
    args = ap.parse_args()

    import torch
    from effort_b200.model import DecodeModel, MistralConfig
    from tools.clocks import ClockSampler

    efforts = [float(e) for e in args.efforts.split(",")] if args.efforts else make_scale()
    card = ClockSampler(index=torch.cuda.current_device())
    n = args.prompt_len + args.tokens
    cfg = MistralConfig(n_layers=args.layers, vocab=args.vocab, max_seq=max(n, 64))
    if args.model_dir:
        model = DecodeModel.from_directory(args.model_dir, cfg)
        source = args.model_dir
    else:
        model = DecodeModel.random_init(cfg, seed=args.seed)
        source = f"random-init Mistral-7B architecture, {args.layers} layers, vocab {args.vocab}, seed {args.seed}"
    g = torch.Generator().manual_seed(args.seed + 1)
    prompt = torch.randint(0, cfg.vocab, (args.prompt_len,), generator=g).tolist()

    t0 = time.time()
    seq = prompt + model.generate(prompt, args.tokens, effort=1.0)
    control, _, _ = model.score(seq, 1.0)
    cont = slice(args.prompt_len - 1, n - 1)          # records whose target is a generated token
    rows = []
    for e in efforts:
        pred, lp, rank = model.score(seq, e)
        rows.append({"effort": e, "match_pct": round(100.0 * float((pred == control).float().mean()), 2),
                     "mean_logprob": round(float(lp[cont].double().mean()), 4),
                     "rank0_share": round(float((rank[cont] == 0).float().mean()), 4)})
    print(json.dumps({
        "gpu": card.name, "power_limit_w": card.power_limit_w, "model": source, "prompt_len": args.prompt_len,
        "tokens": args.tokens, "positions": n, "results": rows, "seconds": round(time.time() - t0, 1),
    }))


if __name__ == "__main__":
    main()
