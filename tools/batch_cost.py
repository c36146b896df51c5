"""Throughput of batch decode (DecodeBatch, DESIGN.md section 4.9) against single-stream stepping, on one GPU, in one
process:

  * the card's name and power limit;
  * the Mistral-7B random model (32 layers, vocab 32000): for each batch size and effort, aggregate tokens/s of
    `--steps` batch steps (n_seq tokens each) with every slot forked from a `--prompt`-token prefill, and tokens/s of
    `--steps` single-stream `step` calls from the same prompt; CUDA events around the steps only, one untimed warm-up of
    both (first eager run, graph capture), then `--rounds` alternated rounds reported as [min, max];
  * the batch size from which a batch step beats stepping the same sequences one after another, per effort.

Prints one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-seq", default="1,4,8,16")
    ap.add_argument("--efforts", default="1.0,0.5,0.25")
    ap.add_argument("--prompt", type=int, default=64)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--vocab", type=int, default=32000)
    args = ap.parse_args()
    sizes = [int(x) for x in args.n_seq.split(",")]
    efforts = [float(x) for x in args.efforts.split(",")]

    import torch
    from effort_b200.model import DecodeBatch, DecodeModel, MistralConfig
    from tools.clocks import ClockSampler

    card = ClockSampler(index=torch.cuda.current_device())
    stream = torch.cuda.Stream()

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e-3   # seconds

    with torch.cuda.stream(stream):
        cfg = MistralConfig(n_layers=args.layers, vocab=args.vocab, max_seq=args.prompt + args.steps + 8)
        model = DecodeModel.random_init(cfg, seed=1234)
        prompt = torch.randint(0, cfg.vocab, (args.prompt,), generator=torch.Generator().manual_seed(4242),
                               dtype=torch.int32).cuda()
        batches = {n: DecodeBatch(model, n) for n in sizes}

        def single_steps(effort, n_steps):
            model.reset()
            model.prefill(prompt, effort)
            torch.cuda.synchronize()
            return timed(lambda: [model.step(None, effort) for _ in range(n_steps)])

        def batch_steps(bt, effort, n_steps):
            model.reset()
            model.prefill(prompt, effort)
            bt.fork()
            torch.cuda.synchronize()
            return timed(lambda: [bt.step(None, effort) for _ in range(n_steps)])

        res, crossover = {}, {}
        for effort in efforts:
            single_steps(effort, 3)   # warm-up: eager step, capture, replay
            for bt in batches.values():
                batch_steps(bt, effort, 3)
            rec = {"single_tok_s": []}
            rec.update({f"batch{n}_tok_s": [] for n in sizes})
            for _ in range(args.rounds):
                rec["single_tok_s"].append(args.steps / single_steps(effort, args.steps))
                for n, bt in batches.items():
                    rec[f"batch{n}_tok_s"].append(n * args.steps / batch_steps(bt, effort, args.steps))
            res[str(effort)] = {k: [round(min(v), 1), round(max(v), 1)] for k, v in rec.items()}
            best_single = max(rec["single_tok_s"])
            wins = [n for n in sizes if min(rec[f"batch{n}_tok_s"]) > best_single]
            crossover[str(effort)] = min(wins) if wins else None

    print(json.dumps({"gpu": card.name, "power_limit_w": card.power_limit_w, "layers": args.layers, "vocab": args.vocab,
                      "prompt": args.prompt, "steps": args.steps, "tok_s_min_max": res,
                      "smallest_batch_faster_than_single": crossover}))


if __name__ == "__main__":
    main()
