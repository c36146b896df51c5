"""Prompt throughput of prefill (effort_model_prefill, DESIGN.md section 4.8) against stepping, on one GPU, in one process:

  * the card's name and power limit;
  * the Mistral-7B random model (32 layers, vocab 32000): prompt tokens/s of `prefill` and of one `step` per token for
    each prompt length and effort, from a reset, after one untimed warm-up of both, alternated `--rounds` times, CUDA
    events around the whole prompt;
  * the multi-token GEMV alone at 4096 -> 14336 (one of the model's w1 matrices) for T = 1, 4, 8, 16 inputs against T
    single-token bucketMul launches, CUDA events around `--reps` repetitions.

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
    ap.add_argument("--prompts", default="128,1024")
    ap.add_argument("--efforts", default="1.0,0.5,0.25")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--vocab", type=int, default=32000)
    ap.add_argument("--reps", type=int, default=200)
    args = ap.parse_args()
    prompts = [int(x) for x in args.prompts.split(",")]
    efforts = [float(x) for x in args.efforts.split(",")]

    import torch
    from effort_b200 import ops
    from effort_b200.model import DecodeModel, MistralConfig
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
        cfg = MistralConfig(n_layers=args.layers, vocab=args.vocab, max_seq=max(2048, max(prompts)))
        model = DecodeModel.random_init(cfg, seed=1234)
        seq = torch.randint(0, cfg.vocab, (max(prompts),), generator=torch.Generator().manual_seed(4242),
                            dtype=torch.int32).cuda()
        toks = [seq[i:i + 1] for i in range(len(seq))]

        def run_prefill(n, effort):
            model.reset()
            model.prefill(seq[:n], effort)

        def run_steps(n, effort):
            model.reset()
            for t in toks[:n]:
                model.step(t, effort)

        prompt = {}
        for n in prompts:
            for effort in efforts:
                run_prefill(n, effort)   # warm-up: first-run eager chunks, graph captures
                run_prefill(n, effort)
                run_steps(min(n, 32), effort)
                rec = {"prefill_tok_s": [], "step_tok_s": []}
                for _ in range(args.rounds):
                    rec["prefill_tok_s"].append(round(n / timed(lambda: run_prefill(n, effort)), 1))
                    rec["step_tok_s"].append(round(n / timed(lambda: run_steps(n, effort)), 1))
                med = {k: sorted(v)[len(v) // 2] for k, v in rec.items()}
                rec["median_speedup"] = round(med["prefill_tok_s"] / med["step_tok_s"], 2)
                prompt[f"{n}@{effort}"] = rec

        w1 = model.layers[0][4]
        gemv = {}
        for effort in efforts:
            for T in (1, 4, 8, 16):
                V = torch.randn(T, w1.inSize, generator=torch.Generator(device="cuda").manual_seed(T), device="cuda")
                out = torch.empty(w1.outSize, dtype=torch.float32, device="cuda")
                rows = [V[t] for t in range(T)]

                def multi():
                    for _ in range(args.reps):
                        ops.bucket_mul_multi(V, w1, effort)

                def single():
                    for _ in range(args.reps):
                        for v in rows:
                            ops.bucketMul(v, w1, None, out, effort)

                multi(); single()
                gemv[f"T{T}@{effort}"] = {"multi_us": round(timed(multi) * 1e6 / args.reps, 1),
                                          "singles_us": round(timed(single) * 1e6 / args.reps, 1)}

    print(json.dumps({"gpu": card.name, "power_limit_w": card.power_limit_w, "layers": args.layers, "vocab": args.vocab,
                      "prompt": prompt, "gemv_4096x14336": gemv}))


if __name__ == "__main__":
    main()
