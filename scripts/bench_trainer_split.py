#!/usr/bin/env python3
"""Times a training step split into Trainer::forward / backward against the whole step, at the headline configuration
(tests/golden/configs/headline.json, 3-D positions, 3 outputs, B = 2^18 by default) with CUDA events:

    python scripts/bench_trainer_split.py [--batch 262144] [--iters 20] [--warmup 5] [--rounds 5] [--out results.json]

  training_step     tcnnb_training_step (fused step + Adam)
  split             forward (inference launch + loss kernel into a ForwardContext) + backward + optimizer_step
  forward           forward alone: what the split adds to a step

Every case runs on its own model. The cases alternate over --rounds rounds; each round times --iters calls back to back and the
mean and spread of the per-round means are printed as one JSON object together with the GPU's name and power limit."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tiny-cuda-nn_b200"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_trainer_ext import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1 << 18)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out")
    args = ap.parse_args()

    import torch

    import tcnn_b200

    if not torch.cuda.is_available():
        raise SystemExit("bench_trainer_split.py measures on the GPU; there is none")
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", "configs", "headline.json")))
    B, n_out = args.batch, 3
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand(B, 3, device="cuda", generator=g)
    y = torch.rand(B, n_out, device="cuda", generator=g)
    models = {name: tcnn_b200.create_from_config(3, n_out, cfg) for name in ("training_step", "split", "forward")}

    def step():
        models["training_step"].trainer.training_step(x, y)

    def split():
        t = models["split"].trainer
        ctx = t.forward(x, y)
        t.backward(ctx, x)
        t.optimizer_step()

    def forward():
        models["forward"].trainer.forward(x, y)

    cases = {"training_step": step, "split": split, "forward": forward}
    for f in cases.values():
        for _ in range(args.warmup):
            f()
    torch.cuda.synchronize()
    per_round = {k: [] for k in cases}
    for _ in range(args.rounds):
        for name, f in cases.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                f()
            e1.record()
            e1.synchronize()
            per_round[name].append(e0.elapsed_time(e1) / args.iters)
    ctx = models["split"].trainer.forward(x, y)
    result = {"gpu": gpu_info(), "batch": B, "iters": args.iters, "rounds": args.rounds,
              "ms_per_step": {k: {"mean": sum(v) / len(v), "min": min(v), "max": max(v)} for k, v in per_round.items()},
              "loss": {"training_step": models["training_step"].trainer.loss(), "split": models["split"].trainer.loss(ctx)}}
    text = json.dumps(result)
    print(text)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
