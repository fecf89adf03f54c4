#!/usr/bin/env python3
"""Times Trainer::training_step's optional arguments at the headline configuration (tests/golden/configs/headline.json, 3-D
positions, 3 outputs, B = 2^18 by default) with CUDA events:

    python scripts/bench_trainer_ext.py [--batch 262144] [--iters 20] [--warmup 5] [--rounds 5] [--out results.json]

  plain            tcnnb_training_step (fused step + Adam)
  data_pdf         the same step with a per-element data_pdf
  external_dL_dy   network inference + the application's own L2 dL/dy (torch) + a step on external_dL_dy
  accumulate_4x    four micro-batches of B / 4: Overwrite, then three Accumulate steps without the optimizer, one optimizer_step

Every case runs on its own model. The cases alternate over --rounds rounds; each round times --iters calls back to back and the
mean and spread of the per-round means are printed as one JSON object together with the GPU's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tiny-cuda-nn_b200"))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


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
        raise SystemExit("bench_trainer_ext.py measures on the GPU; there is none")
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", "configs", "headline.json")))
    B, n_out, loss_scale = args.batch, 3, 128.0
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand(B, 3, device="cuda", generator=g)
    y = torch.rand(B, n_out, device="cuda", generator=g)
    pdf = 0.2 + 4.8 * torch.rand(B, n_out, device="cuda", generator=g)
    models = {name: tcnn_b200.create_from_config(3, n_out, cfg) for name in ("plain", "data_pdf", "external_dL_dy", "accumulate_4x")}
    dy = torch.zeros(B, 16, dtype=torch.float16, device="cuda")
    q = B // 4

    def plain():
        models["plain"].trainer.training_step(x, y)

    def with_pdf():
        models["data_pdf"].trainer.training_step(x, y, data_pdf=pdf)

    def external():
        m = models["external_dL_dy"]
        out = m.network.inference(x)
        dy[:, :n_out] = (loss_scale * 2 / (B * n_out)) * (out - y)
        m.trainer.training_step(x, None, external_dL_dy=dy)

    def accumulate():
        t = models["accumulate_4x"].trainer
        for k in range(4):
            t.training_step(x[k * q : (k + 1) * q], y[k * q : (k + 1) * q], run_optimizer=False, gradient_mode="Overwrite" if k == 0 else "Accumulate")
        t.optimizer_step()

    cases = {"plain": plain, "data_pdf": with_pdf, "external_dL_dy": external, "accumulate_4x": accumulate}
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
    losses = {}
    for name in ("plain", "data_pdf"):
        losses[name] = models[name].trainer.loss()
    result = {"gpu": gpu_info(), "batch": B, "iters": args.iters, "rounds": args.rounds,
              "ms_per_step": {k: {"mean": sum(v) / len(v), "min": min(v), "max": max(v)} for k, v in per_round.items()}, "last_loss": losses}
    text = json.dumps(result)
    print(text)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
