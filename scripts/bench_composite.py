#!/usr/bin/env python3
"""Times factorized grid encodings on the general path with CUDA events, B = 2^18 by default, FFMLP 64x2 behind every encoding:
    python scripts/bench_composite.py [--batch 262144] [--iters 20] [--warmup 5] [--rounds 5]
  grid1        one 3-D HashGrid (L=16, F=2, T=2^19), forced onto the general path (debug_set("general", 1)): the baseline
  sum2         Sum of two such grids (both at dims_to_encode_begin 0)
  concat2      Concatenation of the same two grids (a 64-wide network input)
  planes3      Product of three 2-D planes (L=16, F=2, T=2^19) at dims_to_encode_begin 0, 1, 2 of 4-D positions
For each: training_step (forward + backward + Adam) and inference, alternating over --rounds rounds of --iters calls; mean, min and
max of the per-round means. A separate torch.profiler pass over a few steps reports the device time of the reduce kernels
(reduce_forward_kernel, reduce_product_backward_kernel, sum_input_gradients_kernel) next to that of the grid kernels. One JSON object
with the GPU's name and power limit is printed."""
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


def grid(n_dims, begin=None, log2=19):
    e = {"otype": "HashGrid", "n_levels": 16, "n_features_per_level": 2, "log2_hashmap_size": log2, "base_resolution": 16, "per_level_scale": 1.5, "n_dims_to_encode": n_dims}
    if begin is not None:
        e["dims_to_encode_begin"] = begin
    return e


NET = {"otype": "FullyFusedMLP", "activation": "ReLU", "output_activation": "None", "n_neurons": 64, "n_hidden_layers": 2}
CASES = {
    "grid1": (3, {k: v for k, v in grid(3).items() if k != "n_dims_to_encode"}),
    "sum2": (3, {"otype": "Composite", "reduction": "Sum", "nested": [grid(3, 0), grid(3, 0)]}),
    "concat2": (3, {"otype": "Composite", "nested": [grid(3, 0), grid(3, 0)]}),
    "planes3": (4, {"otype": "Composite", "reduction": "Product", "nested": [grid(2, 0), grid(2, 1), grid(2, 2)]}),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1 << 18)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch

    import tcnn_b200

    if not torch.cuda.is_available():
        raise SystemExit("bench_composite.py measures on the GPU; there is none")
    B = args.batch
    g = torch.Generator(device="cuda").manual_seed(1)
    models, data = {}, {}
    for name, (n_in, enc) in CASES.items():
        cfg = {"loss": {"otype": "RelativeL2"}, "optimizer": {"otype": "Adam", "learning_rate": 1e-2}, "encoding": enc, "network": NET}
        m = tcnn_b200.create_from_config(n_in, 3, cfg)
        if name == "grid1":
            m.debug_set("general", 1)
        models[name] = m
        data[name] = (torch.rand(B, n_in, device="cuda", generator=g), torch.rand(B, 3, device="cuda", generator=g))

    def step(name):
        x, y = data[name]
        models[name].trainer.training_step(x, y)

    def infer(name):
        models[name].network.inference(data[name][0])

    fns = {f"{k}/{kind}": (lambda k=k, f=f: f(k)) for k in CASES for kind, f in (("train", step), ("inference", infer))}
    for f in fns.values():
        for _ in range(args.warmup):
            f()
    torch.cuda.synchronize()
    per_round = {k: [] for k in fns}
    for _ in range(args.rounds):
        for name, f in fns.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                f()
            e1.record()
            e1.synchronize()
            per_round[name].append(e0.elapsed_time(e1) / args.iters)

    # device time per kernel family over 5 training steps of each reduced case
    from torch.profiler import ProfilerActivity, profile

    kernels = {}
    for name in ("sum2", "planes3"):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                step(name)
            torch.cuda.synchronize()
        fam = {}
        for ev in prof.key_averages():
            key = ev.key
            if "reduce_forward_kernel" in key:
                k = "reduce_forward"
            elif "reduce_product_backward_kernel" in key:
                k = "reduce_product_backward"
            elif "sum_input_gradients_kernel" in key:
                k = "sum_input_gradients"
            elif "grid" in key.lower():
                k = "grid_kernels"
            else:
                continue
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            fam[k] = fam.get(k, 0.0) + t / 5 / 1000.0  # ms per step
        kernels[name] = fam
    result = {"gpu": gpu_info(), "batch": B, "iters": args.iters, "rounds": args.rounds,
              "ms": {k: {"mean": sum(v) / len(v), "min": min(v), "max": max(v)} for k, v in per_round.items()},
              "device_ms_per_step": kernels, "loss": {k: m.trainer.loss() for k, m in models.items()}}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
