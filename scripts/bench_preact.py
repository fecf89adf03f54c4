#!/usr/bin/env python3
"""Cost of the pre-activation path: HashGrid + CutlassMLP training steps (the general path) with ReLU against Sine and SiLU, whose
kernels also write the fp16 pre-activations in the forward pass and read them in the backward chain.

    python scripts/bench_preact.py [--batch-log2 18] [--steps 50] [--rounds 5] [--networks 64x2,128x4]

--networks takes n_neurons x n_hidden_layers pairs, e.g. 256x3,256x8 for SIREN / neural-SDF sized networks.

The activations are timed in alternation (one block of --steps steps per activation and round, CUDA events), so that clock and
thermal drift hits all of them alike; the median and range over the rounds are printed, one JSON line per configuration."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tiny-cuda-nn_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import tcnn_b200  # noqa: E402

ENCODING = {"otype": "HashGrid", "n_levels": 16, "n_features_per_level": 2, "log2_hashmap_size": 19, "base_resolution": 16, "per_level_scale": 1.5}
NETWORKS = "64x2,128x4"
# "ReLU*": ReLU forced onto the general path (a 64-wide ReLU network otherwise takes the fused training kernel), the like-for-like
# baseline of the Sine / SiLU steps
ACTIVATIONS = ["ReLU", "ReLU*", "Sine", "SiLU"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch-log2", type=int, default=18)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--networks", default=NETWORKS)
    args = ap.parse_args()
    B = 1 << args.batch_log2
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.rand(B, 3, device="cuda", generator=g)
    y = torch.rand(B, 3, device="cuda", generator=g)
    for width, nh in [tuple(int(v) for v in n.split("x")) for n in args.networks.split(",")]:
        models = {}
        for act in ACTIVATIONS:
            cfg = {"loss": {"otype": "L2"}, "optimizer": {"otype": "Adam", "learning_rate": 1e-3}, "encoding": ENCODING,
                   "network": {"otype": "CutlassMLP", "activation": act.rstrip("*"), "output_activation": "None", "n_neurons": width, "n_hidden_layers": nh}}
            models[act] = tcnn_b200.create_from_config(3, 3, cfg)
            if act.endswith("*"):
                models[act].debug_set("general", 1)
            for _ in range(args.warmup):
                models[act].trainer.training_step(x, y)
        torch.cuda.synchronize()
        times = {act: [] for act in ACTIVATIONS}
        for _ in range(args.rounds):
            for act in ACTIVATIONS:
                start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                start.record()
                for _ in range(args.steps):
                    models[act].trainer.training_step(x, y)
                end.record()
                end.synchronize()
                times[act].append(start.elapsed_time(end) / args.steps)
        res = {"network": f"CutlassMLP {width}x{nh}", "batch": B, "device": torch.cuda.get_device_name()}
        for act in ACTIVATIONS:
            t = np.array(times[act])
            res[act] = {"median_ms": round(float(np.median(t)), 4), "min_ms": round(float(t.min()), 4), "max_ms": round(float(t.max()), 4)}
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
