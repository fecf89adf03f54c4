#!/usr/bin/env python3
"""Networks with more outputs than neurons: stand-alone inference and training steps against the same network with 16 outputs.

    python scripts/bench_wide_out.py [--steps 50] [--rounds 5] [--skip-train] [--reference oracle/_ref/ref_harness]

Inference (tcnn_b200.Network.inference_mixed_precision) at B = 2^18 and 2^21 for FullyFusedMLP 64 x 2, 32 -> {16, 128, 1024} and
CutlassMLP 256 x 4, 64 -> {16, 512, 768}; TFLOP/s counts 2 * B * (sum of the matrices' sizes). Training steps at B = 2^18 for
HashGrid (L = 16, F = 2, T = 2^19) + FullyFusedMLP 64 x 2 -> 128 and + CutlassMLP 256 x 4 -> 512, each next to the same network with
16 outputs forced onto the general path, so that the difference is the output layer's cost.

With the reference harness built (oracle/_ref/ref_harness, the default of --reference when present), every row also carries the
unmodified reference on the same shape: `mlpbench` (inference_mixed_precision, CUDA events) and `bench` (training steps), run
after this library's rounds of the group.

Every configuration of a group is timed in alternation (one block of --steps calls per configuration and round, CUDA events), so
that clock and thermal drift hits all of them alike; median and range over the rounds, one JSON line per group, with the card's
name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tiny-cuda-nn_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import tcnn_b200  # noqa: E402

ENCODING = {"otype": "HashGrid", "n_levels": 16, "n_features_per_level": 2, "log2_hashmap_size": 19, "base_resolution": 16, "per_level_scale": 1.5}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = torch.cuda.get_device_name()
    return out


def ref_run(args, *cmd):
    """The reference harness's JSON line, or None when it is not available."""
    if not args.reference or not os.path.exists(args.reference):
        return None
    out = subprocess.run([args.reference, *map(str, cmd)], capture_output=True, text=True, timeout=600)
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    return json.loads(lines[-1]) if out.returncode == 0 and lines else None


def timed(fns, steps, warmup, rounds):
    for f in fns.values():
        for _ in range(warmup):
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(steps):
                f()
            end.record()
            end.synchronize()
            times[k].append(start.elapsed_time(end) / steps)
    return {k: np.array(v) for k, v in times.items()}


def stat(t):
    return {"median_ms": round(float(np.median(t)), 4), "min_ms": round(float(t.min()), 4), "max_ms": round(float(t.max()), 4)}


def inference_group(otype, width, nh, n_in, outs, B, args):
    fns, flops = {}, {}
    g = torch.Generator(device="cuda").manual_seed(0)
    x = (torch.rand(B, n_in, device="cuda", generator=g) * 2 - 1).half()
    keep = []
    for n_out in outs:
        net = tcnn_b200.Network(n_in, n_out, {"otype": otype, "n_neurons": width, "n_hidden_layers": nh, "activation": "ReLU", "output_activation": "None"})
        p16 = net.initial_params(seed=1).half().contiguous()
        keep.append((net, p16))
        fns[n_out] = lambda net=net, p16=p16: net.inference_mixed_precision(x, p16)
        flops[n_out] = 2.0 * B * net.n_params
    t = timed(fns, args.steps, args.warmup, args.rounds)
    res = {"bench": "inference", "network": f"{otype} {width}x{nh}", "n_in": n_in, "batch": B, "card": card()}
    for n_out in outs:
        res[f"out{n_out}"] = {**stat(t[n_out]), "tflops": round(flops[n_out] / (np.median(t[n_out]) * 1e-3) / 1e12, 1)}
        ref = ref_run(args, "mlpbench", otype, width, nh, n_in, n_out, B, args.steps * args.rounds, args.warmup, 0)
        if ref:
            res[f"out{n_out}"]["reference_ms"] = round(ref["ms_per_batch"], 4)
            res[f"out{n_out}"]["reference_tflops"] = round(flops[n_out] / (ref["ms_per_batch"] * 1e-3) / 1e12, 1)
    print(json.dumps(res), flush=True)


def train_group(otype, width, nh, n_out, B, args):
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.rand(B, 3, device="cuda", generator=g)
    fns = {}
    models = []
    for label, n in (("out16_general", 16), (f"out{n_out}", n_out)):
        cfg = {"loss": {"otype": "L2"}, "optimizer": {"otype": "Adam", "learning_rate": 1e-3}, "encoding": ENCODING,
               "network": {"otype": otype, "activation": "ReLU", "output_activation": "None", "n_neurons": width, "n_hidden_layers": nh}}
        m = tcnn_b200.create_from_config(3, n, cfg)
        m.debug_set("general", 1)
        y = torch.rand(B, n, device="cuda", generator=g)
        models.append((m, y))
        fns[label] = lambda m=m, y=y: m.trainer.training_step(x, y)
    t = timed(fns, args.steps, args.warmup, args.rounds)
    res = {"bench": "training_step", "network": f"HashGrid + {otype} {width}x{nh}", "batch": B, "card": card()}
    for k in fns:
        res[k] = stat(t[k])
    with tempfile.TemporaryDirectory() as tmp:
        for label, n in (("out16_general", 16), (f"out{n_out}", n_out)):
            path = os.path.join(tmp, "config.json")
            json.dump({**cfg, "loss": {"otype": "L2"}}, open(path, "w"))
            ref = ref_run(args, "bench", path, 3, n, B, args.steps * args.rounds, args.warmup, 0)
            if ref:
                res[label]["reference_ms"] = round(ref["ms_per_step"], 4)
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--skip-train", action="store_true")
    default_ref = os.path.join(ROOT, "oracle", "_ref", "ref_harness")
    ap.add_argument("--reference", default=default_ref if os.path.exists(default_ref) else None, help="reference harness binary (oracle/_ref/ref_harness)")
    args = ap.parse_args()
    for B in (1 << 18, 1 << 21):
        inference_group("FullyFusedMLP", 64, 2, 32, (16, 128, 1024), B, args)
        inference_group("CutlassMLP", 256, 4, 64, (16, 512, 768), B, args)
    if not args.skip_train:
        train_group("FullyFusedMLP", 64, 2, 128, 1 << 18, args)
        train_group("CutlassMLP", 256, 4, 512, 1 << 18, args)


if __name__ == "__main__":
    main()
