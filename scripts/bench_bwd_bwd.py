#!/usr/bin/env python3
"""Times the grid encoding's second-order derivatives (tcnnb_encoding_backward_backward_input, csrc/grid_bwd_bwd.cu) with CUDA
events, next to the first-order backward (tcnnb_encoding_backward) on the same inputs. HashGrid L=16 F=2 T=2^19, 3-D, B=2^18 by default.

    python scripts/bench_bwd_bwd.py [--batch 262144] [--iters 50] [--warmup 10] [--out results.json]

Prints one JSON object: the GPU's name and power limit, and the mean milliseconds per call of
  bwd_bwd_params_doutput   dL_dparams + dL_ddLdoutput (the eikonal case)
  bwd_bwd_all              dL_dparams + dL_ddLdoutput + dL_dinput
  bwd_params               first-order dL_dparams
  bwd_params_input         first-order dL_dparams + dL_dinput
Calls of one kind run back to back; the kinds alternate over --rounds rounds and the per-round means are reported with their spread."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tiny-cuda-nn_b200"))

CONFIG = {"otype": "HashGrid", "n_levels": 16, "n_features_per_level": 2, "log2_hashmap_size": 19, "base_resolution": 16, "per_level_scale": 2.0}


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1 << 18)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    import tcnn_b200

    assert torch.cuda.is_available(), "bench_bwd_bwd needs a GPU"
    lib = tcnn_b200.load()
    enc = tcnn_b200.Encoding(3, CONFIG)
    B, W = args.batch, enc.n_output_dims
    g = torch.Generator(device="cuda").manual_seed(0)
    p16 = enc.initial_params(seed=1, scale=50.0).to(torch.float16)
    x = torch.rand(B, 3, device="cuda", generator=g)
    u = (torch.randn(B, W, device="cuda", generator=g) * 0.5).to(torch.float16)
    v = torch.randn(B, 3, device="cuda", generator=g)
    gp = torch.empty(enc.n_params, dtype=torch.float16, device="cuda")
    gd = torch.empty(B, W, dtype=torch.float16, device="cuda")
    gx = torch.empty(B, 3, dtype=torch.float32, device="cuda")
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def bwd_bwd(with_input):
        return lambda: lib.tcnnb_encoding_backward_backward_input(enc._h, s, B, v.data_ptr(), x.data_ptr(), u.data_ptr(), gp.data_ptr(), gd.data_ptr(),
                                                                  gx.data_ptr() if with_input else None, p16.data_ptr())

    def bwd(with_input):
        return lambda: lib.tcnnb_encoding_backward(enc._h, s, B, gx.data_ptr() if with_input else None, u.data_ptr(), gp.data_ptr(), x.data_ptr(), p16.data_ptr())

    kinds = {"bwd_bwd_params_doutput": bwd_bwd(False), "bwd_bwd_all": bwd_bwd(True), "bwd_params": bwd(False), "bwd_params_input": bwd(True)}
    for fn in kinds.values():
        for _ in range(args.warmup):
            assert fn() == 0, lib.tcnnb_last_error().decode()
    torch.cuda.synchronize()
    per_round = {k: [] for k in kinds}
    for _ in range(args.rounds):
        for k, fn in kinds.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.iters):
                fn()
            t1.record()
            t1.synchronize()
            per_round[k].append(t0.elapsed_time(t1) / args.iters)
    result = {"gpu": gpu_info(), "config": CONFIG, "batch": B, "iters": args.iters, "rounds": args.rounds,
              "ms": {k: {"mean": sum(r) / len(r), "min": min(r), "max": max(r)} for k, r in per_round.items()}}
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
