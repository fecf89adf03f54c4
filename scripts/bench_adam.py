"""bench_adam.py -- device time of the Adam kernel at the headline configuration (13 034 160 parameters), next to a plain
device-to-device copy that moves the same number of bytes in the same process.

    python scripts/bench_adam.py [--iters N] [--steps32] [--peaks-out PATH]

The model takes one training step (so that the gradients have the benchmark's sparsity: untouched table entries are skipped),
then trainer.optimizer_step() is timed with CUDA events around each of --iters calls. Achieved GB/s use the algorithmic bytes per
parameter: fp16 gradient read (2), fp32 master weight, first and second moment read + write (24), step counter read + write
(2 x counter width) and fp16 weight write (2) -- 32 B with 16-bit counters, 36 B with 32-bit ones. The copy's rate (read + write
bytes over time) is the achievable HBM rate of this card; it is written to --peaks-out (default MEASURED_PEAKS.json at the
repository root, which bench.py reads) together with the GPU name and power limit. --steps32 forces 32-bit step counters.
"""
import argparse
import json
import os
import struct
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tiny-cuda-nn_b200"))


def counter_bytes(model):
    """Width of the step counters in use: a count above 65535 restored from a snapshot survives only in 32-bit counters."""
    import numpy as np

    blob = bytearray(model.trainer.serialize(with_optimizer=True))
    n = struct.unpack_from("<Q", blob)[0]
    off = 16 + 2 * n + 8 * n
    steps = np.frombuffer(blob, dtype=np.uint32, count=n, offset=off)
    saved = steps.copy()
    steps[:] = 70000
    model.trainer.deserialize(bytes(blob))
    width = 4 if int(np.frombuffer(model.trainer.serialize(with_optimizer=True), dtype=np.uint32, count=1, offset=off)[0]) == 70000 else 2
    steps[:] = saved
    model.trainer.deserialize(bytes(blob))
    return width


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [s.strip() for s in out.stdout.splitlines()[0].split(",")] if out.returncode == 0 and out.stdout.strip() else ("unknown",) * 3
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def time_calls(torch, fn, iters, warmup=20):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for e0, e1 in ev:
        e0.record()
        fn()
        e1.record()
    torch.cuda.synchronize()
    ms = sorted(e0.elapsed_time(e1) for e0, e1 in ev)
    return ms[len(ms) // 2], ms[0], ms[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=500)
    ap.add_argument("--steps32", action="store_true", help="force 32-bit step counters (tcnnb_debug_set adam_steps32)")
    ap.add_argument("--peaks-out", default=os.path.join(ROOT, "MEASURED_PEAKS.json"))
    args = ap.parse_args()

    import torch

    import tcnn_b200

    assert torch.cuda.is_available(), "bench_adam.py needs a GPU"
    torch.cuda.set_device(0)
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", "configs", "headline.json")))
    model = tcnn_b200.create_from_config(3, 3, cfg)
    if args.steps32:
        model.debug_set("adam_steps32", 1)
    g = torch.Generator(device="cuda").manual_seed(1337)
    x = torch.rand(1 << 18, 3, device="cuda", generator=g)
    y = torch.rand(1 << 18, 3, device="cuda", generator=g)
    model.trainer.training_step(x, y)
    torch.cuda.synchronize()
    n = model.trainer.n_params()
    width = counter_bytes(model)
    bytes_per_param = 2 + 24 + 2 * width + 2

    adam_ms, adam_min, adam_max = time_calls(torch, model.trainer.optimizer_step, args.iters)
    half = n * bytes_per_param // 2
    src = torch.empty(half, dtype=torch.uint8, device="cuda")
    dst = torch.empty_like(src)
    copy_ms, copy_min, copy_max = time_calls(torch, lambda: dst.copy_(src), args.iters)
    copy_gbs = 2 * half / (copy_ms * 1e-3) / 1e9
    info = gpu_info()
    line = {"n_params": n, "counter_bytes": width, "bytes_per_param": bytes_per_param, "iters": args.iters,
            "adam_ms": adam_ms, "adam_ms_range": [adam_min, adam_max], "adam_gbs": n * bytes_per_param / (adam_ms * 1e-3) / 1e9,
            "copy_ms": copy_ms, "copy_ms_range": [copy_min, copy_max], "copy_gbs": copy_gbs, **info,
            "library": os.environ.get("TCNNB_LIB", "in-tree")}
    line["adam_share_of_copy_rate"] = line["adam_gbs"] / copy_gbs
    print(json.dumps(line))
    if args.peaks_out:
        peaks = json.load(open(args.peaks_out)) if os.path.exists(args.peaks_out) else {}
        peaks.update({"hbm_gbs": copy_gbs, "hbm_source": "bench_adam.py device-to-device copy", **info})
        with open(args.peaks_out, "w") as f:
            json.dump(peaks, f, indent=1)


if __name__ == "__main__":
    main()
