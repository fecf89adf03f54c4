"""bench_mlp.py -- the reference's benchmarks/mlp/bench_mlp_ours.cu on this library: stand-alone FullyFusedMLP inference throughput
(fp16 in / fp16 out, in = out = width), BASELINE.json configs[4] sweep: width x hidden x batch. One JSON line per point; with
--reference the same points on the unmodified reference (oracle/_ref/ref_harness mlpbench: fully_fused_jit, fully_fused, cutlass).

    python scripts/bench_mlp.py [--widths 16,32,64,128] [--hidden 2,4,8] [--batches 16384,...] [--iters N] [--reference]

Roofline per point (SURVEY.md section 8d): FLOPs/sample = 2 (in*w + (h-1) w^2 + w*out); bytes/sample = 2 (in + out). The line carries
the achieved TFLOP/s against the measured bf16 tensor peak and the achieved GB/s against the measured HBM copy peak, whichever
binds (ridge = 295 FLOP/B from the H100 SXM data sheet: 989 TFLOP/s fp16 over 3.35 TB/s).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tiny-cuda-nn_b200"))


def peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        d = json.load(open(path))
        return float(d["hbm_gbs"]), float(d["bf16_tflops"]), "measured"
    return 3350.0, 989.0, "datasheet"  # H100 SXM: HBM3 GB/s, dense fp16 TFLOP/s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--widths", default="16,32,64,128")
    ap.add_argument("--hidden", default="2,4,8")
    ap.add_argument("--batches", default="16384,262144,4194304")
    ap.add_argument("--iters", type=int, default=0)
    ap.add_argument("--reference", action="store_true")
    args = ap.parse_args()
    import torch

    import tcnn_b200

    hbm, tensor, kind = peaks()
    harness = os.path.join(ROOT, "oracle", "_ref", "ref_harness")
    for width in [int(v) for v in args.widths.split(",")]:
        for hidden in [int(v) for v in args.hidden.split(",")]:
            net = tcnn_b200.Network(width, width, {"otype": "FullyFusedMLP", "n_neurons": width, "n_hidden_layers": hidden, "activation": "ReLU", "output_activation": "None"})
            p16 = net.initial_params(1337).to(torch.float16).contiguous()
            for B in [int(v) for v in args.batches.split(",")]:
                x = torch.rand(B, width, device="cuda").to(torch.float16).contiguous()
                iters = args.iters or max(20, min(2000, (1 << 27) // B))
                for _ in range(max(3, iters // 10)):
                    net.inference_mixed_precision(x, p16)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(iters):
                    net.inference_mixed_precision(x, p16)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / iters
                flops = 2.0 * (width * width * (hidden + 1)) * B
                byts = 2.0 * (width + width) * B
                line = {"impl": "tcnn_b200", "mode": "mlp_inference", "width": width, "n_hidden_layers": hidden, "batch": B, "iters": iters, "ms_per_batch": ms,
                        "samples_per_s": B / (ms * 1e-3), "tflops": flops / (ms * 1e-3) / 1e12, "gbs": byts / (ms * 1e-3) / 1e9,
                        "tensor_frac": flops / (ms * 1e-3) / 1e12 / tensor, "hbm_frac": byts / (ms * 1e-3) / 1e9 / hbm, "peaks": kind}
                if args.reference and os.path.exists(harness):
                    ref = {}
                    for name, otype, jit in (("fully_fused_jit", "FullyFusedMLP", 1), ("fully_fused", "FullyFusedMLP", 0), ("cutlass", "CutlassMLP", 0)):
                        cmd = [harness, "mlpbench", otype, str(width), str(hidden), str(width), str(width), str(B), str(iters), str(max(3, iters // 10)), str(jit)]
                        try:
                            out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
                            js = [l for l in out.stdout.splitlines() if l.startswith("{")]
                            ref[name] = json.loads(js[-1])["samples_per_s"] if js else {"error": (out.stderr or out.stdout)[-200:]}
                        except Exception as e:  # noqa: BLE001
                            ref[name] = {"error": repr(e)}
                    line["reference_samples_per_s"] = ref
                    best = max([v for v in ref.values() if isinstance(v, float)], default=None)
                    line["vs_best_reference_mode"] = line["samples_per_s"] / best if best else None
                print(json.dumps(line), flush=True)
                del x


if __name__ == "__main__":
    main()
