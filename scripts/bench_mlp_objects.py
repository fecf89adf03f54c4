"""The reference's MLP benchmark (benchmarks/mlp/bench_mlp_ours.cu, unmodified) built twice by build(): against include/tiny-cuda-nn/ +
libtcnn_b200 (oracle/_ref/ref_bench_mlp_ours) and against the reference library (oracle/_ref/ref_bench_mlp_ours_tcnn). Runs each once on
one GPU and prints one JSON line with the card's name and power limit beside both results (inference throughput in samples / s, batch
2^20, 32 -> 32x3 -> 32; its three methods "fully_fused_jit", "fully_fused" and "cutlass" -- the JIT method runs without a JIT here).

    python scripts/bench_mlp_objects.py [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILDS = {"tcnn_b200": "ref_bench_mlp_ours", "reference": "ref_bench_mlp_ours_tcnn"}


def gpu_context():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    result = gpu_context()
    for label, name in BUILDS.items():
        exe = os.path.join(ROOT, "oracle", "_ref", name)
        if not os.path.exists(exe):
            sys.exit(f"{exe} is missing: python __graft_entry__.py build (needs the reference's source tree)")
        with tempfile.TemporaryDirectory() as tmp:  # the benchmark writes bench_result_ours.json into its working directory
            r = subprocess.run([exe], cwd=tmp, capture_output=True, text=True, timeout=1800)
            path = os.path.join(tmp, "bench_result_ours.json")
            # the program reports an exception on stdout and exits 0 without writing its result
            if r.returncode != 0 or not os.path.exists(path):
                result[label] = {"error": (r.stdout[-1000:] + r.stderr[-1000:]).strip()}
                continue
            with open(path) as f:
                result[label] = json.load(f)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
