#!/bin/bash
# Regenerates tests/golden/w256_*.npz -- 256-neuron CutlassMLP networks -- from the UNMODIFIED reference (oracle/_ref/ref_harness,
# built by oracle/Makefile). Needs a GPU; run from the repository root:
#   bash tests/golden/make_golden_w256.sh [raw dump dir]
# The raw dumps go to a temporary directory unless one is given; only the arrays the tests read are packed into tests/golden/.
set -e
RAW=${1:-$(mktemp -d)}
H=oracle/_ref/ref_harness
C=tests/golden/configs
mkdir -p "$RAW"
# trainer: <config> <n_in> <n_out> <batch> <n_steps> <outdir> <jit>
$H dump $C/w256_hash3d_relu.json 3 3 512 10 "$RAW/w256_hash3d_relu" 0
# network on its own: <otype> <width> <hidden> <n_in> <n_out> <batch> <outdir> <jit> <activation> <output_activation>
$H mlpdump CutlassMLP 256 3 64 16 2048 "$RAW/w256_net_relu_h3" 0 ReLU None
$H mlpdump CutlassMLP 256 3 64 16 2048 "$RAW/w256_net_sine_h3" 0 Sine None
# not read by tests/test_gpu_cutlass256.py: keep the fixtures small
for d in "$RAW"/w256_hash*; do
	rm -f "$d"/params_step1.f32 "$d"/params_final.f16 "$d"/params_final.f32 "$d"/inference_final.f32 "$d"/loss_values.f32
done
python tests/golden/pack_golden.py "$RAW" tests/golden
