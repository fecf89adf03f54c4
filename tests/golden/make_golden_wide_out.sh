#!/bin/bash
# Regenerates tests/golden/wide_*.npz -- networks whose padded output is wider than their hidden layers -- from the UNMODIFIED
# reference (oracle/_ref/ref_harness, built by oracle/Makefile). Needs a GPU; run from the repository root:
#   bash tests/golden/make_golden_wide_out.sh [raw dump dir]
# The raw dumps go to a temporary directory unless one is given; only the arrays the tests read are packed into tests/golden/.
set -e
RAW=${1:-$(mktemp -d)}
H=oracle/_ref/ref_harness
C=tests/golden/configs
mkdir -p "$RAW"
# trainer: <config> <n_in> <n_out> <batch> <n_steps> <outdir> <jit>
$H dump $C/wide_hash3d_w64.json 3 128 512 10 "$RAW/wide_hash3d_w64" 0
# network on its own: <otype> <width> <hidden> <n_in> <n_out> <batch> <outdir> <jit> <activation> <output_activation>
$H mlpdump FullyFusedMLP 64 2 32 128 1024 "$RAW/wide_net_w64_h2_relu" 0 ReLU None
$H mlpdump FullyFusedMLP 64 2 32 128 1024 "$RAW/wide_net_w64_h2_sigmoid" 0 ReLU Sigmoid
$H mlpdump FullyFusedMLP 16 2 16 48 1024 "$RAW/wide_net_w16_h2_relu" 0 ReLU None
# 256 neurons: a smaller batch keeps the fixtures small (the parameters alone are 0.5 / 0.7 MB)
$H mlpdump CutlassMLP 256 4 64 512 256 "$RAW/wide_net_w256_h4_relu" 0 ReLU None
$H mlpdump CutlassMLP 256 3 64 384 256 "$RAW/wide_net_w256_h3_sine" 0 Sine None
# not read by tests/test_oracle_wide_out.py / test_gpu_wide_output.py: keep the fixtures small
for d in "$RAW"/wide_hash*; do
	rm -f "$d"/params_step1.f32 "$d"/params_final.f16 "$d"/params_final.f32 "$d"/inference_final.f32 "$d"/loss_values.f32
done
python tests/golden/pack_golden.py "$RAW" tests/golden
