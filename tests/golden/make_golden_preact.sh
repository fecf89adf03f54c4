#!/bin/bash
# Regenerates tests/golden/preact_*.npz -- CutlassMLP with the Sine / SiLU hidden activations, whose backward pass needs the stored
# pre-activations -- from the UNMODIFIED reference (oracle/_ref/ref_harness, built by oracle/Makefile). Needs a GPU; run from the
# repository root:
#   bash tests/golden/make_golden_preact.sh [raw dump dir]
# The raw dumps go to a temporary directory unless one is given; only the arrays the tests read are packed into tests/golden/.
set -e
RAW=${1:-$(mktemp -d)}
H=oracle/_ref/ref_harness
C=tests/golden/configs
mkdir -p "$RAW"
# trainer: <config> <n_in> <n_out> <batch> <n_steps> <outdir> <jit>
$H dump $C/preact_hash2d_sine.json 2 3 512 10 "$RAW/preact_hash2d_sine" 0
$H dump $C/preact_hash3d_silu.json 3 3 512 10 "$RAW/preact_hash3d_silu" 0
# network on its own: <otype> <width> <hidden> <n_in> <n_out> <batch> <outdir> <jit> <activation> <output_activation>
$H mlpdump CutlassMLP 64 2 32 16 2048 "$RAW/preact_net_sine_w64_h2" 0 Sine None
$H mlpdump CutlassMLP 128 4 64 32 2048 "$RAW/preact_net_silu_w128_h4" 0 SiLU None
# not read by tests/test_oracle_preact.py / test_gpu_preact.py: keep the fixtures small
for d in "$RAW"/preact_hash*; do
	rm -f "$d"/params_step1.f32 "$d"/params_final.f16 "$d"/params_final.f32 "$d"/inference_final.f32 "$d"/loss_values.f32
done
python tests/golden/pack_golden.py "$RAW" tests/golden
