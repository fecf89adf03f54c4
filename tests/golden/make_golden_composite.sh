#!/bin/bash
# Regenerates tests/golden/composite_{sum_hash3d,product_planes,product_pad,empty}.npz and nrc_top.npz -- Composite encodings with the
# Sum / Product reductions, dims_to_encode_begin, Empty, and the NRC shorthand -- from the UNMODIFIED reference
# (oracle/_ref/ref_harness, built by oracle/Makefile). Needs a GPU; run from the repository root:
#   bash tests/golden/make_golden_composite.sh [raw dump dir]
# The raw dumps go to a temporary directory unless one is given; only the arrays the tests read are packed into tests/golden/.
set -e
RAW=${1:-$(mktemp -d)}
H=oracle/_ref/ref_harness
C=tests/golden/configs
mkdir -p "$RAW"
# trainer: <config> <n_in> <n_out> <batch> <n_steps> <outdir> <jit>
$H dump $C/composite_sum_hash3d.json 3 3 512 10 "$RAW/composite_sum_hash3d" 0
$H dump $C/composite_product_planes.json 4 3 512 10 "$RAW/composite_product_planes" 0
$H dump $C/composite_product_pad.json 4 3 512 10 "$RAW/composite_product_pad" 0
$H dump $C/composite_empty.json 6 3 512 10 "$RAW/composite_empty" 0
$H dump $C/nrc_top.json 9 3 512 10 "$RAW/nrc_top" 0
# not read by tests/test_gpu_composite_reductions.py / tests/test_composite_oracle.py: keep the fixtures small
for d in "$RAW"/composite_* "$RAW"/nrc_top; do
	rm -f "$d"/params_step1.f32 "$d"/params_final.f16 "$d"/params_final.f32 "$d"/inference_final.f32 "$d"/loss_values.f32
done
python tests/golden/pack_golden.py "$RAW" tests/golden
# the grid cases' initial parameters (incompressible noise) are kept as a SHA-256 digest of their fp32 bytes
python tests/golden/digest_params.py tests/golden/composite_sum_hash3d.npz tests/golden/composite_product_planes.npz tests/golden/composite_product_pad.npz \
	tests/golden/composite_empty.npz
