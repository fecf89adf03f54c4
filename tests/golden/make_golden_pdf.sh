#!/bin/bash
# Regenerates tests/golden/pdf_<case>.npz: one step of the UNMODIFIED reference's Trainer::training_step with a data_pdf
# (oracle/_ref/ref_pdf_step, built by __graft_entry__.build() from tests/cpp/ref_pdf_step.cu and the reference library objects).
# Needs a GPU:
#   bash tests/golden/make_golden_pdf.sh <out dir>
#   python tests/golden/pack_golden.py <out dir> tests/golden
#   python tests/golden/add_exact_pdf_grads.py
set -e
OUT=${1:?usage: make_golden_pdf.sh <out dir>}
H=oracle/_ref/ref_pdf_step
C=tests/golden/configs/hash3d_small.json
mkdir -p "$OUT"
# <config> <loss> <n_neurons> <output activation> <batch> <seed> <out>: 64 neurons run on the fused kernel here, 128 on the general
# path; Variance divides by the prediction, so its cases keep the outputs positive
$H $C RelativeL2 64 None 512 21 "$OUT/pdf_relative_l2_w64"
$H $C Variance 64 Exponential 512 22 "$OUT/pdf_variance_w64"
$H $C RelativeL2 128 None 512 23 "$OUT/pdf_relative_l2_w128"
$H $C Variance 128 Exponential 512 24 "$OUT/pdf_variance_w128"
