#!/bin/bash
# Regenerates tests/golden/split_<case>.npz: Trainer::forward then Trainer::backward of the UNMODIFIED reference
# (oracle/_ref/ref_trainer_split, built by __graft_entry__.build() from tests/cpp/ref_trainer_split.cu and the reference library objects).
# Needs a GPU:
#   bash tests/golden/make_golden_split.sh <out dir>
#   python tests/golden/pack_golden.py <out dir> tests/golden
set -e
OUT=${1:?usage: make_golden_split.sh <out dir>}
H=oracle/_ref/ref_trainer_split
C=tests/golden/configs/hash3d_small.json
mkdir -p "$OUT"
# <config> <loss> <n_neurons> <output activation> <batch> <seed> <with pdf> <out>: 64 neurons run on the fused kernel here, 128 on
# the general path
$H $C RelativeL2 64 None 512 31 1 "$OUT/split_relative_l2_pdf_w64"
$H $C L2 128 None 512 32 0 "$OUT/split_l2_w128"
