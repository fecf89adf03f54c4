#!/bin/bash
# Regenerates tests/golden/bwdbwd_<case>.npz: the UNMODIFIED reference's Module::backward_backward_input of a grid encoding
# (oracle/_ref/ref_bwd_bwd, built by __graft_entry__.build() from tests/cpp/ref_bwd_bwd.cu and the reference library objects).
# Needs a GPU:
#   bash tests/golden/make_golden_bwd_bwd.sh <out dir>
#   python tests/golden/pack_golden.py <out dir> tests/golden
set -e
OUT=${1:?usage: make_golden_bwd_bwd.sh <out dir>}
H=oracle/_ref/ref_bwd_bwd
C=tests/golden/configs
mkdir -p "$OUT"
# <config> <n_input_dims> <batch> <seed> <out>
$H $C/bwdbwd_hash3d_f2.json 3 1024 7 "$OUT/bwdbwd_hash3d_f2"
$H $C/bwdbwd_hash3d_f1_smooth.json 3 1024 8 "$OUT/bwdbwd_hash3d_f1_smooth"
$H $C/bwdbwd_dense2d_f4.json 2 1024 9 "$OUT/bwdbwd_dense2d_f4"
$H $C/bwdbwd_hash4d_f8_smooth.json 4 1024 10 "$OUT/bwdbwd_hash4d_f8_smooth"
