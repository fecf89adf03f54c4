#!/bin/bash
# Regenerates tests/golden/net_trainer_<case>.npz: the UNMODIFIED reference's Trainer over create_network<__half>
# (oracle/_ref/ref_network_trainer, built by __graft_entry__.build() from tests/cpp/ref_network_trainer.cu and the reference library
# objects). Needs a GPU:
#   bash tests/golden/make_golden_net_trainer.sh <out dir>
#   python tests/golden/pack_golden.py <out dir> tests/golden
set -e
OUT=${1:?usage: make_golden_net_trainer.sh <out dir>}
H=oracle/_ref/ref_network_trainer
mkdir -p "$OUT"
# <otype> <n_neurons> <n_hidden_layers> <batch> <seed> <out>
$H FullyFusedMLP 64 2 2048 41 "$OUT/net_trainer_ffmlp_w64_h2"
$H CutlassMLP 128 3 2048 42 "$OUT/net_trainer_cutlass_w128_h3"
