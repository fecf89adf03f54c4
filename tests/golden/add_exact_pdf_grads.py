#!/usr/bin/env python3
"""Adds `grads_exact_f32` to tests/golden/pdf_*.npz: the CPU oracle's exact (double-accumulated) step-0 parameter gradients, from the
reference's parameters and batch, with the data_pdf loss gradient of losses/*.h (fp16, x loss scale) as dL/d(output).

Why: the reference sums weight gradients in fp16 (CUTLASS split-K) and table gradients with fp16 atomics; with pdf-weighted
losses its own result lies 1.2e-2 .. 4e-2 (RAE) from the exact sums at B = 512, so the fixed bars between two fp16 implementations do
not apply. The GPU test then states: this library is no further from the exact sums than the reference is.

Usage (CPU only): python tests/golden/add_exact_pdf_grads.py
"""
import glob
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import oracle_binding as ob  # noqa: E402

for path in sorted(glob.glob(os.path.join(HERE, "pdf_*.npz"))):
    z = dict(np.load(path))
    meta = json.loads(bytes(z["meta"]).decode())
    B, n_in, n_out, cfg = meta["batch"], meta["n_input_dims"], meta["n_output_dims"], meta["config"]
    orc = ob.OracleModel(n_in, n_out, cfg)
    orc.params_fp16[:] = z["params_f16"]
    x = z["x_f32"].reshape(B, n_in).copy()
    y = z["y_f32"].reshape(B, n_out).astype(np.float64)
    pdf = z["pdf_f32"].reshape(B, n_out).astype(np.float64)
    enc = orc.encode(x)
    hidden, out = orc.mlp_forward(enc)
    pred = ob.half_bits_to_float(out)[:, :n_out].astype(np.float64)
    n_total = B * n_out
    if cfg["loss"]["otype"] == "RelativeL2":
        grad = 2 * (pred - y) / (pred * pred + 0.01) / pdf
    else:
        assert cfg["loss"]["otype"] == "Variance"
        grad = -(y * y / pdf / n_total) / (pred * pred) * n_total
    dy = np.zeros((B, out.shape[1]), np.float16)
    dy[:, :n_out] = (128.0 * grad / n_total).astype(np.float16)
    dW, d_enc = orc.mlp_backward(enc, hidden, dy.view(np.uint16))
    z["grads_exact_f32"] = np.concatenate([dW, orc.grid_backward(x, d_enc)]).astype(np.float32)
    np.savez_compressed(path, **z)
    print(os.path.basename(path), z["grads_exact_f32"].shape)
