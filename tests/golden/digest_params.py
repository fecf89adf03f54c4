#!/usr/bin/env python3
"""Replace the initial parameters of packed fixtures (tests/golden/<case>.npz, `params_init_f32`) by their SHA-256 digest and count.

Usage: python tests/golden/digest_params.py tests/golden/<case>.npz ...
A freshly initialised grid table is uniform noise that does not compress: for the larger composite fixtures it is most of the file.
The tests compare initial parameters bit for bit, so the digest of the reference's fp32 bytes (`params_init_sha256`, uint8[32]) and
their number (`params_init_count`) pin them as exactly as the array did; the model's own parameters stand in for the array wherever a
test needs the values, once their digest matched.
"""
import hashlib
import sys

import numpy as np

for path in sys.argv[1:]:
    z = np.load(path)
    arrays = {k: z[k] for k in z.files}
    if "params_init_f32" not in arrays:
        continue  # already digested
    p = np.ascontiguousarray(arrays.pop("params_init_f32"), np.float32)
    arrays["params_init_sha256"] = np.frombuffer(hashlib.sha256(p.tobytes()).digest(), np.uint8)
    arrays["params_init_count"] = np.array([p.size], np.int64)
    np.savez_compressed(path, **arrays)
    print(path, "params_init_f32", p.size, "->", arrays["params_init_sha256"].tobytes().hex())
