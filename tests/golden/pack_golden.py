#!/usr/bin/env python3
"""Pack the raw dumps of oracle/ref_harness.cu (gpurun_out/golden/<case>/) into tests/golden/<case>.npz.

Usage: python tests/golden/pack_golden.py gpurun_out/golden tests/golden
The .npz files are the committed fixtures; they were produced by the unmodified reference (built from its sources by
oracle/Makefile) running on the GPU via tests/golden/make_golden.sh.
"""
import glob
import json
import os
import sys

import numpy as np

src, dst = sys.argv[1], sys.argv[2]
DT = {"f32": np.float32, "f16": np.uint16}
for case in sorted(glob.glob(os.path.join(src, "*", "meta.json"))):
    d = os.path.dirname(case)
    name = os.path.basename(d)
    arrays = {"meta": np.frombuffer(open(case, "rb").read(), dtype=np.uint8)}
    jit = name.endswith("_jit")
    for f in sorted(os.listdir(d)):
        stem, ext = os.path.splitext(f)
        if ext[1:] not in DT:
            continue
        if stem == "params_final" and ext == ".f32":
            continue  # the fp16 copy is what the reference serialises (trainer.h:447)
        if jit and stem in ("x", "y", "params_init", "encoded", "params_step1"):
            continue  # identical to the non-JIT case by construction
        arrays[f"{stem}_{ext[1:]}"] = np.fromfile(os.path.join(d, f), dtype=DT[ext[1:]])
    np.savez_compressed(os.path.join(dst, name + ".npz"), **arrays)
    print(name, {k: v.shape for k, v in arrays.items() if k != "meta"})
for p in sorted(glob.glob(os.path.join(src, "probe_*.json"))):
    open(os.path.join(dst, os.path.basename(p)), "w").write(open(p).read())
