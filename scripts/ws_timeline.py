"""Pipeline timeline of the warp-specialised fused kernel (profiling experiment; needs an ABLATION=1 build).

Runs a few headline-config steps with TCNNB_CLOCKS set, then reads the clock64 stamps the kernel left for its last launch:
per CTA, per role (0 = MLP group, 1/2 = memory sub-groups), per tile (first 16 of the CTA), 8 slots.
Prints the median duration of every phase over the steady-state tiles, in microseconds at the SM clock sampled by nvidia-smi.
"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tiny-cuda-nn_b200"))
out = os.path.join(os.environ.get("TCNNB_OUT_DIR", "/tmp"), "ws_clocks.bin")  # phase stamps the library writes (TCNNB_CLOCKS)
os.environ["TCNNB_CLOCKS"] = out
os.environ.setdefault("TCNNB_LIB", os.path.join(ROOT, "tiny-cuda-nn_b200", "ablation", "libtcnn_b200.so"))  # the ABLATION=1 build
import torch

import tcnn_b200

B = 1 << 18
cfg = json.load(open(os.path.join(ROOT, "tests", "golden", "configs", "headline.json")))
model = tcnn_b200.create_from_config(3, 3, cfg)
g = torch.Generator(device="cuda").manual_seed(1)
x, y = torch.rand(B, 3, device="cuda", generator=g), torch.rand(B, 3, device="cuda", generator=g)
for i in range(20):
    model.trainer.training_step(x, y)
torch.cuda.synchronize()
mhz = float(subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"], capture_output=True, text=True).stdout.split()[0])
model.close()

c = np.fromfile(out, dtype=np.int64).reshape(-1, 3, 16, 16).astype(np.float64)
# The buffer has room for 2 x #SMs CTAs (the removed two-CTAs-per-SM shape); the kernel runs #SMs of them. Round 1's version kept the
# all-zero slots, which poisoned every median (VERDICT r01 item 4): drop CTAs that left no stamp, and treat unset stamps as missing.
c = c[(c != 0).any(axis=(1, 2, 3))]
c[c == 0] = np.nan
n_ctas = int(c.shape[0])
us = 1.0 / mhz  # cycles -> microseconds
steady = slice(4, 12)


def med(a):
    a = np.asarray(a, np.float64)
    a = a[np.isfinite(a)]
    return float(np.median(a)) * us if a.size else float("nan")


mlp = c[:, 0]
res = {
    "sm_mhz": mhz,
    "n_ctas_with_stamps": n_ctas,
    "mlp": {
        "tile_period": med((mlp[:, 5:13, 0] - mlp[:, 4:12, 0]).ravel()),
        "wait_enc_full": med((mlp[:, steady, 1] - mlp[:, steady, 0]).ravel()),
        "forward": med((mlp[:, steady, 2] - mlp[:, steady, 1]).ravel()),
        "backward": med((mlp[:, steady, 3] - mlp[:, steady, 2]).ravel()),
        "wait_park_free": med((mlp[:, steady, 4] - mlp[:, steady, 3]).ravel()),
        "park": med((mlp[:, steady, 5] - mlp[:, steady, 4]).ravel()),
        # one forward stage (hidden layer 1) and the first backward stage, split up
        "fwd1_stage_sync": med((mlp[:, steady, 7] - mlp[:, steady, 6]).ravel()),
        "fwd1_mma": med((mlp[:, steady, 9] - mlp[:, steady, 7]).ravel()),  # issue + completion of the wgmma products
        "fwd1_epilogue": med((mlp[:, steady, 10] - mlp[:, steady, 9]).ravel()),
        "bwd1_stage_sync": med((mlp[:, steady, 12] - mlp[:, steady, 11]).ravel()),
        "bwd1_mma": med((mlp[:, steady, 14] - mlp[:, steady, 12]).ravel()),
        "bwd1_epilogue": med((mlp[:, steady, 15] - mlp[:, steady, 14]).ravel()),
    },
}
for g_ in (0, 1):
    m = c[:, 1 + g_]
    ks = [k for k in range(4, 12) if k % 2 == g_]
    res[f"mem{g_}"] = {
        "wait_enc_free": med((m[:, ks, 1] - m[:, ks, 0]).ravel()),
        "gather": med((m[:, ks, 2] - m[:, ks, 1]).ravel()),
        "wait_park_full": med((m[:, ks, 3] - m[:, ks, 2]).ravel()),
        "scatter": med((m[:, ks, 4] - m[:, ks, 3]).ravel()),
        "loop_period": med((m[:, [k + 2 for k in ks], 0] - m[:, ks, 0]).ravel()),
    }
print(json.dumps({"ws_timeline_us": res}))
# one CTA's raw timeline (relative to its first stamp), for eyeballing
cta = c[7]
t0 = np.nanmin(cta)
for role in range(3):
    for k in range(4, 10):
        if np.isfinite(cta[role, k, 0]):
            print(role, k, [round((v - t0) * us, 2) if np.isfinite(v) else None for v in cta[role, k, :16]])
