"""Pins the CPU oracle (oracle/oracle_cpu.cpp, tests/preact_oracle.py) against the unmodified reference at networks whose padded output
is wider than their hidden layers (tests/golden/wide_*.npz, tests/golden/make_golden_wide_out.sh): initial parameters bit for bit
(W_out [padded_out][n_neurons] drawn last from the same pcg32 stream), the network on its own in the oracle's fp16-per-k16 mode
(the reference's FullyFusedMLP rounding) within the reference's bar, and a HashGrid + FullyFusedMLP 64 x 2 trainer with 128 outputs.
CPU only."""
import ctypes
import json
import os

import numpy as np
import pytest

import oracle_binding as ob
import preact_oracle as po
from golden_util import GOLDEN, rae

NET_CASES = ["wide_net_w64_h2_relu", "wide_net_w64_h2_sigmoid", "wide_net_w16_h2_relu", "wide_net_w256_h4_relu", "wide_net_w256_h3_sine"]
TRAINER_CASE, TRAINER_SHAPE = "wide_hash3d_w64", (3, 128, 512)


def load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    d = {k: z[k] for k in z.files if k != "meta"}
    d["meta"] = json.loads(bytes(z["meta"]).decode())
    return d


def trainer_rng(seed=1337):
    """The Trainer's pcg32 (trainer.h:51-87) as the C oracle seeds it, continued in Python."""
    c = ob.Pcg32()
    ob.load().orc_trainer_rng(ctypes.c_uint32(seed), ctypes.byref(c))
    rng = po.Pcg32(0)
    rng.state, rng.inc = c.state, c.inc
    return rng


@pytest.mark.parametrize("name", NET_CASES)
def test_network_fixture_is_wide(name):
    m = load(name)["meta"]
    assert m["padded_output_width"] > m["width"]


@pytest.mark.parametrize("name", NET_CASES)
def test_network_initial_parameters_bit_exact(name):
    g = load(name)
    m = g["meta"]
    in_w = (m["n_in"] + 15) // 16 * 16
    p = po.init_params(m["width"], in_w, m["n_hidden_layers"], m["padded_output_width"], m["activation"], trainer_rng())
    assert p.size == m["n_params"]
    assert np.array_equal(p.astype(np.float16).view(np.uint16), g["params_f16"])


@pytest.mark.parametrize("name", NET_CASES)
def test_network_forward_within_reference_bar(name):
    """The reference's weights and inputs through the oracle -> its outputs (tests/test_common.h:177: RAE < 1e-2 @ p99). ReLU networks
    through orc_mlp_forward in fp16-per-k16 mode, Sine through tests/preact_oracle.py."""
    g = load(name)
    m = g["meta"]
    B, out_pad = m["batch"], m["padded_output_width"]
    x16 = g["x_f16"].reshape(B, m["n_in"])
    ref = g["output_f16"].view(np.float16).reshape(B, out_pad).astype(np.float32)
    if m["activation"] == po.SINE:
        _, _, out = po.forward(m["activation"], g["params_f16"].view(np.float16), x16.view(np.float16), m["width"], m["n_hidden_layers"], out_pad)
        out = out.astype(np.float32)
    else:
        lib = ob.load()
        mlp = ob.Mlp(m["n_in"], m["width"], m["n_hidden_layers"], out_pad, 0, ob.ACT[m["activation"].lower()], ob.ACT[m["output_activation"].lower()], 0)
        assert lib.orc_mlp_setup(ctypes.byref(mlp)) == 0 and mlp.n_params == m["n_params"]
        hid = np.zeros((m["n_hidden_layers"], B, m["width"]), np.uint16)
        o16 = np.zeros((B, out_pad), np.uint16)
        lib.orc_mlp_forward(ctypes.byref(mlp), B, ob.ACCUM_FP16_K16, ob._p(g["params_f16"]), ob._p(np.ascontiguousarray(x16.T)), ob._p(hid), ob._p(o16))
        out = ob.half_bits_to_float(o16)
    assert rae(out, ref, 99.0) < 1e-2, rae(out, ref, 99.0)


def test_trainer_fixture_against_oracle():
    """HashGrid + FullyFusedMLP 64 x 2 -> 128: initial parameters bit for bit, step-0 loss and grid gradients within the reference's
    bars, and the ten-step trajectory within 3 %.

    The network's weight gradients are not held to the reference's: it computes them with split-K GEMMs that accumulate in fp16, and
    at 128 outputs and a fresh grid they are ~3e-6 (about 50 fp16 quanta after the loss scale), so that its sums lie 14 % (W_0), 10 %
    (W_1) and 5.5 % (W_out) RAE @ p99.9 from the exact sums in either accumulation mode of the oracle. tests/test_gpu_wide_output.py
    holds the device to the exact fp32 sums instead. The grid gradients, sums of the fp16 dL/d(encoding), agree to 0.25 %."""
    n_in, n_out, B = TRAINER_SHAPE
    g = load(TRAINER_CASE)
    cfg = json.load(open(os.path.join(GOLDEN, "configs", TRAINER_CASE + ".json")))
    orc = ob.OracleModel(n_in, n_out, cfg, accum_mode=ob.ACCUM_FP16_K16)
    assert orc.n_params == g["meta"]["n_params"]
    assert np.array_equal(orc.params_fp32.view(np.uint32), g["params_init_f32"].view(np.uint32))
    x, y = g["x_f32"].reshape(B, n_in), g["y_f32"].reshape(B, n_out)
    losses = [orc.training_step(x, y, run_optimizer=False)]
    gref = ob.half_bits_to_float(g["grads_step0_f16"])
    got = ob.half_bits_to_float(orc.grads_fp16)
    assert abs(losses[0] - g["meta"]["losses"][0]) <= 1e-3 * abs(g["meta"]["losses"][0])
    assert rae(got[orc.n_mlp :], gref[orc.n_mlp :], 99.9) < 1.2e-2
    for _ in range(g["meta"]["n_steps"]):
        losses.append(orc.training_step(x, y))
    for mine, theirs in zip(losses, g["meta"]["losses"]):  # the step-0 loss, then the loss of each of the ten steps
        assert abs(mine - theirs) <= 3e-2 * abs(theirs), (losses, g["meta"]["losses"])
