"""Pins tests/preact_oracle.py -- the numpy restatement of CutlassMLP with a Sine / SiLU hidden activation -- against the unmodified
reference (tests/golden/preact_*.npz, tests/golden/make_golden_preact.sh) and against float64 finite differences. CPU only."""
import copy
import ctypes
import json
import os

import numpy as np
import pytest

import oracle_binding as ob
import preact_oracle as po
from golden_util import GOLDEN, rae

TRAINER_CASES = {
    # case -> (n_in, n_out, batch)
    "preact_hash2d_sine": (2, 3, 512),
    "preact_hash3d_silu": (3, 3, 512),
}
NET_CASES = ["preact_net_sine_w64_h2", "preact_net_silu_w128_h4"]


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


@pytest.mark.parametrize("name", list(TRAINER_CASES))
def test_initial_parameters_bit_exact(name):
    """SIREN (Sine) / xavier (SiLU) network initialisation, then the grid table from the same pcg32 stream: equal to the reference's
    params_init bit for bit."""
    n_in, n_out, _ = TRAINER_CASES[name]
    g = load(name)
    net = g["meta"]["config"]["network"]
    width, nh, in_w = net["n_neurons"], net["n_hidden_layers"], g["meta"]["encoded_width"]
    p_net = po.init_params(width, in_w, nh, 16, net["activation"], trainer_rng())
    n_mlp = p_net.size
    assert n_mlp == g["meta"]["n_params"] - g["meta"]["n_encoding_params"]
    assert np.array_equal(p_net.view(np.uint32), g["params_init_f32"][:n_mlp].view(np.uint32))
    # the grid's draws continue the stream: the C oracle draws the same number for any activation
    twin = copy.deepcopy(g["meta"]["config"])
    twin["network"]["activation"] = "ReLU"
    orc = ob.OracleModel(n_in, n_out, twin)
    assert orc.n_mlp == n_mlp
    assert np.array_equal(orc.params_fp32[n_mlp:].view(np.uint32), g["params_init_f32"][n_mlp:].view(np.uint32))
    if net["activation"] == "Sine":  # the SIREN bounds differ from xavier's
        assert not np.array_equal(orc.params_fp32[:n_mlp], p_net)
        assert np.abs(p_net[: width * in_w]).max() <= 30.0 / in_w


@pytest.mark.parametrize("name", list(TRAINER_CASES))
def test_forward_within_reference_bar(name):
    """The reference's encoded features through the oracle network -> its fp16 training output and fp32 inference output
    (tests/test_common.h:177: RAE < 1e-2 on the best 99 %; an absolute bar where the outputs are subnormal, values_agree)."""
    n_in, n_out, B = TRAINER_CASES[name]
    g = load(name)
    net = g["meta"]["config"]["network"]
    W = g["meta"]["encoded_width"]
    enc = g["encoded_f16"].view(np.float16).reshape(W, B).T
    p16 = g["params_init_f32"].astype(np.float16)
    n_mlp = g["meta"]["n_params"] - g["meta"]["n_encoding_params"]
    _, _, out = po.forward(net["activation"], p16[:n_mlp], enc, net["n_neurons"], net["n_hidden_layers"], 16)
    ref = g["output_f16"].view(np.float16).reshape(B, 16)
    assert po.values_agree(out[:, :n_out], ref[:, :n_out], 1e-2)
    assert po.values_agree(out[:, :n_out], g["inference_f32"].reshape(B, n_out), 1e-2)


@pytest.mark.parametrize("name", NET_CASES)
def test_network_golden_forward_within_reference_bar(name):
    """`ref_harness mlpdump`: the reference's stand-alone CutlassMLP on its own weights and fp16 inputs."""
    g = load(name)
    m = g["meta"]
    B = m["batch"]
    x = g["x_f16"].view(np.float16).reshape(B, m["n_in"])
    _, _, out = po.forward(m["activation"], g["params_f16"].view(np.float16), x, m["width"], m["n_hidden_layers"], m["padded_output_width"])
    ref = g["output_f16"].view(np.float16).reshape(B, m["padded_output_width"])
    assert rae(out, ref, 99.0) < 1e-2


@pytest.mark.parametrize("act", [po.SINE, po.SILU])
def test_backward_matches_finite_differences(act):
    """backward_f64 of L = sum(dy * out) against central differences of forward_f64, for every parameter and input."""
    rng = np.random.default_rng(3)
    width, nh, in_w, out_pad, B = 8, 2, 5, 3, 7
    n = sum(r * c for r, c in po.matrix_shapes(width, in_w, nh, out_pad))
    params = rng.uniform(-1, 1, n)
    x = rng.uniform(-1, 1, (B, in_w))
    dy = rng.uniform(-1, 1, (B, out_pad))
    dx, dp = po.backward_f64(act, params, x, dy, width, nh, out_pad)

    def loss(p, xx):
        return float((po.forward_f64(act, p, xx, width, nh, out_pad)[1] * dy).sum())

    h = 1e-6
    fd_p = np.array([(loss(params + h * e, x) - loss(params - h * e, x)) / (2 * h) for e in np.eye(n)])
    fd_x = np.array([(loss(params, x + h * e.reshape(B, in_w)) - loss(params, x - h * e.reshape(B, in_w))) / (2 * h) for e in np.eye(B * in_w)]).reshape(B, in_w)
    assert np.allclose(dp, fd_p, rtol=1e-6, atol=1e-8)
    assert np.allclose(dx, fd_x, rtol=1e-6, atol=1e-8)


@pytest.mark.parametrize("act", [po.SINE, po.SILU])
def test_fp16_backward_follows_float64(act):
    """The fp16-rounding mode of the oracle stays within fp16 tolerance of its float64 mode (what the GPU tests lean on)."""
    rng = np.random.default_rng(4)
    width, nh, in_w, out_pad, B = 32, 3, 16, 16, 256
    p16 = po.init_params(width, in_w, nh, out_pad, act, po.Pcg32(7)).astype(np.float16)
    x16 = rng.uniform(-1, 1, (B, in_w)).astype(np.float16)
    dy16 = rng.uniform(-1, 1, (B, out_pad)).astype(np.float16)
    pre, post, out = po.forward(act, p16, x16, width, nh, out_pad)
    assert np.array_equal(post.view(np.uint16), po.act_fwd_pre(act, pre).view(np.uint16))
    _, dx, dp = po.backward(act, p16, x16, pre, post, dy16, width, nh, out_pad)
    p64 = p16.astype(np.float64)
    _, out64 = po.forward_f64(act, p64, x16.astype(np.float64), width, nh, out_pad)
    dx64, dp64 = po.backward_f64(act, p64, x16.astype(np.float64), dy16.astype(np.float64), width, nh, out_pad)
    assert rae(out, out64, 99.0) < 2e-3
    assert rae(dx, dx64, 99.0) < 1e-2
    assert rae(dp, dp64, 99.0) < 1e-2


def test_activation_values():
    """Spot values of the restated activations and derivatives (common_device.h:131-153, 253-277)."""
    z = np.array([0.0, 0.5, -2.0, 3.0], np.float16)
    assert np.array_equal(po.act_fwd_pre(po.SINE, z), np.sin(z.astype(np.float64)).astype(np.float16))
    silu = z.astype(np.float64) / (1 + np.exp(-z.astype(np.float64)))
    assert np.array_equal(po.act_fwd_pre(po.SILU, z), silu.astype(np.float16))
    one = np.ones_like(z)
    assert np.array_equal(po.act_bwd_pre(po.SINE, one, z), np.cos(z.astype(np.float64)).astype(np.float16))
    s = 1 / (1 + np.exp(-z.astype(np.float64)))
    assert np.array_equal(po.act_bwd_pre(po.SILU, one, z), (s * (1 + z.astype(np.float64) * (1 - s))).astype(np.float16))
