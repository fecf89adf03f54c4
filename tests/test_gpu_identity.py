"""BASELINE.json configs[0] as a path of this library: Identity encoding (encodings/identity.h:46-67) + a 64 x 2 network
("CutlassMLP" / "MLP" / "FullyFusedMLP" all run on the wgmma kernels) through create_from_config / trainer->training_step.
Checked against the oracle's MLP stage functions fed with the Identity features, and -- when tests/golden/identity_cutlass.npz
exists -- against vectors dumped by the unmodified reference (its CutlassMLP path, cutlass_mlp.cu:272-308)."""
import ctypes
import json
import os

import numpy as np
import pytest

import oracle_binding as ob
from golden_util import GOLDEN, mlp_gradients_agree, rae

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def f16(t):
    return t.cpu().numpy().view(np.uint16)


def identity_features(x, width=16):
    enc = np.ones((x.shape[0], width), np.float16)
    enc[:, : x.shape[1]] = x.astype(np.float16)
    return enc


@pytest.mark.parametrize("otype,n_in", [("CutlassMLP", 3), ("FullyFusedMLP", 2)])
def test_identity_encoding_training_step_matches_oracle(torch_cuda, otype, n_in):
    torch = torch_cuda
    import tcnn_b200

    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", "configs", "identity_cutlass.json")))
    cfg["network"]["otype"] = otype
    cfg["loss"] = {"otype": "L2"}
    B = 65536  # configs[0]'s batch size
    model = tcnn_b200.create_from_config(n_in, 3, cfg)
    assert model.n_params == model.n_mlp_params == 64 * 16 + 64 * 64 + 16 * 64 and model.encoded_width == 16
    rng = ob.default_rng(7)
    x = ob.generate_random_uniform(rng, B * n_in).reshape(B, n_in)
    y = ob.make_targets(x, 3)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    enc_tap = torch.zeros(B, 64, dtype=torch.float16, device="cuda")
    out_tap = torch.zeros(B, 16, dtype=torch.float16, device="cuda")
    dy_tap = torch.zeros(B, 16, dtype=torch.float16, device="cuda")
    hid_tap = torch.zeros(2, B, 64, dtype=torch.float16, device="cuda")
    model.set_debug_taps(encoded=enc_tap, output=out_tap, dL_doutput=dy_tap, hidden=hid_tap)
    model.trainer.training_step(xd, yd, run_optimizer=False)
    loss = model.trainer.loss()
    torch.cuda.synchronize()
    enc_ref = identity_features(x)
    assert np.array_equal(f16(enc_tap)[:, :16], enc_ref.view(np.uint16)) and (f16(enc_tap)[:, 16:] == 0).all()

    # the oracle's network on the Identity features (a sub-sample: the oracle is a scalar CPU port)
    n = 4096
    lib = ob.load()
    mlp = ob.Mlp(16, 64, 2, 3, 0, ob.ACT["relu"], ob.ACT["none"], 0)
    assert lib.orc_mlp_setup(ctypes.byref(mlp)) == 0
    w16 = f16(model.trainer.params())
    hidden = np.zeros((2, n, 64), np.uint16)
    out = np.zeros((n, 16), np.uint16)
    enc_soa = np.ascontiguousarray(enc_ref[:n].view(np.uint16).T)
    lib.orc_mlp_forward(ctypes.byref(mlp), n, ob.ACCUM_FP32, ob._p(w16), ob._p(enc_soa), ob._p(hidden), ob._p(out))
    assert rae(ob.half_bits_to_float(f16(out_tap)[:n]), ob.half_bits_to_float(out)) < 1e-3
    # full-batch loss from the device's own outputs (L2: mean squared error over B * 3 elements)
    pred = ob.half_bits_to_float(f16(out_tap))[:, :3].astype(np.float64)
    assert abs(loss - float(((pred - y) ** 2).sum() / (B * 3))) <= 1e-4 * loss
    # weight gradients of the whole batch: dL/dy from the device, backward through the oracle in chunks (exact double sums)
    dW = np.zeros(mlp.n_params, np.float64)
    hid_dev, dy_dev = f16(hid_tap), f16(dy_tap)
    for lo in range(0, B, 8192):
        part = np.zeros(mlp.n_params, np.float64)
        e = np.ascontiguousarray(enc_ref[lo : lo + 8192].view(np.uint16).T)
        lib.orc_mlp_backward(ctypes.byref(mlp), 8192, ob.ACCUM_FP32, ob._p(w16), ob._p(e), ob._p(np.ascontiguousarray(hid_dev[:, lo : lo + 8192])),
                             ob._p(np.ascontiguousarray(dy_dev[lo : lo + 8192])), ob._p(part), None)
        dW += part
    g_dev = ob.half_bits_to_float(f16(model.trainer.param_gradients()))
    assert rae(g_dev, dW.astype(np.float16).astype(np.float64), 99.9) < 1.2e-2  # tests/test_common.h:218

    model.set_debug_taps()
    losses = []
    for _ in range(30):
        model.trainer.training_step(xd, yd)
        losses.append(model.trainer.loss())
    assert losses[-1] < 0.7 * losses[0] and np.isfinite(losses).all(), losses[::5]
    inf = model.network.inference(xd)
    assert inf.shape == (B, 3) and torch.isfinite(inf).all()


@pytest.mark.skipif(not os.path.exists(os.path.join(GOLDEN, "identity_cutlass.npz")), reason="tests/golden/identity_cutlass.npz not generated yet")
def test_identity_cutlass_against_reference_golden_vectors(torch_cuda):
    torch = torch_cuda
    import tcnn_b200
    from golden_util import load_case

    g = load_case("identity_cutlass")
    cfg = g["meta"]["config"]
    B, n_in, n_out = g["meta"]["batch"], g["meta"]["n_in"], g["meta"]["n_out"]
    model = tcnn_b200.create_from_config(n_in, n_out, cfg)
    x, y = g["x_f32"].reshape(B, n_in), g["y_f32"].reshape(B, n_out)
    xd, yd = torch.from_numpy(x.copy()).cuda(), torch.from_numpy(y.copy()).cuda()
    p0 = model.trainer.params_full_precision().cpu().numpy()
    assert np.array_equal(p0.view(np.uint32), g["params_init_f32"].view(np.uint32))  # same xavier stream as the reference's CutlassMLP
    out_tap = torch.zeros(B, 16, dtype=torch.float16, device="cuda")
    model.set_debug_taps(output=out_tap)
    inf = model.network.inference(xd).cpu().numpy()
    assert rae(inf, g["inference_f32"].reshape(B, n_out), 99.0) < 1e-2
    model.trainer.training_step(xd, yd, run_optimizer=False)
    loss0 = model.trainer.loss()
    assert abs(loss0 - g["meta"]["losses"][0]) <= 2e-3 * g["meta"]["losses"][0]
    grads = ob.half_bits_to_float(f16(model.trainer.param_gradients()))
    assert mlp_gradients_agree(grads, ob.half_bits_to_float(g["grads_step0_f16"]), 2e-2)
    losses = [loss0]
    for _ in range(g["meta"]["n_steps"]):
        model.trainer.training_step(xd, yd)
        losses.append(model.trainer.loss())
    for mine, theirs in zip(losses, g["meta"]["losses"]):
        assert abs(mine - theirs) <= 5e-2 * abs(theirs), (losses, g["meta"]["losses"])
