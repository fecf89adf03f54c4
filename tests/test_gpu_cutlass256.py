"""256-neuron CutlassMLP networks (csrc/mlp_fused.cu mlp_forward256_kernel: every product in two N = 128 halves, weights through a
ring of half-matrix stages; csrc/mlp_wgrad.cu mlp_wgrad256_kernel: the weight gradients in two 128-row halves, one per CTA of a pair)
against the CPU oracle, tests/preact_oracle.py, torch restatements and the unmodified reference (tests/golden/w256_*.npz), through
the network tier, the trainer, the module tier and the torch modules."""
import ctypes
import json
import os

import numpy as np
import pytest

import oracle_binding as ob
import preact_oracle as po
from golden_util import GOLDEN, rae
from test_gpu_preact import test_network_matches_oracle as preact_network_check

pytestmark = pytest.mark.gpu

W = 256


def f16(t):
    return t.detach().cpu().numpy().view(np.uint16)


def h16(t):
    return t.detach().cpu().numpy().astype(np.float16)


def net_cfg(n_hidden, act="ReLU", out_act="None", otype="CutlassMLP", width=W):
    return {"otype": otype, "n_neurons": width, "n_hidden_layers": n_hidden, "activation": act, "output_activation": out_act}


def oracle_mlp(n_hidden, in_w, out_pad, act, out_act, weights16):
    lib = ob.load()
    mlp = ob.Mlp(in_w, W, n_hidden, out_pad, 0, ob.ACT[act.lower()], ob.ACT[out_act.lower()], 0)
    assert lib.orc_mlp_setup(ctypes.byref(mlp)) == 0
    assert mlp.n_params == weights16.size and mlp.padded_out_width == out_pad
    return lib, mlp


def torch_forward(x16, p16, in_w, n_hidden, out_pad, act="ReLU"):
    """fp32 evaluation of the chain with fp16 rounding after every layer (as the kernels round)."""
    import torch

    h, w, off = x16.float(), p16.float(), 0
    for l, (r, c) in enumerate([(W, in_w)] + [(W, W)] * (n_hidden - 1) + [(out_pad, W)]):
        z = h @ w[off : off + r * c].view(r, c).t()
        off += r * c
        h = (torch.relu(z) if act == "ReLU" and l < n_hidden else z).half().float()
    return h


FORWARD_SHAPES = [
    # hidden, n_in, n_out, activation, output_activation, batch
    (1, 32, 16, "ReLU", "None", 2048),
    (3, 64, 16, "ReLU", "None", 132 * 128 * 3 + 256),  # uneven rounds per CTA
    (8, 256, 256, "ReLU", "None", 2048),               # weight ring over 9 matrices, the widest input and output (two output halves)
    (4, 128, 48, "Tanh", "Sigmoid", 1024),
]


@pytest.mark.parametrize("n_hidden,n_in,n_out,act,out_act,B", FORWARD_SHAPES)
def test_network_forward_matches_oracle(torch_cuda, n_hidden, n_in, n_out, act, out_act, B):
    """The bars of test_gpu_network.test_network_forward_matches_oracle."""
    torch = torch_cuda
    import tcnn_b200

    net = tcnn_b200.Network(n_in, n_out, net_cfg(n_hidden, act, out_act))
    out_pad = (n_out + 15) // 16 * 16
    assert net.n_params == W * n_in + (n_hidden - 1) * W * W + out_pad * W and net.width == W
    p16 = net.initial_params(seed=11).half().contiguous()
    g = torch.Generator(device="cuda").manual_seed(5)
    x = (torch.rand(B, n_in, device="cuda", generator=g) * 2 - 1).half().contiguous()
    out, hidden = net.forward(x, p16)
    out_inf = net.inference_mixed_precision(x, p16)
    torch.cuda.synchronize()
    assert torch.equal(out, out_inf)
    n_check = min(B, 4096)
    sel = np.r_[0 : n_check // 2, B - n_check // 2 : B]
    lib, mlp = oracle_mlp(n_hidden, n_in, out_pad, act, out_act, f16(p16))
    hid_ref = np.zeros((n_hidden, len(sel), W), np.uint16)
    out_ref = np.zeros((len(sel), out_pad), np.uint16)
    lib.orc_mlp_forward(ctypes.byref(mlp), len(sel), ob.ACCUM_FP32, ob._p(f16(p16)), ob._p(np.ascontiguousarray(f16(x)[sel].T)), ob._p(hid_ref), ob._p(out_ref))
    hid_dev = f16(hidden)[:, sel]
    a, b = ob.half_bits_to_float(hid_dev), ob.half_bits_to_float(hid_ref)
    exact = act == "ReLU"
    assert np.abs(a[0] - b[0]).max() <= 2.0**-9 * max(1.0, np.abs(b[0]).max())
    assert (hid_dev[0] != hid_ref[0]).mean() < (0.02 if exact else 0.2)
    assert rae(a, b) < (1e-3 if exact else 3e-3)
    o_dev, o_ref = ob.half_bits_to_float(f16(out)[sel]), ob.half_bits_to_float(out_ref)
    assert np.isfinite(o_dev).all()
    assert rae(o_dev, o_ref, 99.0) < 2e-3
    assert np.abs(o_dev - o_ref).max() <= 1e-2 * max(1.0, np.abs(o_ref).max())
    if B > 4096:  # every row of a large batch was written
        ref = torch_forward(x, p16, n_in, n_hidden, out_pad)
        assert rae(out.float().cpu().numpy(), ref.cpu().numpy(), 99.0) < 2e-3


BACKWARD_SHAPES = [
    # hidden, n_in, n_out, activation, batch
    (3, 64, 16, "ReLU", 1024),
    (2, 256, 192, "Tanh", 2048),                 # dL/d(input) and the output matrix both in two halves; fan-in 256 weight gradients
    (1, 128, 16, "ReLU", 1024),                  # dL/d(input) in one half
    (4, 32, 16, "ReLU", 132 * 128 * 3 + 256),    # 66 CTA pairs: several CTAs flush each row half of every matrix
]


@pytest.mark.parametrize("n_hidden,n_in,n_out,act,B", BACKWARD_SHAPES)
def test_network_backward_matches_oracle(torch_cuda, n_hidden, n_in, n_out, act, B):
    """The bars of test_gpu_general.test_network_backward_matches_oracle."""
    torch = torch_cuda
    import tcnn_b200

    net = tcnn_b200.Network(n_in, n_out, net_cfg(n_hidden, act))
    out_pad = net.padded_output_width
    p16 = net.initial_params(seed=3).half().contiguous()
    g = torch.Generator(device="cuda").manual_seed(7)
    x = (torch.rand(B, n_in, device="cuda", generator=g) * 2 - 1).half().contiguous()
    dy = ((torch.rand(B, out_pad, device="cuda", generator=g) * 2 - 1) * 0.25).half().contiguous()
    out, hidden = net.forward(x, p16)
    dx, dp = net.backward(x, out, hidden, dy, p16)
    dx_only, none = net.backward(x, out, hidden, dy, p16, want_param_grad=False)
    torch.cuda.synchronize()
    assert none is None and torch.equal(dx_only, dx)

    lib, mlp = oracle_mlp(n_hidden, n_in, out_pad, act, "None", f16(p16))
    n_check = min(B, 2048)
    sel = np.r_[0 : n_check // 2, B - n_check // 2 : B]
    dW_sel = np.zeros(net.n_params, np.float64)
    dx_ref = np.zeros((n_in, len(sel)), np.uint16)
    lib.orc_mlp_backward(ctypes.byref(mlp), len(sel), ob.ACCUM_FP32, ob._p(f16(p16)), ob._p(np.ascontiguousarray(f16(x)[sel].T)), ob._p(np.ascontiguousarray(f16(hidden)[:, sel])),
                         ob._p(np.ascontiguousarray(f16(dy)[sel])), ob._p(dW_sel), ob._p(dx_ref))
    a, b = ob.half_bits_to_float(f16(dx)[sel]), ob.half_bits_to_float(dx_ref.T)
    assert rae(a, b, 99.9) < (2e-3 if act == "ReLU" else 5e-3), rae(a, b, 99.9)
    if B <= 4096:
        dW = np.zeros(net.n_params, np.float64)
        lib.orc_mlp_backward(ctypes.byref(mlp), B, ob.ACCUM_FP32, ob._p(f16(p16)), ob._p(np.ascontiguousarray(f16(x).T)), ob._p(np.ascontiguousarray(f16(hidden))), ob._p(f16(dy)),
                             ob._p(dW), None)
        got = dp.float().cpu().numpy()
        want = dW.astype(np.float16).astype(np.float32)
        assert rae(got, want, 99.9) < 3e-3, rae(got, want, 99.9)
        assert np.abs(got - want).max() <= 2e-2 * np.abs(want).max()
    else:
        # split the batch in two multiples of 256: the gradients add up (the big call spreads the tiles over every CTA pair)
        h = (B // 2) // 256 * 256
        parts = []
        for lo, hi in ((0, h), (h, B)):
            o2, hid2 = net.forward(x[lo:hi].contiguous(), p16)
            parts.append(net.backward(x[lo:hi].contiguous(), o2, hid2, dy[lo:hi].contiguous(), p16, want_input_grad=False)[1].float())
        total = (parts[0] + parts[1]).cpu().numpy()
        assert rae(dp.float().cpu().numpy(), total, 99.9) < 2e-3


@pytest.mark.parametrize("n_hidden,n_in,n_out,act,B", [(3, 64, 16, po.SINE, 2048), (2, 256, 32, po.SILU, 2048), (4, 32, 16, po.SILU, 132 * 128 * 2 + 512)])
def test_preact_network_matches_oracle(torch_cuda, n_hidden, n_in, n_out, act, B):
    """Sine / SiLU at 256 neurons with every check of test_gpu_preact.test_network_matches_oracle: SIREN / xavier initial parameters
    bit-equal to preact_oracle.init_params (fan-in 256), stage-by-stage layers, the backward pass fed the device's own buffers."""
    preact_network_check(torch_cuda, W, n_hidden, n_in, n_out, act, B)


TRAINER_CONFIGS = {
    "hash_f2_w256x3": (3, 3, 512, {"encoding": {"otype": "HashGrid", "n_levels": 16, "n_features_per_level": 2, "log2_hashmap_size": 14, "base_resolution": 16, "per_level_scale": 1.5},
                                   "network": net_cfg(3)}),
    "hash_f8_w256x2": (2, 1, 256, {"encoding": {"otype": "HashGrid", "n_levels": 16, "n_features_per_level": 8, "log2_hashmap_size": 12, "base_resolution": 8, "per_level_scale": 1.5},
                                   "network": net_cfg(2)}),
}
for _c in TRAINER_CONFIGS.values():
    _c[3]["loss"] = {"otype": "RelativeL2"}
    _c[3]["optimizer"] = {"otype": "Adam", "learning_rate": 1e-2, "beta1": 0.9, "beta2": 0.99, "epsilon": 1e-15, "l2_reg": 1e-6}


def make_batch(n_in, n_out, B, seed=1337):
    rng = ob.default_rng(seed)
    x = ob.generate_random_uniform(rng, B * n_in).reshape(B, n_in)
    return x, ob.make_targets(x, n_out)


@pytest.mark.parametrize("name", list(TRAINER_CONFIGS))
def test_trainer_matches_oracle(torch_cuda, name):
    """The bars of test_gpu_general.test_general_path_step_matches_oracle."""
    torch = torch_cuda
    import tcnn_b200

    n_in, n_out, B, cfg = TRAINER_CONFIGS[name]
    model = tcnn_b200.create_from_config(n_in, n_out, cfg)
    orc = ob.OracleModel(n_in, n_out, cfg, scales=model.grid_levels()["scales"])
    assert model.n_params == orc.n_params
    assert np.array_equal(model.trainer.params_full_precision().cpu().numpy(), orc.params_fp32)
    x, y = make_batch(n_in, n_out, B)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()

    model.trainer.training_step(xd, yd, run_optimizer=False)
    loss_dev = model.trainer.loss()
    grads = model.trainer.param_gradients().float().cpu().numpy()
    loss_ref = orc.training_step(x, y, run_optimizer=False)
    gref = ob.half_bits_to_float(orc.grads_fp16)
    assert abs(loss_dev - loss_ref) <= 1e-3 * abs(loss_ref)
    n_mlp = orc.n_mlp
    assert rae(grads[:n_mlp], gref[:n_mlp], 99.9) < 1.2e-2
    assert ((grads[n_mlp:] != 0) != (gref[n_mlp:] != 0)).mean() < 2e-3
    assert rae(grads[n_mlp:], gref[n_mlp:], 99.9) < 1.2e-2
    assert rae(model.network.inference(xd).cpu().numpy(), orc.inference(x), 99.0) < 1e-2

    dev_losses, ref_losses = [], []
    for _ in range(10):
        model.trainer.training_step(xd, yd)
        dev_losses.append(model.trainer.loss())
        ref_losses.append(orc.training_step(x, y))
    assert dev_losses[-1] < dev_losses[0]
    for a, b in zip(dev_losses, ref_losses):
        assert abs(a - b) <= 3e-2 * abs(b) + 1e-6, (dev_losses, ref_losses)


def torch_identity_mlp(params, x, n_in_pad, n_hidden, n_out):
    """float32 autograd restatement of an Identity-encoded ReLU network with the module's fp16 weights."""
    import torch

    h = torch.cat([x, torch.ones(x.shape[0], n_in_pad - x.shape[1], device=x.device)], 1).half().float()
    p = params.half().float()
    off = 0
    for l, (r, c) in enumerate(po.matrix_shapes(W, n_in_pad, n_hidden, (n_out + 15) // 16 * 16)):
        h = h @ p[off : off + r * c].view(r, c).t()
        off += r * c
        if l < n_hidden:
            h = torch.relu(h)
    return h[:, :n_out]


def test_torch_modules(torch_cuda):
    """torch_modules.Network (parameter and input gradients) and NetworkWithInputEncoding (Identity) against a float32 torch autograd
    restatement with the same fp16 weights; the module tier with a HashGrid in front and dL/d(position) against the oracle, and
    NetworkWithInputEncoding(HashGrid) with the input requiring grad against the module tier."""
    torch = torch_cuda
    import tcnn_b200
    import tcnn_b200.torch_modules as tm

    B, n_in, n_out, nh = 4096, 5, 3, 3
    g = torch.Generator(device="cuda").manual_seed(2)
    x = (torch.rand(B, n_in, device="cuda", generator=g) * 2 - 1).requires_grad_(True)
    target = torch.rand(B, n_out, device="cuda", generator=g)

    net = tm.Network(n_in, n_out, net_cfg(nh))
    y = net(x)
    ((y.float() - target) ** 2).mean().backward()
    p_ref = net.params.detach().clone().requires_grad_(True)
    x_ref = x.detach().clone().requires_grad_(True)
    y_ref = torch_identity_mlp(p_ref, x_ref, 16, nh, n_out)
    ((y_ref - target) ** 2).mean().backward()
    assert rae(y.float().detach().cpu().numpy(), y_ref.detach().cpu().numpy(), 99.0) < 5e-3
    assert rae(net.params.grad.cpu().numpy(), p_ref.grad.cpu().numpy(), 99.0) < 2e-2
    assert rae(x.grad.cpu().numpy(), x_ref.grad.cpu().numpy(), 99.0) < 2e-2

    model = tm.NetworkWithInputEncoding(n_in, n_out, {"otype": "Identity"}, net_cfg(nh))
    ((model(x.detach()).float() - target) ** 2).mean().backward()
    p2 = model.params.detach().clone().requires_grad_(True)
    ((torch_identity_mlp(p2, x.detach(), 16, nh, n_out) - target) ** 2).mean().backward()
    assert rae(model.params.grad.cpu().numpy(), p2.grad.cpu().numpy(), 99.0) < 2e-2

    # a grid in front, dL/d(position) through it: the module tier (tcnn::cpp::Module) against the oracle's backward pass
    n_in, n_out, Bg, cfg = TRAINER_CONFIGS["hash_f2_w256x3"]
    xs, _ = make_batch(n_in, n_out, Bg)
    native = tcnn_b200.Module(n_in, n_out, cfg["encoding"], cfg["network"])
    p16 = native.initial_params(seed=1337).half().contiguous()
    dy = torch.zeros(Bg, 16, dtype=torch.float16, device="cuda")
    dy[:, :n_out] = ((torch.rand(Bg, n_out, device="cuda", generator=g) * 2 - 1) * 0.1).half()
    scaled = (dy.float() * 128.0).half()
    native.fwd(torch.from_numpy(xs).cuda(), p16)
    dp, dx = native.bwd(torch.from_numpy(xs).cuda(), p16, scaled, want_input_grad=True)
    torch.cuda.synchronize()
    orc = ob.OracleModel(n_in, n_out, cfg, scales=tcnn_b200.create_from_config(n_in, n_out, cfg).grid_levels()["scales"])
    orc.set_params_full_precision(p16.float().cpu().numpy())
    want = orc.backward_from_dy(xs, f16(scaled))
    got = dp.float().cpu().numpy()
    assert rae(got[: orc.n_mlp], want[: orc.n_mlp], 99.9) < 1.2e-2
    assert rae(got[orc.n_mlp :], want[orc.n_mlp :], 99.9) < 1.2e-2
    enc = orc.encode(xs)
    hidden, _ = orc.mlp_forward(enc)
    _, d_enc = orc.mlp_backward(enc, hidden, np.ascontiguousarray(f16(scaled)))
    assert rae(dx.cpu().numpy(), orc.grid_input_gradient(xs, d_enc), 99.0) < 2e-2

    # NetworkWithInputEncoding(HashGrid) with the input requiring grad: autograd must deliver the native module's gradients of the
    # loss-scaled dL/d(output), divided by the loss scale (the bars of test_gpu_parity.test_torch_autograd_layer_on_the_module_tier).
    # As in the reference's modules.py, the parameter gradient comes back in the parameters' fp16 working precision: with a fresh
    # grid in front the network's weight gradients are ~1e-5, fp16 subnormals, so the expected values are rounded the same way.
    mod = tm.NetworkWithInputEncoding(n_in, n_out, cfg["encoding"], cfg["network"])
    xg = torch.from_numpy(xs).cuda().requires_grad_(True)
    dy1 = torch.zeros(Bg, 16, dtype=torch.float16, device="cuda")
    dy1[:, :n_out] = (torch.rand(Bg, n_out, device="cuda", generator=g) * 2 - 1).half()
    mod(xg).backward(dy1[:, :n_out])
    p16m = mod.params.detach().half().contiguous()
    x_dev = torch.from_numpy(xs).cuda()
    mod.native_tcnn_module.fwd(x_dev, p16m)
    dp1, dx1 = mod.native_tcnn_module.bwd(x_dev, p16m, (dy1.float() * mod.loss_scale).half(), want_input_grad=True)
    torch.cuda.synchronize()
    a = mod.params.grad.cpu().numpy()
    b = (dp1.float() / mod.loss_scale).half().float().cpu().numpy()
    assert rae(a[: orc.n_mlp], b[: orc.n_mlp], 99.9) < 2e-3 and rae(a[orc.n_mlp :], b[orc.n_mlp :], 99.9) < 5e-3
    assert rae(xg.grad.cpu().numpy(), (dx1 / mod.loss_scale).cpu().numpy(), 99.9) < 5e-3



def test_snapshot_roundtrip(torch_cuda):
    torch = torch_cuda
    import tcnn_b200

    n_in, n_out, B, cfg = TRAINER_CONFIGS["hash_f2_w256x3"]
    a = tcnn_b200.create_from_config(n_in, n_out, cfg)
    x, y = make_batch(n_in, n_out, B)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    for _ in range(3):
        a.trainer.training_step(xd, yd)
    blob = a.trainer.serialize(with_optimizer=True)
    b = tcnn_b200.create_from_config(n_in, n_out, cfg, seed=7)
    b.trainer.deserialize(blob)
    assert torch.equal(a.trainer.params(), b.trainer.params())
    assert torch.equal(a.network.inference(xd), b.network.inference(xd))


@pytest.mark.parametrize("name,act", [("w256_net_relu_h3", "ReLU"), ("w256_net_sine_h3", po.SINE)])
def test_network_against_reference_golden_vectors(torch_cuda, name, act):
    """`ref_harness mlpdump` of the unmodified reference's CutlassMLP 256 x 3: its weights and inputs -> its outputs within
    tests/test_common.h:177 (RAE < 1e-2 @ p99)."""
    torch = torch_cuda
    import tcnn_b200

    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    m = json.loads(bytes(z["meta"]).decode())
    assert m["width"] == W
    net = tcnn_b200.Network(m["n_in"], m["n_out"], net_cfg(m["n_hidden_layers"], m["activation"], otype=m["otype"]))
    assert net.n_params == m["n_params"] and net.padded_output_width == m["padded_output_width"]
    B = m["batch"]
    p16 = torch.from_numpy(z["params_f16"].view(np.float16).copy()).cuda()
    x = torch.from_numpy(z["x_f16"].view(np.float16).reshape(B, m["n_in"]).copy()).cuda()
    out = net.inference_mixed_precision(x, p16)
    torch.cuda.synchronize()
    assert rae(h16(out), z["output_f16"].view(np.float16).reshape(B, m["padded_output_width"]), 99.0) < 1e-2


def outputs_agree(a, b):
    """preact_oracle.values_agree, whose absolute bar (mean <= 2.5, max <= 16 quanta of 2^-24) also applies when every reference output
    is an fp16 subnormal (< 2^-14): a fresh grid (entries ~1e-4) in front of a 256-wide ReLU network outputs a few hundred quanta, where
    the reference's fp16 accumulation inside the MMA is quantisation noise of a few quanta."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if po.values_agree(a, b, 1e-2):
        return True
    d, q = np.abs(a - b), 2.0**-24
    return bool(np.abs(b).max() < 2.0**-14 and d.mean() <= 2.5 * q and d.max() <= 16 * q)


def test_trainer_against_reference_golden_vectors(torch_cuda):
    """`ref_harness dump` of HashGrid + CutlassMLP 256 x 2: initial parameters, outputs, loss and the ten-step trajectory with the bars of
    test_gpu_preact.test_trainer_against_reference_golden_vectors (its step-0 gradient comparison is left out, see below)."""
    torch = torch_cuda
    import tcnn_b200

    name, n_in, n_out, B = "w256_hash3d_relu", 3, 3, 512
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    g = {k: z[k] for k in z.files if k != "meta"}
    meta = json.loads(bytes(z["meta"]).decode())
    model = tcnn_b200.create_from_config(n_in, n_out, json.load(open(os.path.join(GOLDEN, "configs", name + ".json"))))
    x, y = g["x_f32"].reshape(B, n_in), g["y_f32"].reshape(B, n_out)
    xd, yd = torch.from_numpy(x.copy()).cuda(), torch.from_numpy(y.copy()).cuda()
    assert np.array_equal(model.trainer.params_full_precision().cpu().numpy().view(np.uint32), g["params_init_f32"].view(np.uint32))

    out_tap = torch.zeros(B, 16, dtype=torch.float16, device="cuda")
    model.set_debug_taps(output=out_tap)
    assert outputs_agree(model.network.inference(xd).cpu().numpy(), g["inference_f32"].reshape(B, n_out))
    model.trainer.training_step(xd, yd, run_optimizer=False)
    loss0 = model.trainer.loss()
    torch.cuda.synchronize()
    assert outputs_agree(h16(out_tap)[:, :n_out], g["output_f16"].view(np.float16).reshape(B, 16)[:, :n_out])
    assert abs(loss0 - meta["losses"][0]) <= 1e-3 * meta["losses"][0]
    # The step-0 gradients are not compared with the reference's: they are compared with the fp32 oracle in test_trainer_matches_oracle.
    # On this fixture the oracle (fp32 accumulation) is 3.1 % (network), 12 % (first matrix) and 12 % (grid) RAE @p99.9 from the
    # reference's gradients, and the oracle's own fp16-accumulating mode is 10 % (first matrix) and 9.5 % (grid) from its fp32
    # mode: the reference's fp16 sums of 256-wide products account for a gap of that size, in the grid gradients too (they are
    # sums of the fp16 dL/d(encoding) the network's backward pass produces).

    model.trainer.training_step(xd, yd)
    losses = [loss0, model.trainer.loss()]
    for _ in range(meta["n_steps"] - 1):
        model.trainer.training_step(xd, yd)
        losses.append(model.trainer.loss())
    for mine, theirs in zip(losses, meta["losses"]):
        assert abs(mine - theirs) <= 3e-2 * abs(theirs), (losses, meta["losses"])


def test_errors(torch_cuda):
    import tcnn_b200

    grid = {"otype": "HashGrid", "n_levels": 8, "n_features_per_level": 2, "log2_hashmap_size": 12}
    # FullyFusedMLP keeps the reference's widths and text
    with pytest.raises(tcnn_b200.TcnnError, match="FullyFusedMLP only supports 16, 32, 64, and 128 neurons, but got 256. Use CutlassMLP instead"):
        tcnn_b200.Network(16, 16, net_cfg(2, otype="FullyFusedMLP"))
    with pytest.raises(tcnn_b200.TcnnError, match="but got 256"):
        tcnn_b200.create_from_config(3, 3, {"encoding": grid, "network": net_cfg(2, otype="FullyFusedMLP")})
    for otype in ("CutlassMLP", "MLP"):
        for width in (192, 512):
            with pytest.raises(tcnn_b200.TcnnError, match=f"only supports 16, 32, 64, and 128 neurons, but got {width}"):
                tcnn_b200.Network(16, 16, net_cfg(2, otype=otype, width=width))
            with pytest.raises(tcnn_b200.TcnnError, match=f"only supports 16, 32, 64, and 128 neurons, but got {width}"):
                tcnn_b200.create_from_config(3, 3, {"encoding": grid, "network": net_cfg(2, otype=otype, width=width)})
        assert tcnn_b200.Network(16, 16, net_cfg(2, otype=otype)).width == W
        for act in (po.SINE, po.SILU):
            assert tcnn_b200.Network(16, 16, net_cfg(2, act, otype=otype)).n_forward_activations == 4
    # the network input of a 256-neuron network is at most 256 wide
    with pytest.raises(tcnn_b200.TcnnError, match="at most 64 \\(128 / 256 for 128 / 256 neurons\\)"):
        tcnn_b200.Network(272, 16, net_cfg(2))
    with pytest.raises(tcnn_b200.TcnnError, match="at most 64 \\(128 / 256 for 128 / 256 neurons\\)"):
        tcnn_b200.Module(272, 16, {"otype": "Identity"}, net_cfg(2))
    assert tcnn_b200.Network(256, 16, net_cfg(2)).input_width == 256
