"""CutlassMLP with a Sine / SiLU hidden activation on the GPU: the stand-alone network kernels keep the fp16 pre-activations next to
the post-activations (csrc/mlp_fused.cu, PRE) and take the derivative at them. Checked against tests/preact_oracle.py, against the
unmodified reference (tests/golden/preact_*.npz), through the network tier, the trainer and the torch modules."""
import json
import os

import numpy as np
import pytest

import oracle_binding as ob
import preact_oracle as po
from golden_util import GOLDEN, mlp_gradients_agree, rae

pytestmark = pytest.mark.gpu


def f16(t):
    return t.detach().cpu().numpy().view(np.uint16)


def h16(t):
    return t.detach().cpu().numpy().astype(np.float16)


def net_cfg(act, width, n_hidden, otype="CutlassMLP", out_act="None"):
    return {"otype": otype, "n_neurons": width, "n_hidden_layers": n_hidden, "activation": act, "output_activation": out_act}


def ulp16(v):
    """Spacing of fp16 at |v| (subnormal spacing below 2^-14)."""
    e = np.floor(np.log2(np.maximum(np.abs(np.asarray(v, np.float64)), 2.0**-14)))
    return 2.0 ** (e - 10)


def close_to(dev, ref, z, act):
    """The device evaluates the reference's expressions with the fast-math hardware functions (__sinf / __cosf / __expf, as the
    reference's build does): within one fp16 ulp of the exact value plus their absolute error, which grows with |z| for Sine (range
    reduction in fp32)."""
    dev, ref, z = (np.asarray(a, np.float64) for a in (dev, ref, z))
    slack = 2e-6 * (1 + np.abs(z)) if act == po.SINE else 2e-6 * np.abs(ref)
    return np.abs(dev - ref) <= ulp16(ref) + slack


def is_function_of(keys16, values16):
    """Every stored key (fp16 bits) maps to ONE stored value: the value was computed from the stored key alone."""
    pairs = np.unique((np.asarray(keys16).view(np.uint16).ravel().astype(np.uint32) << 16) | np.asarray(values16).view(np.uint16).ravel().astype(np.uint32))
    return np.unique(pairs >> 16).size == pairs.size


def all_finite_fp16():
    bits = np.r_[np.arange(0x0000, 0x7C00), np.arange(0x8000, 0xFC00)].astype(np.uint16)
    return bits.view(np.float16)


@pytest.mark.parametrize("act", [po.SINE, po.SILU])
@pytest.mark.parametrize("width", [16, 32, 64, 128])
def test_activation_and_derivative_bit_exact(torch_cuda, act, width):
    """Every finite fp16 value as a pre-activation. W_0 = I makes z_0 = x exactly; W_out[j][k] = (k % 16 == j) makes the gradient
    that reaches hidden layer 0 exactly dL/dy[k % 16]; dL/dx = W_0^T g_0 = g_0. A first backward pass with dL/dy = 1 reads out the
    device's fp16 factor (half)act'(z) for every z; a second one with random dL/dy must then give g_0 = dL/dy * factor (an fp16
    product) bit for bit. The stored post-activations and the factors are close to the exact act(z) / act'(z)."""
    torch = torch_cuda
    import tcnn_b200

    net = tcnn_b200.Network(width, 16, net_cfg(act, width, 1))
    assert net.n_forward_activations == 2
    vals = all_finite_fp16()
    B = (vals.size + width * 256 - 1) // (width * 256) * 256
    x = np.zeros(B * width, np.float16)
    x[: vals.size] = vals
    x = x.reshape(B, width)
    w0 = np.eye(width, dtype=np.float16)
    wo = (np.arange(width)[None, :] % 16 == np.arange(16)[:, None]).astype(np.float16)
    p16 = torch.from_numpy(np.concatenate([w0.ravel(), wo.ravel()])).cuda()
    assert p16.numel() == net.n_params
    xd = torch.from_numpy(x).cuda()
    dy = (torch.rand(B, 16, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1)) * 2 - 1).half()
    out, hidden = net.forward(xd, p16)
    factor, _ = net.backward(xd, out, hidden, torch.ones_like(dy), p16, want_param_grad=False)
    dx, _ = net.backward(xd, out, hidden, dy, p16, want_param_grad=False)
    assert torch.equal(out, net.inference_mixed_precision(xd, p16))
    torch.cuda.synchronize()
    post, pre = h16(hidden[0]), h16(hidden[1])
    assert np.array_equal(pre.astype(np.float64), x.astype(np.float64))  # (an input -0 accumulates to +0)
    factor = h16(factor)
    g_expect = (h16(dy)[:, np.arange(width) % 16] * factor).astype(np.float16)  # fp16 product
    # exact in value: dL/dx = W_0^T g_0 passes through an fp32 sum, which turns a -0 of g_0 (an underflowed product) into +0
    bad = np.nonzero(h16(dx).astype(np.float64) != g_expect.astype(np.float64))
    assert bad[0].size == 0, (bad[0].size, [(float(pre[i, j]), float(h16(dy)[i, j % 16]), float(factor[i, j]), float(h16(dx)[i, j]), float(g_expect[i, j])) for i, j in zip(*bad)][:8])
    assert is_function_of(pre, post) and is_function_of(pre, factor)
    moderate = np.abs(pre.astype(np.float64)) <= (64 if act == po.SINE else 1e4)
    assert close_to(post, po.act_f64(act, pre), pre, act)[moderate].all()
    assert close_to(factor, po.act_deriv_f64(act, pre), pre, act)[moderate].all()


SHAPES = [
    # width, hidden, n_in, n_out, activation, batch
    (16, 2, 16, 16, po.SINE, 2048),
    (16, 3, 32, 16, po.SILU, 1024),
    (32, 3, 32, 32, po.SINE, 148 * 128 * 3 + 256),   # uneven slots
    (32, 2, 16, 16, po.SILU, 2048),
    (64, 2, 64, 64, po.SINE, 148 * 128 * 9),         # 4 slots, 2+ rounds
    (64, 4, 32, 16, po.SILU, 4096),
    (128, 3, 64, 16, po.SINE, 2048),
    (128, 8, 128, 128, po.SILU, 148 * 128 * 2 + 512),  # 9 matrices > 7 stages: weights stream through the ring
    (128, 8, 128, 32, po.SINE, 2048),
]


@pytest.mark.parametrize("width,n_hidden,n_in,n_out,act,B", SHAPES)
def test_network_matches_oracle(torch_cuda, width, n_hidden, n_in, n_out, act, B):
    torch = torch_cuda
    import tcnn_b200

    net = tcnn_b200.Network(n_in, n_out, net_cfg(act, width, n_hidden))
    out_pad = net.padded_output_width
    assert net.n_forward_activations == 2 * n_hidden
    p32 = net.initial_params(seed=11)
    # SIREN / xavier from the same pcg32 stream as the reference's CutlassMLP::initialize_params
    ref_init = po.init_params(width, n_in, n_hidden, out_pad, act, po.Pcg32(11))
    assert np.array_equal(p32.cpu().numpy().view(np.uint32), ref_init.view(np.uint32))
    p16 = p32.half().contiguous()
    g = torch.Generator(device="cuda").manual_seed(5)
    x = (torch.rand(B, n_in, device="cuda", generator=g) * 2 - 1).half()
    dy = (torch.rand(B, out_pad, device="cuda", generator=g) * 2 - 1).half()
    out, hidden = net.forward(x, p16)
    dx, dp = net.backward(x, out, hidden, dy, p16)
    assert torch.equal(out, net.inference_mixed_precision(x, p16))
    torch.cuda.synchronize()
    n_check = min(B, 4096)
    sel = np.r_[0 : n_check // 2, B - n_check // 2 : B]
    hid = h16(hidden)[:, sel]
    post, pre = hid[:n_hidden], hid[n_hidden:]
    xs, dys, w16 = h16(x)[sel], h16(dy)[sel], h16(p16)
    # hidden = act(pre-activations), computed from the stored fp16 z alone, in every layer
    assert is_function_of(pre, post)
    assert close_to(post, po.act_f64(act, pre), pre, act).all()
    # stage by stage, each oracle layer fed with the device's previous one: one fp16 rounding of an fp32 (device) / float64 (oracle) sum
    mats = po.split_weights(w16, width, n_in, n_hidden, out_pad)
    ins = [xs] + list(post)
    for l in range(n_hidden + 1):
        ref = (ins[l].astype(np.float64) @ mats[l].T).astype(np.float16).astype(np.float64)
        dev = (pre[l] if l < n_hidden else h16(out)[sel]).astype(np.float64)
        assert np.abs(dev - ref).max() <= 2.0**-10 * max(1.0, np.abs(ref).max()), l
        assert (dev != ref).mean() < 0.05, l
    _, _, out_ref = po.forward(act, w16, xs, width, n_hidden, out_pad)  # and the whole chain from the inputs
    assert rae(h16(out)[sel], out_ref, 99.0) < 2e-2
    # backward: the oracle fed with the device's own forward buffers
    _, dx_ref, dp_ref = po.backward(act, w16, xs, pre, post, dys, width, n_hidden, out_pad)
    assert rae(h16(dx)[sel], dx_ref, 99.0) < 1e-2
    if B == n_check:  # weight gradients sum over the whole batch
        assert mlp_gradients_agree(h16(dp).astype(np.float64), dp_ref, 2e-2)
    # every row of a large batch: the weight gradients against a torch fp32 evaluation from the device's own buffers
    else:
        hb = [x.float()] + [hidden[l].float() for l in range(n_hidden)]
        gb, up, off = [None] * n_hidden, dy.float(), []
        mats = po.split_weights(w16, width, n_in, n_hidden, out_pad, np.float32)
        for l in range(n_hidden - 1, -1, -1):
            z = hidden[n_hidden + l].double()
            d = torch.cos(z) if act == po.SINE else torch.sigmoid(z) * (1 + z * (1 - torch.sigmoid(z)))
            up = (up.float() @ torch.from_numpy(mats[l + 1]).cuda()).half() * d.half()
            gb[l] = up.float()
        dW = [gb[l].t() @ hb[l] for l in range(n_hidden)] + [dy.float().t() @ hb[n_hidden]]
        ref = torch.cat([w.reshape(-1) for w in dW]).cpu().numpy()
        assert mlp_gradients_agree(h16(dp).astype(np.float64), ref.astype(np.float64), 2e-2)


NET_GOLDEN = ["preact_net_sine_w64_h2", "preact_net_silu_w128_h4"]


@pytest.mark.parametrize("name", NET_GOLDEN)
def test_network_against_reference_golden_vectors(torch_cuda, name):
    """`ref_harness mlpdump` of the unmodified reference's CutlassMLP (Sine 64 x 2, SiLU 128 x 4): its weights and inputs -> its
    outputs within tests/test_common.h:177 (RAE < 1e-2 @ p99)."""
    torch = torch_cuda
    import tcnn_b200

    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    m = json.loads(bytes(z["meta"]).decode())
    net = tcnn_b200.Network(m["n_in"], m["n_out"], net_cfg(m["activation"], m["width"], m["n_hidden_layers"], m["otype"]))
    assert net.n_params == m["n_params"] and net.padded_output_width == m["padded_output_width"]
    B = m["batch"]
    p16 = torch.from_numpy(z["params_f16"].view(np.float16).copy()).cuda()
    x = torch.from_numpy(z["x_f16"].view(np.float16).reshape(B, m["n_in"]).copy()).cuda()
    out = net.inference_mixed_precision(x, p16)
    torch.cuda.synchronize()
    ref = z["output_f16"].view(np.float16).reshape(B, m["padded_output_width"])
    assert rae(h16(out), ref, 99.0) < 1e-2


TRAINER_GOLDEN = {"preact_hash2d_sine": (2, 3, 512), "preact_hash3d_silu": (3, 3, 512)}


@pytest.mark.parametrize("name", list(TRAINER_GOLDEN))
def test_trainer_against_reference_golden_vectors(torch_cuda, name):
    """The assertions of test_gpu_parity.test_against_reference_golden_vectors on HashGrid + CutlassMLP Sine 64 x 2 / SiLU 128 x 3 (the
    general path). Outputs use values_agree: the SiLU network behind a fresh grid outputs subnormal fp16 values."""
    torch = torch_cuda
    import tcnn_b200

    n_in, n_out, B = TRAINER_GOLDEN[name]
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    g = {k: z[k] for k in z.files if k != "meta"}
    meta = json.loads(bytes(z["meta"]).decode())
    cfg = json.load(open(os.path.join(GOLDEN, "configs", name + ".json")))
    model = tcnn_b200.create_from_config(n_in, n_out, cfg)
    x, y = g["x_f32"].reshape(B, n_in), g["y_f32"].reshape(B, n_out)
    xd, yd = torch.from_numpy(x.copy()).cuda(), torch.from_numpy(y.copy()).cuda()

    p0 = model.trainer.params_full_precision().cpu().numpy()
    assert np.array_equal(p0.view(np.uint32), g["params_init_f32"].view(np.uint32))  # SIREN / xavier + grid, bit for bit

    out_tap = torch.zeros(B, 16, dtype=torch.float16, device="cuda")
    model.set_debug_taps(output=out_tap)
    inf = model.network.inference(xd).cpu().numpy()
    assert po.values_agree(inf, g["inference_f32"].reshape(B, n_out), 1e-2)

    model.trainer.training_step(xd, yd, run_optimizer=False)
    loss0 = model.trainer.loss()
    torch.cuda.synchronize()
    a = h16(out_tap)[:, :n_out]
    assert po.values_agree(a, g["output_f16"].view(np.float16).reshape(B, 16)[:, :n_out], 1e-2)
    assert abs(loss0 - meta["losses"][0]) <= 1e-3 * meta["losses"][0]

    grads = ob.half_bits_to_float(f16(model.trainer.param_gradients()))
    ref = ob.half_bits_to_float(g["grads_step0_f16"])
    n_mlp = model.n_mlp_params
    assert mlp_gradients_agree(grads[:n_mlp], ref[:n_mlp], 2e-2)
    assert rae(grads[n_mlp:], ref[n_mlp:], 99.9) < 1.2e-2

    model.trainer.training_step(xd, yd)
    losses = [loss0, model.trainer.loss()]
    for _ in range(meta["n_steps"] - 1):
        model.trainer.training_step(xd, yd)
        losses.append(model.trainer.loss())
    for mine, theirs in zip(losses, meta["losses"]):
        assert abs(mine - theirs) <= 3e-2 * abs(theirs), (losses, meta["losses"])


def torch_mlp(act, params, x, n_in_pad, width, n_hidden, n_out):
    """float32 autograd restatement: Identity encoding (padding features 1), fp16 weights, act on every hidden layer."""
    import torch

    ones = torch.ones(x.shape[0], n_in_pad - x.shape[1], device=x.device)
    h = torch.cat([x, ones], 1).half().float()
    p = params.half().float()
    off = 0
    out_pad = (n_out + 15) // 16 * 16
    for rows, cols in po.matrix_shapes(width, n_in_pad, n_hidden, out_pad):
        w = p[off : off + rows * cols].view(rows, cols)
        off += rows * cols
        h = h @ w.t()
        if rows == width and off < p.numel():
            h = torch.sin(h) if act == po.SINE else torch.nn.functional.silu(h)
    return h[:, :n_out]


@pytest.mark.parametrize("act", [po.SINE, po.SILU])
def test_torch_modules_gradients(torch_cuda, act):
    """torch_modules.Network (parameter and input gradients) and NetworkWithInputEncoding (Identity encoding, parameter gradients) on
    CutlassMLP Sine / SiLU against a float32 torch autograd restatement with the same fp16 weights."""
    torch = torch_cuda
    import tcnn_b200.torch_modules as tm

    B, n_in, n_out, width, nh = 4096, 5, 3, 64, 3
    cfg = net_cfg(act, width, nh)
    g = torch.Generator(device="cuda").manual_seed(2)
    x = (torch.rand(B, n_in, device="cuda", generator=g) * 2 - 1).requires_grad_(True)
    target = torch.rand(B, n_out, device="cuda", generator=g)

    net = tm.Network(n_in, n_out, cfg)
    y = net(x)
    ((y.float() - target) ** 2).mean().backward()
    p_ref = net.params.detach().clone().requires_grad_(True)
    x_ref = x.detach().clone().requires_grad_(True)
    y_ref = torch_mlp(act, p_ref, x_ref, 16, width, nh, n_out)
    ((y_ref - target) ** 2).mean().backward()
    assert rae(y.float().detach().cpu().numpy(), y_ref.detach().cpu().numpy(), 99.0) < 5e-3
    assert rae(net.params.grad.cpu().numpy(), p_ref.grad.cpu().numpy(), 99.0) < 2e-2
    assert rae(x.grad.cpu().numpy(), x_ref.grad.cpu().numpy(), 99.0) < 2e-2

    model = tm.NetworkWithInputEncoding(n_in, n_out, {"otype": "Identity"}, cfg)
    y2 = model(x.detach())
    ((y2.float() - target) ** 2).mean().backward()
    p2 = model.params.detach().clone().requires_grad_(True)
    ((torch_mlp(act, p2, x.detach(), 16, width, nh, n_out) - target) ** 2).mean().backward()
    assert rae(model.params.grad.cpu().numpy(), p2.grad.cpu().numpy(), 99.0) < 2e-2


def test_siren_fits_a_sinusoidal_image(torch_cuda):
    """A small SIREN (CutlassMLP Sine 64 x 3) fitted to a 2-D sinusoidal image through torch_modules.Network: the loss falls 10x."""
    torch = torch_cuda
    import tcnn_b200.torch_modules as tm

    net = tm.Network(2, 1, net_cfg(po.SINE, 64, 3))
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    g = torch.Generator(device="cuda").manual_seed(0)

    def image(x):
        return (0.5 + 0.5 * torch.sin(2 * np.pi * 3 * x[:, :1]) * torch.cos(2 * np.pi * 2 * x[:, 1:])).float()

    xs = torch.rand(1 << 14, 2, device="cuda", generator=g)
    first = None
    for _ in range(300):
        x = torch.rand(1 << 14, 2, device="cuda", generator=g)
        loss = ((net(x).float() - image(x)) ** 2).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
    with torch.no_grad():
        final = float(((net(xs).float() - image(xs)) ** 2).mean())
        first = float(((tm.Network(2, 1, net_cfg(po.SINE, 64, 3))(xs).float() - image(xs)) ** 2).mean())
    assert final * 10 <= first, (first, final)


def test_errors(torch_cuda):
    import tcnn_b200

    enc = {"otype": "HashGrid", "n_levels": 8, "n_features_per_level": 2, "log2_hashmap_size": 12}
    for act in (po.SINE, po.SILU):
        with pytest.raises(tcnn_b200.TcnnError, match="Unsupported activation"):
            tcnn_b200.Network(16, 16, net_cfg(act, 64, 2, otype="FullyFusedMLP"))
        with pytest.raises(tcnn_b200.TcnnError, match="Unsupported activation"):
            tcnn_b200.create_from_config(3, 3, {"encoding": enc, "network": net_cfg(act, 64, 2, otype="FullyFusedMLP")})
        for otype in ("CutlassMLP", "MLP", "FullyFusedMLP"):
            with pytest.raises(tcnn_b200.TcnnError, match="output_activation"):
                tcnn_b200.Network(16, 16, net_cfg("ReLU", 64, 2, otype=otype, out_act=act))
        with pytest.raises(tcnn_b200.TcnnError, match="output_activation"):
            tcnn_b200.create_from_config(3, 3, {"encoding": enc, "network": net_cfg("ReLU", 64, 2, out_act=act)})
        # accepted as the hidden activation of a CutlassMLP / MLP, in every tier
        assert tcnn_b200.Network(16, 16, net_cfg(act, 64, 2, otype="MLP")).n_forward_activations == 4
        tcnn_b200.create_from_config(3, 3, {"encoding": enc, "network": net_cfg(act, 64, 2)})
    assert tcnn_b200.Network(16, 16, net_cfg("Tanh", 64, 2)).n_forward_activations == 2
