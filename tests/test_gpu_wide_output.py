"""Networks whose padded output is wider than their hidden layers (feature fields, many-class heads): the WIDE kernels of
csrc/mlp_fused.cu (the output matrix in chunks of n_neurons rows, forward; the first backward product in K-blocks) and csrc/mlp_wgrad.cu
(the output matrix's weight gradients in several passes) against the fp32-accumulate CPU oracle, tests/preact_oracle.py and torch
restatements, through the network tier, the general path of the trainer and the torch modules."""
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


def f16(t):
    return t.detach().cpu().numpy().view(np.uint16)


def net_cfg(width, n_hidden, act="ReLU", out_act="None"):
    otype = "CutlassMLP" if width == 256 else "FullyFusedMLP"
    return {"otype": otype, "n_neurons": width, "n_hidden_layers": n_hidden, "activation": act, "output_activation": out_act}


def oracle_mlp(width, n_hidden, in_w, out_pad, act, out_act, n_params):
    lib = ob.load()
    mlp = ob.Mlp(in_w, width, n_hidden, out_pad, 0, ob.ACT[act.lower()], ob.ACT[out_act.lower()], 0)
    assert lib.orc_mlp_setup(ctypes.byref(mlp)) == 0
    assert mlp.n_params == n_params and mlp.padded_out_width == out_pad
    return lib, mlp


FORWARD_SHAPES = [
    # width, hidden, n_in, n_out, activation, output_activation, batch
    (16, 2, 16, 32, "ReLU", "None", 2048),                 # just above the width
    (16, 2, 16, 1024, "ReLU", "None", 1024),               # 64 chunks: weight ring
    (32, 3, 32, 48, "ReLU", "None", 2048),
    (32, 2, 32, 512, "Tanh", "Sigmoid", 1024),
    (64, 2, 32, 128, "ReLU", "None", 132 * 64 * 4 + 256),   # uneven rounds per CTA
    (64, 2, 32, 200, "ReLU", "Sigmoid", 2048),             # 208: not a multiple of the chunk
    (64, 3, 64, 1024, "ReLU", "None", 1024),
    (128, 2, 64, 144, "ReLU", "None", 2048),
    (128, 8, 64, 256, "ReLU", "None", 2048),               # ring mode: 8 hidden + 2 output chunks > 6 resident stages
    (128, 2, 128, 1000, "Sigmoid", "None", 1024),
    (256, 4, 64, 272, "ReLU", "None", 2048),               # the last chunk is one half
    (256, 4, 64, 512, "ReLU", "None", 2048),
    (256, 8, 256, 1024, "ReLU", "Exponential", 1024),      # deep: every matrix streams
]


@pytest.mark.parametrize("width,n_hidden,n_in,n_out,act,out_act,B", FORWARD_SHAPES)
def test_forward_matches_oracle(torch_cuda, width, n_hidden, n_in, n_out, act, out_act, B):
    """forward / inference_mixed_precision / inference (fp32, trimmed) against orc_mlp_forward in fp32-accumulate mode."""
    torch = torch_cuda
    import tcnn_b200

    net = tcnn_b200.Network(n_in, n_out, net_cfg(width, n_hidden, act, out_act))
    out_pad = (n_out + 15) // 16 * 16
    assert net.padded_output_width == out_pad and net.n_params == width * n_in + (n_hidden - 1) * width * width + out_pad * width
    p16 = net.initial_params(seed=11).half().contiguous()
    g = torch.Generator(device="cuda").manual_seed(5)
    x = (torch.rand(B, n_in, device="cuda", generator=g) * 2 - 1).half().contiguous()
    out, hidden = net.forward(x, p16)
    out_inf = net.inference_mixed_precision(x, p16)
    out32 = net.inference(x.float(), p16)
    torch.cuda.synchronize()
    assert torch.equal(out, out_inf)
    assert out32.shape == (B, n_out) and torch.equal(out32, out[:, :n_out].float())
    n_check = min(B, 4096)
    sel = np.r_[0 : n_check // 2, B - n_check // 2 : B]
    lib, mlp = oracle_mlp(width, n_hidden, n_in, out_pad, act, out_act, net.n_params)
    hid_ref = np.zeros((n_hidden, len(sel), width), np.uint16)
    out_ref = np.zeros((len(sel), out_pad), np.uint16)
    lib.orc_mlp_forward(ctypes.byref(mlp), len(sel), ob.ACCUM_FP32, ob._p(f16(p16)), ob._p(np.ascontiguousarray(f16(x)[sel].T)), ob._p(hid_ref), ob._p(out_ref))
    o_dev, o_ref = ob.half_bits_to_float(f16(out)[sel]), ob.half_bits_to_float(out_ref)
    assert np.isfinite(o_dev).all()
    assert rae(o_dev, o_ref, 99.0) < 2e-3, rae(o_dev, o_ref, 99.0)
    assert np.abs(o_dev - o_ref).max() <= 1e-2 * max(1.0, np.abs(o_ref).max())


BACKWARD_SHAPES = [
    # width, hidden, n_in, n_out, activation, output_activation, batch
    (16, 2, 16, 32, "ReLU", "None", 2048),
    (16, 2, 32, 1024, "ReLU", "None", 1024),       # dL/d(input) 32 wide; 64 K-chunks through the ring
    (32, 2, 32, 80, "Tanh", "None", 2048),         # two wgrad passes of 64, the second 16 wide
    (64, 2, 32, 128, "ReLU", "None", 2048),
    (64, 3, 64, 1000, "ReLU", "Sigmoid", 1024),    # output activation's transfer at 1008 columns
    (128, 2, 64, 144, "ReLU", "None", 2048),
    (128, 8, 64, 256, "ReLU", "None", 2048),       # ring mode
    (128, 2, 128, 1024, "ReLU", "None", 1024),
    (256, 4, 64, 272, "ReLU", "None", 2048),
    (256, 4, 64, 512, "ReLU", "None", 2048),
    (256, 6, 256, 1024, "Tanh", "None", 1024),     # deep 256-wide: four K-blocks per half
]


def check_backward(torch, width, n_hidden, n_in, n_out, act, out_act, B, exact_grads=True):
    import tcnn_b200

    net = tcnn_b200.Network(n_in, n_out, net_cfg(width, n_hidden, act, out_act))
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
    # the oracle's backward starts after the output activation: hand it dL/dy through the same transfer
    dy_eff = dy
    if out_act != "None":
        yo = out.float()
        dy_eff = (dy.float() * {"Sigmoid": yo * (1 - yo)}[out_act]).half()
    lib, mlp = oracle_mlp(width, n_hidden, n_in, out_pad, act, "None", net.n_params)
    n_check = min(B, 2048)
    sel = np.r_[0 : n_check // 2, B - n_check // 2 : B]
    dW_sel = np.zeros(net.n_params, np.float64)
    dx_ref = np.zeros((n_in, len(sel)), np.uint16)
    lib.orc_mlp_backward(ctypes.byref(mlp), len(sel), ob.ACCUM_FP32, ob._p(f16(p16)), ob._p(np.ascontiguousarray(f16(x)[sel].T)), ob._p(np.ascontiguousarray(f16(hidden)[:, sel])),
                         ob._p(np.ascontiguousarray(f16(dy_eff)[sel])), ob._p(dW_sel), ob._p(dx_ref))
    a, b = ob.half_bits_to_float(f16(dx)[sel]), ob.half_bits_to_float(dx_ref.T)
    assert rae(a, b, 99.0) < 2e-3 or (act != "ReLU" and rae(a, b, 99.0) < 5e-3), rae(a, b, 99.0)
    if exact_grads:
        dW = np.zeros(net.n_params, np.float64)
        lib.orc_mlp_backward(ctypes.byref(mlp), B, ob.ACCUM_FP32, ob._p(f16(p16)), ob._p(np.ascontiguousarray(f16(x).T)), ob._p(np.ascontiguousarray(f16(hidden))),
                             ob._p(f16(dy_eff)), ob._p(dW), None)
        got = dp.float().cpu().numpy()
        want = dW.astype(np.float16).astype(np.float32)
        assert rae(got, want, 99.9) < 3e-3, rae(got, want, 99.9)
        assert np.abs(got - want).max() <= 2e-2 * np.abs(want).max()
        # the output matrix alone, and its last chunk / pass with the padding rows on its own
        n_out_params, n_tail = out_pad * width, (out_pad - (out_pad - 1) // width * width) * width
        assert rae(got[-n_out_params:], want[-n_out_params:], 99.9) < 3e-3
        assert rae(got[-n_tail:], want[-n_tail:], 99.9) < 3e-3
        assert np.abs(got[-n_tail:] - want[-n_tail:]).max() <= 2e-2 * max(np.abs(want[-n_tail:]).max(), 1e-30)
    return net, x, dy, p16, dp


@pytest.mark.parametrize("width,n_hidden,n_in,n_out,act,out_act,B", BACKWARD_SHAPES)
def test_backward_matches_oracle(torch_cuda, width, n_hidden, n_in, n_out, act, out_act, B):
    """dL/d(input) and the weight gradients (fp16 of the fp32 sums) against orc_mlp_backward with exact sums."""
    check_backward(torch_cuda, width, n_hidden, n_in, n_out, act, out_act, B)


@pytest.mark.parametrize("width,n_out", [(64, 512), (128, 1024), (256, 768)])
def test_weight_gradients_are_batch_linear(torch_cuda, width, n_out):
    """At 2^16 samples every CTA sums several tiles per pass; the gradients of two halves of the batch add up to the whole."""
    torch = torch_cuda
    B = 1 << 16
    net, x, dy, p16, dp = check_backward(torch, width, 2, 32, n_out, "ReLU", "None", B, exact_grads=False)
    h = B // 2
    parts = []
    for lo, hi in ((0, h), (h, B)):
        o2, hid2 = net.forward(x[lo:hi].contiguous(), p16)
        parts.append(net.backward(x[lo:hi].contiguous(), o2, hid2, dy[lo:hi].contiguous(), p16, want_input_grad=False)[1].float())
    total = (parts[0] + parts[1]).cpu().numpy()
    assert rae(dp.float().cpu().numpy(), total, 99.0) < 2e-3


@pytest.mark.parametrize("width,n_hidden,n_in,n_out,act,B", [(64, 2, 32, 128, po.SINE, 2048), (128, 3, 64, 400, po.SILU, 2048), (256, 3, 64, 384, po.SINE, 2048),
                                                            (32, 2, 32, 512, po.SILU, 1024)])
def test_preact_network_matches_oracle(torch_cuda, width, n_hidden, n_in, n_out, act, B):
    """Sine / SiLU with wide outputs: every check of test_gpu_preact.test_network_matches_oracle."""
    preact_network_check(torch_cuda, width, n_hidden, n_in, n_out, act, B)


def make_batch(n_in, n_out, B, seed=1337):
    rng = ob.default_rng(seed)
    x = ob.generate_random_uniform(rng, B * n_in).reshape(B, n_in)
    return x, ob.make_targets(x, n_out)


TRAINER_CASE = "wide_hash3d_w64"  # HashGrid (T = 2^10) + FullyFusedMLP 64 x 2 -> 128, L2 (tests/golden/make_golden_wide_out.sh)
TRAINER_CFG = json.load(open(os.path.join(GOLDEN, "configs", TRAINER_CASE + ".json")))


def load_golden(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    d = {k: z[k] for k in z.files if k != "meta"}
    d["meta"] = json.loads(bytes(z["meta"]).decode())
    return d


def test_trainer_general_path(torch_cuda):
    """HashGrid + FullyFusedMLP 64 x 2 with 128 outputs takes the general path: the step's loss and gradients against
    orc_training_step, ten steps against the oracle's trajectory; data_pdf and external dL/dy through training_step."""
    torch = torch_cuda
    import tcnn_b200

    n_in, n_out, B = 3, 128, 2048
    model = tcnn_b200.create_from_config(n_in, n_out, TRAINER_CFG)
    assert model.network.padded_output_width() == 128
    orc = ob.OracleModel(n_in, n_out, TRAINER_CFG, scales=model.grid_levels()["scales"])
    assert model.n_params == orc.n_params
    assert np.array_equal(model.trainer.params_full_precision().cpu().numpy(), orc.params_fp32)
    x, y = make_batch(n_in, n_out, B)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()

    # the general path: the same launches as the network with 16 outputs forced onto it (the wide kernels add none)
    narrow = tcnn_b200.create_from_config(n_in, 16, TRAINER_CFG)
    narrow.debug_set("general", 1)
    launches = []
    for m, yy in ((narrow, yd[:, :16].contiguous()), (model, yd)):
        m.trainer.training_step(xd, yy, run_optimizer=False)
        torch.cuda.synchronize()
        before = tcnn_b200.kernel_launch_count()
        m.trainer.training_step(xd, yy, run_optimizer=False)
        torch.cuda.synchronize()
        launches.append(tcnn_b200.kernel_launch_count() - before)
    assert launches[0] == launches[1] and launches[1] > 1, launches

    model.trainer.training_step(xd, yd, run_optimizer=False)
    loss_dev = model.trainer.loss()
    grads = model.trainer.param_gradients().float().cpu().numpy()
    loss_ref = orc.training_step(x, y, run_optimizer=False)
    gref = ob.half_bits_to_float(orc.grads_fp16)
    assert abs(loss_dev - loss_ref) <= 1e-3 * abs(loss_ref)
    n_mlp = orc.n_mlp
    assert rae(grads[:n_mlp], gref[:n_mlp], 99.9) < 1.2e-2
    assert rae(grads[n_mlp:], gref[n_mlp:], 99.9) < 1.2e-2
    assert rae(model.network.inference(xd).cpu().numpy(), orc.inference(x), 99.0) < 1e-2

    # a uniform pdf of 1/2 doubles the loss and every gradient (doubling, unlike halving, loses nothing to fp16 subnormals)
    pdf = torch.full((B, n_out), 0.5, device="cuda")
    model.trainer.training_step(xd, yd, run_optimizer=False, data_pdf=pdf)
    g_pdf = model.trainer.param_gradients().float().cpu().numpy()
    assert abs(model.trainer.loss() - 2 * loss_dev) <= 1e-3 * abs(loss_dev)
    assert rae(g_pdf, 2 * grads, 99.0) < 1e-2
    # external dL/dy: the gradients are linear in it
    gen = torch.Generator(device="cuda").manual_seed(3)
    ext = ((torch.rand(B, n_out, device="cuda", generator=gen) * 2 - 1) * 64).half()
    model.trainer.training_step(xd, None, run_optimizer=False, external_dL_dy=ext)
    g1 = model.trainer.param_gradients().float().cpu().numpy()
    model.trainer.training_step(xd, None, run_optimizer=False, external_dL_dy=(ext.float() * 2).half())
    g2 = model.trainer.param_gradients().float().cpu().numpy()
    assert np.abs(g1[:n_mlp]).max() > 0 and np.isfinite(g1).all()
    assert rae(g2[:n_mlp], 2 * g1[:n_mlp], 99.0) < 1e-2

    dev_losses, ref_losses = [], []
    for _ in range(10):
        model.trainer.training_step(xd, yd)
        dev_losses.append(model.trainer.loss())
        ref_losses.append(orc.training_step(x, y))
    assert dev_losses[-1] < dev_losses[0]
    for a, b in zip(dev_losses, ref_losses):
        assert abs(a - b) <= 3e-2 * abs(b) + 1e-6, (dev_losses, ref_losses)


NET_FIXTURES = ["wide_net_w64_h2_relu", "wide_net_w64_h2_sigmoid", "wide_net_w16_h2_relu", "wide_net_w256_h4_relu", "wide_net_w256_h3_sine"]


@pytest.mark.parametrize("name", NET_FIXTURES)
def test_network_against_reference_golden_vectors(torch_cuda, name):
    """`ref_harness mlpdump` of the unmodified reference: its initial parameters from this library's initialisation (the trainer's
    pcg32 stream, seed 1337) bit for bit, and its weights and inputs -> its outputs within tests/test_common.h:177 (RAE < 1e-2 @ p99)."""
    torch = torch_cuda
    import tcnn_b200

    g = load_golden(name)
    m = g["meta"]
    net = tcnn_b200.Network(m["n_in"], m["n_out"], {"otype": m["otype"], "n_neurons": m["width"], "n_hidden_layers": m["n_hidden_layers"], "activation": m["activation"],
                                                     "output_activation": m["output_activation"]})
    assert net.n_params == m["n_params"] and net.padded_output_width == m["padded_output_width"]
    B = m["batch"]
    p16 = torch.from_numpy(g["params_f16"].view(np.float16).copy()).cuda()
    x = torch.from_numpy(g["x_f16"].view(np.float16).reshape(B, m["n_in"]).copy()).cuda()
    out = net.inference_mixed_precision(x, p16)
    torch.cuda.synchronize()
    ref = g["output_f16"].view(np.float16).reshape(B, m["padded_output_width"]).astype(np.float32)
    assert rae(out.float().cpu().numpy(), ref, 99.0) < 1e-2


def test_trainer_against_reference_golden_vectors(torch_cuda):
    """`ref_harness dump` of HashGrid + FullyFusedMLP 64 x 2 -> 128: initial parameters bit for bit, inference, the step-0 loss and the
    ten-step trajectory within 3 %. The step-0 weight gradients are held to the fp32 oracle (test_trainer_general_path): the
    reference's fp16-accumulating split-K GEMMs put its own ones 5-14 % from the exact sums here (tests/test_oracle_wide_out.py)."""
    torch = torch_cuda
    import tcnn_b200

    n_in, n_out, B = 3, 128, 512
    g = load_golden(TRAINER_CASE)
    model = tcnn_b200.create_from_config(n_in, n_out, TRAINER_CFG)
    assert np.array_equal(model.trainer.params_full_precision().cpu().numpy().view(np.uint32), g["params_init_f32"].view(np.uint32))
    xd = torch.from_numpy(g["x_f32"].reshape(B, n_in).copy()).cuda()
    yd = torch.from_numpy(g["y_f32"].reshape(B, n_out).copy()).cuda()
    # a fresh grid in front: the outputs are fp16 subnormals (~1e-5), where the reference's bar is absolute (values_agree)
    out, ref = model.network.inference(xd).cpu().numpy().astype(np.float64), g["inference_f32"].reshape(B, n_out).astype(np.float64)
    d, q = np.abs(out - ref), 2.0**-24
    assert po.values_agree(out, ref, 1e-2) or (np.abs(ref).max() < 2.0**-14 and d.mean() <= 2.5 * q and d.max() <= 16 * q), (rae(out, ref, 99.0), d.max() / q)
    model.trainer.training_step(xd, yd, run_optimizer=False)
    losses = [model.trainer.loss()]
    for _ in range(g["meta"]["n_steps"]):
        model.trainer.training_step(xd, yd)
        losses.append(model.trainer.loss())
    assert abs(losses[0] - g["meta"]["losses"][0]) <= 1e-3 * g["meta"]["losses"][0]
    for mine, theirs in zip(losses, g["meta"]["losses"]):
        assert abs(mine - theirs) <= 3e-2 * abs(theirs), (losses, g["meta"]["losses"])


def test_network_with_hashgrid_encoding(torch_cuda):
    """torch_modules.NetworkWithInputEncoding(3, 128, HashGrid, FullyFusedMLP 64 x 2) with the positions requiring grad: outputs,
    parameter gradients and dL/d(position) are those of the native module (whose dL/d(position) test_module_tier_grid_wide_output holds
    to the oracle) for the loss-scaled dL/dy, divided by the loss scale (the bars of test_gpu_cutlass256.test_torch_modules)."""
    torch = torch_cuda
    import tcnn_b200.torch_modules as tm

    n_in, n_out, B = 3, 128, 2048
    mod = tm.NetworkWithInputEncoding(n_in, n_out, TRAINER_CFG["encoding"], TRAINER_CFG["network"])
    g = torch.Generator(device="cuda").manual_seed(6)
    xs, _ = make_batch(n_in, n_out, B)
    xg = torch.from_numpy(xs).cuda().requires_grad_(True)
    dy = (torch.rand(B, n_out, device="cuda", generator=g) * 2 - 1).half()
    y = mod(xg)
    y.backward(dy)
    p16 = mod.params.detach().half().contiguous()
    x_dev = torch.from_numpy(xs).cuda()
    out_native = mod.native_tcnn_module.fwd(x_dev, p16)
    dp, dx = mod.native_tcnn_module.bwd(x_dev, p16, (dy.float() * mod.loss_scale).half(), want_input_grad=True)
    torch.cuda.synchronize()
    if isinstance(out_native, tuple):
        out_native = out_native[0]
    assert torch.equal(y.detach(), out_native[:, :n_out].to(y.dtype))
    n_mlp = 64 * 16 + 64 * 64 + 128 * 64
    a = mod.params.grad.cpu().numpy()
    b = (dp.float() / mod.loss_scale).half().float().cpu().numpy()
    assert rae(a[:n_mlp], b[:n_mlp], 99.9) < 2e-3 and rae(a[n_mlp:], b[n_mlp:], 99.9) < 5e-3
    assert rae(xg.grad.cpu().numpy(), (dx / mod.loss_scale).cpu().numpy(), 99.9) < 5e-3


def torch_mlp(params, x, n_in_pad, width, n_hidden, n_out):
    """float32 autograd restatement of an Identity-encoded ReLU network with the module's fp16 weights."""
    import torch

    h = torch.cat([x, torch.ones(x.shape[0], n_in_pad - x.shape[1], device=x.device)], 1).half().float()
    p = params.half().float()
    off = 0
    for l, (r, c) in enumerate(po.matrix_shapes(width, n_in_pad, n_hidden, (n_out + 15) // 16 * 16)):
        h = h @ p[off : off + r * c].view(r, c).t()
        off += r * c
        if l < n_hidden:
            h = torch.relu(h)
    return h[:, :n_out]


@pytest.mark.parametrize("width,n_hidden,n_in,n_out", [(256, 4, 64, 512), (64, 2, 3, 128)])
def test_torch_modules(torch_cuda, width, n_hidden, n_in, n_out):
    """torch_modules.Network and NetworkWithInputEncoding(Identity): outputs, parameter and input gradients against a float32 torch
    restatement with the same fp16 weights (the loss scale rounds dL/dy to fp16, as test_gpu_cutlass256.test_torch_modules notes)."""
    torch = torch_cuda
    import tcnn_b200.torch_modules as tm

    B = 4096
    g = torch.Generator(device="cuda").manual_seed(2)
    x = (torch.rand(B, n_in, device="cuda", generator=g) * 2 - 1).requires_grad_(True)
    target = torch.rand(B, n_out, device="cuda", generator=g)
    in_pad = (n_in + 15) // 16 * 16

    net = tm.Network(n_in, n_out, net_cfg(width, n_hidden))
    # the loss is summed over the outputs, so that dL/dy x the loss scale stays out of fp16's subnormal range at 512 outputs
    y = net(x)
    assert y.shape == (B, n_out)
    ((y.float() - target) ** 2).sum(1).mean().backward()
    p_ref = net.params.detach().clone().requires_grad_(True)
    x_ref = x.detach().clone().requires_grad_(True)
    y_ref = torch_mlp(p_ref, x_ref, in_pad, width, n_hidden, n_out)
    ((y_ref - target) ** 2).sum(1).mean().backward()
    assert rae(y.float().detach().cpu().numpy(), y_ref.detach().cpu().numpy(), 99.0) < 5e-3
    assert rae(net.params.grad.cpu().numpy(), p_ref.grad.cpu().numpy(), 99.0) < 2e-2
    assert rae(x.grad.cpu().numpy(), x_ref.grad.cpu().numpy(), 99.0) < 2e-2

    model = tm.NetworkWithInputEncoding(n_in, n_out, {"otype": "Identity"}, net_cfg(width, n_hidden))
    ((model(x.detach()).float() - target) ** 2).sum(1).mean().backward()
    p2 = model.params.detach().clone().requires_grad_(True)
    ((torch_mlp(p2, x.detach(), in_pad, width, n_hidden, n_out) - target) ** 2).sum(1).mean().backward()
    assert rae(model.params.grad.cpu().numpy(), p2.grad.cpu().numpy(), 99.0) < 2e-2


def test_module_tier_grid_wide_output(torch_cuda):
    """The module tier (tcnn::cpp::Module) with HashGrid + FullyFusedMLP 64 x 2 and 128 outputs: parameter gradients and
    dL/d(position) against the oracle's backward pass from the same loss-scaled dL/d(output)."""
    torch = torch_cuda
    import tcnn_b200

    n_in, n_out, Bg = 3, 128, 2048
    cfg = TRAINER_CFG
    g = torch.Generator(device="cuda").manual_seed(4)
    xs, _ = make_batch(n_in, n_out, Bg)
    native = tcnn_b200.Module(n_in, n_out, cfg["encoding"], cfg["network"])
    p16 = native.initial_params(seed=1337).half().contiguous()
    dy = ((torch.rand(Bg, n_out, device="cuda", generator=g) * 2 - 1) * 0.1).half()
    scaled = (dy.float() * 128.0).half().contiguous()
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


def test_output_width_limit(torch_cuda):
    import tcnn_b200

    for cfg in (net_cfg(64, 2), net_cfg(256, 2)):
        with pytest.raises(RuntimeError, match="padded network output width must be at most 1024"):
            tcnn_b200.Network(32, 1025, cfg)
        net = tcnn_b200.Network(32, 1024, cfg)
        assert net.padded_output_width == 1024
