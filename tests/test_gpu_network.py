"""GPU parity of the stand-alone FullyFusedMLP kernel (csrc/mlp_fused.cu: TMA-staged weights, activations threaded through
registers as the A operand of wgmma) against the CPU oracle's restatement of kernel_mlp_fused (oracle_cpu.cpp orc_mlp_forward,
fully_fused_mlp.cu:499-557), through the C ABI's network tier (tcnnb_network_*)."""
import ctypes

import numpy as np
import pytest

import oracle_binding as ob
from golden_util import rae

pytestmark = pytest.mark.gpu


def oracle_forward(width, n_hidden, in_w, out_pad, act, out_act, weights16, x16):
    """x16: [B][in_w] fp16 bits -> (hidden [n_hidden][B][width], out [B][out_pad]) fp16 bits, fp32 accumulation."""
    lib = ob.load()
    mlp = ob.Mlp(in_w, width, n_hidden, out_pad, 0, ob.ACT[act.lower()], ob.ACT[out_act.lower()], 0)
    assert lib.orc_mlp_setup(ctypes.byref(mlp)) == 0
    assert mlp.n_params == weights16.size and mlp.padded_out_width == out_pad
    B = x16.shape[0]
    hidden = np.zeros((n_hidden, B, width), np.uint16)
    out = np.zeros((B, out_pad), np.uint16)
    lib.orc_mlp_forward(ctypes.byref(mlp), B, ob.ACCUM_FP32, ob._p(weights16), ob._p(np.ascontiguousarray(x16.T)), ob._p(hidden), ob._p(out))
    return hidden, out


def f16(t):
    return t.cpu().numpy().view(np.uint16)


SHAPES = [
    # width, hidden, n_in, n_out, activation, output_activation, batch
    (128, 4, 128, 128, "ReLU", "None", 1024),            # BASELINE configs[2]/[4] shape: 5 resident 32 KB matrices
    (128, 4, 128, 128, "ReLU", "None", 148 * 128 * 5 + 256),  # several tiles per slot, uneven slots
    (128, 8, 128, 128, "ReLU", "None", 148 * 128 * 2 + 512),  # 9 matrices > 7 stages: weights stream through the ring
    (128, 2, 64, 16, "ReLU", "None", 2048),
    (128, 3, 32, 48, "Tanh", "Sigmoid", 1024),
    (64, 2, 64, 64, "ReLU", "None", 148 * 128 * 9),      # 4 slots, 2+ rounds
    (64, 4, 32, 16, "ReLU", "None", 4096),
    (64, 8, 64, 64, "LeakyReLU", "None", 2048),
    (32, 3, 32, 32, "ReLU", "None", 2048),
    (32, 2, 16, 16, "Softplus", "Exponential", 1024),
    (16, 2, 16, 16, "ReLU", "None", 2048),
    (16, 4, 64, 16, "Squareplus", "None", 1024),
]


@pytest.mark.parametrize("width,n_hidden,n_in,n_out,act,out_act,B", SHAPES)
def test_network_forward_matches_oracle(torch_cuda, width, n_hidden, n_in, n_out, act, out_act, B):
    torch = torch_cuda
    import tcnn_b200

    cfg = {"otype": "FullyFusedMLP", "n_neurons": width, "n_hidden_layers": n_hidden, "activation": act, "output_activation": out_act}
    net = tcnn_b200.Network(n_in, n_out, cfg)
    out_pad = (n_out + 15) // 16 * 16
    assert net.n_params == width * n_in + (n_hidden - 1) * width * width + out_pad * width
    assert net.padded_output_width == out_pad and net.input_width == n_in
    p32 = net.initial_params(seed=11)
    # xavier bounds per matrix (fully_fused_mlp.cu:868-892)
    w0 = p32[: width * n_in]
    assert float(w0.abs().max()) <= np.sqrt(6.0 / (width + n_in)) + 1e-6 and float(w0.abs().max()) > 0.5 * np.sqrt(6.0 / (width + n_in))
    p16 = p32.to(torch.float16).contiguous()
    g = torch.Generator(device="cuda").manual_seed(5)
    x = (torch.rand(B, n_in, device="cuda", generator=g) * 2 - 1).to(torch.float16).contiguous()
    out, hidden = net.forward(x, p16)
    out_inf = net.inference_mixed_precision(x, p16)
    torch.cuda.synchronize()
    assert torch.equal(out, out_inf)
    n_check = min(B, 4096)  # the oracle is a scalar CPU port: head and tail of the batch
    sel = np.r_[0 : n_check // 2, B - n_check // 2 : B]
    hid_ref, out_ref = oracle_forward(width, n_hidden, n_in, out_pad, act, out_act, f16(p16), f16(x)[sel])
    hid_dev = f16(hidden)[:, sel]
    a, b = ob.half_bits_to_float(hid_dev), ob.half_bits_to_float(hid_ref)
    exact = act in ("ReLU", "LeakyReLU", "None")
    # fp32-accumulated dot products rounded once to fp16: the first layer is at most 1 ulp apart (summation order); deeper layers
    # inherit the rare 1-ulp flips of their inputs
    assert np.abs(a[0] - b[0]).max() <= 2.0 ** -9 * max(1.0, np.abs(b[0]).max())
    assert (hid_dev[0] != hid_ref[0]).mean() < (0.02 if exact else 0.2)
    assert rae(a, b) < (1e-3 if exact else 3e-3)
    o_dev, o_ref = ob.half_bits_to_float(f16(out)[sel]), ob.half_bits_to_float(out_ref)
    assert np.isfinite(o_dev).all()
    assert rae(o_dev, o_ref, 99.0) < 2e-3
    assert np.abs(o_dev - o_ref).max() <= 1e-2 * max(1.0, np.abs(o_ref).max())
    # every row of a large batch was written (no tile skipped): compare a cheap statistic against a torch fp32 evaluation
    if B > 4096:
        h = x.float()
        off = 0
        dims = [(width, n_in)] + [(width, width)] * (n_hidden - 1) + [(out_pad, width)]
        for i, (r, c) in enumerate(dims):
            wmat = p16[off : off + r * c].view(r, c).float()
            off += r * c
            h = h @ wmat.t()
            if i < n_hidden:
                h = torch.relu(h).half().float() if act == "ReLU" else torch.nn.functional.leaky_relu(h, 0.01).half().float()
        assert rae(out.float().cpu().numpy(), h.cpu().numpy(), 99.0) < 5e-3


def test_network_identity_inference_matches_oracle(torch_cuda):
    """cpp::create_network semantics (src/cpp_api.cu:160-162): fp32 inputs through the Identity encoding -- features beyond
    n_input_dims are ONE (identity.h:62-66) -- fp32 outputs trimmed to n_output_dims. BASELINE configs[0] shape (64 x 2, 3 -> 3)."""
    torch = torch_cuda
    import tcnn_b200

    for otype in ("CutlassMLP", "FullyFusedMLP"):
        net = tcnn_b200.Network(3, 3, {"otype": otype, "n_neurons": 64, "n_hidden_layers": 2, "activation": "ReLU", "output_activation": "None"})
        assert net.input_width == 16 and net.padded_output_width == 16 and net.n_params == 64 * 16 + 64 * 64 + 16 * 64
        p16 = net.initial_params(seed=3).to(torch.float16).contiguous()
        B = 65536
        x = torch.rand(B, 3, device="cuda")
        out = net.inference(x, p16)
        torch.cuda.synchronize()
        enc = np.ones((B, 16), np.float16)
        enc[:, :3] = x.cpu().numpy().astype(np.float16)
        _, out_ref = oracle_forward(64, 2, 16, 16, "ReLU", "None", f16(p16), enc.view(np.uint16)[:4096])
        a = out.cpu().numpy()[:4096]
        b = ob.half_bits_to_float(out_ref)[:, :3]
        assert a.shape == (4096, 3) and rae(a, b, 99.0) < 2e-3
    with pytest.raises(tcnn_b200.TcnnError, match="multiple of 16"):
        net.inference_mixed_precision(x.half(), p16)
    with pytest.raises(tcnn_b200.TcnnError, match="16, 32, 64, and 128"):
        tcnn_b200.Network(16, 16, {"otype": "FullyFusedMLP", "n_neurons": 48})
    with pytest.raises(tcnn_b200.TcnnError, match="multiple of 256"):
        net.inference(x[:100], p16)


import glob  # noqa: E402
import json  # noqa: E402
import os  # noqa: E402

from golden_util import GOLDEN  # noqa: E402

MLP_GOLDEN = sorted(os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(GOLDEN, "mlp_*.npz")) if not p.endswith("_jit.npz"))


@pytest.mark.parametrize("name", MLP_GOLDEN)
def test_network_against_reference_golden_vectors(torch_cuda, name):
    """tests/golden/mlp_*.npz: weights, fp16 inputs and fp16 outputs of the UNMODIFIED reference's Network<__half>::inference_mixed_precision
    (`ref_harness mlpdump`: create_network<T>(json), FullyFusedMLP 128 x 4 / 64 x 2 / 32 x 3 Tanh->Sigmoid, CutlassMLP 64 x 2) on the GPU.
    Same weights, same inputs -> outputs within the reference's own forward bar (tests/test_common.h:177: RAE < 1e-2 @ p99); the
    difference is the accumulator: fp16 inside HMMA there, fp32 in registers (wgmma) here."""
    torch = torch_cuda
    import tcnn_b200

    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(bytes(z["meta"]).decode())
    cfg = {"otype": meta["otype"], "n_neurons": meta["width"], "n_hidden_layers": meta["n_hidden_layers"], "activation": meta["activation"], "output_activation": meta["output_activation"]}
    net = tcnn_b200.Network(meta["n_in"], meta["n_out"], cfg)
    assert net.n_params == meta["n_params"] and net.padded_output_width == meta["padded_output_width"]
    B = meta["batch"]
    p16 = torch.from_numpy(z["params_f16"].view(np.float16).copy()).cuda()
    x = torch.from_numpy(z["x_f16"].view(np.float16).reshape(B, meta["n_in"]).copy()).cuda()
    out = net.inference_mixed_precision(x, p16)
    torch.cuda.synchronize()
    a = out.float().cpu().numpy()
    b = ob.half_bits_to_float(z["output_f16"]).reshape(B, meta["padded_output_width"])
    assert rae(a, b, 99.0) < 1e-2
    assert np.abs(a - b).max() <= 2e-2 * max(1.0, np.abs(b).max())
    jit = os.path.join(GOLDEN, name + "_jit.npz")
    if os.path.exists(jit):  # the reference's JIT-fused mode on the same weights and inputs
        bj = ob.half_bits_to_float(np.load(jit)["output_f16"]).reshape(B, meta["padded_output_width"])
        assert rae(a, bj, 99.0) < 1e-2
    # and the oracle, which this kernel must match to fp16 rounding
    _, o_ref = oracle_forward(meta["width"], meta["n_hidden_layers"], meta["n_in"], meta["padded_output_width"], meta["activation"], meta["output_activation"], z["params_f16"],
                              z["x_f16"].reshape(B, meta["n_in"]))
    assert rae(a, ob.half_bits_to_float(o_ref), 99.0) < 2e-3
