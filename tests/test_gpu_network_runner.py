"""What the stand-alone network kernels (mlp_fused.cu / mlp_wgrad.cu) do when a tier drives them: the network tier (tcnnb_network_*),
the general path's trainer step and inference, and the module tier on the general path. Pinned here: how many kernels each call
launches, that the network tier's Identity encoding is exactly the fp16 rows its fp16 calls take, and which error each bad input
raises, in which order."""
import ctypes

import numpy as np
import pytest

from golden_util import rae

pytestmark = pytest.mark.gpu

B = 1024
NET = {"otype": "FullyFusedMLP", "n_neurons": 64, "n_hidden_layers": 2, "activation": "ReLU", "output_activation": "None"}
SINE = {"otype": "CutlassMLP", "n_neurons": 64, "n_hidden_layers": 2, "activation": "Sine", "output_activation": "None"}
GRID = {"otype": "HashGrid", "n_levels": 8, "n_features_per_level": 2, "log2_hashmap_size": 14, "base_resolution": 16, "per_level_scale": 1.5}
NET128 = dict(NET, n_neurons=128)
TRAIN = {"loss": {"otype": "L2"}, "optimizer": {"otype": "Adam", "learning_rate": 1e-3}, "encoding": GRID, "network": NET128}


def launches(fn):
    import tcnn_b200

    before = tcnn_b200.kernel_launch_count()
    fn()
    return tcnn_b200.kernel_launch_count() - before


def identity_rows(torch, x, width):
    """The Identity encoding of fp32 rows: x as fp16, the padding columns ONE (encodings/identity.h:46-67)."""
    enc = torch.ones(x.shape[0], width, dtype=torch.float16, device=x.device)
    enc[:, : x.shape[1]] = x.half()
    return enc.contiguous()


@pytest.fixture(scope="module")
def calls(torch_cuda):
    """name -> a call of one entry point on a 64 x 2 network (3 -> 3 for fp32 inputs, 16 -> 3 for fp16 inputs), B = 1024."""
    torch = torch_cuda
    import tcnn_b200

    g = torch.Generator(device="cuda").manual_seed(1)
    x32 = torch.rand(B, 3, device="cuda", generator=g)
    dy = ((torch.rand(B, 16, device="cuda", generator=g) * 2 - 1) * 0.25).half().contiguous()
    nets = {}
    for name, n_in, cfg in [("net3", 3, NET), ("net16", 16, NET), ("sig16", 16, dict(NET, output_activation="Sigmoid")), ("sine16", 16, SINE)]:
        net = tcnn_b200.Network(n_in, 3, cfg)
        nets[name] = (net, net.initial_params(seed=2).half().contiguous())
    x16 = identity_rows(torch, x32, 16)
    fwd = {k: nets[k][0].forward(x16, nets[k][1]) for k in ("net16", "sig16", "sine16")}

    def backward(k, **kw):
        net, p = nets[k]
        out, hidden = fwd[k]
        return lambda: net.backward(x16, out, hidden, dy, p, **kw)

    net3, p3 = nets["net3"]
    net16, p16 = nets["net16"]
    sine, psine = nets["sine16"]
    model = tcnn_b200.create_from_config(3, 3, TRAIN)
    y = torch.rand(B, 3, device="cuda", generator=g)
    module = tcnn_b200.Module(3, 3, GRID, NET128)
    pm = module.initial_params(seed=4).half().contiguous()
    module_sig = tcnn_b200.Module(3, 3, GRID, dict(NET128, output_activation="Sigmoid"))
    pm_sig = module_sig.initial_params(seed=4).half().contiguous()
    return {
        "network.inference": lambda: net3.inference(x32, p3),
        "network.module_inference": lambda: net3.module_inference(x32, p3),
        "network.inference_mixed_precision": lambda: net16.inference_mixed_precision(x16, p16),
        "network.forward": lambda: net16.forward(x16, p16),
        "network.backward": backward("net16"),
        "network.backward.input_only": backward("net16", want_param_grad=False),
        "network.backward.params_only": backward("net16", want_input_grad=False),
        "network.backward.output_activation": backward("sig16"),
        "network.module_backward": lambda: net3.module_backward(x32, dy, p3),
        "network.module_backward.params_only": lambda: net3.module_backward(x32, dy, p3, want_input_grad=False),
        "network.module_backward.input_only": lambda: net3.module_backward(x32, dy, p3, want_param_grad=False),
        "network.sine.forward": lambda: sine.forward(x16, psine),
        "network.sine.backward": backward("sine16"),
        "general.training_step": lambda: model.trainer.training_step(x32, y),
        "general.inference": lambda: model.network.inference(x32),
        "general.module.fwd": lambda: module.fwd(x32, pm),
        "general.module.bwd": lambda: module.bwd(x32, pm, dy, want_input_grad=True),
        "general.module.bwd.output_activation": lambda: module_sig.bwd(x32, pm_sig, dy, want_input_grad=True),
    }


# Kernel launches per call. Network tier: one forward kernel; backward = [output activation] + dgrad chain + weight gradients +
# fp32 -> fp16 finalize; module_backward adds the Identity encoding, its forward pass and dL/d(input). General path: grid forward,
# network forward, loss, dgrad, weight gradients, table scatter, Adam / finalize, grid input gradient.
LAUNCHES = {
    "network.inference": 1,
    "network.module_inference": 1,
    "network.inference_mixed_precision": 1,
    "network.forward": 1,
    "network.backward": 3,
    "network.backward.input_only": 1,
    "network.backward.params_only": 3,
    "network.backward.output_activation": 4,
    "network.module_backward": 6,
    "network.module_backward.params_only": 5,
    "network.module_backward.input_only": 4,
    "network.sine.forward": 1,
    "network.sine.backward": 3,
    "general.training_step": 7,
    "general.inference": 2,
    "general.module.fwd": 2,
    "general.module.bwd": 7,
    "general.module.bwd.output_activation": 8,
}


@pytest.mark.parametrize("name", sorted(LAUNCHES))
def test_launch_count_per_call(calls, name):
    calls[name]()  # first call: scratch allocations
    assert launches(calls[name]) == LAUNCHES[name]


@pytest.mark.parametrize("out_act", ["None", "Sigmoid"])
def test_module_backward_is_backward_on_identity_rows(torch_cuda, out_act):
    """module_backward (fp32 inputs) == backward on the Identity-encoded fp16 rows of the same inputs: dL/d(input) bit for bit (the
    fp32 cast of the first n_input_dims columns), dL/d(params) up to the order of the fp32 atomic sums."""
    torch = torch_cuda
    import tcnn_b200

    cfg = dict(NET, output_activation=out_act)
    net3, net16 = tcnn_b200.Network(3, 3, cfg), tcnn_b200.Network(16, 3, cfg)
    assert net3.n_params == net16.n_params
    p = net3.initial_params(seed=9).half().contiguous()
    n = 1 << 14
    g = torch.Generator(device="cuda").manual_seed(8)
    x32 = torch.rand(n, 3, device="cuda", generator=g) * 2 - 1
    dy = ((torch.rand(n, 16, device="cuda", generator=g) * 2 - 1) * 0.25).half().contiguous()
    dx, dp = net3.module_backward(x32, dy, p)
    x16 = identity_rows(torch, x32, 16)
    out, hidden = net16.forward(x16, p)
    dx16, dp16 = net16.backward(x16, out, hidden, dy, p)
    dx_again, dp_again = net3.module_backward(x32, dy, p)  # the weight-gradient accumulator starts from zero every call
    torch.cuda.synchronize()
    assert dx.abs().max() > 0
    assert torch.equal(dx.view(torch.int32), dx16[:, :3].float().contiguous().view(torch.int32))
    assert torch.equal(dx_again, dx)
    assert rae(dp.float().cpu().numpy(), dp16.float().cpu().numpy()) < 1e-3
    assert rae(dp_again.float().cpu().numpy(), dp.float().cpu().numpy()) < 1e-3


def test_network_errors_and_their_order(torch_cuda):
    torch = torch_cuda
    import tcnn_b200

    lib = tcnn_b200.load()
    s = tcnn_b200._stream_handle(None)
    net3, net16, sig16 = tcnn_b200.Network(3, 3, NET), tcnn_b200.Network(16, 3, NET), tcnn_b200.Network(16, 3, dict(NET, output_activation="Sigmoid"))
    p = net16.initial_params(seed=1).half().contiguous()
    x32 = torch.rand(B, 3, device="cuda")
    x16 = torch.rand(B, 16, device="cuda").half()
    out, hidden = sig16.forward(x16, p)
    dy = torch.zeros(B, 16, dtype=torch.float16, device="cuda")
    dx32 = torch.empty(B, 3, device="cuda")
    dx16 = torch.empty(B, 16, dtype=torch.float16, device="cuda")
    dp = torch.empty(net16.n_params, dtype=torch.float16, device="cuda")
    P, P1 = p.data_ptr(), p.data_ptr() + 2  # P1: misaligned
    X32, X16, O, H, DY, DX32, DX16, DP = (t.data_ptr() for t in (x32, x16, out, hidden, dy, dx32, dx16, dp))

    def err(fn, *args):
        assert fn(*args) != 0
        return lib.tcnnb_last_error().decode()

    BATCH = "batch size 1000 must be a non-zero multiple of 256"
    NULL_P, ALIGN_P = "network: params is null.", "network: params must be 16-byte aligned."
    FP16 = "network: fp16 inputs need n_input_dims to be a multiple of 16."
    BWD_NULL = "network: backward needs the forward pass's input and hidden activations and dL_doutput."
    BWD_OUT = "network: backward through an output activation needs the forward pass's output."

    h = lambda net: net._h  # noqa: E731
    # inference / module_inference (fp32 inputs through the Identity encoding)
    for fn in (lib.tcnnb_network_inference, lib.tcnnb_network_module_inference):
        assert err(fn, h(net3), s, 1000, None, O, None) == "network: input / output is null."
        assert err(fn, h(net3), s, 1000, X32, O, None) == BATCH
        assert err(fn, h(net3), s, B, X32, O, None) == NULL_P
        assert err(fn, h(net3), s, B, X32, O, P1) == ALIGN_P
    assert err(lib.tcnnb_network_module_inference, h(net3), s, 1000, X32, O + 2, None) == "network: output must be 16-byte aligned."
    # inference_mixed_precision
    fn = lib.tcnnb_network_inference_mixed_precision
    assert err(fn, h(net3), s, 1000, None, O, None) == ("network: fp16 inputs need n_input_dims to be a multiple of 16 (got 3); use tcnnb_network_inference "
                                                         "(Identity encoding pads the input).")
    assert err(fn, h(net16), s, 1000, None, O, None) == "network: input / output is null."
    assert err(fn, h(net16), s, 1000, X16 + 2, O, None) == "network: input / output must be 16-byte aligned."
    assert err(fn, h(net16), s, 1000, X16, O, None) == BATCH
    assert err(fn, h(net16), s, B, X16, O, None) == NULL_P
    assert err(fn, h(net16), s, B, X16, O, P1) == ALIGN_P
    # forward
    fn = lib.tcnnb_network_forward
    assert err(fn, h(net3), s, 1000, None, O, H, None) == FP16
    assert err(fn, h(net16), s, 1000, None, O, H, None) == "network: input is null."
    assert err(fn, h(net16), s, 1000, X16, O, H + 2, None) == "network: input / output / hidden must be 16-byte aligned."
    assert err(fn, h(net16), s, 1000, X16, O, H, None) == BATCH
    assert err(fn, h(net16), s, B, X16, O, H, P1) == ALIGN_P
    # backward
    fn = lib.tcnnb_network_backward
    assert err(fn, h(net3), s, 1000, None, None, None, None, None, DX16, DP) == FP16
    assert err(fn, h(sig16), s, 1000, None, None, None, None, None, DX16 + 2, DP) == "network: all arrays must be 16-byte aligned."
    assert fn(h(sig16), s, 1000, None, None, None, None, None, None, None) == 0  # nothing asked for: nothing checked
    assert err(fn, h(sig16), s, 1000, None, None, None, None, None, DX16, None) == BATCH
    assert err(fn, h(sig16), s, B, None, None, None, None, None, DX16, None) == NULL_P
    assert err(fn, h(sig16), s, B, X16, None, None, DY, P1, None, DP) == ALIGN_P
    assert err(fn, h(sig16), s, B, X16, None, None, DY, P, DX16, DP) == BWD_NULL
    assert err(fn, h(sig16), s, B, X16, O, H, None, P, DX16, None) == BWD_NULL
    assert err(fn, h(sig16), s, B, X16, None, H, DY, P, None, DP) == BWD_OUT
    # module_backward
    fn = lib.tcnnb_network_module_backward
    assert fn(h(net3), s, 1000, None, None, None, None, None) == 0  # nothing asked for: nothing checked
    assert err(fn, h(net3), s, 1000, DX32, None, DP, X32, None) == "network: input / dL_doutput is null."
    assert err(fn, h(net3), s, 1000, DX32, DY, DP + 2, X32, None) == "network: dL_doutput / dL_dparams must be 16-byte aligned."
    assert err(fn, h(net3), s, 1000, DX32, DY, DP, X32, None) == BATCH
    assert err(fn, h(net3), s, B, DX32, DY, None, X32, None) == NULL_P
    assert err(fn, h(net3), s, B, None, DY, DP, X32, P1) == ALIGN_P
    # create
    for n_in, n_out in ((0, 3), (3, 0)):
        with pytest.raises(tcnn_b200.TcnnError) as e:
            tcnn_b200.Network(n_in, n_out, NET)
        assert str(e.value) == "network: n_input_dims and n_output_dims must be positive."
    with pytest.raises(tcnn_b200.TcnnError) as e:
        tcnn_b200.Network(0, 3, dict(NET, otype="Foo"))
    assert str(e.value) == "Invalid network type: Foo"
