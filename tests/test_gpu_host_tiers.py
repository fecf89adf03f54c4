"""The C-ABI tiers share one network description (csrc/network_config.h) and one encoding-plan runner (csrc/encoding_plan.cu): the
trainer and module tiers apply the network tier's width rule, the module tier's dL/d(input) goes through the plan where it is built,
and the launch counter counts every kernel a grid backward pass launches."""
import pytest

from golden_util import rae

pytestmark = pytest.mark.gpu

GRID = {"otype": "HashGrid", "n_levels": 8, "n_features_per_level": 2, "log2_hashmap_size": 14, "base_resolution": 16, "per_level_scale": 1.5}
WIDTH_MESSAGE = "only supports 16, 32, 64, and 128 neurons, but got 48"


@pytest.mark.parametrize("otype", ["CutlassMLP", "MLP"])
def test_every_tier_applies_the_network_width_rule(torch_cuda, otype):
    import tcnn_b200

    net = {"otype": otype, "n_neurons": 48, "n_hidden_layers": 2}
    with pytest.raises(tcnn_b200.TcnnError, match=WIDTH_MESSAGE):
        tcnn_b200.Network(3, 3, net)
    with pytest.raises(tcnn_b200.TcnnError, match=WIDTH_MESSAGE):
        tcnn_b200.create_from_config(3, 3, {"encoding": GRID, "network": net})
    with pytest.raises(tcnn_b200.TcnnError, match=WIDTH_MESSAGE):
        tcnn_b200.Module(3, 3, GRID, net)


def test_module_input_gradient_through_identity(torch_cuda):
    """128 neurons run on the general path, which computes dL/d(input) through the plan's Identity segment: it equals the network
    tier's Identity module. The fused kernel (64 neurons) does not hand out checked dL/d(encoded) rows for Identity: rejected."""
    torch = torch_cuda
    import tcnn_b200

    B = 1024
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.rand(B, 3, device="cuda", generator=g)
    dy = ((torch.rand(B, 16, device="cuda", generator=g) * 2 - 1) * 0.5).to(torch.float16).contiguous()

    cfg = {"otype": "FullyFusedMLP", "n_neurons": 128, "n_hidden_layers": 2, "activation": "ReLU", "output_activation": "None"}
    module = tcnn_b200.Module(3, 3, {"otype": "Identity"}, cfg)
    net = tcnn_b200.Network(3, 3, cfg)
    assert module.n_params == net.n_params
    p16 = net.initial_params(seed=5).to(torch.float16).contiguous()
    dp, dx = module.bwd(x, p16, dy, want_input_grad=True)
    dx_net, dp_net = net.module_backward(x, dy, p16)
    torch.cuda.synchronize()
    assert torch.isfinite(dx).all() and dx.abs().max() > 0
    assert rae(dx.cpu().numpy(), dx_net.cpu().numpy(), 99.9) < 1e-3
    assert rae(dp.float().cpu().numpy(), dp_net.float().cpu().numpy(), 99.9) < 1e-3

    fused = tcnn_b200.Module(3, 3, {"otype": "Identity"}, dict(cfg, n_neurons=64))
    p64 = fused.initial_params(seed=5).to(torch.float16).contiguous()
    fused.bwd(x, p64, dy)  # parameter gradients alone stay available
    with pytest.raises(tcnn_b200.TcnnError, match="Identity encoding"):
        fused.bwd(x, p64, dy, want_input_grad=True)


@pytest.mark.parametrize("F,B,max_level,launches", [
    (1, 1024, 1.0, 2),      # scatter into the fp32 accumulator + cast to fp16
    (2, 1 << 18, 1.0, 2),   # scatter with replicated coarse levels + replica reduce
    (2, 1 << 18, 0.5, 1),   # a partial max_level scatters without replicas
])
def test_grid_backward_counts_every_launch(torch_cuda, F, B, max_level, launches):
    torch = torch_cuda
    import tcnn_b200

    enc = tcnn_b200.Encoding(3, dict(GRID, n_features_per_level=F))
    enc.set_max_level(max_level)
    p16 = enc.initial_params(seed=1).to(torch.float16).contiguous()
    x = torch.rand(B, 3, device="cuda")
    dy = torch.ones(B, enc.n_output_dims, dtype=torch.float16, device="cuda")
    before = tcnn_b200.kernel_launch_count()
    enc.bwd(x, p16, dy)
    assert tcnn_b200.kernel_launch_count() - before == launches
    torch.cuda.synchronize()
