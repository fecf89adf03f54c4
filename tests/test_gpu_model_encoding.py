"""How the trainer and module tiers see their encoding: which kernels run a configuration (the fused kernel or the general path of
encoding kernels and stand-alone network kernels), and what the C ABI reports about the encoding (width, parameter count,
hyperparams, level table)."""
import pytest

pytestmark = pytest.mark.gpu

B = 1024  # below the spatial-binning threshold: a fused training step is the fused kernel and Adam, nothing else
NET = {"otype": "FullyFusedMLP", "n_neurons": 64, "n_hidden_layers": 2}
HASH = {"otype": "HashGrid", "n_levels": 16, "n_features_per_level": 2, "log2_hashmap_size": 14, "base_resolution": 16, "per_level_scale": 1.5}

# (n_input_dims, n_output_dims, encoding, network, path)
PATHS = {
    "hash_3d": (3, 3, HASH, NET, "fused"),
    "dense_2d": (2, 3, {"otype": "DenseGrid", "n_levels": 8, "base_resolution": 8}, NET, "fused"),
    "64_features": (3, 3, dict(HASH, n_levels=32, per_level_scale=1.2), NET, "fused"),
    "identity_3d": (3, 3, {"otype": "Identity"}, NET, "fused"),
    "128_neurons": (3, 3, HASH, dict(NET, n_neurons=128), "general"),
    "7_hidden_layers": (3, 3, HASH, dict(NET, n_hidden_layers=7), "general"),
    "17_outputs": (3, 17, HASH, NET, "general"),
    "4_features_per_level": (3, 3, dict(HASH, n_features_per_level=4), NET, "general"),
    "grid_4d": (4, 3, HASH, NET, "general"),
    "nearest": (3, 3, dict(HASH, interpolation="Nearest"), NET, "general"),
    "identity_4d": (4, 3, {"otype": "Identity"}, NET, "general"),
    "composite_of_one_grid": (3, 3, {"otype": "Composite", "nested": [HASH]}, NET, "general"),
    "frequency": (3, 3, {"otype": "Frequency", "n_frequencies": 4}, NET, "general"),
}


def training_step_launches(torch, n_in, n_out, encoding, network):
    import tcnn_b200

    model = tcnn_b200.create_from_config(n_in, n_out, {"encoding": encoding, "network": network})
    x = torch.rand(B, n_in, device="cuda")
    y = torch.rand(B, n_out, device="cuda")
    before = tcnn_b200.kernel_launch_count()
    model.trainer.training_step(x, y)
    launches = tcnn_b200.kernel_launch_count() - before
    torch.cuda.synchronize()
    model.close()
    return launches


@pytest.mark.parametrize("name", list(PATHS))
def test_path_at_the_fused_kernel_limits(torch_cuda, name):
    n_in, n_out, encoding, network, path = PATHS[name]
    launches = training_step_launches(torch_cuda, n_in, n_out, encoding, network)
    if path == "fused":
        assert launches == 2  # the fused kernel and Adam
    else:
        assert launches > 2


def test_encoding_wider_than_the_fused_kernel_is_rejected(torch_cuda):
    """33 levels x 2 features pad to 80 columns: too wide for the fused kernel, and the general path's network backward cannot
    hand dL/d(encoded) rows wider than its 64-neuron layers back to the grid."""
    import tcnn_b200

    with pytest.raises(tcnn_b200.TcnnError, match="encoding wider than 64 features"):
        tcnn_b200.create_from_config(3, 3, {"encoding": dict(HASH, n_levels=33, per_level_scale=1.2), "network": NET})


@pytest.mark.parametrize("network,path", [(NET, "fused"), (dict(NET, n_neurons=128), "general")])
def test_module_forward_path(torch_cuda, network, path):
    torch = torch_cuda
    import tcnn_b200

    module = tcnn_b200.Module(3, 3, HASH, network)
    params = module.initial_params(seed=1).to(torch.float16).contiguous()
    x = torch.rand(B, 3, device="cuda")
    before = tcnn_b200.kernel_launch_count()
    module.fwd(x, params)
    launches = tcnn_b200.kernel_launch_count() - before
    torch.cuda.synchronize()
    if path == "fused":
        assert launches == 1
    else:
        assert launches > 1


# 4 levels with per_level_scale 2: level scales 7, 15, 31, 63 are exact, tables of 8^3 entries and then 2^12 (hashed)
GRID = {"otype": "HashGrid", "n_levels": 4, "n_features_per_level": 2, "log2_hashmap_size": 12, "base_resolution": 8, "per_level_scale": 2.0}
GRID_LEVELS = {"n_levels": 4, "offsets": [0, 512, 4608, 8704, 12800], "scales": [7.0, 15.0, 31.0, 63.0], "resolutions": [8, 16, 32, 64]}
NO_LEVELS = {"n_levels": 0, "offsets": [0], "scales": [], "resolutions": []}
MLP_PARAMS_16 = 64 * 16 + 64 * 64 + 16 * 64  # 64 x 2 network behind a 16-wide encoding, 16 padded outputs
MLP_PARAMS_32 = 64 * 32 + 64 * 64 + 16 * 64
GRID_PARAMS = 12800 * 2

# (n_input_dims, encoding, encoded_width, n_params, hyperparams()["encoding"], grid_levels())
ENCODINGS = {
    "grid": (3, GRID, 16, MLP_PARAMS_16 + GRID_PARAMS,
             {"otype": "Grid", "type": "Hash", "n_levels": 4, "n_features_per_level": 2, "base_resolution": 8, "log2_hashmap_size": 12, "per_level_scale": 2.0,
              "interpolation": "Linear", "hash": "CoherentPrime"},
             GRID_LEVELS),
    "identity": (3, {"otype": "Identity", "scale": 0.5, "offset": 0.25}, 16, MLP_PARAMS_16, {"otype": "Identity", "scale": 0.5, "offset": 0.25}, NO_LEVELS),
    "composite_of_one_grid": (3, {"otype": "Composite", "nested": [GRID]}, 16, MLP_PARAMS_16 + GRID_PARAMS, {"otype": "Composite", "n_nested": 1, "n_output_dims": 16},
                              NO_LEVELS),
    # 8 grid features, 16 spherical-harmonics coefficients, padded to 32
    "composite_grid_sh": (6, {"otype": "Composite", "nested": [dict(GRID, n_dims_to_encode=3), {"otype": "SphericalHarmonics", "degree": 4}]}, 32,
                          MLP_PARAMS_32 + GRID_PARAMS, {"otype": "Composite", "n_nested": 2, "n_output_dims": 32}, NO_LEVELS),
}


@pytest.mark.parametrize("name", list(ENCODINGS))
def test_encoding_as_the_abi_reports_it(torch_cuda, name):
    import tcnn_b200

    n_in, encoding, width, n_params, hyper, levels = ENCODINGS[name]
    model = tcnn_b200.create_from_config(n_in, 3, {"encoding": encoding, "network": NET})
    assert model.encoded_width == width
    assert model.n_params == n_params
    h = model.hyperparams()
    assert h["encoding"] == hyper
    assert h["encoded_width"] == width
    assert model.grid_levels() == levels
    if name == "grid":
        assert model.grid_levels() == tcnn_b200.Encoding(3, GRID).grid_levels()
    model.close()
