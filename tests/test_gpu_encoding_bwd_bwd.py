"""GPU checks of the grid encoding's second-order derivatives (csrc/grid_bwd_bwd.cu, tcnnb_encoding_backward_backward_input,
tcnn.Encoding under create_graph=True) against the double-precision oracle (tests/cpp/grid_bwd_bwd_oracle.cpp, pinned on the CPU by
tests/test_oracle_bwd_bwd.py) and against the reference's own results (tests/golden/bwdbwd_*.npz)."""
import ctypes
import itertools
import json
import os

import numpy as np
import pytest

import grid_bwd_bwd_oracle as bb
import oracle_binding as ob
from golden_util import GOLDEN, rae

pytestmark = pytest.mark.gpu

CONFIGS = [
    # (n_input_dims, encoding config) -- the grid configurations of test_gpu_encoding.py
    (3, {"otype": "HashGrid", "n_levels": 8, "n_features_per_level": 1, "log2_hashmap_size": 12, "base_resolution": 8, "per_level_scale": 1.5}),
    (3, {"otype": "HashGrid", "n_levels": 8, "n_features_per_level": 2, "log2_hashmap_size": 12, "base_resolution": 8, "per_level_scale": 1.5}),
    (3, {"otype": "HashGrid", "n_levels": 8, "n_features_per_level": 4, "log2_hashmap_size": 12, "base_resolution": 8, "per_level_scale": 1.5}),
    (3, {"otype": "HashGrid", "n_levels": 6, "n_features_per_level": 8, "log2_hashmap_size": 11, "base_resolution": 4, "per_level_scale": 2.0}),
    (2, {"otype": "HashGrid", "n_levels": 10, "n_features_per_level": 4, "log2_hashmap_size": 10, "base_resolution": 16, "per_level_scale": 1.5}),
    (4, {"otype": "HashGrid", "n_levels": 6, "n_features_per_level": 2, "log2_hashmap_size": 12, "base_resolution": 4, "per_level_scale": 1.5}),
    (4, {"otype": "HashGrid", "n_levels": 4, "n_features_per_level": 1, "log2_hashmap_size": 10, "base_resolution": 3, "per_level_scale": 2.0}),
    (3, {"otype": "DenseGrid", "n_levels": 4, "n_features_per_level": 4, "base_resolution": 4, "per_level_scale": 1.5}),
    (3, {"otype": "TiledGrid", "n_levels": 5, "n_features_per_level": 2, "base_resolution": 5, "per_level_scale": 1.5}),
    (3, {"otype": "HashGrid", "n_levels": 8, "n_features_per_level": 2, "log2_hashmap_size": 12, "base_resolution": 8, "per_level_scale": 1.5, "interpolation": "Nearest"}),
    (3, {"otype": "HashGrid", "n_levels": 8, "n_features_per_level": 4, "log2_hashmap_size": 12, "base_resolution": 8, "per_level_scale": 1.5, "interpolation": "Smoothstep"}),
    (2, {"otype": "HashGrid", "n_levels": 8, "n_features_per_level": 1, "log2_hashmap_size": 12, "base_resolution": 8, "per_level_scale": 1.5, "interpolation": "Nearest"}),
]
CASES = [(n, c, 1.0) for n, c in CONFIGS] + [
    (3, {"otype": "HashGrid", "n_levels": 8, "n_features_per_level": 2, "log2_hashmap_size": 12, "base_resolution": 8, "per_level_scale": 1.5, "interpolation": "Smoothstep"}, 0.5),
]
OUTPUTS = ("params", "doutput", "input")


def f16(t):
    return t.cpu().numpy().view(np.uint16)


def native_bwd_bwd(torch, enc, x, p16, v, u, want, prefill=float("nan")):
    """The C ABI with the asked outputs pre-filled (NaN by default: every non-null output must be overwritten)."""
    import tcnn_b200

    B = x.shape[0]
    gp = torch.full((enc.n_params,), prefill, dtype=torch.float16, device="cuda") if "params" in want else None
    gd = torch.full((B, enc.n_output_dims), prefill, dtype=torch.float16, device="cuda") if "doutput" in want else None
    gx = torch.full((B, enc.n_input_dims), prefill, dtype=torch.float32, device="cuda") if "input" in want else None
    rc = tcnn_b200.load().tcnnb_encoding_backward_backward_input(enc._h, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream), B, v.data_ptr(), x.data_ptr(), u.data_ptr(),
                                                                 gp.data_ptr() if gp is not None else None, gd.data_ptr() if gd is not None else None,
                                                                 gx.data_ptr() if gx is not None else None, p16.data_ptr())
    tcnn_b200._check(rc)
    torch.cuda.synchronize()
    return gp, gd, gx


def assert_input_like(dev, ref):
    """The bars of the first-order input gradient (test_gpu_encoding.py)."""
    assert np.isfinite(dev).all()
    assert rae(dev, ref, 99.0) < 1e-3
    assert np.abs(dev - ref).max() <= 1e-3 * np.abs(ref).max()


def assert_params_like(dev, ref):
    """The bars of the first-order scatter: fp16 atomics against exact sums."""
    assert np.isfinite(dev).all()
    assert rae(dev, ref.astype(np.float16).astype(np.float64), 99.9) < 1.2e-2


def case_id(c):
    n, cfg, ml = c
    return f"D{n}_F{cfg['n_features_per_level']}_{cfg['otype']}_{cfg.get('interpolation', 'Linear')}" + ("_maxlevel0.5" if ml < 1 else "")


@pytest.mark.parametrize("n_in,enc_cfg,max_level", CASES, ids=[case_id(c) for c in CASES])
def test_device_matches_oracle(torch_cuda, n_in, enc_cfg, max_level):
    torch = torch_cuda
    import tcnn_b200

    enc = tcnn_b200.Encoding(n_in, enc_cfg)
    levels = enc.grid_levels()
    orc = ob.OracleModel(n_in, 1, {"encoding": enc_cfg, "network": {"n_neurons": 16, "n_hidden_layers": 1}}, scales=levels["scales"])
    F, L = enc_cfg["n_features_per_level"], enc_cfg["n_levels"]
    if max_level < 1:
        enc.set_max_level(max_level)
    p16 = enc.initial_params(seed=9, scale=50.0).to(torch.float16).contiguous()
    B = 2048
    rng = ob.default_rng(31)
    x = ob.generate_random_uniform(rng, B * n_in).reshape(B, n_in)
    g = torch.Generator(device="cuda").manual_seed(3)
    u = (torch.randn(B, L * F, device="cuda", generator=g) * 0.5).to(torch.float16).contiguous()
    v = torch.randn(B, n_in, device="cuda", generator=g).contiguous()
    xd = torch.from_numpy(x).cuda()
    u_soa = np.zeros((orc.grid.padded_width, B), np.uint16)
    u_soa[: L * F] = f16(u).T
    ref_p, ref_d, ref_x = bb.grid_backward_backward_input(orc.grid, x, f16(p16), u_soa, v.cpu().numpy(), max_level=max_level)
    nearest = enc_cfg.get("interpolation") == "Nearest"
    if nearest:
        assert not ref_p.any() and not ref_d.any() and not ref_x.any()
    else:
        assert np.abs(ref_p).max() > 0 and np.abs(ref_d).max() > 0 and np.abs(ref_x).max() > 0
    # every output alone and in every combination, into NaN-filled buffers
    for k in (1, 2, 3):
        for want in itertools.combinations(OUTPUTS, k):
            gp, gd, gx = native_bwd_bwd(torch, enc, xd, p16, v, u, want)
            if gp is not None:
                dev = ob.half_bits_to_float(f16(gp)).astype(np.float64)
                if nearest:
                    assert (f16(gp) == 0).all(), want
                else:
                    assert_params_like(dev, ref_p)
            if gd is not None:
                dev = ob.half_bits_to_float(f16(gd)).astype(np.float64)
                if nearest:
                    assert (f16(gd) == 0).all(), want
                else:
                    assert_input_like(dev, ref_d)
            if gx is not None:
                dev = gx.cpu().numpy().astype(np.float64)
                if nearest:
                    assert (dev == 0).all(), want
                else:
                    assert_input_like(dev, ref_x)
    # the Python surface returns the same
    dd, gp, gx = enc.bwd_bwd_input(xd, p16, v, u, want_doutput=True, want_params=True, want_input=True)
    torch.cuda.synchronize()
    if not nearest:
        assert_input_like(ob.half_bits_to_float(f16(dd)).astype(np.float64), ref_d)
        assert_params_like(ob.half_bits_to_float(f16(gp)).astype(np.float64), ref_p)
        assert_input_like(gx.cpu().numpy().astype(np.float64), ref_x)


# tests/golden/make_golden_bwd_bwd.sh: Linear and Smoothstep, D = 2, 3, 4, F = 1, 2, 4, 8, hashed and dense
GOLDEN_CASES = ["bwdbwd_hash3d_f2", "bwdbwd_hash3d_f1_smooth", "bwdbwd_dense2d_f4", "bwdbwd_hash4d_f8_smooth"]


@pytest.mark.parametrize("case", GOLDEN_CASES)
def test_device_matches_the_reference_dump(torch_cuda, case):
    torch = torch_cuda
    import tcnn_b200

    z = np.load(os.path.join(GOLDEN, case + ".npz"))
    meta = json.loads(bytes(z["meta"]).decode())
    D, B, W = meta["n_input_dims"], meta["batch"], meta["width"]
    enc = tcnn_b200.Encoding(D, meta["encoding"])
    assert enc.n_output_dims == W and enc.n_params == meta["n_params"]
    x = torch.from_numpy(z["x_f32"].reshape(B, D)).cuda()
    p16 = torch.from_numpy(z["params_f16"].view(np.float16)).cuda()
    u = torch.from_numpy(z["dL_doutput_f16"].view(np.float16).reshape(B, W)).cuda()
    v = torch.from_numpy(z["dL_ddLdinput_f32"].reshape(B, D)).cuda()
    gp, gd, gx = native_bwd_bwd(torch, enc, x, p16, v, u, OUTPUTS)
    ref_p = z["dL_dparams_f16"].view(np.float16).astype(np.float64)
    ref_d = z["dL_ddLdoutput_f16"].view(np.float16).astype(np.float64).reshape(B, W)
    ref_x = z["dL_dinput_f32"].astype(np.float64).reshape(B, D)
    assert np.abs(ref_p).max() > 0 and np.abs(ref_d).max() > 0 and np.abs(ref_x).max() > 0
    assert_params_like(ob.half_bits_to_float(f16(gp)).astype(np.float64), ref_p)
    assert_input_like(ob.half_bits_to_float(f16(gd)).astype(np.float64), ref_d)
    assert_input_like(gx.cpu().numpy().astype(np.float64), ref_x)


EIKONAL_GRID = {"otype": "HashGrid", "n_levels": 8, "n_features_per_level": 2, "log2_hashmap_size": 14, "base_resolution": 4, "per_level_scale": 1.5}


def test_torch_eikonal_gradients_match_the_oracle(torch_cuda):
    """g = dL/dx with create_graph=True, then an eikonal loss on g: the table and the input receive the second-order gradients that
    the oracle gives for the same dL_doutput (loss-scaled, as the layer sends it) and dL_ddLdinput."""
    torch = torch_cuda
    import tcnn_b200.torch_modules as tcnn

    torch.manual_seed(0)
    enc = tcnn.Encoding(3, EIKONAL_GRID, seed=5)
    with torch.no_grad():
        enc.params.uniform_(-1e-2, 1e-2)  # a trained-looking table: gradients of order one
    W = enc.n_output_dims
    w = torch.randn(W, 1, device="cuda")
    B = 1024
    x = torch.rand(B, 3, device="cuda", requires_grad=True)
    y = enc(x).float() @ w
    (g,) = torch.autograd.grad(y.sum(), x, create_graph=True)
    loss = ((g.norm(dim=-1) - 1.0) ** 2).mean()
    loss.backward()
    assert enc.params.grad is not None and x.grad is not None
    assert float(enc.params.grad.abs().max()) > 0  # the eikonal term reaches the grid

    # the oracle composed by hand: the layer's dL_doutput is fp16(w * loss_scale) on every row; v = d(loss)/dg
    ls = enc.loss_scale
    levels = enc.native_tcnn_module.grid_levels()
    orc = ob.OracleModel(3, 1, {"encoding": EIKONAL_GRID, "network": {"n_neurons": 16, "n_hidden_layers": 1}}, scales=levels["scales"])
    table = f16(enc.params.detach().to(torch.float16))
    scaled = (w[:, 0] * ls).to(torch.float16)
    u_soa = np.zeros((orc.grid.padded_width, B), np.uint16)
    u_soa[:W] = np.repeat(f16(scaled)[:, None], B, axis=1)
    xn = x.detach().cpu().numpy()
    gd = g.detach().cpu().numpy().astype(np.float64)
    dx_ref = orc.grid_input_gradient(xn, u_soa, table) / ls
    assert np.abs(gd - dx_ref).max() <= 1e-3 * np.abs(dx_ref).max()
    n = np.linalg.norm(gd, axis=1, keepdims=True)
    v = (2.0 * (n - 1.0) * gd / n / B).astype(np.float32)
    ref_p, _, ref_x = bb.grid_backward_backward_input(orc.grid, xn, table, u_soa, v, want=("params", "input"))
    assert_params_like(enc.params.grad.cpu().numpy().astype(np.float64) * ls, ref_p)
    assert_input_like(x.grad.cpu().numpy().astype(np.float64), ref_x / ls)


def test_torch_sdf_fit_of_a_sphere_lowers_the_eikonal_loss(torch_cuda):
    torch = torch_cuda
    import tcnn_b200.torch_modules as tcnn

    torch.manual_seed(1)
    enc = tcnn.Encoding(3, EIKONAL_GRID, seed=7)
    mlp = torch.nn.Sequential(torch.nn.Linear(enc.n_output_dims, 64), torch.nn.Softplus(beta=10.0), torch.nn.Linear(64, 1)).cuda()
    opt = torch.optim.Adam(list(enc.parameters()) + list(mlp.parameters()), lr=1e-2)

    def losses(x):
        x = x.requires_grad_(True)
        f = mlp(enc(x).float())
        (g,) = torch.autograd.grad(f.sum(), x, create_graph=True)
        sdf = (x - 0.5).norm(dim=-1, keepdim=True) - 0.3
        return ((f - sdf) ** 2).mean(), ((g.norm(dim=-1) - 1.0) ** 2).mean()

    probe = torch.rand(4096, 3, device="cuda")
    eik0 = float(losses(probe.clone())[1].detach())
    for _ in range(150):
        fit, eik = losses(torch.rand(2048, 3, device="cuda"))
        opt.zero_grad()
        (fit + 0.1 * eik).backward()
        opt.step()
    eik1 = float(losses(probe.clone())[1].detach())
    assert eik1 < 0.5 * eik0, (eik0, eik1)


def test_other_objects_do_not_support_double_backward(torch_cuda):
    torch = torch_cuda
    import tcnn_b200
    import tcnn_b200.torch_modules as tcnn

    x = torch.rand(256, 3, device="cuda")
    v = torch.rand(256, 3, device="cuda")
    composite = {"otype": "Composite", "nested": [dict(EIKONAL_GRID, n_dims_to_encode=3)]}
    for cfg, name in ((composite, "Composite"), ({"otype": "Identity"}, "Identity"), ({"otype": "Frequency", "n_frequencies": 2}, "Frequency")):
        enc = tcnn_b200.Encoding(3, cfg)
        p16 = (enc.initial_params(1) if enc.n_params else torch.zeros(8, device="cuda")).to(torch.float16)
        u = torch.zeros(256, enc.n_output_dims, dtype=torch.float16, device="cuda")
        with pytest.raises(tcnn_b200.TcnnError, match=f"{name} does not support double backward"):
            enc.bwd_bwd_input(x, p16, v, u)
    net_cfg = {"otype": "FullyFusedMLP", "activation": "ReLU", "output_activation": "None", "n_neurons": 64, "n_hidden_layers": 2}
    with pytest.raises(tcnn_b200.TcnnError, match="does not support double backward"):
        tcnn_b200.Module(3, 1, EIKONAL_GRID, net_cfg).bwd_bwd_input(x, None, v, None)
    with pytest.raises(tcnn_b200.TcnnError, match="does not support double backward"):
        tcnn_b200.Network(16, 1, net_cfg).bwd_bwd_input(x, None, v, None)
    # through autograd: a second-order term of a non-grid encoding fails loudly instead of being dropped
    layer = tcnn.Encoding(3, {"otype": "Frequency", "n_frequencies": 2})
    xr = x.clone().requires_grad_(True)
    (g,) = torch.autograd.grad(layer(xr).float().sum(), xr, create_graph=True)
    with pytest.raises(Exception, match="does not support double backward"):
        (g ** 2).sum().backward()
