"""GPU parity of Composite's Sum / Product reductions, dims_to_encode_begin (overlapping input ranges), Empty and the NRC shorthand
(encodings/composite.h, encodings/empty.h, src/encoding.cu:93-115) through every tier: the encoding tier (tcnnb_encoding_*), the trainer
(create_from_config on the general path), the module tier and the torch modules. Oracles: tests/composite_oracle.py (numpy: layout,
plain encodings, the reductions in float32), the C oracle for grids and the network (tests/oracle_binding.py), and the vectors the
unmodified reference wrote (tests/golden/{composite_sum_hash3d,composite_product_planes,composite_product_pad,composite_empty,nrc_top}.npz)."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

import composite_oracle as co
import oracle_binding as ob
from golden_util import GOLDEN, rae

pytestmark = pytest.mark.gpu


def hg(n_dims, begin=None, log2=14, base=16, L=8, F=2):
    e = {"otype": "HashGrid", "n_levels": L, "n_features_per_level": F, "log2_hashmap_size": log2, "base_resolution": base, "per_level_scale": 1.5, "n_dims_to_encode": n_dims}
    if begin is not None:
        e["dims_to_encode_begin"] = begin
    return e


CONFIGS = {
    # grid-only reductions (bit-exact forward)
    "sum_hash3d": (3, {"otype": "Composite", "reduction": "Sum", "nested": [hg(3, 0, 14, 8), hg(3, 0, 12, 16)]}),
    "product_planes": (4, {"otype": "Composite", "reduction": "Product", "nested": [hg(2, 0), hg(2, 1), hg(2, 2)]}),
    # a grid x Identity: zero padding times one padding; Identity is exact, so bit-exact too
    "product_pad": (4, {"otype": "Composite", "reduction": "product", "nested": [hg(4, 0, L=2), {"otype": "Identity", "n_dims_to_encode": 4, "dims_to_encode_begin": 0}]}),
    # F = 4 next to a 6-wide TriangleWave padded to 8, overlapping ranges in reverse order
    "sum_f4_wave": (3, {"otype": "Composite", "reduction": "SUM", "nested": [hg(2, 1, L=2, F=4), {"otype": "TriangleWave", "n_frequencies": 3, "n_dims_to_encode": 2, "dims_to_encode_begin": 0}]}),
    # odd width 3 in the encoding tier (scalar reduce kernels), overlapping plain encodings
    "sum_plain_odd": (4, {"otype": "Composite", "reduction": "Sum", "nested": [{"otype": "Identity", "scale": 2.0, "n_dims_to_encode": 3, "dims_to_encode_begin": 0},
                                                                             {"otype": "TriangleWave", "n_frequencies": 1, "n_dims_to_encode": 3, "dims_to_encode_begin": 1}]}),
    "product_plain_odd": (4, {"otype": "Composite", "reduction": "Product", "nested": [{"otype": "Identity", "offset": 0.5, "n_dims_to_encode": 3, "dims_to_encode_begin": 1},
                                                                                     {"otype": "OneBlob", "n_bins": 1, "n_dims_to_encode": 3, "dims_to_encode_begin": 0}]}),
    # Concatenation with begin: overlapping ranges, out of order, and Empty
    "concat_begin_empty": (6, {"otype": "Composite", "nested": [hg(3, 2), {"otype": "Empty", "n_dims_to_encode": 2, "dims_to_encode_begin": 0}, {"otype": "Identity", "n_dims_to_encode": 2, "dims_to_encode_begin": 1}]}),
    "nrc": (9, {"otype": "NRC"}),
}
GRID_ONLY_OR_IDENTITY = ("sum_hash3d", "product_planes", "product_pad")


def f16(t):
    return t.cpu().numpy().view(np.uint16)


def make_x(n_in, B, seed=1337):
    rng = ob.default_rng(seed)
    return ob.generate_random_uniform(rng, B * n_in).reshape(B, n_in)


def grid_oracle(e, n_dims):
    import tcnn_b200

    sub = {k: v for k, v in e.items() if k not in ("n_dims_to_encode", "dims_to_encode_begin")}
    scales = tcnn_b200.Encoding(n_dims, sub).grid_levels()["scales"]
    return ob.OracleModel(n_dims, 1, {"encoding": sub, "network": {"n_neurons": 16, "n_hidden_layers": 1}}, scales=scales)


class Oracle:
    """The whole encoding on the host: numpy for layout / plain encodings / reductions, the C oracle for grids."""

    def __init__(self, n_in, cfg, alignment, x, enc_params16):
        self.rows, self.segs, self.width, self.red = co.encode_nested(x, cfg, alignment)
        self.x = x
        self.grids = {}
        off = 0
        for k, (t, e, in_begin, n_dims, out_begin, n_out, n_pad, pad_first) in enumerate(self.segs):
            if t in co.GRIDS:
                orc = grid_oracle(e, n_dims)
                n_p = orc.grid.n_params
                orc.params_fp16[orc.n_mlp :] = enc_params16[off : off + n_p]
                xs = np.ascontiguousarray(x[:, in_begin : in_begin + n_dims])
                self.rows[:, out_begin : out_begin + n_out] = ob.half_bits_to_float(orc.encode(xs)[:n_out].T)
                self.grids[k] = (orc, xs, off)
                off += n_p
        self.n_params = off
        assert not np.isnan(self.rows).any()
        self.slabs = [self.rows] if self.red == "concatenation" else co.slabs_of(self.rows, len(self.segs), self.width)

    def forward(self):
        """fp16 [n][width]"""
        if self.red == "concatenation":
            return self.rows.astype(np.float16)
        return co.reduce_forward(self.slabs, self.red)

    def nested_dy(self, dy):
        """dL/d(nested) per segment, float32 [n][n_out] (columns of its own features)."""
        per = co.reduce_backward(dy, self.slabs, self.red) if self.red != "concatenation" else None
        out = []
        for k, (t, e, in_begin, n_dims, out_begin, n_out, n_pad, pad_first) in enumerate(self.segs):
            first = n_pad if pad_first else 0
            if per is None:
                out.append(dy.astype(np.float16).astype(np.float32)[:, out_begin + first : out_begin + first + n_out])
            else:
                out.append(per[k].astype(np.float32)[:, first : first + n_out])
        return out

    def backward(self, dy):
        """(param gradients per grid: {seg: (offset, grads)}, summed input gradient)"""
        gx = np.zeros(self.x.shape, np.float32)
        gp = {}
        for k, ((t, e, in_begin, n_dims, out_begin, n_out, n_pad, pad_first), dys) in enumerate(zip(self.segs, self.nested_dy(dy))):
            if k in self.grids:
                orc, xs, off = self.grids[k]
                dy_soa = np.zeros((orc.grid.padded_width, xs.shape[0]), np.uint16)
                dy_soa[:n_out] = dys.astype(np.float16).view(np.uint16).T
                gx[:, in_begin : in_begin + n_dims] += orc.grid_input_gradient(xs, dy_soa)
                gp[k] = (off, orc.grid_backward(xs, dy_soa))
            else:
                gx[:, in_begin : in_begin + n_dims] += co.plain_input_gradient(t, e, self.x[:, in_begin : in_begin + n_dims], dys)
        return gp, gx


def encoding_setup(torch, name, B=1024, seed=9):
    import tcnn_b200

    n_in, cfg = CONFIGS[name]
    enc = tcnn_b200.Encoding(n_in, cfg)
    x = make_x(n_in, B)
    p16 = enc.initial_params(seed=seed, scale=3000.0).to(torch.float16).contiguous() if enc.n_params else torch.zeros(8, dtype=torch.float16, device="cuda")
    orc = Oracle(n_in, cfg, 0, x, f16(p16))
    assert enc.n_output_dims == orc.width and orc.n_params == enc.n_params
    return enc, x, torch.from_numpy(x).cuda(), p16, orc


@pytest.mark.parametrize("name", list(CONFIGS))
def test_encoding_tier_forward_and_backward_match_the_oracles(torch_cuda, name):
    torch = torch_cuda
    enc, x, xd, p16, orc = encoding_setup(torch, name)
    B = x.shape[0]
    out = enc.fwd(xd, p16)
    want = orc.forward()
    if name in GRID_ONLY_OR_IDENTITY:
        assert np.array_equal(f16(out), want.view(np.uint16)), "reduced features differ from the float32 reduction of the nested outputs"
    else:
        got = out.float().cpu().numpy()
        w = want.astype(np.float32)
        assert (np.abs(got - w) <= 4e-3 * np.maximum(1.0, np.abs(w))).all(), np.abs(got - w).max()
        assert (got.astype(np.float16) != w.astype(np.float16)).mean() < 0.05
    g = torch.Generator(device="cuda").manual_seed(3)
    dy = (torch.randn(B, orc.width, device="cuda", generator=g) * 0.5).to(torch.float16).contiguous()
    gp, gx = enc.bwd(xd, p16, dy, want_params=enc.n_params > 0, want_input=True)
    torch.cuda.synchronize()
    # the oracle's dL/d(nested) from the DEVICE's nested outputs is what the C grid oracle sees: with bit-identical nested outputs the
    # reduction's backward is bit-exact, so the grid gradients carry only the scatter's own reordering
    gp_ref, gx_ref = orc.backward(dy.cpu().numpy().astype(np.float32))
    for k, (off, g_ref) in gp_ref.items():
        n_p = len(g_ref)
        g_dev = ob.half_bits_to_float(f16(gp))[off : off + n_p]
        assert rae(g_dev, g_ref, 99.9) < 1.2e-2, (k, rae(g_dev, g_ref, 99.9))
    gx_dev = gx.cpu().numpy()
    scale = max(1.0, float(np.abs(gx_ref).max()))
    assert np.abs(gx_dev - gx_ref).max() <= 5e-3 * scale, (np.abs(gx_dev - gx_ref).max(), scale)


@pytest.mark.parametrize("name", ["product_planes", "sum_f4_wave"])
def test_backward_does_not_read_an_earlier_forward(torch_cuda, name):
    """fwd(A), fwd(B), bwd(A) == fwd(A), bwd(A): the Product's nested outputs are recomputed inside the backward call."""
    torch = torch_cuda
    enc, x, xd, p16, orc = encoding_setup(torch, name)
    xb = torch.from_numpy(make_x(x.shape[1], x.shape[0], seed=77)).cuda()
    dy = (torch.randn(x.shape[0], orc.width, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4)) * 0.5).to(torch.float16).contiguous()
    enc.fwd(xd, p16)
    gp1, gx1 = enc.bwd(xd, p16, dy, want_params=True, want_input=True)
    enc.fwd(xd, p16)
    enc.fwd(xb, p16)
    gp2, gx2 = enc.bwd(xd, p16, dy, want_params=True, want_input=True)
    torch.cuda.synchronize()
    assert torch.equal(gx1, gx2)
    assert rae(gp1.float().cpu().numpy(), gp2.float().cpu().numpy(), 100.0) < 1e-3


def net_cfg(width=64, hidden=2):
    return {"otype": "FullyFusedMLP", "activation": "ReLU", "output_activation": "None", "n_neurons": width, "n_hidden_layers": hidden}


OPT = {"otype": "Adam", "learning_rate": 1e-2, "beta1": 0.9, "beta2": 0.99, "epsilon": 1e-15, "l2_reg": 1e-6}


def mlp_oracle(width, n_mlp, w16, enc16, B, dy_out=None, y=None):
    """C-oracle FFMLP 64x2: (output fp16 bits [B][16], loss values, dL/d(encoded) fp16 bits SoA [width][B], dW)."""
    lib = ob.load()
    mlp = ob.Mlp(width, 64, 2, 16, 0, ob.ACT["relu"], ob.ACT["none"], 0)
    assert lib.orc_mlp_setup(ctypes.byref(mlp)) == 0 and mlp.n_params == n_mlp
    enc_soa = np.ascontiguousarray(enc16.view(np.uint16).T)
    hidden = np.zeros((2, B, 64), np.uint16)
    out = np.zeros((B, 16), np.uint16)
    w16 = np.ascontiguousarray(w16)
    lib.orc_mlp_forward(ctypes.byref(mlp), B, ob.ACCUM_FP32, ob._p(w16), ob._p(enc_soa), ob._p(hidden), ob._p(out))
    values = np.zeros((B, 16), np.float32)
    if dy_out is None:
        dy_out = np.zeros((B, 16), np.uint16)
        lib.orc_loss(ob.LOSS_RELATIVE_L2, B, 16, y.shape[1], ctypes.c_float(128.0), ob._p(out), ob._p(y), ob._p(values), ob._p(dy_out))
    dW = np.zeros(n_mlp, np.float64)
    d_enc = np.zeros_like(enc_soa)
    lib.orc_mlp_backward(ctypes.byref(mlp), B, ob.ACCUM_FP32, ob._p(w16), ob._p(enc_soa), ob._p(hidden), ob._p(np.ascontiguousarray(dy_out)), ob._p(dW), ob._p(d_enc))
    return out, values, d_enc, dW


@pytest.mark.parametrize("name", ["sum_hash3d", "product_planes", "product_pad", "concat_begin_empty", "nrc"])
def test_trainer_general_path_matches_the_oracles(torch_cuda, name):
    torch = torch_cuda
    import tcnn_b200

    n_in, enc_cfg = CONFIGS[name]
    n_out, B = 3, 512
    model = tcnn_b200.create_from_config(n_in, n_out, {"loss": {"otype": "RelativeL2"}, "optimizer": OPT, "encoding": enc_cfg, "network": net_cfg()})
    x = make_x(n_in, B)
    y = ob.make_targets(x[:, :3].copy(), n_out)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    gx = torch.zeros(B, n_in, device="cuda")
    model.trainer.training_step(xd, yd, run_optimizer=False, dL_dinput=gx)
    loss_dev = model.trainer.loss()
    grads = ob.half_bits_to_float(f16(model.trainer.param_gradients()))
    p16 = f16(model.trainer.params())
    n_mlp = model.n_mlp_params
    orc = Oracle(n_in, enc_cfg, 16, x, p16[n_mlp:])
    assert orc.width == model.encoded_width and n_mlp + orc.n_params == model.n_params
    enc16 = orc.forward()
    _, values, d_enc, dW = mlp_oracle(orc.width, n_mlp, p16[:n_mlp], enc16, B, y=y)
    assert abs(loss_dev - values.sum()) <= 2e-3 * values.sum(), (loss_dev, values.sum())
    assert rae(grads[:n_mlp], dW.astype(np.float16).astype(np.float32), 99.9) < 2e-2
    gp_ref, gx_ref = orc.backward(ob.half_bits_to_float(d_enc.T))
    for k, (off, g_ref) in gp_ref.items():
        g_dev = grads[n_mlp + off : n_mlp + off + len(g_ref)]
        assert rae(g_dev, g_ref, 99.9) < 2e-2, (k, rae(g_dev, g_ref, 99.9))
    # dL/dinput: from the loss-scaled dL/d(encoded), as the fused path delivers it
    scale = max(1e-3, float(np.abs(gx_ref).max()))
    assert np.abs(gx.cpu().numpy() - gx_ref).max() <= 2e-2 * scale, (np.abs(gx.cpu().numpy() - gx_ref).max(), scale)
    losses = []
    for _ in range(10):
        model.trainer.training_step(xd, yd)
        losses.append(model.trainer.loss())
    if name != "product_planes":  # (a product of three freshly initialised tables, O(1e-4) each, is zero in fp16: as in the reference, nothing trains)
        assert losses[-1] < 0.8 * losses[0], losses
    inf = model.network.inference(xd)
    assert torch.isfinite(inf).all()


def test_module_tier_position_gradient_through_a_product_of_planes(torch_cuda):
    torch = torch_cuda
    import tcnn_b200

    n_in, enc_cfg = CONFIGS["product_planes"]
    B = 512
    mod = tcnn_b200.Module(n_in, 3, enc_cfg, net_cfg())
    p16 = mod.initial_params(seed=5).to(torch.float16).contiguous()
    x = make_x(n_in, B)
    xd = torch.from_numpy(x).cuda()
    out = mod.fwd(xd, p16)
    g = torch.Generator(device="cuda").manual_seed(6)
    dy = (torch.randn(B, mod.n_output_dims, device="cuda", generator=g) * 16).to(torch.float16)
    dy[:, 3:] = 0
    dy = dy.contiguous()
    grads, gx = mod.bwd(xd, p16, dy, output=out, want_input_grad=True)
    torch.cuda.synchronize()
    p = f16(p16)
    # the network's parameters come first; the three planes' tables after them
    grid_params = sum(grid_oracle(e, 2).grid.n_params for e in enc_cfg["nested"])
    n_mlp = mod.n_params - grid_params
    orc = Oracle(n_in, enc_cfg, 16, x, p[n_mlp:])
    enc16 = orc.forward()
    out_ref, _, d_enc, _ = mlp_oracle(orc.width, n_mlp, p[:n_mlp], enc16, B, dy_out=f16(dy))
    assert rae(ob.half_bits_to_float(f16(out)[:, :3]), ob.half_bits_to_float(out_ref[:, :3]), 99.0) < 1e-2
    _, gx_ref = orc.backward(ob.half_bits_to_float(d_enc.T))
    scale = max(1e-3, float(np.abs(gx_ref).max()))
    assert np.abs(gx.cpu().numpy() - gx_ref).max() <= 2e-2 * scale, (np.abs(gx.cpu().numpy() - gx_ref).max(), scale)


def test_torch_encoding_gradients_against_autograd_of_the_reduction(torch_cuda):
    torch = torch_cuda
    import tcnn_b200.torch_modules as tcnn

    n_in, cfg = CONFIGS["product_planes"]
    B = 1024
    enc = tcnn.Encoding(n_in, cfg, seed=3)
    with torch.no_grad():
        enc.params.mul_(3000.0)  # table values of O(0.3): products well inside fp16's normal range
    x = torch.from_numpy(make_x(n_in, B)).cuda().requires_grad_(True)
    w = torch.randn(B, enc.n_output_dims, device="cuda", generator=torch.Generator(device="cuda").manual_seed(8))
    y = enc(x)
    (y.float() * w).sum().backward()
    torch.cuda.synchronize()
    p16 = enc.params.detach().to(torch.float16)
    orc = Oracle(n_in, cfg, 0, x.detach().cpu().numpy(), f16(p16))
    assert np.array_equal(f16(y.detach()), orc.forward().view(np.uint16))
    # dL/d(nested) by fp32 torch autograd of the reduction agrees with the oracle's float32 restatement to its fp16 rounding
    slabs = [torch.from_numpy(s.copy()).requires_grad_(True) for s in orc.slabs]
    prod = slabs[0] * slabs[1] * slabs[2]
    dy16 = (w.cpu() * 128.0).to(torch.float16)
    (prod * dy16.float()).sum().backward()
    mine = co.reduce_backward(dy16.numpy().astype(np.float32), orc.slabs, "product")
    for s, m in zip(slabs, mine):
        assert np.abs(s.grad.numpy() - m.astype(np.float32)).max() <= 1e-3 * max(1.0, float(np.abs(s.grad.numpy()).max()))
    gp_ref, gx_ref = orc.backward(dy16.numpy().astype(np.float32))
    gx_ref = gx_ref / 128.0
    gx_dev = x.grad.cpu().numpy()
    scale = max(1e-3, float(np.abs(gx_ref).max()))
    assert np.abs(gx_dev - gx_ref).max() <= 1e-2 * scale, (np.abs(gx_dev - gx_ref).max(), scale)
    gparams = enc.params.grad.cpu().numpy()
    for k, (off, g_ref) in gp_ref.items():
        assert rae(gparams[off : off + len(g_ref)], g_ref / 128.0, 99.9) < 2e-2


def test_torch_network_with_input_encoding_trains_a_sum_composite(torch_cuda):
    torch = torch_cuda
    import tcnn_b200
    import tcnn_b200.torch_modules as tcnn

    n_in, cfg = CONFIGS["sum_hash3d"]
    model = tcnn.NetworkWithInputEncoding(n_in, 3, cfg, net_cfg())
    x = torch.from_numpy(make_x(n_in, 1000)).cuda()  # not a multiple of 256: padded by the module
    target = torch.sin(x * 6.0)
    native = tcnn_b200.Module(n_in, 3, cfg, net_cfg())
    ref = native.fwd(torch.nn.functional.pad(x, [0, 0, 0, 24]).contiguous(), model.params.detach().to(torch.float16).contiguous())[:1000, :3]
    assert torch.equal(model(x), ref)
    opt = torch.optim.Adam(model.parameters(), lr=1e-2)
    losses = []
    for _ in range(30):
        opt.zero_grad()
        loss = ((model(x).float() - target) ** 2).mean()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert model.params.grad is not None and torch.isfinite(model.params.grad).all()
    assert losses[-1] < 0.5 * losses[0], losses


def test_snapshot_round_trip(torch_cuda):
    torch = torch_cuda
    import tcnn_b200

    n_in, enc_cfg = CONFIGS["product_planes"]
    cfg = {"loss": {"otype": "RelativeL2"}, "optimizer": OPT, "encoding": enc_cfg, "network": net_cfg()}
    a = tcnn_b200.create_from_config(n_in, 3, cfg)
    x = make_x(n_in, 512)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(ob.make_targets(x[:, :3].copy(), 3)).cuda()
    for _ in range(3):
        a.trainer.training_step(xd, yd)
    blob = a.trainer.serialize(with_optimizer=True)
    b = tcnn_b200.create_from_config(n_in, 3, cfg, seed=4242)
    b.trainer.deserialize(blob)
    assert torch.equal(a.trainer.params(), b.trainer.params())
    assert torch.equal(a.network.inference(xd), b.network.inference(xd))
    a.trainer.training_step(xd, yd)
    b.trainer.training_step(xd, yd)
    assert a.trainer.loss() == b.trainer.loss()


FIXTURES = ["composite_sum_hash3d", "composite_product_planes", "composite_product_pad", "composite_empty", "nrc_top"]


@pytest.mark.parametrize("case", FIXTURES)
def test_against_reference_fixtures(torch_cuda, case):
    torch = torch_cuda
    import tcnn_b200

    z = np.load(os.path.join(GOLDEN, case + ".npz"))
    meta = json.loads(bytes(z["meta"]).decode())
    cfg = json.load(open(os.path.join(GOLDEN, "configs", case + ".json")))
    n_in, n_out, B = meta["n_in"], meta["n_out"], meta["batch"]
    model = tcnn_b200.create_from_config(n_in, n_out, cfg)
    x, y = z["x_f32"].reshape(B, n_in), z["y_f32"].reshape(B, n_out)
    xd, yd = torch.from_numpy(x.copy()).cuda(), torch.from_numpy(y.copy()).cuda()
    p0 = model.trainer.params_full_precision().cpu().numpy()
    # same pcg32 stream through the nested encodings: bit for bit, against the array or (grid cases, tests/golden/digest_params.py) the
    # SHA-256 of its fp32 bytes
    if "params_init_f32" in z.files:
        assert np.array_equal(p0.view(np.uint32), z["params_init_f32"].view(np.uint32))
    else:
        assert p0.size == int(z["params_init_count"][0])
        assert hashlib.sha256(np.ascontiguousarray(p0, np.float32).tobytes()).digest() == z["params_init_sha256"].tobytes()
    # encoded features: the encoding tier on the reference's parameters, against the reference's rows (in front of its network)
    W = meta["encoded_width"]
    assert model.encoded_width == W
    enc_ref = z["encoded_f16"].view(np.float16)
    enc_ref = enc_ref.reshape(W, B).T if meta.get("encoded_layout", "AoS") == "SoA" else enc_ref.reshape(B, W)
    n_mlp = model.n_mlp_params
    p16 = torch.from_numpy(p0[n_mlp:].astype(np.float16)).cuda() if model.n_params > n_mlp else torch.zeros(8, dtype=torch.float16, device="cuda")
    if case == "composite_empty":
        # 16 grid columns + 1 Identity column is odd: the encoding tier cannot hold it behind an F = 2 grid. The grid alone, then Identity
        # (exact) and the ones of the padding
        grid_cfg = {k: v for k, v in cfg["encoding"]["nested"][0].items() if k != "n_dims_to_encode"}
        got = np.ones((B, W), np.float16)
        got[:, :16] = tcnn_b200.Encoding(3, grid_cfg).fwd(torch.from_numpy(x[:, :3].copy()).cuda(), p16).cpu().numpy()
        got[:, 16] = x[:, 5].astype(np.float16)
        w = W
    else:
        enc = tcnn_b200.Encoding(n_in, cfg["encoding"])
        got = enc.fwd(xd, p16).cpu().numpy()
        w = min(W, enc.n_output_dims)
    if case == "nrc_top":  # fast-math sin / floor in the triangle wave: a few fp16 ulps
        assert np.abs(got[:, :w].astype(np.float32) - enc_ref[:, :w].astype(np.float32)).max() < 4e-3
    else:
        assert np.array_equal(got[:, :w].view(np.uint16), np.ascontiguousarray(enc_ref[:, :w]).view(np.uint16))
    inf = model.network.inference(xd).cpu().numpy()
    inf_ref = z["inference_f32"].reshape(B, n_out)
    # outputs at the bottom of fp16 (a product of O(1e-4) tables): a relative measure is meaningless, a few subnormal quanta apart
    assert rae(inf, inf_ref, 99.0) < 1e-2 or np.abs(inf - inf_ref).max() <= 4 * 2.0 ** -24, (rae(inf, inf_ref, 99.0), np.abs(inf - inf_ref).max())
    model.trainer.training_step(xd, yd, run_optimizer=False)
    loss0 = model.trainer.loss()
    assert abs(loss0 - meta["losses"][0]) <= 2e-3 * meta["losses"][0]
    grads = ob.half_bits_to_float(f16(model.trainer.param_gradients()))
    ref = ob.half_bits_to_float(z["grads_step0_f16"])
    assert rae(grads[:n_mlp], ref[:n_mlp], 99.9) < 2e-2
    if model.n_params > n_mlp:
        # the reference sums table gradients with fp16 atomics. The 4-D grid of composite_product_pad sends 16 corners per sample into
        # two small levels, so its sums lie ~3 % from any other order's (the C oracle's exact sums agree with ours to 1.2e-2 above)
        assert rae(grads[n_mlp:], ref[n_mlp:], 99.9) < (4e-2 if case == "composite_product_pad" else 1.2e-2)
        assert ((grads[n_mlp:] != 0) != (ref[n_mlp:] != 0)).mean() < 2e-3
    losses = [loss0]
    for _ in range(meta["n_steps"]):
        model.trainer.training_step(xd, yd)
        losses.append(model.trainer.loss())
    for mine, theirs in zip(losses[1:], meta["losses"][1:]):
        assert abs(mine - theirs) <= 3e-2 * abs(theirs), (losses, meta["losses"])


ERRORS = [
    ("Invalid reduction type: Mean", 3, {"otype": "Composite", "reduction": "Mean", "nested": [{"otype": "Identity"}]}),
    ("must have equal output widths", 3, {"otype": "Composite", "reduction": "Sum", "nested": [hg(3), {"otype": "Identity", "n_dims_to_encode": 3, "dims_to_encode_begin": 0}]}),
    ("reads input dims [2, 4)", 3, {"otype": "Composite", "nested": [{"otype": "Identity", "n_dims_to_encode": 2, "dims_to_encode_begin": 2}]}),
    ("may only leave 'n_dims_to_encode' unspecified", 3, {"otype": "Composite", "nested": [{"otype": "Identity", "n_dims_to_encode": 1, "dims_to_encode_begin": 0}, {"otype": "Identity"}]}),
    ("nested inside a Composite", 3, {"otype": "Composite", "nested": [{"otype": "Composite", "nested": [{"otype": "Identity"}]}]}),
    ("nested inside a Composite", 9, {"otype": "Composite", "nested": [{"otype": "NRC"}]}),
]


@pytest.mark.parametrize("i", range(len(ERRORS)))
def test_invalid_configurations_raise_in_every_tier(torch_cuda, i):
    import tcnn_b200

    msg, n_in, cfg = ERRORS[i]
    with pytest.raises(ValueError):
        co.layout(n_in, cfg, 16)
    with pytest.raises(tcnn_b200.TcnnError, match=None) as e:
        tcnn_b200.Encoding(n_in, cfg)
    assert msg in str(e.value)
    with pytest.raises(tcnn_b200.TcnnError) as e:
        tcnn_b200.create_from_config(n_in, 3, {"encoding": cfg, "network": net_cfg()})
    assert msg in str(e.value)
    with pytest.raises(tcnn_b200.TcnnError) as e:
        tcnn_b200.Module(n_in, 3, cfg, net_cfg())
    assert msg in str(e.value)


def test_composite_double_backward_still_throws(torch_cuda):
    torch = torch_cuda
    enc, x, xd, p16, orc = encoding_setup(torch, "product_planes", B=256)
    dy = torch.ones(256, orc.width, dtype=torch.float16, device="cuda")
    import tcnn_b200

    with pytest.raises(tcnn_b200.TcnnError, match="Composite does not support double backward."):
        enc.bwd_bwd_input(xd, p16, torch.ones(256, 4, device="cuda"), dy)
