"""GPU parity at the sizes bench.py actually runs: the BINNED, MULTI-TILE warp-specialised kernel (>= 3 tiles per CTA, enc / park
buffer reuse, the scatter of tile k-2 overlapping the gather of tile k) against

  (1) vectors the UNMODIFIED reference dumped at T = 2^19 with B = 2^16 and 2^18 (`ref_harness dumpbig`, tests/golden/big_*.npz:
      loss trajectory, per-sample heads, [all network weights | every stride-th grid parameter] samples of gradients and
      post-step parameters, touched-set counts) -- same bars as test_against_reference_golden_vectors;
  (2) the CPU oracle on 65 536 samples of the headline configuration (3.5 tiles per CTA), encoded features bit-exact for every sample;
  (3) itself with the binning pass off: identical touched sets.
Plus the configurations round 1 claimed without a GPU test: padded level counts (12 and 5 levels), Tiled grids with an odd
base resolution (unaligned level offsets), Dense grids, Smoothstep, 5 and 6 hidden layers.
"""
import glob
import json
import os

import numpy as np
import pytest

import oracle_binding as ob
from golden_util import GOLDEN, load_case, mlp_gradients_agree, rae

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG_DIR = os.path.join(ROOT, "tests", "golden", "configs")
BIG_CASES = sorted(os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(GOLDEN, "big_*.npz")))


def load_cfg(name):
    return json.load(open(os.path.join(CFG_DIR, name + ".json")))


def f16(t):
    return t.cpu().numpy().view(np.uint16)


def make_batch(n_in, n_out, B, seed=1337):
    rng = ob.default_rng(seed)
    x = ob.generate_random_uniform(rng, B * n_in).reshape(B, n_in)
    return x, ob.make_targets(x, n_out)


def param_sample(a, n_net, stride):
    """[all network weights | every stride-th grid parameter], the layout `ref_harness dumpbig` writes."""
    return np.concatenate([a[:n_net], a[n_net::stride]])


@pytest.mark.skipif(not BIG_CASES, reason="tests/golden/big_*.npz not generated yet (tests/golden/make_golden.sh)")
@pytest.mark.parametrize("name", BIG_CASES)
def test_benchmarked_size_against_reference(torch_cuda, name):
    torch = torch_cuda
    import tcnn_b200

    g = load_case(name)
    meta = g["meta"]
    n_in, n_out, B, stride, H = meta["n_in"], meta["n_out"], meta["batch"], meta["stride"], meta["n_head"]
    cfg = meta["config"]
    n_net = meta["n_network_params"]
    model = tcnn_b200.create_from_config(n_in, n_out, cfg)
    assert model.n_params == meta["n_params"] and model.n_mlp_params == n_net
    assert B // 128 >= 3 * 148, "the point of this test: several tiles per CTA"

    # the batch is regenerated from the seed; its sums pin it to the one the reference trained on
    x, y = make_batch(n_in, n_out, B, meta["input_seed"])
    assert abs(float(x.sum(dtype=np.float64)) - meta["sum_x"]) <= 1e-9 * abs(meta["sum_x"])
    assert abs(float(y.sum(dtype=np.float64)) - meta["sum_y"]) <= 1e-6 * abs(meta["sum_y"])
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()

    p0 = model.trainer.params_full_precision().cpu().numpy()
    assert np.array_equal(param_sample(p0, n_net, stride).view(np.uint32), g["params_init_f32"].view(np.uint32))

    enc_tap = torch.zeros(B, 64, dtype=torch.float16, device="cuda")
    out_tap = torch.zeros(B, 16, dtype=torch.float16, device="cuda")
    lv_tap = torch.zeros(B, n_out, dtype=torch.float32, device="cuda")
    model.set_debug_taps(encoded=enc_tap, output=out_tap, loss_values=lv_tap)

    inf = model.network.inference(xd).cpu().numpy()
    assert rae(inf[:H], g["inference_head_f32"].reshape(H, n_out), 99.0) < 1e-2  # tests/test_common.h:177

    model.trainer.training_step(xd, yd, run_optimizer=False)
    loss0 = model.trainer.loss()
    torch.cuda.synchronize()
    W = meta["encoded_width"]
    # encoded features of the first H samples == the reference's kernel_grid output, bit for bit (through the binning permutation)
    assert np.array_equal(f16(enc_tap)[:H, :W].T, g["encoded_head_f16"].reshape(W, H))
    a = ob.half_bits_to_float(f16(out_tap))[:H, :n_out]
    b = ob.half_bits_to_float(g["output_head_f16"].reshape(H, 16))[:, :n_out]
    assert rae(a, b, 99.0) < 1e-2
    assert abs(loss0 - meta["losses"][0]) <= 1e-3 * meta["losses"][0]
    assert rae(lv_tap.cpu().numpy()[:H], g["loss_values_head_f32"].reshape(H, 16)[:, :n_out], 99.0) < 1e-2

    grads = ob.half_bits_to_float(f16(model.trainer.param_gradients()))
    gs = param_sample(grads, n_net, stride)
    ref = ob.half_bits_to_float(g["grads_step0_f16"])
    # network weight gradients: fp32 (wgmma) vs fp16 split-K accumulation in the reference -> the relaxed 2e-2 bar, this row only
    assert mlp_gradients_agree(gs[:n_net], ref[:n_net], 2e-2)
    # Grid gradients. At these batch sizes every coarse entry receives hundreds of fp16 atomic addends and the REFERENCE's result is
    # itself 1-2e-2 (RAE) away from the exact sums (`grads_exact_f32`: the oracle's double-accumulated sums, added to the fixture by
    # tests/golden/add_exact_grads.py), so the small-batch bar of tests/test_common.h:218 cannot hold between two fp16-atomic
    # implementations. The bar here: this library is no further from the exact sums than the reference is (25 % slack for the
    # different summation order), and the two agree to within the sum of their distances from the truth.
    exact = g["grads_exact_f32"]
    ref_err = rae(ref[n_net:], exact[n_net:], 99.9)
    own_err = rae(gs[n_net:], exact[n_net:], 99.9)
    assert own_err <= max(1.2e-2, 1.25 * ref_err), (own_err, ref_err)
    assert rae(gs[n_net:], ref[n_net:], 99.9) <= max(1.2e-2, 1.1 * (own_err + ref_err)), (own_err, ref_err)
    assert ((gs[n_net:] != 0) != (ref[n_net:] != 0)).mean() < 2e-3
    n_nonzero = int((grads[n_net:] != 0).sum())
    assert abs(n_nonzero - meta["n_grid_grad_nonzero"]) <= 2e-3 * meta["n_grid_grad_nonzero"], (n_nonzero, meta["n_grid_grad_nonzero"])

    lr = cfg["optimizer"]["learning_rate"]
    model.set_debug_taps()
    model.trainer.training_step(xd, yd)
    losses = [loss0, model.trainer.loss()]
    p1 = model.trainer.params_full_precision().cpu().numpy()
    d = np.abs(param_sample(p1, n_net, stride) - g["params_step1_f32"])
    assert np.percentile(d, 99) < 2e-2 * lr and d.mean() < 1e-2 * lr
    n_moved = int((p1[n_net:] != p0[n_net:]).sum())
    assert abs(n_moved - meta["n_grid_params_moved_step1"]) <= 2e-3 * meta["n_grid_params_moved_step1"]
    for _ in range(meta["n_steps"] - 1):
        model.trainer.training_step(xd, yd)
        losses.append(model.trainer.loss())
    for mine, theirs in zip(losses, meta["losses"]):
        assert abs(mine - theirs) <= 3e-2 * abs(theirs), (losses, meta["losses"])
    out = model.network.inference(xd).cpu().numpy()
    assert rae(out[:H], g["inference_final_head_f32"].reshape(H, n_out), 99.0) < 5e-2
    pf = ob.half_bits_to_float(param_sample(f16(model.trainer.params()), n_net, stride))
    assert np.abs(pf - ob.half_bits_to_float(g["params_final_f16"])).mean() < 0.05 * lr * meta["n_steps"]


def test_multi_tile_binned_kernel_matches_oracle(torch_cuda):
    """65 536 samples of the headline configuration (T = 2^19): 512 tiles on 132 persistent CTAs (H100) -> 3-4 tiles per CTA, binning on.
    Every sample's encoding is bit-exact with the oracle; gradients within the reference's bars of the oracle's exact sums; the
    binned and the unbinned step touch exactly the same table entries."""
    torch = torch_cuda
    import tcnn_b200

    cfg = load_cfg("headline")
    B = 1 << 16
    model = tcnn_b200.create_from_config(3, 3, cfg)
    orc = ob.OracleModel(3, 3, cfg, scales=model.grid_levels()["scales"])
    x, y = make_batch(3, 3, B, seed=4242)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    enc_tap = torch.zeros(B, 64, dtype=torch.float16, device="cuda")
    out_tap = torch.zeros(B, 16, dtype=torch.float16, device="cuda")
    denc_tap = torch.zeros(B, 64, dtype=torch.float16, device="cuda")
    model.set_debug_taps(encoded=enc_tap, output=out_tap, dL_dencoded=denc_tap)
    model.trainer.training_step(xd, yd, run_optimizer=False)
    loss = model.trainer.loss()
    g_binned = ob.half_bits_to_float(f16(model.trainer.param_gradients()))
    W = 32
    enc_dev = f16(enc_tap)
    enc_ref, idx = orc.encode(x, want_indices=True)
    assert np.array_equal(enc_dev[:, :W].T, enc_ref), "encoded features differ"
    # the set of table entries any sample indexes (from the oracle's integer indices): gradients elsewhere must stay exactly zero
    offsets = np.asarray(orc.grid.offsets[: orc.grid.n_levels], np.int64)
    indexed = np.zeros(orc.grid.n_params // 2, bool)
    indexed[(idx.astype(np.int64) + offsets[None, :, None]).ravel()] = True
    indexed = np.repeat(indexed, 2)  # F = 2 parameters per entry
    del idx
    _, out_ref = orc.mlp_forward(np.ascontiguousarray(enc_dev[:, :W].T))
    a, b = ob.half_bits_to_float(f16(out_tap)), ob.half_bits_to_float(out_ref)
    assert rae(a[:, :3], b[:, :3]) < 1e-3
    ref_loss = orc.training_step(x, y, run_optimizer=False)
    assert abs(loss - ref_loss) <= 1e-3 * abs(ref_loss)
    g_ref = ob.half_bits_to_float(orc.grads_fp16)
    n_mlp = orc.n_mlp
    assert rae(g_binned[:n_mlp], g_ref[:n_mlp], 99.9) < 1.2e-2
    # grid scatter of the DEVICE's dL/d(encoded) (isolates the scatter from MLP rounding): exact sums vs fp16 reductions
    g_scatter = orc.grid_backward(x, np.ascontiguousarray(f16(denc_tap)[:, :W].T))
    gd = g_binned[n_mlp:].astype(np.float64)
    assert rae(gd, g_scatter.astype(np.float16).astype(np.float64), 99.9) < 1.2e-2
    assert (gd[~indexed] == 0).all(), "gradient written to an entry no sample indexes"
    # entries whose exact sum is non-zero are non-zero on the device too, up to sums that round to zero in fp16
    assert ((gd == 0) & (np.abs(g_scatter) > 2.0 ** -20)).mean() < 1e-4

    # binning off: same sums in a different order -> same touched set, values within fp16 reduction noise
    model.debug_set("binning", 0)
    model.trainer.training_step(xd, yd, run_optimizer=False)
    loss_u = model.trainer.loss()
    g_unbinned = ob.half_bits_to_float(f16(model.trainer.param_gradients()))
    model.debug_set("binning", 1)
    assert abs(loss_u - loss) <= 1e-4 * abs(loss)
    # identical touched sets up to sums that cancel to exactly zero in one order only
    assert ((g_unbinned[n_mlp:] != 0) != (g_binned[n_mlp:] != 0)).mean() < 1e-4
    assert ((g_unbinned[n_mlp:] != 0) & ~indexed).sum() == 0
    assert rae(g_unbinned[n_mlp:], g_binned[n_mlp:], 99.9) < 5e-3


def _variant(base, **enc_or_net):
    cfg = load_cfg(base)
    for k, v in enc_or_net.items():
        section, key = k.split("__")
        cfg[section][key] = v
    return cfg


VARIANTS = {
    # 12 levels -> 24 features padded to 32, 5 levels -> 10 padded to 16: the padding columns of the first-layer tile must be zero
    "levels12": (3, _variant("hash3d_small", encoding__n_levels=12)),
    "levels5": (3, _variant("hash3d_small", encoding__n_levels=5)),
    # Tiled grid, base_resolution 5: levels of 125 entries -> level offsets that are not multiples of 4 (no merged reductions)
    "tiled_odd": (3, _variant("hash3d_small", encoding__otype="TiledGrid", encoding__base_resolution=5, encoding__n_levels=6)),
    "tiled2d_odd": (2, _variant("image2d", encoding__otype="TiledGrid", encoding__base_resolution=3, encoding__n_levels=8)),
    "dense": (3, _variant("hash3d_small", encoding__otype="DenseGrid", encoding__base_resolution=4, encoding__n_levels=5, encoding__per_level_scale=1.5)),
    "smoothstep": (3, _variant("hash3d_small", encoding__interpolation="Smoothstep")),
    "hidden5": (3, _variant("hash3d_small", network__n_hidden_layers=5)),
    "hidden6_wide_enc": (3, _variant("hash3d_small", network__n_hidden_layers=6, encoding__n_levels=24, encoding__log2_hashmap_size=12)),
}


@pytest.mark.parametrize("name", list(VARIANTS))
def test_configuration_variants_match_oracle(torch_cuda, name):
    torch = torch_cuda
    import tcnn_b200

    n_in, cfg = VARIANTS[name]
    B = 1024
    model = tcnn_b200.create_from_config(n_in, 3, cfg)
    levels = model.grid_levels()
    orc = ob.OracleModel(n_in, 3, cfg, scales=levels["scales"])
    assert model.n_params == orc.n_params and levels["offsets"] == list(orc.grid.offsets[: orc.grid.n_levels + 1])
    assert np.array_equal(model.trainer.params_full_precision().cpu().numpy().view(np.uint32), orc.params_fp32.view(np.uint32))
    x, y = make_batch(n_in, 3, B, seed=77)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    enc_tap = torch.full((B, 64), float("nan"), dtype=torch.float16, device="cuda")
    model.set_debug_taps(encoded=enc_tap)
    model.trainer.training_step(xd, yd, run_optimizer=False)
    loss = model.trainer.loss()
    torch.cuda.synchronize()
    W = orc.grid.padded_width
    n_feat = orc.grid.n_levels * 2
    assert np.array_equal(f16(enc_tap)[:, :n_feat].T, orc.encode(x)[:n_feat]), "encoded features differ"
    ref_loss = orc.training_step(x, y, run_optimizer=False)
    assert np.isfinite(loss) and abs(loss - ref_loss) <= 2e-3 * abs(ref_loss) + 1e-7, (loss, ref_loss)
    g_dev = ob.half_bits_to_float(f16(model.trainer.param_gradients()))
    g_ref = ob.half_bits_to_float(orc.grads_fp16)
    assert np.isfinite(g_dev).all()
    n_mlp = orc.n_mlp
    # first-layer weight gradients of the padding columns are exactly zero (the padded features are zero, grid.h:757-766)
    w0 = g_dev[: cfg["network"]["n_neurons"] * W].reshape(cfg["network"]["n_neurons"], W)
    assert (w0[:, n_feat:] == 0).all()
    assert rae(g_dev[:n_mlp], g_ref[:n_mlp], 99.9) < 1.2e-2
    assert rae(g_dev[n_mlp:], g_ref[n_mlp:], 99.9) < 1.2e-2
    assert ((g_dev[n_mlp:] != 0) != (g_ref[n_mlp:] != 0)).mean() < 2e-3
    dev_losses, ref_losses = [], []
    model.set_debug_taps()
    for _ in range(5):
        model.trainer.training_step(xd, yd)
        dev_losses.append(model.trainer.loss())
        ref_losses.append(orc.training_step(x, y))
    for a, b in zip(dev_losses, ref_losses):
        assert abs(a - b) <= 3e-2 * abs(b) + 1e-6, (dev_losses, ref_losses)
    assert rae(model.network.inference(xd).cpu().numpy(), orc.inference(x), 99.0) < 5e-2


def test_pipelined_host_steps_equal_synchronous_steps(torch_cuda):
    """tcnnb_training_step_host_submit / _wait with two steps in flight == the same steps one at a time (same losses, same
    parameters up to the order of the fp16 reductions), pageable and page-locked caller buffers alike; misuse fails loudly."""
    torch = torch_cuda
    import tcnn_b200

    cfg = load_cfg("hash3d_small")
    B = 32768
    batches = [make_batch(3, 3, B, seed=100 + i) for i in range(4)]
    a = tcnn_b200.create_from_config(3, 3, cfg)
    b = tcnn_b200.create_from_config(3, 3, cfg)
    ref_losses = [a.training_step_host(x, y) for x, y in batches]
    pinned = [(torch.from_numpy(x).pin_memory().numpy(), torch.from_numpy(y).pin_memory().numpy()) for x, y in batches[:2]] + batches[2:]
    got = []
    prev = b.training_step_host_submit(*pinned[0])
    for x, y in pinned[1:]:
        cur = b.training_step_host_submit(x, y)
        got.append(b.training_step_host_wait(prev))
        prev = cur
    t3 = b.training_step_host_submit(*pinned[0])
    with pytest.raises(tcnn_b200.TcnnError, match="already in flight"):
        b.training_step_host_submit(*pinned[1])
    got.append(b.training_step_host_wait(prev))
    b.training_step_host_wait(t3)
    with pytest.raises(tcnn_b200.TcnnError, match="not in flight"):
        b.training_step_host_wait(t3)
    for u, v in zip(got, ref_losses):
        assert abs(u - v) <= 2e-3 * abs(v), (got, ref_losses)
    a.training_step_host(*batches[0])
    pa = a.trainer.params_full_precision().cpu().numpy()
    pb = b.trainer.params_full_precision().cpu().numpy()
    assert np.abs(pa - pb).mean() < 0.05 * cfg["optimizer"]["learning_rate"]
