"""The fused training kernel fetches a hashed level's corner pair with one 8-byte load when both entries share an aligned slot
and the level's base is 16-byte aligned (LevelInfo::wide_ok), and with two 4-byte loads otherwise. These tests run training
steps on configurations whose hashed levels take the 4-byte path because their base is NOT 16-byte aligned: with
log2_hashmap_size = 1 every level is a hashed table of two entries, so every other level starts at an offset of 2 (mod 4)
entries, while the levels in between take the merged load. The encoding must stay bit-exact with the oracle on both kinds of
level, and the table gradients must stay within the usual bars.

(A hashed level's table is min(next_multiple(res^D, 8), 2^log2_hashmap_size) entries and is hashed only when that is below
res^D, so hashed tables are powers of two: the fused kernel never meets a hashed level with another size.)
"""
import math

import numpy as np
import pytest

import oracle_binding as ob

pytestmark = pytest.mark.gpu


def rae(a, b, percentile=100.0):
    """tests/test_common.h:59-117: |a-b| / (|a|+|b|)/2 + eps with eps scaled by the mean magnitude, best-p% trimmed mean."""
    a = np.asarray(a, np.float64).ravel()
    b = np.asarray(b, np.float64).ravel()
    eps = 1e-2 * 0.5 * (np.abs(a).mean() + np.abs(b).mean()) + 1e-30
    e = np.abs(a - b) / (0.5 * (np.abs(a) + np.abs(b)) + eps)
    if percentile < 100.0:
        e = np.sort(e)[: max(1, int(len(e) * percentile / 100.0))]
    return float(e.mean())


def config(n_levels):
    return {
        "loss": {"otype": "RelativeL2"},
        "optimizer": {"otype": "Adam", "learning_rate": 1e-2, "beta1": 0.9, "beta2": 0.99, "epsilon": 1e-15, "l2_reg": 1e-6},
        "encoding": {"otype": "HashGrid", "n_levels": n_levels, "n_features_per_level": 2, "log2_hashmap_size": 1, "base_resolution": 4, "per_level_scale": 1.5},
        "network": {"otype": "FullyFusedMLP", "activation": "ReLU", "output_activation": "None", "n_neurons": 64, "n_hidden_layers": 2},
    }


@pytest.mark.parametrize("n_in,n_levels,B", [(3, 16, 256), (2, 12, 256)])
def test_unaligned_hashed_levels_train_like_the_oracle(torch_cuda, n_in, n_levels, B):
    torch = torch_cuda
    import tcnn_b200

    n_out = 3
    cfg = config(n_levels)
    model = tcnn_b200.create_from_config(n_in, n_out, cfg)
    levels = model.grid_levels()
    orc = ob.OracleModel(n_in, n_out, cfg, scales=levels["scales"])
    offsets = levels["offsets"]
    assert offsets == list(orc.grid.offsets[: n_levels + 1])
    # every level is hashed (two entries, far fewer than res^D) and every other one starts off a 16-byte boundary
    sizes = [offsets[i + 1] - offsets[i] for i in range(n_levels)]
    res = [math.ceil(s) + 1 for s in levels["scales"]]
    assert all(sizes[i] == 2 and sizes[i] < res[i] ** n_in for i in range(n_levels))
    assert sum(o % 4 != 0 for o in offsets[:n_levels]) == n_levels // 2

    rng = ob.default_rng(4242)
    x = ob.generate_random_uniform(rng, B * n_in).reshape(B, n_in)
    y = ob.make_targets(x, n_out)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    enc_tap = torch.zeros(B, 64, dtype=torch.float16, device="cuda")
    denc_tap = torch.zeros(B, 64, dtype=torch.float16, device="cuda")
    model.set_debug_taps(encoded=enc_tap, dL_dencoded=denc_tap)
    model.trainer.training_step(xd, yd, run_optimizer=False)
    torch.cuda.synchronize()
    W = orc.grid.padded_width

    enc_dev = enc_tap.cpu().numpy().view(np.uint16)
    assert np.array_equal(enc_dev[:, :W].T, orc.encode(x)), "encoded features differ"

    # table gradients of the device's dL/d(encoded): fp16 atomics against the oracle's exact sums
    denc_dev = np.ascontiguousarray(denc_tap.cpu().numpy().view(np.uint16)[:, :W].T)
    g_ref = orc.grid_backward(x, denc_dev)
    grads = ob.half_bits_to_float(model.trainer.param_gradients().cpu().numpy().view(np.uint16))
    g_dev = grads[orc.n_mlp :].astype(np.float64)
    touched = g_ref != 0
    assert (g_dev[~touched] == 0).all()
    assert rae(g_dev, g_ref.astype(np.float16).astype(np.float64), 99.9) < 1.2e-2

