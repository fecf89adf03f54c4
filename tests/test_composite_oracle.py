"""The numpy restatement of Composite's reductions, dims_to_encode_begin, Empty and NRC (tests/composite_oracle.py): layout rules,
errors, the reduction's backward pass against finite differences, and the encoded features of the reference's fixtures
(tests/golden/{composite_sum_hash3d,composite_product_planes,composite_product_pad,composite_empty,nrc_top}.npz, written by the
unmodified reference with tests/golden/make_golden_composite.sh). CPU only."""
import json
import os

import numpy as np
import pytest

import composite_oracle as co
from golden_util import GOLDEN

HG = {"otype": "HashGrid", "n_levels": 8, "n_features_per_level": 2, "log2_hashmap_size": 14, "base_resolution": 16, "per_level_scale": 1.5}


def test_sum_and_product_pad_every_nested_encoding_to_one_width():
    cfg = {"otype": "Composite", "reduction": "Sum", "nested": [dict(HG, n_dims_to_encode=3, dims_to_encode_begin=0), dict(HG, n_dims_to_encode=3, dims_to_encode_begin=0, log2_hashmap_size=12)]}
    segs, width, red = co.layout(3, cfg, 16)
    assert red == "sum" and width == 16 and [(s[2], s[3], s[4], s[5], s[6]) for s in segs] == [(0, 3, 0, 16, 0), (0, 3, 16, 16, 0)]
    # grid (4 columns) x Identity (4 columns): equal widths; the network's alignment pads both to 16, zeros behind the grid, ones behind Identity
    cfg = {"otype": "Composite", "reduction": "product", "nested": [dict(HG, n_dims_to_encode=4, n_levels=2, dims_to_encode_begin=0), {"otype": "Identity", "n_dims_to_encode": 4, "dims_to_encode_begin": 0}]}
    segs, width, _ = co.layout(4, cfg, 16)
    assert width == 16 and [(s[4], s[5], s[6]) for s in segs] == [(0, 4, 12), (16, 4, 12)]
    x = np.full((2, 4), 0.5, np.float32)
    rows, _, _, _ = co.encode_nested(x, cfg, 16)
    rows[:, :4] = 0.25  # stand-in grid features
    out = co.reduce_forward(co.slabs_of(rows, 2, 16), "product").astype(np.float32)
    assert (out[:, :4] == np.float32(np.float16(0.125))).all() and (out[:, 4:] == 0).all()
    # without a consumer alignment (the encoding tier) an odd common width stays odd: Identity and one-frequency TriangleWave over 3 dims
    cfg = {"otype": "Composite", "reduction": "Sum", "nested": [{"otype": "Identity", "n_dims_to_encode": 3, "dims_to_encode_begin": 0}, {"otype": "TriangleWave", "n_frequencies": 1, "n_dims_to_encode": 3, "dims_to_encode_begin": 0}]}
    assert co.layout(3, cfg, 0)[1] == 3 and co.layout(3, cfg, 16)[1] == 16
    # grids of F = 4 force the lcm: a 6-wide TriangleWave pads to 8 next to an 8-wide grid
    cfg = {"otype": "Composite", "reduction": "Sum", "nested": [dict(HG, n_dims_to_encode=2, n_levels=2, n_features_per_level=4), {"otype": "TriangleWave", "n_frequencies": 3, "n_dims_to_encode": 2, "dims_to_encode_begin": 0}]}
    segs, width, _ = co.layout(2, cfg, 0)
    assert width == 8 and segs[1][5:7] == (6, 2)


def test_dims_to_encode_begin_sets_the_offset_and_later_entries_continue_from_it():
    cfg = {"otype": "Composite", "nested": [{"otype": "Identity", "n_dims_to_encode": 2, "dims_to_encode_begin": 3}, {"otype": "Identity", "n_dims_to_encode": 1},
                                            {"otype": "Frequency", "n_frequencies": 1, "n_dims_to_encode": 3, "dims_to_encode_begin": 0}]}
    segs, width, _ = co.layout(6, cfg, 0)
    assert [(s[2], s[3]) for s in segs] == [(3, 2), (5, 1), (0, 3)] and width == 2 + 1 + 6
    # with a begin anywhere, the total may exceed n_in (overlap) ...
    cfg = {"otype": "Composite", "reduction": "Product", "nested": [dict(HG, n_dims_to_encode=2, dims_to_encode_begin=b) for b in (0, 1, 2)]}
    segs, width, _ = co.layout(4, cfg, 16)
    assert [(s[2], s[3], s[4]) for s in segs] == [(0, 2, 0), (1, 2, 16), (2, 2, 32)] and width == 16
    # ... and begin is read only together with n_dims_to_encode: the NRC expansion of 9 dims
    segs, width, _ = co.layout(9, {"otype": "NRC"}, 16)
    assert [(s[0], s[2], s[3], s[4], s[5], s[6]) for s in segs] == [("trianglewave", 0, 3, 0, 36, 0), ("oneblob", 3, 5, 36, 20, 0), ("identity", 8, 1, 56, 1, 7)] and width == 64


def test_nrc_shorthand_defaults_and_overrides():
    e = co.expand({"otype": "oneblobfrequency"})
    assert e["nested"][0]["n_frequencies"] == 12 and e["nested"][1]["n_bins"] == 4
    e = co.expand({"otype": "NRC", "n_frequencies": 4, "n_bins": 8})
    assert e["nested"][0]["n_frequencies"] == 4 and e["nested"][1]["n_bins"] == 8
    # exactly 8 dims: the Identity has nothing left and is skipped
    segs, width, _ = co.layout(8, {"otype": "NRC"}, 16)
    assert [s[0] for s in segs] == ["trianglewave", "oneblob"] and width == 64


def test_empty_has_no_columns_and_pads_with_ones():
    cfg = {"otype": "Composite", "nested": [dict(HG, n_dims_to_encode=3), {"otype": "Empty", "n_dims_to_encode": 2}, {"otype": "Identity", "n_dims_to_encode": 1}]}
    segs, width, _ = co.layout(6, cfg, 16)
    assert [(s[0], s[2], s[3], s[4], s[5], s[6]) for s in segs] == [("hashgrid", 0, 3, 0, 16, 0), ("empty", 3, 2, 16, 0, 0), ("identity", 5, 1, 16, 1, 15)] and width == 32
    rows, _, _, _ = co.encode_nested(np.full((2, 6), 0.25, np.float32), cfg, 16)
    assert (rows[:, 16] == 0.25).all() and (rows[:, 17:] == 1).all()
    # top level, in front of a network: 16 columns of ones; in the encoding tier: no columns
    segs, width, _ = co.layout(3, {"otype": "Empty"}, 16)
    assert width == 16 and segs[0][6] == 16
    assert co.layout(3, {"otype": "Empty"}, 0)[1] == 0
    # last in a concatenation, Empty carries the final padding
    segs, width, _ = co.layout(3, {"otype": "Composite", "nested": [{"otype": "Identity", "n_dims_to_encode": 1}, {"otype": "Empty"}]}, 16)
    assert width == 16 and segs[1][6] == 15


ERRORS = [
    ("Invalid reduction type: Mean", 3, {"otype": "Composite", "reduction": "Mean", "nested": [{"otype": "Identity"}]}),
    ("must have equal output widths", 3, {"otype": "Composite", "reduction": "Sum", "nested": [dict(HG, n_dims_to_encode=3), {"otype": "Identity", "n_dims_to_encode": 3, "dims_to_encode_begin": 0}]}),
    ("reads input dims [2, 4)", 3, {"otype": "Composite", "nested": [{"otype": "Identity", "n_dims_to_encode": 2, "dims_to_encode_begin": 2}]}),
    ("may only leave 'n_dims_to_encode' unspecified", 3, {"otype": "Composite", "nested": [{"otype": "Identity", "n_dims_to_encode": 1, "dims_to_encode_begin": 0}, {"otype": "Identity"}]}),
    ("may only leave 'n_dims_to_encode' unspecified", 3, {"otype": "Composite", "nested": [{"otype": "Identity"}, {"otype": "Identity"}]}),
    ("nested inside a Composite", 3, {"otype": "Composite", "nested": [{"otype": "Composite", "nested": [{"otype": "Identity"}]}]}),
    ("nested inside a Composite", 9, {"otype": "Composite", "nested": [{"otype": "NRC"}]}),
    ("must not encode more dims 4 than composite 3", 3, {"otype": "Composite", "nested": [{"otype": "Identity", "n_dims_to_encode": 4}]}),
]


@pytest.mark.parametrize("i", range(len(ERRORS)))
def test_invalid_configurations_raise(i):
    msg, n_in, cfg = ERRORS[i]
    with pytest.raises(ValueError, match=None) as e:
        co.layout(n_in, cfg, 16)
    assert msg in str(e.value), str(e.value)


@pytest.mark.parametrize("reduction", ["sum", "product"])
def test_reduce_backward_matches_finite_differences(reduction):
    rng = np.random.default_rng(5)
    K, n, w = 3, 16, 5
    slabs = [rng.uniform(-1.5, 1.5, size=(n, w)) for _ in range(K)]
    dy = rng.normal(size=(n, w))
    grads = co.reduce_backward(dy, slabs, reduction, exact=True)
    eps = 1e-6
    for k in range(K):
        num = np.zeros((n, w))
        for j in range(w):
            plus = [s.copy() for s in slabs]
            minus = [s.copy() for s in slabs]
            plus[k][:, j] += eps
            minus[k][:, j] -= eps
            num[:, j] = ((co.reduce_forward(plus, reduction, exact=True) - co.reduce_forward(minus, reduction, exact=True)) * dy).sum(1) / (2 * eps)
        assert np.abs(num - grads[k]).max() < 1e-6
    # the fp16 variant: the reference's rounding, one per value
    g16 = co.reduce_backward(dy.astype(np.float16), [s.astype(np.float16) for s in slabs], reduction)
    assert all(g.dtype == np.float16 for g in g16)
    assert max(np.abs(g.astype(np.float64) - e).max() for g, e in zip(g16, co.reduce_backward(dy.astype(np.float16).astype(np.float64), [s.astype(np.float16).astype(np.float64) for s in slabs], reduction, exact=True))) < 1e-2


def test_product_of_zero_is_exact_and_sum_is_ordered():
    a = np.array([[0.0, 1e-3]], np.float16)
    b = np.array([[7.0, 3.0]], np.float16)
    g = co.reduce_backward(np.ones((1, 2), np.float16), [a, b], "product")
    assert g[0][0, 0] == 7 and g[1][0, 0] == 0
    # fp32 accumulation, rounded once: 2048 + 1 + 1 in fp16 steps would stay 2048
    s = co.reduce_forward([np.array([[2048.0]], np.float16), np.array([[1.0]], np.float16), np.array([[1.0]], np.float16)], "sum")
    assert s[0, 0] == 2050


FIXTURES = ["composite_sum_hash3d", "composite_product_planes", "composite_product_pad", "composite_empty", "nrc_top"]


@pytest.mark.parametrize("case", FIXTURES)
def test_oracle_layout_and_plain_features_match_the_reference_fixture(case):
    path = os.path.join(GOLDEN, case + ".npz")
    z = np.load(path)
    meta = json.loads(bytes(z["meta"]).decode())
    cfg = json.load(open(os.path.join(GOLDEN, "configs", case + ".json")))
    B, n_in = meta["batch"], meta["n_in"]
    x = z["x_f32"].reshape(B, n_in)
    W = meta["encoded_width"]
    enc_ref = z["encoded_f16"].view(np.float16).astype(np.float32)
    enc_ref = enc_ref.reshape(W, B).T if meta.get("encoded_layout", "AoS") == "SoA" else enc_ref.reshape(B, W)
    rows, segs, width, red = co.encode_nested(x, cfg["encoding"], 16)
    assert width == W
    if red == "concatenation":
        want = rows
    else:
        # a reduced column is known where no grid feature enters it; grid padding is zero, so a Product column with one is zero
        slabs = co.slabs_of(rows, len(segs), width)
        known = np.all([~np.isnan(s) for s in slabs], axis=0)
        want = np.full((B, width), np.nan, np.float32)
        red_vals = co.reduce_forward([np.nan_to_num(s) for s in slabs], red).astype(np.float32)
        want[known] = red_vals[known]
        if red == "product":
            zero = np.any([(s == 0) for s in slabs], axis=0)
            want[zero] = 0.0
    plain = ~np.isnan(want)
    if case == "nrc_top":
        assert plain.all()
    if case == "composite_product_pad":
        assert plain[:, 4:].all() and (want[:, 4:] == 0).all()
    if not plain.any():  # nothing but grid features: the GPU tests compare those
        return
    # fast-math sin / fp16 rounding: a few fp16 ulps of values in [-1, 1]; identity and padding are exact
    assert np.abs(want[plain] - enc_ref[plain]).max() < 4e-3
    assert (want[plain].astype(np.float16) != enc_ref[plain].astype(np.float16)).mean() < 0.05
