"""CPU checks of the numpy oracle of the parameter-free encodings (oracle/feature_encodings.py) -- the checker has to be right before
the GPU kernels are compared with it: spherical harmonics against scipy on unit vectors, analytic input gradients against central
differences, OneBlob's partition of unity, Composite's column layout, and -- when the fixtures exist -- the features the unmodified
reference wrote on the GPU (tests/golden/composite_*.npz)."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import feature_encodings as fe  # noqa: E402


def test_spherical_harmonics_match_scipy_on_unit_vectors():
    import scipy.special as sp

    rng = np.random.default_rng(0)
    v = rng.normal(size=(200, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    x = ((v + 1) / 2).astype(np.float64)
    got = fe.spherical_harmonics(x, 8).astype(np.float64)
    theta, phi = np.arccos(v[:, 2]), np.arctan2(v[:, 1], v[:, 0])
    for l in range(8):
        for m in range(-l, l + 1):
            if hasattr(sp, "sph_harm_y"):
                Y = sp.sph_harm_y(l, abs(m), theta, phi)
            else:
                Y = sp.sph_harm(abs(m), l, phi, theta)
            want = Y.real if m == 0 else (np.sqrt(2) * Y.real if m > 0 else np.sqrt(2) * Y.imag)  # Condon-Shortley phase kept, as the reference's polynomials
            assert np.abs(got[:, l * (l + 1) + m] - want).max() < 2e-5, (l, m)
    # the three first-order terms as the reference writes them (common_device.h:485-487): -c y, c z, -c x
    c = 0.48860251190291987
    assert np.allclose(got[:, 1], -c * v[:, 1], atol=1e-6) and np.allclose(got[:, 2], c * v[:, 2], atol=1e-6) and np.allclose(got[:, 3], -c * v[:, 0], atol=1e-6)


def _numeric_grad(f, x, dL_dy, eps=1e-4):
    g = np.zeros_like(x, dtype=np.float64)
    for d in range(x.shape[1]):
        xp, xm = x.copy(), x.copy()
        xp[:, d] += eps
        xm[:, d] -= eps
        g[:, d] = ((f(xp).astype(np.float64) - f(xm).astype(np.float64)) * dL_dy).sum(1) / (2 * eps)
    return g


@pytest.mark.parametrize("name", ["frequency", "oneblob", "spherical_harmonics"])
def test_input_gradients_match_central_differences(name):
    rng = np.random.default_rng(1)
    x = rng.uniform(0.05, 0.95, size=(64, 3)).astype(np.float64)
    if name == "frequency":
        f = lambda v: fe.frequency(v.astype(np.float32), 4)  # noqa: E731
        grad = lambda v, g: fe.frequency_input_gradient(v.astype(np.float32), g.astype(np.float32), 4)  # noqa: E731
        width, tol = 3 * 8, 2e-2
    elif name == "oneblob":
        f = lambda v: fe.oneblob(v.astype(np.float32), 8)  # noqa: E731
        grad = lambda v, g: fe.oneblob_input_gradient(v.astype(np.float32), g.astype(np.float32), 8)  # noqa: E731
        width, tol = 3 * 8, 2e-2
    else:
        f = lambda v: fe.spherical_harmonics(v, 6)  # noqa: E731
        grad = lambda v, g: fe.spherical_harmonics_input_gradient(v, g, 6)  # noqa: E731
        width, tol = 36, 2e-3
    dL_dy = rng.normal(size=(64, width))
    eps = 1e-3 if name != "spherical_harmonics" else 1e-5
    num = _numeric_grad(f, x, dL_dy, eps)
    ana = grad(x, dL_dy).astype(np.float64)
    assert np.abs(num - ana).max() <= tol * max(1.0, np.abs(ana).max()), np.abs(num - ana).max()


def test_oneblob_is_a_partition_of_unity_and_triangle_wave_is_bounded():
    rng = np.random.default_rng(2)
    x = rng.uniform(0, 1, size=(256, 2)).astype(np.float32)
    ob = fe.oneblob(x, 16)
    assert np.allclose(ob[:, :16].sum(1), 1.0, atol=1e-5) and np.allclose(ob[:, 16:].sum(1), 1.0, atol=1e-5) and (ob >= -1e-6).all()
    tw = fe.triangle_wave(x, 12)
    assert tw.min() >= -1.0 - 1e-6 and tw.max() <= 1.0 + 1e-6
    g = fe.triangle_wave_input_gradient(x, np.ones_like(tw), 12)
    assert np.isfinite(g).all()


def test_composite_layout_follows_the_reference_rules():
    # the reference's "NRC" / "OneBlobFrequency" shorthand (src/encoding.cu:97-120) for 10 input dims, in front of a network (alignment 16)
    nrc = {"otype": "Composite", "nested": [{"n_dims_to_encode": 3, "otype": "TriangleWave", "n_frequencies": 12}, {"n_dims_to_encode": 5, "otype": "OneBlob", "n_bins": 4}, {"otype": "Identity"}]}
    segs, width = fe.composite_layout(10, nrc, 16)
    assert [(s[0], s[2], s[3], s[4], s[5], s[6]) for s in segs] == [("trianglewave", 0, 3, 0, 36, 0), ("oneblob", 3, 5, 36, 20, 0), ("identity", 8, 2, 56, 2, 6)] and width == 64
    # a grid behind an odd-width encoding starts at a multiple of its n_features_per_level; spherical harmonics pad in FRONT
    cfg = {"otype": "Composite", "nested": [{"n_dims_to_encode": 3, "otype": "Frequency", "n_frequencies": 1, "n_dims": 0},
                                            {"n_dims_to_encode": 3, "otype": "HashGrid", "n_levels": 2, "n_features_per_level": 4}]}
    segs, width = fe.composite_layout(6, cfg, 16)
    assert segs[0][5] == 6 and segs[0][6] == 2 and segs[1][4] == 8 and width == 16
    cfg = {"otype": "Composite", "nested": [{"n_dims_to_encode": 3, "otype": "HashGrid", "n_levels": 4, "n_features_per_level": 2}, {"otype": "SphericalHarmonics", "degree": 3}]}
    enc, segs, width = fe.encode_plain(np.full((2, 6), 0.25, np.float32), cfg, 16)
    assert width == 32 and segs[1][4] == 8 and segs[1][6] == 15 and segs[1][7]
    assert (enc[:, 8:23] == 1.0).all() and np.isnan(enc[:, :8]).all() and np.isfinite(enc[:, 23:]).all()


GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.mark.parametrize("case", ["composite_nrc", "composite_grid_sh", "frequency_top"])
def test_oracle_matches_reference_dump(case):
    path = os.path.join(GOLDEN, case + ".npz")
    if not os.path.exists(path):
        pytest.skip("fixture not generated yet (tests/golden/make_golden.sh on a GPU box)")
    import json

    z = np.load(path)
    meta = json.loads(bytes(z["meta"]).decode())
    cfg = json.load(open(os.path.join(GOLDEN, "configs", case + ".json")))
    x = z["x_f32"].reshape(-1, meta["n_in"])
    enc_ref = z["encoded_f16"].view(np.float16).astype(np.float32)
    B = x.shape[0]
    enc_ref = enc_ref.reshape(meta["encoded_width"], B).T if meta.get("encoded_layout", "AoS") == "SoA" else enc_ref.reshape(B, meta["encoded_width"])
    enc, segs, width = fe.encode_plain(x, cfg["encoding"], 16)
    assert width == meta["encoded_width"]
    plain = ~np.isnan(enc)
    # fast-math sin / fp16 rounding: a few fp16 ulps of values in [-1, 1]
    assert np.abs(enc[plain] - enc_ref[plain]).max() < 4e-3
    assert (enc[plain].astype(np.float16) != enc_ref[plain].astype(np.float16)).mean() < 0.05
