"""oracle/feature_encodings.py -- numpy restatement of the reference's parameter-free encodings and of Composite's column layout.

TEST INFRASTRUCTURE ONLY (see oracle/README.md): imported by tests/ to check csrc/feature_encodings.cu; the product never imports it.
Each function cites the reference lines it restates. fp32 arithmetic like the kernels (the reference compiles them with
--use_fast_math, so sin / cos are approximations there: comparisons use a tolerance of a few fp16 ulps, stated in the tests).

Pinned by: tests/golden/composite_*.npz (encoded features dumped from the unmodified reference on the GPU, tests/golden/make_golden.sh)
and, for the spherical harmonics, scipy.special on unit vectors (tests/test_feature_oracle.py).
"""
import math

import numpy as np

F32 = np.float32


def identity(x, scale=1.0, offset=0.0):
    """encodings/identity.h:46-67: y_j = x_j * scale + offset."""
    return (x.astype(F32) * F32(scale) + F32(offset)).astype(F32)


def frequency(x, n_frequencies):
    """encodings/frequency.h:46-82: for input d, frequency f: sin(2^f pi x), sin(2^f pi x + pi/2); column d * 2F + 2f + k."""
    n, D = x.shape
    out = np.zeros((n, D * n_frequencies * 2), F32)
    for d in range(D):
        for f in range(n_frequencies):
            arg = (x[:, d].astype(F32) * F32(2.0 ** f)) * F32(math.pi)
            out[:, d * 2 * n_frequencies + 2 * f] = np.sin(arg, dtype=F32)
            out[:, d * 2 * n_frequencies + 2 * f + 1] = np.sin(arg + F32(math.pi / 2), dtype=F32)
    return out


def frequency_input_gradient(x, dL_dy, n_frequencies):
    """encodings/frequency.h:78-103: dy/dx = 2^f pi cos(.), summed over the outputs of an input."""
    n, D = x.shape
    out = np.zeros((n, D), F32)
    for d in range(D):
        for f in range(n_frequencies):
            arg = (x[:, d].astype(F32) * F32(2.0 ** f)) * F32(math.pi)
            k = F32(2.0 ** f) * F32(math.pi)
            out[:, d] += dL_dy[:, d * 2 * n_frequencies + 2 * f] * k * np.cos(arg, dtype=F32)
            out[:, d] += dL_dy[:, d * 2 * n_frequencies + 2 * f + 1] * k * np.cos(arg + F32(math.pi / 2), dtype=F32)
    return out


def triangle_wave(x, n_frequencies):
    """encodings/triangle_wave.h:46-82: v = 2^(f-1) x + f / 4; y = |v - floor(v) - 1/2| * 4 - 1; column d * F + f."""
    n, D = x.shape
    out = np.zeros((n, D * n_frequencies), F32)
    for d in range(D):
        for f in range(n_frequencies):
            val = x[:, d].astype(F32) * F32(2.0 ** (f - 1)) + F32(f * 0.25)
            out[:, d * n_frequencies + f] = np.abs(val - np.floor(val) - F32(0.5)) * F32(4) - F32(1)
    return out


def triangle_wave_input_gradient(x, dL_dy, n_frequencies):
    """encodings/triangle_wave.h:78-105: slope -+ 2^(f+1) by the parity of floor(2 v)."""
    n, D = x.shape
    out = np.zeros((n, D), F32)
    for d in range(D):
        for f in range(n_frequencies):
            val = x[:, d].astype(F32) * F32(2.0 ** (f - 1)) + F32(f * 0.25)
            sign = np.where(np.floor(val * F32(2)).astype(np.int64) % 2 == 0, F32(-1), F32(1))
            out[:, d] += dL_dy[:, d * n_frequencies + f] * sign * F32(2.0 ** (f + 1))
    return out


def _quartic_cdf(x, inv_radius):
    """common_device.h:1090-1095."""
    u = (x * F32(inv_radius)).astype(F32)
    u2 = u * u
    u4 = u2 * u2
    return np.clip(F32(15.0 / 16.0) * u * (F32(1) - F32(2.0 / 3.0) * u2 + F32(1.0 / 5.0) * u4) + F32(0.5), F32(0), F32(1)).astype(F32)


def _quartic_cdf_deriv(x, inv_radius):
    """common_device.h:1080-1088."""
    u = (x * F32(inv_radius)).astype(F32)
    tmp = np.maximum(F32(1) - u * u, F32(0))
    return (F32(15.0 / 16.0) * tmp * tmp * F32(inv_radius)).astype(F32)


def _wrapped(fn, boundary, x, n_bins):
    b = F32(boundary)
    return fn(b - x, n_bins) + fn(b - x - F32(1), n_bins) + fn(b - x + F32(1), n_bins)


def oneblob(x, n_bins):
    """encodings/oneblob.h:47-120: bin b of input d = CDF(right boundary) - CDF(left boundary) of a quartic kernel of radius 1 / n_bins
    centred on x, wrapping around [0, 1) (three kernel images); column d * n_bins + b."""
    n, D = x.shape
    out = np.zeros((n, D * n_bins), F32)
    for d in range(D):
        xd = x[:, d].astype(F32)
        left = _wrapped(_quartic_cdf, 0.0, xd, n_bins)
        for b in range(n_bins):
            right = _wrapped(_quartic_cdf, (b + 1) / n_bins, xd, n_bins)
            out[:, d * n_bins + b] = right - left
            left = right
    return out


def oneblob_input_gradient(x, dL_dy, n_bins):
    """encodings/oneblob.h:122-160."""
    n, D = x.shape
    out = np.zeros((n, D), F32)
    for d in range(D):
        xd = x[:, d].astype(F32)
        left = _wrapped(_quartic_cdf_deriv, 0.0, xd, n_bins)
        for b in range(n_bins):
            right = _wrapped(_quartic_cdf_deriv, (b + 1) / n_bins, xd, n_bins)
            out[:, d] += dL_dy[:, d * n_bins + b] * (left - right)
            left = right
    return out


def _sh_terms(degree, x, y, z):
    """Real spherical harmonics as the polynomials the reference hard-codes (common_device.h:476-..., generated from the recurrences of
    Sloan, 'Stupid Spherical Harmonics Tricks', appendix A1): Y_l^m = K_l^m P_l^m(z) {sqrt2 Re, 1, sqrt2 Im}(x + i y)^|m| with the
    Legendre factors as polynomials in z. float64 here. Returns [(index, value, d/dx, d/dy, d/dz)]."""
    x, y, z = (np.asarray(v, np.float64) for v in (x, y, z))
    terms = []
    c, s = np.ones_like(x), np.zeros_like(x)
    c_prev, s_prev = np.zeros_like(x), np.zeros_like(x)
    pmm = 1.0
    for m in range(degree):
        if m > 0:
            c_prev, s_prev = c, s
            c, s = x * c_prev - y * s_prev, x * s_prev + y * c_prev
            pmm *= 1.0 - 2.0 * m
        dc_dx, dc_dy, ds_dx, ds_dy = m * c_prev, -m * s_prev, m * s_prev, m * c_prev
        p2 = p1 = dp2 = dp1 = None
        for l in range(m, degree):
            if l == m:
                p, dp = np.full_like(x, pmm), np.zeros_like(x)
            elif l == m + 1:
                p, dp = (2 * m + 1) * z * p1, (2 * m + 1) * p1
            else:
                p = ((2 * l - 1) * z * p1 - (l + m - 1) * p2) / (l - m)
                dp = ((2 * l - 1) * (p1 + z * dp1) - (l + m - 1) * dp2) / (l - m)
            p2, dp2, p1, dp1 = p1, dp1, p, dp
            K = math.sqrt((2 * l + 1) * math.factorial(l - m) / (4 * math.pi * math.factorial(l + m)))
            base = l * (l + 1)
            if m == 0:
                terms.append((base, K * p, np.zeros_like(x), np.zeros_like(x), K * dp))
            else:
                K *= math.sqrt(2.0)
                terms.append((base + m, K * p * c, K * p * dc_dx, K * p * dc_dy, K * dp * c))
                terms.append((base - m, K * p * s, K * p * ds_dx, K * p * ds_dy, K * dp * s))
    return terms


def spherical_harmonics(x, degree):
    """encodings/spherical_harmonics.h:44-72: direction d = 2 x - 1 (NOT normalised), degree^2 coefficients."""
    d = x.astype(np.float64) * 2.0 - 1.0
    out = np.zeros((x.shape[0], degree * degree), np.float64)
    for idx, v, _, _, _ in _sh_terms(degree, d[:, 0], d[:, 1], d[:, 2]):
        out[:, idx] = v
    return out.astype(F32)


def spherical_harmonics_input_gradient(x, dL_dy, degree):
    """encodings/spherical_harmonics.h:74-100: 2 * sum_k dL_dy_k grad Y_k."""
    d = x.astype(np.float64) * 2.0 - 1.0
    out = np.zeros((x.shape[0], 3), np.float64)
    for idx, _, gx, gy, gz in _sh_terms(degree, d[:, 0], d[:, 1], d[:, 2]):
        w = dL_dy[:, idx].astype(np.float64)
        out[:, 0] += w * gx
        out[:, 1] += w * gy
        out[:, 2] += w * gz
    return (2.0 * out).astype(F32)


def composite_layout(n_in, config, alignment, grid_features=None):
    """Column layout of an encoding configuration (encodings/composite.h:135-215, encoding.h:70-72): list of
    (otype, config, in_begin, n_in, out_begin, n_out, n_pad, pad_first), and the padded width. Grids: n_out = n_levels * n_features_per_level."""
    otype = config.get("otype", "OneBlob").lower()
    nested = config["nested"] if otype == "composite" else [dict(config, n_dims_to_encode=n_in)]
    total = sum(e.get("n_dims_to_encode", 0) for e in nested)
    segs, offset = [], 0
    for e in nested:
        dims = e.get("n_dims_to_encode", n_in - total)
        if dims > 0:
            t = e.get("otype", "OneBlob").lower()
            if t in ("grid", "hashgrid", "densegrid", "tiledgrid"):
                n_out, align = e.get("n_levels", 16) * e.get("n_features_per_level", 2), e.get("n_features_per_level", 2)
            elif t == "identity":
                n_out, align = dims, 1
            elif t == "frequency":
                n_out, align = dims * e.get("n_frequencies", 12) * 2, 1
            elif t == "trianglewave":
                n_out, align = dims * e.get("n_frequencies", 12), 1
            elif t == "oneblob":
                n_out, align = dims * e.get("n_bins", 16), 1
            elif t == "sphericalharmonics":
                n_out, align = e.get("degree", 4) ** 2, 1
            else:
                raise ValueError(t)
            segs.append([t, e, offset, dims, 0, n_out, 0, t == "sphericalharmonics", align])
        offset += dims
    so_far = 0
    for i, sg in enumerate(segs):
        sg[4] = so_far
        if i + 1 < len(segs):
            a = segs[i + 1][8]
        else:
            a = max(alignment, 1)
            while a % sg[8]:
                a *= 2
        padded = -(-(so_far + sg[5]) // a) * a - so_far
        sg[6] = padded - sg[5]
        so_far += padded
    return [tuple(sg[:8]) for sg in segs], so_far


def encode_plain(x, config, alignment):
    """Encoded rows [n][width] fp32 of every NON-grid nested encoding (grid columns are left NaN for the caller to fill), with the
    padding columns as the reference writes them: ONE (zero behind a grid), SphericalHarmonics' padding in front of its coefficients."""
    segs, width = composite_layout(x.shape[1], config, alignment)
    out = np.full((x.shape[0], width), np.nan, F32)
    for t, e, in_begin, n_in, out_begin, n_out, n_pad, pad_first in segs:
        xs = x[:, in_begin : in_begin + n_in]
        if t in ("grid", "hashgrid", "densegrid", "tiledgrid"):
            out[:, out_begin + n_out : out_begin + n_out + n_pad] = 0.0
            continue
        if t == "identity":
            v = identity(xs, e.get("scale", 1.0), e.get("offset", 0.0))
        elif t == "frequency":
            v = frequency(xs, e.get("n_frequencies", 12))
        elif t == "trianglewave":
            v = triangle_wave(xs, e.get("n_frequencies", 12))
        elif t == "oneblob":
            v = oneblob(xs, e.get("n_bins", 16))
        else:
            v = spherical_harmonics(xs, e.get("degree", 4))
        if pad_first:
            out[:, out_begin : out_begin + n_pad] = 1.0
            out[:, out_begin + n_pad : out_begin + n_pad + n_out] = v
        else:
            out[:, out_begin : out_begin + n_out] = v
            out[:, out_begin + n_out : out_begin + n_out + n_pad] = 1.0
    return out, segs, width
