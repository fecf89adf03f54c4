"""Numpy restatement of the Composite encoding's full configuration space, on top of oracle/feature_encodings.py's per-encoding
functions: the Sum / Product reductions (encodings/composite.h:47-133, 189-211), "dims_to_encode_begin" (composite.h:147-186), the
Empty encoding (encodings/empty.h) and the "NRC" / "OneBlobFrequency" shorthand (src/encoding.cu:93-115).

TEST INFRASTRUCTURE ONLY: imported by tests/test_composite_oracle.py and tests/test_gpu_composite_reductions.py. Grids stay on the C
oracle (tests/oracle_binding.py); their columns are left NaN here for the caller to fill. Two deliberate departures from the reference,
which the native code shares: `begin + n_dims_to_encode > n_in` is an error (the reference reads out of bounds), and the input
gradient of a dimension that several nested encodings read is the SUM of their contributions (the reference's nested backward passes
overwrite it from concurrent streams).
"""
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import feature_encodings as fe  # noqa: E402

F32 = np.float32
GRIDS = ("grid", "hashgrid", "densegrid", "tiledgrid")
REDUCTIONS = ("concatenation", "sum", "product")


def _next_multiple(v, d):
    return -(-v // d) * d


def expand(config):
    """The NRC / OneBlobFrequency shorthand as the Composite it stands for; every other configuration unchanged."""
    otype = config.get("otype", "OneBlob").lower()
    if otype in ("nrc", "oneblobfrequency"):
        return {"otype": "Composite", "nested": [
            {"n_dims_to_encode": 3, "otype": "TriangleWave", "n_frequencies": config.get("n_frequencies", 12)},
            {"n_dims_to_encode": 5, "otype": "OneBlob", "n_bins": config.get("n_bins", 4)},
            {"otype": "Identity"}]}
    return config


def _features(t, e, dims):
    """(n_out, required output alignment) of one nested encoding."""
    if t in GRIDS:
        return e.get("n_levels", 16) * e.get("n_features_per_level", 2), e.get("n_features_per_level", 2)
    if t == "identity":
        return dims, 1
    if t == "frequency":
        return dims * e.get("n_frequencies", 12) * 2, 1
    if t == "trianglewave":
        return dims * e.get("n_frequencies", 12), 1
    if t == "oneblob":
        return dims * e.get("n_bins", 16), 1
    if t == "sphericalharmonics":
        return e.get("degree", 4) ** 2, 1
    if t == "empty":
        return 0, 1
    if t in ("composite", "nrc", "oneblobfrequency"):
        raise ValueError(f"Encoding '{e.get('otype')}' nested inside a Composite is not built")
    raise ValueError(f"Encoding '{e.get('otype')}' not found")


def layout(n_in, config, alignment):
    """Segments (otype, config, in_begin, n_in, out_begin, n_out, n_pad, pad_first), the encoding's width and its reduction.
    Concatenation: out_begin is the column in the encoded rows. Sum / Product: every segment is `width` columns wide and out_begin =
    k * width is its column in the UNREDUCED rows [n][K * width]."""
    config = expand(config)
    otype = config.get("otype", "OneBlob").lower()
    reduction = "concatenation"
    if otype == "composite":
        nested = config.get("nested")
        if not isinstance(nested, list):
            raise ValueError("Must provide an array of nested encodings to CompositeEncoding.")
        reduction = config.get("reduction", "Concatenation").lower()
        if reduction not in REDUCTIONS:
            raise ValueError(f"Invalid reduction type: {config['reduction']}")
        any_begin = any("dims_to_encode_begin" in e for e in nested)
        total = sum(e.get("n_dims_to_encode", 0) for e in nested)
        if not any_begin and total > n_in:
            raise ValueError(f"CompositeEncoding: nested encodings must not encode more dims {total} than composite {n_in}")
        if sum("n_dims_to_encode" not in e for e in nested) > (0 if any_begin else 1):
            raise ValueError("CompositeEncoding: may only leave 'n_dims_to_encode' unspecified for a single nested encoding")
    else:
        nested = [dict(config, n_dims_to_encode=n_in)]
    segs, offset = [], 0
    for e in nested:
        dims = e.get("n_dims_to_encode", n_in - sum(f.get("n_dims_to_encode", 0) for f in nested))
        if "n_dims_to_encode" in e and "dims_to_encode_begin" in e:
            offset = e["dims_to_encode_begin"]
        if offset + dims > n_in:
            raise ValueError(f"CompositeEncoding: nested encoding reads input dims [{offset}, {offset + dims}) of a composite over {n_in}")
        if dims > 0:
            t = e.get("otype", "OneBlob").lower()
            n_out, align = _features(t, e, dims)
            segs.append([t, e, offset, dims, 0, n_out, 0, t == "sphericalharmonics", align])
        offset += dims
    if reduction == "concatenation":
        so_far = 0
        for i, sg in enumerate(segs):
            sg[4] = so_far
            if i + 1 < len(segs):
                a = segs[i + 1][8]
            else:
                a = math.lcm(max(alignment, 1), sg[8])
            padded = _next_multiple(so_far + sg[5], a) - so_far
            sg[6] = padded - sg[5]
            so_far += padded
        width = so_far
        if width == 0 and alignment:
            segs[-1][6] = width = alignment
    else:
        a = 1
        for sg in segs:
            a = math.lcm(a, sg[8])
        widths = [_next_multiple(sg[5], a) for sg in segs]
        if len(set(widths)) != 1:
            raise ValueError(f"CompositeEncoding: the nested encodings of a {reduction.capitalize()} reduction must have equal output widths, got {widths}")
        width = _next_multiple(widths[0], math.lcm(max(alignment, 1), a)) or alignment
        for k, sg in enumerate(segs):
            sg[4], sg[6] = k * width, width - sg[5]
    return [tuple(sg[:8]) for sg in segs], width, reduction


def encode_nested(x, config, alignment):
    """The nested encodings' rows as the reference writes them before any reduction: [n][width] under Concatenation, [n][K * width]
    under Sum / Product. Padding columns: ONE (zero behind a grid, in front of the coefficients for SphericalHarmonics); grid feature
    columns NaN."""
    segs, width, reduction = layout(x.shape[1], config, alignment)
    cols = width if reduction == "concatenation" else width * len(segs)
    out = np.full((x.shape[0], cols), np.nan, F32)
    for t, e, in_begin, n_in, out_begin, n_out, n_pad, pad_first in segs:
        xs = x[:, in_begin : in_begin + n_in]
        if t in GRIDS:
            out[:, out_begin + n_out : out_begin + n_out + n_pad] = 0.0
            continue
        if t == "empty":
            out[:, out_begin : out_begin + n_pad] = 1.0
            continue
        if t == "identity":
            v = fe.identity(xs, e.get("scale", 1.0), e.get("offset", 0.0))
        elif t == "frequency":
            v = fe.frequency(xs, e.get("n_frequencies", 12))
        elif t == "trianglewave":
            v = fe.triangle_wave(xs, e.get("n_frequencies", 12))
        elif t == "oneblob":
            v = fe.oneblob(xs, e.get("n_bins", 16))
        else:
            v = fe.spherical_harmonics(xs, e.get("degree", 4))
        if pad_first:
            out[:, out_begin : out_begin + n_pad] = 1.0
            out[:, out_begin + n_pad : out_begin + n_pad + n_out] = v
        else:
            out[:, out_begin : out_begin + n_out] = v
            out[:, out_begin + n_out : out_begin + n_out + n_pad] = 1.0
    return out, segs, width, reduction


def slabs_of(rows, n_segs, width):
    """Unreduced rows [n][K * width] -> list of K arrays [n][width]."""
    return [rows[:, k * width : (k + 1) * width] for k in range(n_segs)]


def reduce_forward(slabs, reduction, exact=False):
    """composite.h:47-104: an fp32 accumulator starting at 0 (Sum) / 1 (Product) takes the fp16 slabs in nested order, rounded to fp16
    once. exact=True: the same in float64 without rounding (for finite differences)."""
    dt = np.float64 if exact else F32
    acc = np.full(slabs[0].shape, 1.0 if reduction == "product" else 0.0, dt)
    for s in slabs:
        v = np.asarray(s, np.float16).astype(dt) if not exact else np.asarray(s, dt)
        acc = acc * v if reduction == "product" else acc + v
    return acc if exact else acc.astype(np.float16)


def reduce_backward(dL_dy, slabs, reduction, exact=False):
    """composite.h:67-84 / 106-133: Sum hands dL/dy to every nested encoding; Product gives nested k fp16(float(dL_dy) *
    prod_{l != k} slab_l), multiplied in ascending l in fp32."""
    dt = np.float64 if exact else F32
    conv = (lambda a: np.asarray(a, dt)) if exact else (lambda a: np.asarray(a, np.float16).astype(F32))
    K = len(slabs)
    out = []
    for k in range(K):
        r = conv(dL_dy)
        if reduction == "product":
            for l in range(K - 1):
                r = r * conv(slabs[l if l < k else l + 1])
        out.append(r if exact else r.astype(np.float16))
    return out


def plain_input_gradient(t, e, xs, dys):
    """dL/d(input) of one non-grid nested encoding from dL/d(its n_out feature columns)."""
    if t == "identity":
        return dys * F32(e.get("scale", 1.0))
    if t == "frequency":
        return fe.frequency_input_gradient(xs, dys, e.get("n_frequencies", 12))
    if t == "trianglewave":
        return fe.triangle_wave_input_gradient(xs, dys, e.get("n_frequencies", 12))
    if t == "oneblob":
        return fe.oneblob_input_gradient(xs, dys, e.get("n_bins", 16))
    if t == "sphericalharmonics":
        return fe.spherical_harmonics_input_gradient(xs, dys, e.get("degree", 4))
    return np.zeros_like(xs, dtype=F32)  # empty
