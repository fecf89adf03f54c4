"""A numpy restatement of the reference's CutlassMLP with a Sine / SiLU hidden activation: the activations whose derivative needs the
stored pre-activations (cutlass_mlp.cu:53 m_can_fuse_activation; forward_impl :162-209 keeps z and act(z) per hidden layer;
backward_impl :266-304 takes the derivative at z through activation_backward_gpu / warp_activation_backward_in, common_device.h:253-277),
and its parameter initialisation (cutlass_mlp.cu:362-371: SIREN for Sine, xavier otherwise; gpu_matrix.h:292-377).

Layout as everywhere in this library: W_0 [width][in_width], (n_hidden - 1) x [width][width], W_out [out_pad][width], row-major;
rows of activations are [batch][features].

Two modes:
  * `forward` / `backward` with fp16 rounding where the device rounds: fp16 operands, each product summed in float64 and rounded to
    fp16 once per layer; act(z) and act'(z) are the correctly rounded fp16 values of the float64 functions, the backward product is an
    fp16 product (the kernels, csrc/fused_common.cuh act_fwd_pre_h / act_bwd_pre_h, evaluate the same expressions with the fast-math
    hardware functions, as the reference's build does: within about one fp16 ulp of these);
  * `forward_f64` / `backward_f64`: everything in float64 -- for finite-difference checks of the backward pass.
"""
import numpy as np

SINE, SILU = "Sine", "SiLU"


class Pcg32:
    """pcg32 as the reference seeds and draws it (random.h, pcg32(initstate, initseq = 1), next_float)."""

    MULT = 0x5851F42D4C957F2D
    MASK = (1 << 64) - 1

    def __init__(self, initstate, initseq=1):
        self.state = 0
        self.inc = ((initseq << 1) | 1) & self.MASK
        self.next_uint()
        self.state = (self.state + initstate) & self.MASK
        self.next_uint()

    def next_uint(self):
        old = self.state
        self.state = (old * self.MULT + self.inc) & self.MASK
        xorshifted = (((old >> 18) ^ old) >> 27) & 0xFFFFFFFF
        rot = old >> 59
        return ((xorshifted >> rot) | (xorshifted << ((-rot) & 31))) & 0xFFFFFFFF

    def next_floats(self, n):
        u = np.fromiter((self.next_uint() for _ in range(n)), dtype=np.uint32, count=n)
        return ((u >> np.uint32(9)) | np.uint32(0x3F800000)).view(np.float32) - np.float32(1.0)


def matrix_shapes(width, in_width, n_hidden, out_pad):
    """(rows = fan_out, cols = fan_in) of every weight matrix in parameter order."""
    return [(width, in_width)] + [(width, width)] * (n_hidden - 1) + [(out_pad, width)]


def init_params(width, in_width, n_hidden, out_pad, activation, rng, scale=1.0):
    """CutlassMLP::initialize_params (cutlass_mlp.cu:362-371) in fp32: per matrix, uniform in [-bound, bound) from consecutive draws,
    bound = scale * 30 / fan_in for the first matrix of a Sine network (initialize_siren_uniform_first, gpu_matrix.h:360-377),
    scale * sqrt(6 / fan_in) for its other matrices (initialize_siren_uniform, :343-358), scale * sqrt(6 / (fan_in + fan_out))
    otherwise (initialize_xavier_uniform, :292-306). Every expression in float32, in the reference's order."""
    out = []
    for m, (rows, cols) in enumerate(matrix_shapes(width, in_width, n_hidden, out_pad)):
        s = np.float32(scale)
        if activation != SINE:
            s = np.float32(s * np.sqrt(np.float32(6.0) / np.float32(rows + cols)))
        elif m == 0:
            s = np.float32(s * (np.float32(30.0) / np.float32(cols)))
        else:
            s = np.float32(s * np.sqrt(np.float32(6.0) / np.float32(cols)))
        f = rng.next_floats(rows * cols)
        out.append((f * np.float32(2.0)) * s - s)
    return np.concatenate(out).astype(np.float32)


def split_weights(params, width, in_width, n_hidden, out_pad, dtype=np.float64):
    mats, off = [], 0
    for rows, cols in matrix_shapes(width, in_width, n_hidden, out_pad):
        mats.append(np.asarray(params[off : off + rows * cols], dtype).reshape(rows, cols))
        off += rows * cols
    assert off == params.size
    return mats


def _logistic(z):
    with np.errstate(over="ignore"):
        return 1.0 / (1.0 + np.exp(-z))


def act_f64(act, z):
    z = np.asarray(z, np.float64)
    return np.sin(z) if act == SINE else z * _logistic(z)


def act_deriv_f64(act, z):
    """common_device.h:253-277: cos(z); logistic(z) + z * logistic(z) * (1 - logistic(z))."""
    z = np.asarray(z, np.float64)
    if act == SINE:
        return np.cos(z)
    lz = _logistic(z)
    return lz + z * (lz * (1.0 - lz))


def act_fwd_pre(act, z16):
    """fp16 z -> fp16 act(z), correctly rounded."""
    return act_f64(act, np.asarray(z16, np.float16)).astype(np.float16)


def act_bwd_pre(act, grad16, z16):
    """warp_activation_backward_in<__half>: grad * (half)act'(z), the product in fp16."""
    d = act_deriv_f64(act, np.asarray(z16, np.float16)).astype(np.float16)
    with np.errstate(over="ignore", invalid="ignore"):
        return (np.asarray(grad16, np.float16) * d).astype(np.float16)


def _dot16(a16, w):
    """[B][K] fp16 . [N][K]^T summed in float64, rounded to fp16 once."""
    with np.errstate(over="ignore"):
        return (np.asarray(a16, np.float64) @ np.asarray(w, np.float64).T).astype(np.float16)


def forward(act, params16, x16, width, n_hidden, out_pad):
    """-> (pre [n_hidden][B][width], post [n_hidden][B][width], out [B][out_pad]), all fp16 (np.float16)."""
    x16 = np.asarray(x16, np.float16)
    mats = split_weights(np.asarray(params16, np.float16), width, x16.shape[1], n_hidden, out_pad)
    pre, post, h = [], [], x16
    for l in range(n_hidden):
        z = _dot16(h, mats[l])
        pre.append(z)
        h = act_fwd_pre(act, z)
        post.append(h)
    return np.stack(pre), np.stack(post), _dot16(h, mats[-1])


def backward(act, params16, x16, pre16, post16, dy16, width, n_hidden, out_pad):
    """From the forward pass's fp16 buffers (pass the device's own to check a stage on its own): -> (g [n_hidden][B][width] fp16,
    dL/dx [B][in_width] fp16, dL/dparams float64 in parameter order). dW_l = g_l^T . h_{l-1} summed in float64."""
    x16 = np.asarray(x16, np.float16)
    mats = split_weights(np.asarray(params16, np.float16), width, x16.shape[1], n_hidden, out_pad)
    g = [None] * n_hidden
    up = np.asarray(dy16, np.float16)
    for l in range(n_hidden - 1, -1, -1):
        g[l] = act_bwd_pre(act, _dot16(up, mats[l + 1].T), pre16[l])
        up = g[l]
    dx = _dot16(up, mats[0].T)
    ins = [x16] + [post16[l] for l in range(n_hidden)]
    outs = list(g) + [np.asarray(dy16, np.float16)]
    dW = [np.asarray(o, np.float64).T @ np.asarray(i, np.float64) for o, i in zip(outs, ins)]
    return np.stack(g), dx, np.concatenate([d.ravel() for d in dW])


def forward_f64(act, params, x, width, n_hidden, out_pad):
    mats = split_weights(params, width, x.shape[1], n_hidden, out_pad)
    zs, h = [], np.asarray(x, np.float64)
    for l in range(n_hidden):
        zs.append(h @ mats[l].T)
        h = act_f64(act, zs[-1])
    return zs, h @ mats[-1].T


def backward_f64(act, params, x, dy, width, n_hidden, out_pad):
    """-> (dL/dx, dL/dparams) of L = sum(dy * out), in float64."""
    mats = split_weights(params, width, x.shape[1], n_hidden, out_pad)
    zs, _ = forward_f64(act, params, x, width, n_hidden, out_pad)
    hs = [np.asarray(x, np.float64)] + [act_f64(act, z) for z in zs]
    up, dW = np.asarray(dy, np.float64), [None] * (n_hidden + 1)
    dW[n_hidden] = up.T @ hs[n_hidden]
    for l in range(n_hidden - 1, -1, -1):
        up = (up @ mats[l + 1]) * act_deriv_f64(act, zs[l])
        dW[l] = up.T @ hs[l]
    return up @ mats[0], np.concatenate([d.ravel() for d in dW])


def values_agree(a, b, rae_bar, percentile=99.0):
    """The reference's forward bar (tests/test_common.h:177: RAE < rae_bar on the best `percentile` %), except where the values sit at
    the bottom of fp16: a SiLU network behind a freshly initialised grid (table entries ~1e-4) outputs a few dozen subnormal quanta
    (2^-24), where the reference's fp16 accumulation inside the MMA is quantisation noise of a few quanta. Then the bar is absolute:
    mean <= 2.5 quanta, max <= 16 quanta (the rule golden_util.mlp_gradients_agree applies to weight gradients)."""
    from golden_util import rae

    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    if rae(a, b, percentile) < rae_bar:
        return True
    q = 2.0**-24
    if np.abs(b).mean() < 64 * q:
        d = np.abs(a - b)
        return d.mean() <= 2.5 * q and d.max() <= 16 * q
    return False
