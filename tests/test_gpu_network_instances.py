"""Every instance of the stand-alone network kernels (csrc/mlp_fused.cu, csrc/mlp_wgrad.cu) past one round per CTA, layer by layer
against float64 sums.

The stand-alone kernels run every network the fused training kernel does not take: widths 128 and 256, Sine / SiLU, outputs wider
than the layers, more than 6 hidden layers, and the general path of every tier. mlp_forward_kernel runs min(#groups, #SMs)
persistent CTAs; a CTA's consumer warpgroups take 64-sample units round by round, so from the second round on they reuse the weight
stages, and when a chain has more steps than fit in shared memory (the ring: max_stages<W>() = 32 / 32 / 28 / 7 stages at width
16 / 32 / 64 / 128, three half-matrix stages at 256) they walk the mbarrier parities of g = round * n_steps + step; a consumer with
no unit left in the last round only releases the stages. mlp_wgrad_kernel gives every CTA a contiguous range of 128-sample tiles
and adds its fp32 sums to the accumulator with red.add.

The cases below launch every instance -- mlp_forward_kernel<W, GENERIC_ACT, BWD, PRE, WIDE> for W = 16 / 32 / 64 / 128, both WIDE
and the six (GENERIC_ACT, BWD, PRE) combinations; the same six of mlp_forward256_kernel and mlp_forward256_wide_kernel;
mlp_wgrad_kernel<W, WIDE>; mlp_wgrad256{,_wide}_kernel -- with B = 2^17 + 256 (2 052 units of 64 samples, 1 026 wgrad tiles: at
least 2 rounds per CTA and a ragged last round on an H100), and the ring at every width, with and without WIDE, forward and backward
(with and without dL/d(input): one step fewer, another ring phase).

Each case drives the network tier (tcnn_b200.Network), with g_l = dL/d(pre-activation of hidden layer l) tapped from the backward
chain (set_debug_grad_hidden), and checks every element of every row against references computed in float64 on the GPU from the
DEVICE's own input to each stage:

  1. forward, layer by layer: z = W h_prev from the device's h_prev, |fp32 accumulation error| <= e = c(K) sum_k |W_jk h_k| with
     c(K) = max((K / 16 + 1) 2^-24, 2^-22) for K chained k16 wgmma steps; the device value lies in [act(fp16(z - e)),
     act(fp16(z + e))] (one more fp16 ulp either side for the fast-math transcendental activations), and the fraction not bit-equal
     to act(fp16(z)) is at most the mean plus five standard deviations of the chance 2 e / ulp that z lies that close to a rounding
     boundary. Sine / SiLU: the stored z meets that bar, and the post-activation equals act(z_dev) to one fp16 ulp plus the fast-math
     error of __sinf / __expf. Output layer: every padded column. inference_mixed_precision equals the forward output bit for bit;
  2. backward, layer by layer from the tapped g_l: g_{l-1} = fp16(fp16(W_l^T g_l) * f'), f' from the stored forward value as
     act_bwd_pack / act_bwd_pre_pack compute it; dL/d(input) = fp16(W_0^T g_0). The first product starts from the output
     activation's transfer act_bwd(dL/d(output), y), evaluated elementwise in float64 (its fp16 rounding steps reproduced);
  3. weight gradients over the whole batch, every entry: |dev - sum_b g h| <= ulp16(ref) + c_w sum_b |g h|, c_w = (8 k16 steps per
     tile x tiles per CTA + 1 + the CTAs whose sums red.add meets) 2^-24 -- one dropped or doubled tile fails it;
  4. a second backward gives bit-identical g_l and dL/d(input) (the dL/dparams within the bar: the red.add order varies); a backward
     without dL/d(input) gives bit-identical g_l and dL/dparams within the bar;
  5. non-vacuity: every hidden layer and every g_l has an RMS in [2^-6, 2^6], at least 25 % nonzero elements, no inf or NaN;
  6. (the `fp32` case) the Identity paths: inference (fp32 in, fp32 out), module_inference and module_backward on the unpadded input
     against a twin network fed the Identity-encoded rows, bit for bit (dL/dparams within the bar).

The premise test (no GPU) restates the dispatch and the kernels' limits, pins them to the sources, and asserts that the case list
reaches every instance and the ring at every width.
"""
import os
from types import SimpleNamespace

import pytest

from test_gpu_fused_instances import TRANSCENDENTAL, act_bwd_factor, act_fwd, check_interval, rn16, ulp16

gpu = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tiny-cuda-nn_b200", "csrc")
B = (1 << 17) + 256  # 2 052 units of 64 samples, 1 026 tiles of 128
UNIT = 64
TILE = 128
H100_SMS = 132
MLPF_MAX_STAGES = 32
SMEM = 227 * 1024
PRE_ACTS = ("Sine", "SiLU")

# name: (width, hidden layers, input dims, output dims, activation, output activation, extras)
#   scale: initial_params(scale=...) so that deep chains keep their magnitude; fp32: the Identity fp32 paths on a 3-dim input
CASES = {
    "w16_relu": (16, 3, 32, 16, "ReLU", "None", {"scale": 2 ** 0.5}),
    # 33 ReLU layers 16 wide leave most neurons dead; LeakyReLU keeps every element alive
    "w16_leaky_ring_sigmoid_out": (16, 33, 16, 13, "LeakyReLU", "Sigmoid", {"scale": 2 ** 0.5}),
    "w16_silu": (16, 2, 16, 8, "SiLU", "None", {}),
    "w16_wide_relu_ring": (16, 1, 16, 1024, "ReLU", "None", {}),
    "w16_wide48_leaky": (16, 2, 16, 48, "LeakyReLU", "None", {}),
    "w16_wide_sine": (16, 2, 16, 100, "Sine", "None", {}),
    "w32_relu_ring": (32, 33, 32, 32, "ReLU", "None", {"scale": 2 ** 0.5}),
    "w32_sigmoid_exp_out": (32, 2, 32, 16, "Sigmoid", "Exponential", {}),
    "w32_sine": (32, 3, 32, 32, "Sine", "None", {}),
    "w32_wide_relu_ring": (32, 2, 32, 1024, "ReLU", "None", {}),
    "w32_wide64_softplus": (32, 2, 32, 64, "Softplus", "None", {}),
    "w32_wide_silu_tanh_out": (32, 2, 32, 200, "SiLU", "Tanh", {}),
    "w64_relu_ring": (64, 29, 64, 64, "ReLU", "None", {"scale": 2 ** 0.5}),
    "w64_tanh_fp32": (64, 2, 3, 3, "Tanh", "None", {"fp32": True}),
    "w64_sine": (64, 2, 64, 16, "Sine", "None", {}),
    "w64_wide_relu_ring": (64, 14, 64, 1024, "ReLU", "None", {"scale": 2 ** 0.5}),
    "w64_wide_squareplus": (64, 2, 64, 128, "Squareplus", "Sigmoid", {}),
    "w64_wide_silu": (64, 2, 64, 80, "SiLU", "None", {}),
    "w128_relu_ring": (128, 8, 128, 128, "ReLU", "None", {"scale": 2 ** 0.5}),
    "w128_leaky_exp_out": (128, 3, 64, 32, "LeakyReLU", "Exponential", {}),
    "w128_sine": (128, 2, 128, 64, "Sine", "None", {}),
    "w128_wide_relu_ring": (128, 7, 64, 256, "ReLU", "None", {"scale": 2 ** 0.5}),
    "w128_wide_sigmoid": (128, 2, 64, 160, "Sigmoid", "None", {}),
    "w128_wide_silu": (128, 2, 64, 144, "SiLU", "None", {}),
    "w256_relu": (256, 3, 64, 64, "ReLU", "None", {"scale": 2 ** 0.5}),
    "w256_tanh_sigmoid_out": (256, 2, 256, 128, "Tanh", "Sigmoid", {}),
    "w256_sine": (256, 2, 128, 200, "Sine", "None", {}),
    "w256_wide_relu": (256, 2, 64, 512, "ReLU", "None", {"scale": 2 ** 0.5}),
    "w256_wide_softplus": (256, 2, 64, 300, "Softplus", "None", {}),
    "w256_wide_silu": (256, 2, 64, 1000, "SiLU", "None", {}),
}


def case(name):
    W, nh, n_in, n_out, act, out_act, extra = CASES[name]
    in_w = (n_in + 15) // 16 * 16
    out_pad = (n_out + 15) // 16 * 16
    return SimpleNamespace(name=name, W=W, nh=nh, n_in=n_in, n_out=n_out, in_w=in_w, out_pad=out_pad, act=act, out_act=out_act,
                           scale=extra.get("scale", 1.0), fp32=extra.get("fp32", False))


def net_config(c):
    otype = "CutlassMLP" if c.W == 256 or c.act in PRE_ACTS else "FullyFusedMLP"
    return {"otype": otype, "n_neurons": c.W, "n_hidden_layers": c.nh, "activation": c.act, "output_activation": c.out_act}


# ---- restatements of the host-side rules (pinned to the sources by the premise test)


def stage_bytes(W):
    """MlpCfg<W>::STAGE_BYTES."""
    kblocks = (W + 63) // 64
    return max(kblocks * W * 128, 2048)


def max_stages(W):
    """mlp_fused.cu max_stages<W>()."""
    return min((SMEM - 1024) // stage_bytes(W), MLPF_MAX_STAGES)


def wgs(W):
    """Consumer warpgroups of the forward / backward-chain kernel (MlpCfg<W>::WGS, Mlp256::WGS)."""
    return 1 if W == 256 else (2 if W == 128 else 4)


def fwd_wide(c):
    return c.out_pad > c.W


def forward_instance(c, bwd):
    """(kernel, W, GENERIC_ACT, BWD, PRE, WIDE) of the chain a forward (bwd = False) or backward pass launches (launch_width /
    launch_width256); the backward chain sees no output activation (split_backward)."""
    pre = c.act in PRE_ACTS
    if pre:
        flags = (True, bwd, True)
    elif bwd:
        flags = (c.act != "ReLU", True, False)
    else:
        flags = (c.act != "ReLU" or c.out_act != "None", False, False)
    if c.W == 256:
        return ("mlp_forward256_wide_kernel" if fwd_wide(c) else "mlp_forward256_kernel", 256) + flags + (None,)
    return ("mlp_forward_kernel", c.W) + flags + (fwd_wide(c),)


def wgrad_instance(c):
    """launch_wgrad_width / launch_wgrad256: WIDE when dL/d(output) is wider than an accumulator."""
    if c.W == 256:
        return ("mlp_wgrad256_wide_kernel" if c.out_pad > 256 else "mlp_wgrad256_kernel", 256, None)
    return ("mlp_wgrad_kernel", c.W, c.out_pad > 64 * ((c.W + 63) // 64))


def chain_steps(c, bwd, input_grad=True):
    """launch_impl / launch_impl256 n_layers: NH + 1 + n_oc - 1 weight steps, one fewer for a backward chain without dL/d(input).
    At 256 the backward chain walks the output matrix's K-blocks inside its first step."""
    if c.W == 256:
        n_oc = (c.out_pad + 255) // 256 if not bwd else 1
    else:
        n_oc = (c.out_pad + c.W - 1) // c.W if fwd_wide(c) else 1
    return c.nh + n_oc - (1 if bwd and not input_grad else 0)


def ring(c, bwd, input_grad=True):
    """The weights stream through the stages (always at 256: a matrix is 128 KB)."""
    return c.W == 256 or chain_steps(c, bwd, input_grad) > max_stages(c.W)


def units_per_cta(W, n_sms):
    """Units of 64 samples of every CTA of the chain kernel: CTA x takes units x, x + grid, ..."""
    n_units = B // UNIT
    grid = min((n_units + wgs(W) - 1) // wgs(W), n_sms)
    return [(n_units - x + grid - 1) // grid for x in range(grid)]


def wgrad_tiles_per_cta(W, n_sms):
    """Tiles of 128 samples of every CTA (of every CTA pair at 256) of the weight-gradient kernel."""
    n_tiles = B // TILE
    grid = min(n_tiles, n_sms // 2 if W == 256 else n_sms)
    return [(x + 1) * n_tiles // grid - x * n_tiles // grid for x in range(grid)]


def kernel_limits_ok(c):
    """mlp_forward_supported / mlp_wgrad_supported for the case's shapes (dL/d(input) included)."""
    max_in = 64 * ((c.W + 63) // 64)
    return (c.nh >= 1 and c.nh + 1 <= 64 and c.in_w % 16 == 0 and 0 < c.in_w <= max_in and c.out_pad <= 1024 and B % 256 == 0
            and c.in_w <= max(c.W, 32) and c.nh * B < 2 ** 31)


def test_premise_every_instance_past_one_round_per_cta():
    with open(os.path.join(CSRC, "mlp_fused.cu")) as f:
        fused = f.read()
    with open(os.path.join(CSRC, "mlp_wgrad.cu")) as f:
        wgrad = f.read()
    with open(os.path.join(CSRC, "network.cu")) as f:
        network = f.read()
    # the configuration of the chain kernels restated in stage_bytes / max_stages / wgs
    for s in ("constexpr uint32_t MLPF_MAX_STAGES = 32;", "constexpr uint32_t UNIT_M = 64;", "static constexpr uint32_t WGS = W == 128 ? 2 : 4;",
              "static constexpr uint32_t KBLOCKS = (W + 63) / 64;", "static constexpr uint32_t KBLOCK_BYTES = W * 128;",
              "static constexpr uint32_t STAGE_BYTES = KBLOCKS * KBLOCK_BYTES < 2048 ? 2048 : KBLOCKS * KBLOCK_BYTES;",
              "return (uint32_t)((227u * 1024u - 1024u) / MlpCfg<W>::STAGE_BYTES) < MLPF_MAX_STAGES ? (uint32_t)((227u * 1024u - 1024u) / MlpCfg<W>::STAGE_BYTES) : MLPF_MAX_STAGES;",
              "static constexpr uint32_t WGS = 1;", "static constexpr uint32_t STAGES = 3;"):
        assert s in fused, s
    # the dispatch restated in forward_instance / chain_steps / ring / units_per_cta
    for s in ("if (activation_needs_preact(p.activation)) return p.backward ? launch_impl<W, true, true, true, WIDE>(p, n_sms, stream) : launch_impl<W, true, false, true, WIDE>(p, n_sms, stream);",
              "if (p.backward) return p.activation != ACT_RELU ? launch_impl<W, true, true, false, WIDE>(p, n_sms, stream) : launch_impl<W, false, true, false, WIDE>(p, n_sms, stream);",
              "return generic ? launch_impl<W, true, false, false, WIDE>(p, n_sms, stream) : launch_impl<W, false, false, false, WIDE>(p, n_sms, stream);",
              "return p.out_width > W ? launch_width<W, true>(p, n_sms, stream) : launch_width<W, false>(p, n_sms, stream);",
              "if (activation_needs_preact(p.activation)) return p.backward ? launch_impl256<true, true, true, WIDE>(p, n_sms, stream) : launch_impl256<true, false, true, WIDE>(p, n_sms, stream);",
              "if (p.backward) return p.activation != ACT_RELU ? launch_impl256<true, true, false, WIDE>(p, n_sms, stream) : launch_impl256<false, true, false, WIDE>(p, n_sms, stream);",
              "return generic ? launch_impl256<true, false, false, WIDE>(p, n_sms, stream) : launch_impl256<false, false, false, WIDE>(p, n_sms, stream);",
              "case 256: return p.out_width > 256 ? launch_width256<true>(p, n_sms, stream) : launch_width256<false>(p, n_sms, stream);",
              "const uint32_t n_oc = WIDE ? (p.out_width + W - 1) / W : 1;  // steps of the output matrix",
              "const uint32_t n_oc = (WIDE && !BWD) ? (p.out_width + C::W - 1) / C::W : 1;",
              "kp.resident = n_layers <= max_stages<W>() ? 1 : 0;", "kp.resident = 0;"):
        assert s in fused, s
    assert fused.count("const bool generic = p.activation != ACT_RELU || p.output_activation != ACT_NONE;") == 2
    assert fused.count("const uint32_t n_layers = p.n_hidden_layers + ((BWD && !p.output_fp16) ? 0 : 1) + n_oc - 1;") == 2
    assert fused.count("const uint32_t n_groups = (p.batch_size / UNIT_M + C::WGS - 1) / C::WGS;") == 2
    assert fused.count("n_groups < n_sms ? n_groups : n_sms") == 2
    assert fused.count("const uint32_t n_my = blockIdx.x < n_units ? (n_units - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;") == 3
    # the limits restated in kernel_limits_ok
    for s in ("if (p.n_hidden_layers + 1 > 64)", "const uint32_t max_in = 64 * ((p.width + 63) / 64);",
              "if (p.in_width == 0 || p.in_width % 16 != 0 || p.in_width > max_in)", "if (p.out_width > MLP_MAX_OUTPUT_WIDTH)",
              "if (p.output_fp16 && p.in_width > (p.width < 32 ? 32u : p.width))"):
        assert s in fused, s
    # the weight-gradient dispatch and grid restated in wgrad_instance / wgrad_tiles_per_cta
    for s in ("return p.out_width > WgradCfg<W>::KB * 64 ? launch_wgrad_width<W, true>(p, n_sms, stream, n_launches) : launch_wgrad_width<W, false>(p, n_sms, stream, n_launches);",
              "auto kernel = p.out_width > C::W ? mlp_wgrad256_wide_kernel : mlp_wgrad256_kernel;",
              "const uint32_t n_tiles = B / TILE_M, n_pairs = n_tiles < n_sms / 2 ? n_tiles : n_sms / 2;",
              "err = launch_pdl(kernel, n_tiles < n_sms ? n_tiles : n_sms, C::THREADS, smem, stream, kp, mx, mh, mg, mgo);",
              "const uint32_t tile_begin = (uint32_t)((uint64_t)blockIdx.x * n_tiles / gridDim.x), tile_end = (uint32_t)((uint64_t)(blockIdx.x + 1) * n_tiles / gridDim.x);",
              "const uint32_t tile_begin = (uint32_t)((uint64_t)pair * n_tiles / n_pairs), tile_end = (uint32_t)((uint64_t)(pair + 1) * n_tiles / n_pairs);",
              "d.output_activation = ACT_NONE;", "const uint32_t acc = (!first_tile || kk > 0) ? 1u : 0u;"):
        assert s in wgrad, s
    # the network tier runs on every SM, and the tap replaces the scratch rows of g_l
    assert "n.n_sms = require_sm90();" in network
    assert "if (s.grad_hidden_tap) {\n\t\ta.grad_hidden = s.grad_hidden_tap;" in network

    fwd, wg = set(), set()
    ring_reached = set()
    for name in CASES:
        c = case(name)
        assert kernel_limits_ok(c), name
        fwd.add(forward_instance(c, False))
        fwd.add(forward_instance(c, True))
        wg.add(wgrad_instance(c))
        if ring(c, False) and ring(c, True) and ring(c, True, input_grad=False):
            ring_reached.add((c.W, fwd_wide(c)))
    six = [(False, False, False), (True, False, False), (True, False, True), (False, True, False), (True, True, False), (True, True, True)]
    want = {("mlp_forward_kernel", W) + f + (wide,) for W in (16, 32, 64, 128) for wide in (False, True) for f in six}
    want |= {(k, 256) + f + (None,) for k in ("mlp_forward256_kernel", "mlp_forward256_wide_kernel") for f in six}
    assert fwd == want, sorted(want - fwd)
    assert len(fwd) == 60
    assert wg == {("mlp_wgrad_kernel", W, wide) for W in (16, 32, 64, 128) for wide in (False, True)} | {("mlp_wgrad256_kernel", 256, None), ("mlp_wgrad256_wide_kernel", 256, None)}
    assert ring_reached == {(W, wide) for W in (16, 32, 64, 128, 256) for wide in (False, True)}, ring_reached
    # width 16 with 32-64 outputs: the WIDE chain and the non-WIDE weight gradients
    c = case("w16_wide48_leaky")
    assert fwd_wide(c) and not wgrad_instance(c)[2]
    # stages of the weight ring at widths 16 / 32 / 64 / 128
    assert [max_stages(W) for W in (16, 32, 64, 128)] == [32, 32, 28, 7]
    # two or more rounds per CTA and a ragged last round, and two or more weight-gradient tiles per CTA, on a 132-SM H100 (the GPU
    # test asserts the same on the device it runs on)
    for W in (16, 32, 64, 128, 256):
        u = units_per_cta(W, H100_SMS)
        assert min(u) >= 2 * wgs(W), W
        assert W == 256 or any(n % wgs(W) for n in u), W
        assert min(wgrad_tiles_per_cta(W, H100_SMS)) >= 2


# ---- float64 references on the GPU


def c_of(K):
    """Relative bound of an fp32 wgmma accumulation over K = 16 k products: one rounding per chained k16 step, never below the fused
    kernel test's 2^-22."""
    return max((K // 16 + 1) * 2.0 ** -24, 2.0 ** -22)


SIN_ERR = 2.0 ** -21.41  # __sinf / __cosf absolute error on [-pi, pi] (CUDA C Programming Guide, intrinsic functions)


def pre_act(act, z):
    """Sine / SiLU on float64 values, and the bound of the fast-math fp32 evaluation's absolute error."""
    import torch

    if act == "Sine":
        # outside [-pi, pi] the argument reduction by 2 pi in fp32 adds up to |z| 2^-23
        return torch.sin(z), SIN_ERR + z.abs() * 2.0 ** -23
    sig = torch.sigmoid(z)
    # __expf: 2 + 1.173 |z| ulp; __fdividef and the product: a few ulp more (fp32 ulp <= 2^-23 relative)
    return z * sig, (z * sig).abs() * (8.0 + 1.2 * z.abs()) * 2.0 ** -23 + 2.0 ** -126


def pre_act_bwd_factor(act, z):
    """act'(z) as act_bwd_pre_h evaluates it (fast math in fp32, rounded to fp16): (low, high, value)."""
    import torch

    if act == "Sine":
        v, d = torch.cos(z), SIN_ERR + z.abs() * 2.0 ** -23
    else:
        s = torch.sigmoid(z)
        v = s + z * s * (1.0 - s)
        d = (8.0 + 1.2 * z.abs()) * (1.0 + z.abs()) * 2.0 ** -23
    return rn16(v - d), rn16(v + d), rn16(v)


def interval_forward(what, act, h_prev, Wm, dev, pre_z_dev=None):
    """dev = act(fp16(h_prev W^T)) for the device's h_prev [B][k] and W [n][k] (the fp32 sum within e = c(K) sum |W h|)."""
    import torch

    z = h_prev @ Wm.T
    e = c_of(Wm.shape[1]) * (h_prev.abs() @ Wm.abs().T)
    p = torch.clamp(2.0 * e / ulp16(z), max=1.0)
    if act in PRE_ACTS:
        # the stored pre-activation meets the bar of a plain product; the post-activation is act(z_dev) to one fp16 ulp and the
        # fast-math error
        check_interval(what + " (pre-activation)", pre_z_dev, rn16(z - e), rn16(z + e), rn16(z), p)
        y, d = pre_act(act, pre_z_dev)
        bar = ulp16(y.abs() + d) + d
        bad = (dev - y).abs() > bar
        assert not bad.any(), f"{what}: {int(bad.sum())} post-activations off act(z_dev), first {torch.nonzero(bad)[0].tolist()}"
        return flip_ratio(pre_z_dev, z, e, torch.ones_like(z, dtype=torch.bool))
    lo, hi, mid = act_fwd(act, rn16(z - e)), act_fwd(act, rn16(z + e)), act_fwd(act, rn16(z))
    if act in TRANSCENDENTAL:
        lo, hi = lo - ulp16(lo), hi + ulp16(hi)
        p = torch.clamp(p + 2.0 ** -8, max=1.0)
    check_interval(what, dev, lo, hi, mid, p)
    if act in ("None", "ReLU"):
        return flip_ratio(dev, z, e, dev > 0 if act == "ReLU" else torch.ones_like(z, dtype=torch.bool))
    return 0.0


def interval_backward(what, act, s, e, f, dev):
    """dev = fp16(fp16(s') * factor) for the device's fp32 sum s' within e of s; factor from the stored forward value f (post-
    activation, or the pre-activation z for Sine / SiLU; None: no activation)."""
    import torch

    if f is None:
        flo = fhi = fmid = torch.ones_like(s)
    elif act in PRE_ACTS:
        flo, fhi, fmid = pre_act_bwd_factor(act, f)
    else:
        flo, fhi, fmid = act_bwd_factor(act, f)
    glo, ghi = rn16(s - e), rn16(s + e)
    corners = torch.stack([glo * flo, glo * fhi, ghi * flo, ghi * fhi])
    lo, hi = rn16(corners.min(0).values), rn16(corners.max(0).values)
    mid = rn16(rn16(s) * fmid)
    p = torch.clamp(2.0 * e / ulp16(s) + (fhi != flo).double(), max=1.0)
    check_interval(what, dev, lo, hi, mid, p)
    if f is None or act == "ReLU":
        return flip_ratio(dev, s, e, torch.ones_like(s, dtype=torch.bool) if f is None else f > 0)
    return 0.0


def output_transfer(act, dy, y):
    """act_bwd_h(act, dL/d(output), y) elementwise (launch_activation_backward_output): (low, high) of the fp16 result over the fp32
    evaluation errors of the factor."""
    if act == "None":
        return dy, dy
    flo, fhi, _ = act_bwd_factor(act, y)
    a, b = rn16(dy * flo), rn16(dy * fhi)
    return a.minimum(b), a.maximum(b)


def non_vacuous(what, t):
    import torch

    assert torch.isfinite(t).all(), f"{what}: inf or NaN"
    rms = float(t.pow(2).mean().sqrt())
    assert 2.0 ** -6 <= rms <= 2.0 ** 6, f"{what}: RMS {rms:.3e} outside [2^-6, 2^6]"
    nz = float((t != 0).double().mean())
    assert nz >= 0.25, f"{what}: only {nz:.1%} of the elements nonzero"


def ratio(dev, ref, bar):
    return float(((dev - ref).abs() / bar).max())


def flip_ratio(dev, s, e, mask):
    """A lower bound of the largest |fp32 accumulation error| / e among the elements where the device's value is fp16(s') for its fp32
    sum s' (`mask`): where dev is not fp16(s), s' lies beyond the rounding boundary between the two, at least that far from s."""
    mid = rn16(s)
    sel = mask & (dev != mid)
    if not sel.any():
        return 0.0
    return float((((dev + mid) * 0.5 - s).abs() / e)[sel].max())


class Weights:
    """The parameter layout: W_0 [W][in_w], (NH - 1) x [W][W], W_out [out_pad][W]."""

    def __init__(self, c, p16):
        P = p16.double()
        self.mats, off = [], 0
        for rows, cols in [(c.W, c.in_w)] + [(c.W, c.W)] * (c.nh - 1) + [(c.out_pad, c.W)]:
            self.mats.append(P[off : off + rows * cols].view(rows, cols))
            off += rows * cols
        assert off == P.numel()


def check_case(torch, c):
    import tcnn_b200

    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    u = units_per_cta(c.W, n_sms)
    assert min(u) >= 2 * wgs(c.W), "premise: every CTA of the chain kernel runs two or more rounds"
    assert c.W == 256 or any(n % wgs(c.W) for n in u), "premise: a ragged last round"
    assert min(wgrad_tiles_per_cta(c.W, n_sms)) >= 2, "premise: two or more weight-gradient tiles per CTA"

    net = tcnn_b200.Network(c.in_w, c.n_out, net_config(c))
    twin = None
    try:
        assert (net.input_width, net.padded_output_width, net.width, net.n_hidden_layers) == (c.in_w, c.out_pad, c.W, c.nh)
        pre = c.act in PRE_ACTS
        assert net.n_forward_activations == (2 if pre else 1) * c.nh
        p16 = net.initial_params(seed=7, scale=c.scale).half().contiguous()
        Ws = Weights(c, p16).mats
        g = torch.Generator(device="cuda").manual_seed(4242)
        x16 = (torch.rand(B, c.in_w, device="cuda", generator=g) * 2 - 1).half()
        if c.fp32:
            x32 = (torch.rand(B, c.n_in, device="cuda", generator=g) * 2 - 1).contiguous()
            x16 = torch.ones(B, c.in_w, dtype=torch.float16, device="cuda")
            x16[:, : c.n_in] = x32.half()  # the Identity encoding: fp16(x), padding ONE
        x16 = x16.contiguous()
        dy16 = (torch.rand(B, c.out_pad, device="cuda", generator=g) * 2 - 1).half().contiguous()
        ratios = {"forward": 0.0, "backward": 0.0}

        # 1. forward, layer by layer
        out, hidden = net.forward(x16, p16)
        torch.cuda.synchronize()
        h = hidden.double()
        h_prev = x16.double()
        for l in range(c.nh):
            non_vacuous(f"hidden[{l}]", h[l])
            r = interval_forward(f"hidden[{l}]", c.act, h_prev, Ws[l], h[l], h[c.nh + l] if pre else None)
            ratios["forward"] = max(ratios["forward"], r)
            h_prev = h[l]
        y = out.double()
        assert torch.isfinite(y).all()
        ratios["forward"] = max(ratios["forward"], interval_forward("output", c.out_act, h_prev, Ws[c.nh], y))
        inf16 = net.inference_mixed_precision(x16, p16)
        assert torch.equal(inf16.view(torch.int16), out.view(torch.int16)), "inference_mixed_precision differs from forward"

        # 2. backward, layer by layer from the tapped g_l
        def backward(input_grad):
            tap = torch.full((c.nh, B, c.W), float("nan"), dtype=torch.float16, device="cuda")
            net.set_debug_grad_hidden(tap)
            try:
                dx, dp = net.backward(x16, out, hidden, dy16, p16, want_input_grad=input_grad, want_param_grad=True)
                torch.cuda.synchronize()
            finally:
                net.set_debug_grad_hidden(None)
            return tap, dx, dp

        tap, dx, dp = backward(True)
        gl = tap.double()
        t_lo, t_hi = output_transfer(c.out_act, dy16.double(), y)
        t = 0.5 * (t_lo + t_hi)
        s = t @ Ws[c.nh]
        e = c_of(c.out_pad) * (t.abs() @ Ws[c.nh].abs()) + (t_hi - t_lo) @ Ws[c.nh].abs()
        def fwd_of(l):
            """What f' of hidden layer l is computed from: the pre-activation for Sine / SiLU, else the post-activation."""
            return h[c.nh + l] if pre else h[l]

        rb = [interval_backward(f"g[{c.nh - 1}]", c.act, s, e, fwd_of(c.nh - 1), gl[c.nh - 1])]
        for l in range(c.nh - 1, 0, -1):
            s = gl[l] @ Ws[l]
            e = c_of(c.W) * (gl[l].abs() @ Ws[l].abs())
            rb.append(interval_backward(f"g[{l - 1}]", c.act, s, e, fwd_of(l - 1), gl[l - 1]))
        for l in range(c.nh):
            non_vacuous(f"g[{l}]", gl[l])
        s = gl[0] @ Ws[0]
        rb.append(interval_backward("dL/d(input)", "None", s, c_of(c.W) * (gl[0].abs() @ Ws[0].abs()), None, dx.double()))
        ratios["backward"] = max(rb)

        # 3. weight gradients over the whole batch
        tiles = wgrad_tiles_per_cta(c.W, n_sms)
        c_w = (8 * max(tiles) + 1 + len(tiles)) * 2.0 ** -24
        ops = [(gl[0], x16.double())] + [(gl[l], h[l - 1]) for l in range(1, c.nh)] + [(t, h[c.nh - 1])]
        refs, bars = [], []
        for a, b in ops:
            refs.append((a.T @ b).flatten())
            bars.append(c_w * (a.abs().T @ b.abs()).flatten())
        bars[-1] = bars[-1] + ((t_hi - t_lo).T @ h[c.nh - 1].abs()).flatten()
        ref = torch.cat(refs)
        bar = ulp16(ref) + torch.cat(bars)

        def check_dw(what, dp):
            dev = dp.double()
            bad = (dev - ref).abs() > bar
            assert not bad.any(), (f"{what}: {int(bad.sum())} of {ref.numel()} weight gradients off the whole-batch sums, first {torch.nonzero(bad)[0].item()}: "
                                   f"dev {dev[bad][0].item()!r} ref {ref[bad][0].item()!r} bar {bar[bad][0].item()!r}")
            return ratio(dev, ref, bar)

        ratios["wgrad"] = check_dw("dL/dparams", dp)

        # 4. determinism, and the backward chain without dL/d(input)
        tap2, dx2, dp2 = backward(True)
        assert torch.equal(tap2.view(torch.int16), tap.view(torch.int16)), "a second backward gives other g_l"
        assert torch.equal(dx2.view(torch.int16), dx.view(torch.int16)), "a second backward gives another dL/d(input)"
        check_dw("dL/dparams (second backward)", dp2)
        tap3, dx3, dp3 = backward(False)
        assert dx3 is None
        assert torch.equal(tap3.view(torch.int16), tap.view(torch.int16)), "a backward without dL/d(input) gives other g_l"
        check_dw("dL/dparams (backward without dL/d(input))", dp3)

        # 6. the Identity fp32 paths against a twin network fed the encoded rows
        if c.fp32:
            twin = net
            net = tcnn_b200.Network(c.n_in, c.n_out, net_config(c))
            assert net.n_params == twin.n_params
            o32 = net.inference(x32, p16)
            assert torch.equal(o32, out[:, : c.n_out].float()), "inference (fp32) differs from the fp16 forward of the encoded rows"
            o16 = net.module_inference(x32, p16)
            assert torch.equal(o16.view(torch.int16), out.view(torch.int16)), "module_inference differs from the forward of the encoded rows"
            tap4 = torch.full((c.nh, B, c.W), float("nan"), dtype=torch.float16, device="cuda")
            net.set_debug_grad_hidden(tap4)
            try:
                dx32, dp4 = net.module_backward(x32, dy16, p16)
                torch.cuda.synchronize()
            finally:
                net.set_debug_grad_hidden(None)
            assert torch.equal(tap4.view(torch.int16), tap.view(torch.int16)), "module_backward gives other g_l"
            assert torch.equal(dx32, dx[:, : c.n_in].float()), "module_backward's dL/d(input) differs from the twin's"
            check_dw("dL/dparams (module_backward)", dp4)
        return ratios
    finally:
        net.close()
        if twin is not None:
            twin.close()


@gpu
@pytest.mark.parametrize("name", list(CASES))
def test_network_instance_layer_by_layer(torch_cuda, name):
    ratios = check_case(torch_cuda, case(name))
    print(f"\n{name}: largest measured error / bar: " + ", ".join(f"{k} {v:.3f}" for k, v in ratios.items()))
