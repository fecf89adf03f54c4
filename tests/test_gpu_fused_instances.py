"""Every instance of the fused training kernel (csrc/fused_ws.cu) past one tile per CTA, stage by stage against float64 sums.

fused_ws_kernel runs min(B / 128, #SMs) persistent CTAs, each over a contiguous range of 128-sample tiles. From a CTA's second
tile on it reuses state that a one-tile batch never exercises: the encoded-tile ring and its mbarrier parities, the two park
buffers, the sample index and targets fetched one tile ahead, the CTA's fp32 weight-gradient sums kept in shared memory across
tiles (or, for 5-6 hidden layers, added to the global accumulator after every tile), and reads through the binning permutation.
The kernel is compiled as 12 instances, (D, TRAIN, GENERIC_ACT, PDF); the cases below reach each of them with B = 2^17 + 256
(1 026 tiles: 7-8 per CTA on a 132-SM H100), at widths 16 / 32 / 64 and depths 1-6.

Each case runs one step without the optimizer, every debug tap NaN-filled first, and checks, with references computed in
float64 on the GPU from the DEVICE's own input to each stage (so that every stage is isolated):

  1. every tap row is written;
  2. every per-sample row equals the unbinned step's bit for bit (the taps are written in caller order);
  3. a step without taps gives the same loss (fp32 summation order) and gradients that meet the same bars;
  4. the encoded features equal the CPU oracle's bit for bit (Identity: fp16(fp32(x * scale + offset)), padding ONE);
  5. forward, layer by layer: z = W h_prev from the device's h_prev, |fp32 accumulation error| <= 2^-22 sum_k |W_jk h_k|,
     rounded to fp16 and passed through the activation as act_fwd_h does it. The activations are monotone, so the device's
     value must lie in [act(fp16(z - e)), act(fp16(z + e))], one more fp16 ulp either side for the fast-math transcendental
     ones. The fraction of elements that are not bit-equal to act(fp16(z)) is bounded by the chance that z lies within e of a
     rounding boundary (2 e / ulp, plus 2^-8 for a transcendental) -- its mean plus five standard deviations;
  6. the loss values against the loss formulas on the device's output (data_pdf included) to 2^-18 of their terms, the loss
     equal to their sum, and dL/d(output) = act_bwd(fp16(loss_scale * grad / n_total), y) with the fp32 evaluation of the
     gradient bounded by 2^-19 relative; padding columns exactly zero;
  7. backward, layer by layer, the same way: g_{l-1} = fp16(fp16(W_l^T g_l) * f'), the factor f' as act_bwd_h computes it
     from the stored forward value (its fp32 evaluation bounded where it is not exact), dL/d(encoded) = fp16(W_0^T g_0);
  8. the network weight gradients over the whole batch: |dev - sum_b g_l[b] h_{l-1}[b]| <= ulp16(ref) + 2^-20 sum_b |g h|
     (fp32 accumulation and the final fp16 cast) for every entry -- one dropped or doubled tile fails it. W_0's columns of
     padded grid features are exactly zero;
  9. the table gradients against the exact float64 scatter of the device's dL/d(encoded) (the oracle's grid_backward): nothing
     outside the entries the batch indexes, every entry within the worst-case bound of fp16 accumulation
     (n_e 2^-11 + 2^-10) S_e + n_e 2^-24, where n_e is the number of addends and S_e = sum |addend| = grid_backward(x,
     |dL/d(encoded)|) (Linear and Smoothstep weights are non-negative); RAE < 1.2e-2 @ p99.9 on the hashed levels; the binned
     step no further from the exact sums than the unbinned one (25 % slack); touched sets equal up to exact cancellation;
 10. (cases marked `infer`) network.inference on the same batch equals the step's output tap bit for bit: the TRAIN = false
     instance against the TRAIN = true one;
 11. (the module-tier case) dL/d(input) against the oracle's grid_input_gradient on the device's dL/d(encoded).

The premise test (no GPU) restates the dispatch rule and the fused kernel's limits and pins them to the sources, so that a change
of either fails it instead of letting the cases drift back to one tile per CTA or off the fused kernel.
"""
import json
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest

import oracle_binding as ob
from golden_util import GOLDEN, rae

gpu = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tiny-cuda-nn_b200", "csrc")
B = (1 << 17) + 256  # 1 026 tiles of 128 samples
TILE = 128
H100_SMS = 132
N_OUT = 3
LOSS_SCALE = 128.0
SEED = 4242
TRANSCENDENTAL = {"Exponential", "Sigmoid", "Squareplus", "Softplus", "Tanh"}

# name: (D, width, hidden layers, activation, output activation, extras)
#   loss (default L2), pdf (data_pdf in [0.2, 5]), enc ("identity" / "levels24" / "smoothstep"), module (module tier, caller's
#   dL/dy and the grid's input gradient), infer (network.inference against the step's output)
CASES = {
    "leaky": (3, 64, 2, "LeakyReLU", "None", {}),
    "sigmoid": (3, 64, 2, "Sigmoid", "None", {}),
    "tanh_sigmoid": (3, 64, 3, "Tanh", "Sigmoid", {}),
    "squareplus": (3, 64, 2, "Squareplus", "None", {}),
    "softplus_exp": (3, 64, 2, "Softplus", "Exponential", {"infer": True}),
    "linear": (3, 64, 2, "None", "None", {}),
    "relu_sigmoid_out": (3, 64, 2, "ReLU", "Sigmoid", {}),
    "w16_sigmoid": (3, 16, 3, "Sigmoid", "None", {}),
    "w32_softplus": (3, 32, 2, "Softplus", "None", {}),
    "w16_relu": (3, 16, 2, "ReLU", "None", {}),
    "w32_relu": (3, 32, 1, "ReLU", "None", {}),
    "deep5": (3, 64, 5, "ReLU", "None", {}),
    "deep6_tanh": (3, 64, 6, "Tanh", "None", {"enc": "levels24"}),
    "smoothstep_tanh": (3, 64, 2, "Tanh", "None", {"enc": "smoothstep"}),
    "identity_sigmoid": (3, 64, 2, "Sigmoid", "None", {"enc": "identity"}),
    "image_relu": (2, 64, 2, "ReLU", "None", {"infer": True}),
    "image_sigmoid": (2, 64, 2, "Sigmoid", "None", {"infer": True}),
    "pdf_rel_l2": (3, 64, 2, "ReLU", "None", {"loss": "RelativeL2", "pdf": True, "infer": True}),
    "pdf_variance": (3, 64, 2, "ReLU", "Exponential", {"loss": "Variance", "pdf": True}),
    "pdf_image": (2, 64, 2, "ReLU", "None", {"pdf": True}),
    "pdf_image_sigmoid": (2, 64, 2, "Sigmoid", "Exponential", {"pdf": True}),
    "ext_dy_module": (3, 64, 2, "ReLU", "Sigmoid", {"module": True}),
}


def case(name):
    D, width, nh, act, out_act, extra = CASES[name]
    return SimpleNamespace(name=name, D=D, width=width, nh=nh, act=act, out_act=out_act, loss=extra.get("loss", "L2"), pdf=extra.get("pdf", False),
                           enc=extra.get("enc"), module=extra.get("module", False), infer=extra.get("infer", False))


def make_config(c):
    with open(os.path.join(GOLDEN, "configs", ("hash3d_small" if c.D == 3 else "image2d") + ".json")) as f:
        cfg = json.load(f)
    cfg["loss"] = {"otype": c.loss}
    cfg["network"].update(n_neurons=c.width, n_hidden_layers=c.nh, activation=c.act, output_activation=c.out_act)
    if c.enc == "identity":
        cfg["encoding"] = {"otype": "Identity", "scale": 0.5, "offset": 0.25}
    elif c.enc == "levels24":
        cfg["encoding"]["n_levels"] = 24  # 48 features: wider than 32, so the parked dL/d(encoded) rows get tiles of their own
    elif c.enc == "smoothstep":
        cfg["encoding"]["interpolation"] = "Smoothstep"
    return cfg


# ---- restatements of the host-side rules (pinned to the sources by the premise test)


def encoded_width(c, cfg):
    """build_encoding_plan(..., 16): the encoding's features padded to a multiple of 16."""
    n = c.D if c.enc == "identity" else cfg["encoding"]["n_levels"] * cfg["encoding"]["n_features_per_level"]
    return (n + 15) // 16 * 16


def base_smem_bytes(nh, enc_width, train):
    """fused_step.h fused_ws_base_smem_bytes."""
    return (2 + nh + ((1 if enc_width <= 32 else 3) if train else 0)) * TILE * 128 + nh * 64 * 128 + 16 * 128 + 128


def dw_in_smem(nh, enc_width):
    """fused_step.h fused_ws_dw_in_smem: the CTA's weight-gradient sums stay in shared memory across tiles."""
    return base_smem_bytes(nh, enc_width, True) + nh * 64 * 64 * 4 + 64 * 16 * 4 <= 227 * 1024


def smem_bytes(nh, enc_width, train):
    """fused_ws.cu fused_ws_smem_bytes."""
    return base_smem_bytes(nh, enc_width, train) + (nh * 64 * 64 * 4 + 64 * 16 * 4 if train and dw_in_smem(nh, enc_width) else 0)


def fused_kernel_unsupported(c, cfg):
    """model.cu fused_kernel_unsupported: None when the fused kernel runs the configuration."""
    enc = cfg["encoding"]
    grid = enc["otype"] in ("HashGrid", "DenseGrid", "TiledGrid", "Grid")
    if not grid and enc["otype"] != "Identity":
        return "encoding"
    if c.act in ("Sine", "SiLU"):
        return "pre-activation"
    if c.width > 64:
        return "width"
    if c.nh > 6:
        return "depth"
    if N_OUT > 16:
        return "outputs"
    if grid and enc.get("n_features_per_level", 2) != 2:
        return "features per level"
    if c.D not in (2, 3):
        return "input dims"
    w = encoded_width(c, cfg)
    if w > 64 or (grid and enc["n_levels"] > 32):
        return "encoding width"
    if smem_bytes(c.nh, w, True) > 227 * 1024:
        return "shared memory"
    if grid and enc.get("interpolation", "Linear") == "Nearest":
        return "Nearest"
    return None


def instances(c):
    """(D, TRAIN, GENERIC_ACT, PDF) of the kernels the case launches (fused_ws.cu launch_ws_act / launch_ws_pdf)."""
    generic = c.act != "ReLU" or c.out_act != "None"
    pdf = c.pdf and not c.module  # the module tier hands a caller's dL/dy: no pdf
    out = [(c.D, True, generic, pdf)]
    if c.infer:
        out.append((c.D, False, generic, False))
    return out


def test_premise_every_instance_past_one_tile_per_cta():
    with open(os.path.join(CSRC, "fused_ws.cu")) as f:
        ws = f.read()
    with open(os.path.join(CSRC, "model.cu")) as f:
        model = f.read()
    with open(os.path.join(CSRC, "fused_step.h")) as f:
        step_h = f.read()
    # the dispatch rule restated in instances()
    assert "const bool generic = p.activation != ACT_RELU || p.output_activation != ACT_NONE;" in ws
    assert "if (TRAIN && p.data_pdf && !p.ext_dy) return launch_ws_act<D, TRAIN, TRAIN>(p, n_ctas, stream);" in ws
    assert "return launch_ws_act<D, TRAIN, false>(p, n_ctas, stream);" in ws
    assert len(re.findall(r"launch_ws_pdf<([23]), (true|false)>", ws)) == 4
    # one CTA per SM, each over a contiguous range of tiles
    assert model.count("launch_fused_ws(p, m.n_in, true,std::min(batch / TILE_M, (uint32_t)m.n_sms), stream)") == 1
    assert model.count("launch_fused_ws(p, m.n_in, false,std::min(batch / TILE_M, (uint32_t)m.n_sms), stream)") == 1
    assert "const uint32_t cta_first = (uint32_t)(((uint64_t)blockIdx.x * n_tiles) / gridDim.x);" in ws
    # the limits restated in fused_kernel_unsupported / smem_bytes
    body = model[model.index("static const char* fused_kernel_unsupported"):]
    body = body[: body.index("\n}\n")]
    assert len(re.findall(r"\breturn \"", body)) == 10, body
    for limit in ("mlp.width > 64", "mlp.n_hidden_layers > 6", "mlp.padded_out_width != 16", "grid->n_features_per_level != 2", "n_in != 2 && n_in != 3",
                  "plan.width > 64 || (grid && grid->n_levels > MAX_LEVELS)", "fused_ws_smem_bytes(mlp.n_hidden_layers, plan.width, true) > 227 * 1024",
                  "grid->interpolation == INTERP_NEAREST", "activation_needs_preact(mlp.activation)"):
        assert limit in body, limit
    assert "const uint32_t tiles = 2 + n_hidden_layers + (train ? (enc_width <= 32 ? 1 : 3) : 0);" in step_h
    assert "return tiles * TILE_M * 128 + n_hidden_layers * 64 * 128 + 16 * 128 + 128;" in step_h
    assert "return n_hidden_layers * 64 * 64 * 4 + 64 * 16 * 4;" in step_h

    reached = set()
    for name in CASES:
        c = case(name)
        cfg = make_config(c)
        assert fused_kernel_unsupported(c, cfg) is None, name
        reached.update(instances(c))
    assert reached == {(D, t, g, p) for D in (2, 3) for t in (True, False) for g in (True, False) for p in ((True, False) if t else (False,))}
    assert len(reached) == 12
    # 7-8 tiles per CTA on a 132-SM H100
    assert B % 256 == 0 and B // TILE >= 4 * H100_SMS
    # both ways of keeping the weight-gradient sums: in shared memory across tiles, and flushed after every tile
    widths = {name: encoded_width(case(name), make_config(case(name))) for name in CASES}
    assert not dw_in_smem(5, widths["deep5"]) and not dw_in_smem(6, widths["deep6_tanh"]) and dw_in_smem(3, widths["tanh_sigmoid"])
    assert widths["deep6_tanh"] == 48 and widths["identity_sigmoid"] == 16


# ---- float64 references on the GPU


def ulp16(x):
    """Spacing of the fp16 numbers at |x| (2^-24 below the normal range)."""
    import torch

    _, e = torch.frexp(x)
    e = torch.where(x == 0, torch.full_like(e, -100), e)
    k = torch.clamp(e - 1, min=-14).to(torch.int64) - 10
    return ((k + 1023) << 52).view(torch.float64)  # 2^k built from its bits: exact, where pow() need not be


def rn16(x):
    """float64 -> the nearest fp16 value (ties to even), once; as float64."""
    import torch

    u = ulp16(x)
    return torch.round(x / u) * u


LEAKY = float(np.float16(0.01))


def act_fwd(act, x):
    """act_fwd_h (fused_common.cuh) on fp16 values, exact math, rounded to fp16."""
    import torch

    if act == "ReLU":
        return torch.clamp(x, min=0.0)
    if act == "LeakyReLU":
        return torch.where(x > 0, x, rn16(x * LEAKY))
    if act == "None":
        return x
    if act == "Exponential":
        return rn16(torch.exp(x))
    if act == "Sigmoid":
        return rn16(torch.sigmoid(x))
    if act == "Squareplus":
        v = x * 10.0
        return rn16(0.5 * (v + torch.sqrt(v * v + 4.0)) / 10.0)
    if act == "Softplus":
        return rn16(torch.nn.functional.softplus(x * 10.0) / 10.0)
    assert act == "Tanh"
    return rn16(torch.tanh(x))


def act_bwd_factor(act, f):
    """The fp16 factor act_bwd_h multiplies the gradient by, from the stored forward value f: (low, high) over the fp32
    evaluation errors where it is not exact, and the value itself."""
    import torch

    if act == "ReLU":
        v = (f > 0).double()
        return v, v, v
    if act == "LeakyReLU":
        v = torch.where(f > 0, torch.ones_like(f), torch.full_like(f, LEAKY))
        return v, v, v
    if act == "None":
        v = torch.ones_like(f)
        return v, v, v
    if act == "Exponential":
        return f, f, f
    if act == "Sigmoid":
        v = rn16(f * rn16(1.0 - f))  # 1 - f is exact in fp32
        return v, v, v
    if act == "Tanh":
        phi, d = 1.0 - f * f, 2.0 ** -24  # f^2 exact in fp32, one rounding of the difference
    elif act == "Squareplus":
        y2 = (10.0 * f) ** 2
        phi = y2 / (y2 + 1.0)
        d = phi * 2.0 ** -21  # y^2, + 1 and the fast-math division
    else:
        assert act == "Softplus"
        phi, d = -torch.expm1(-10.0 * f), 2.0 ** -21  # 1 - __expf(-10 f): absolute error of the fast exp near 1
    return rn16(phi - d), rn16(phi + d), rn16(phi)


def check_interval(what, dev, lo, hi, mid, p_flip):
    """dev within [lo, hi] everywhere; the fraction of elements not bit-equal to mid within the ceiling from p_flip."""
    import torch

    bad = ~((dev >= lo) & (dev <= hi))
    if bad.any():
        i = torch.nonzero(bad)[0].tolist()
        t = tuple(i)
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the bar, first {t}: dev {dev[t].item()!r} "
                             f"bar [{lo[t].item()!r}, {hi[t].item()!r}] ref {mid[t].item()!r}")
    n = dev.numel()
    p = float(p_flip.mean())
    ceiling = p + 5.0 * (p / n) ** 0.5 + 1.0 / n
    neq = float((dev != mid).double().mean())
    assert neq <= ceiling, f"{what}: {neq:.3e} of the elements differ from the rounded reference, ceiling {ceiling:.3e}"


def check_forward(what, act, h_prev, W, dev):
    """dev = act(fp16(W h_prev)) for the device's h_prev; W [64][k] (rows beyond the network's width are zero)."""
    import torch

    z = h_prev @ W.T
    e = 2.0 ** -22 * (h_prev.abs() @ W.abs().T)
    lo, hi, mid = act_fwd(act, rn16(z - e)), act_fwd(act, rn16(z + e)), act_fwd(act, rn16(z))
    p = torch.clamp(2.0 * e / ulp16(z), max=1.0)
    if act in TRANSCENDENTAL:
        lo, hi = lo - ulp16(lo), hi + ulp16(hi)
        p = torch.clamp(p + 2.0 ** -8, max=1.0)
    check_interval(what, dev, lo, hi, mid, p)


def backward_bounds(act, s, e, f):
    """fp16(fp16(s') * factor(f)) for the device's fp32 sum s' within e of s: (low, high, value at s, flip chance)."""
    import torch

    flo, fhi, fmid = act_bwd_factor(act, f)
    glo, ghi = rn16(s - e), rn16(s + e)
    corners = torch.stack([glo * flo, glo * fhi, ghi * flo, ghi * fhi])
    lo, hi = rn16(corners.min(0).values), rn16(corners.max(0).values)
    mid = rn16(rn16(s) * fmid)
    p = torch.clamp(2.0 * e / ulp16(s), max=1.0)
    if act in ("Tanh", "Squareplus", "Softplus"):
        p = torch.clamp(p + (fhi != flo).double(), max=1.0)
    return lo, hi, mid, p


def check_backward(what, act, g, W, f, dev):
    """dev = act_bwd(fp16(g W), f) for the device's g [B][n] and W [n][k]; f [B][k] the forward values (None: no activation)."""
    s = g @ W
    e = 2.0 ** -22 * (g.abs() @ W.abs())
    lo, hi, mid, p = backward_bounds(act, s, e, f if f is not None else s)
    check_interval(what, dev, lo, hi, mid, p)


def pad_rows(W, rows=64):
    import torch

    out = torch.zeros(rows, W.shape[1], dtype=W.dtype, device=W.device)
    out[: W.shape[0]] = W
    return out


def pad_cols(a, cols=64):
    import torch

    out = torch.zeros(a.shape[0], cols, dtype=a.dtype, device=a.device)
    out[:, : a.shape[1]] = a
    return out


def loss_reference(name, pred, tgt, pdf, n_total):
    """losses/*.h with data_pdf (1 without one): per-element value, d(value)/d(pred) x n_total, and the magnitude of the value's
    terms (the scale of its fp32 rounding)."""
    d = pred - tgt
    if name == "L2":
        v = d * d / pdf / n_total
        return v, 2 * d / pdf, v.abs()
    if name == "RelativeL2":
        psq = pred * pred + 0.01
        v = d * d / psq / pdf / n_total
        return v, 2 * d / psq / pdf, v.abs()
    assert name == "Variance"
    factor = tgt * tgt / pdf / n_total
    return factor / pred - factor / pdf, -factor / (pred * pred) * n_total, (factor / pred).abs() + (factor / pdf).abs()


# ---- one model, three steps


class Run:
    def __init__(self, torch, c):
        import tcnn_b200

        self.torch, self.c = torch, c
        self.cfg = make_config(c)
        self.model = tcnn_b200.create_from_config(c.D, N_OUT, self.cfg)
        self.mod = tcnn_b200.Module(c.D, N_OUT, self.cfg["encoding"], self.cfg["network"]) if c.module else None
        self.grid = c.enc != "identity"
        self.n_mlp = self.model.n_mlp_params
        self.in_w = self.model.encoded_width
        assert self.in_w == encoded_width(c, self.cfg)
        self.n_feat = self.in_w if not self.grid else self.cfg["encoding"]["n_levels"] * 2
        self.p16 = self.model.trainer.params().clone()  # the module tier gets the trainer's initial parameters
        rng = ob.default_rng(SEED)
        x = ob.generate_random_uniform(rng, B * c.D).reshape(B, c.D)
        self.x = np.ascontiguousarray(x)
        self.xd = torch.from_numpy(self.x).cuda()
        self.yd = torch.from_numpy(ob.make_targets(self.x, N_OUT)).cuda()
        g = torch.Generator(device="cuda").manual_seed(SEED)
        self.pdf = (0.2 + 4.8 * torch.rand(B, N_OUT, device="cuda", generator=g)).contiguous() if c.pdf else None
        self.dy_in = None
        if c.module:
            dy = torch.zeros(B, 16, device="cuda")
            dy[:, :N_OUT] = (torch.rand(B, N_OUT, device="cuda", generator=g) * 2 - 1) * 4
            self.dy_in = dy.to(torch.float16).contiguous()

    def close(self):
        import tcnn_b200

        for h in (self.model, self.mod):
            if h is not None:
                tcnn_b200.TrainableModel.set_debug_taps(h)
                h.close()

    def step(self, binned, taps_on, input_grad=False):
        """One step without the optimizer; the module handle is a model of the same C ABI, so the model's debug calls take it."""
        import tcnn_b200

        torch, c = self.torch, self.c
        nan = float("nan")
        taps = {}
        if taps_on:
            taps = dict(encoded=torch.full((B, 64), nan, dtype=torch.float16, device="cuda"),
                        hidden=torch.full((c.nh, B, 64), nan, dtype=torch.float16, device="cuda"),
                        output=torch.full((B, 16), nan, dtype=torch.float16, device="cuda"),
                        dL_doutput=torch.full((B, 16), nan, dtype=torch.float16, device="cuda"),
                        grad_hidden=torch.full((c.nh, B, 64), nan, dtype=torch.float16, device="cuda"),
                        dL_dencoded=torch.full((B, 64), nan, dtype=torch.float16, device="cuda"),
                        loss_values=torch.full((B, N_OUT), nan, dtype=torch.float32, device="cuda"))
        h = self.mod if c.module else self.model
        tcnn_b200.TrainableModel.debug_set(h, "binning", int(binned))
        tcnn_b200.TrainableModel.set_debug_taps(h, **taps)
        dinput, loss = None, None
        try:
            n0 = tcnn_b200.kernel_launch_count()
            if c.module:
                r = self.mod.bwd(self.xd, self.p16, self.dy_in, want_input_grad=input_grad)
                grads, dinput = r if input_grad else (r, None)
            else:
                self.model.trainer.training_step(self.xd, self.yd, run_optimizer=False, data_pdf=self.pdf)
                loss = self.model.trainer.loss()
            launches = tcnn_b200.kernel_launch_count() - n0
            if not c.module:
                grads = self.model.trainer.param_gradients().clone()
            torch.cuda.synchronize()
        finally:
            tcnn_b200.TrainableModel.set_debug_taps(h)
            tcnn_b200.TrainableModel.debug_set(h, "binning", 1)
        # premise: the fused kernel ran (after the binning pass when the batch is binned); the module tier adds the fp16 cast of
        # the network's gradients
        want = 1 + (3 if binned and self.grid else 0) + (1 if c.module else 0)
        if not input_grad:
            assert launches == want, (launches, want)
        return SimpleNamespace(taps=taps, loss=loss, grads=grads, dinput=dinput)


def written(run, name):
    return {"encoded": run.n_feat, "loss_values": N_OUT}.get(name)


def check_case(torch, run):
    c = run.c
    A = run.step(True, True)  # binned
    U = run.step(False, True)  # unbinned
    N = run.step(True, False, input_grad=c.module)  # no taps (module tier: with the grid's input gradient)

    # 1. coverage, 2. binned == unbinned per sample
    names = [k for k in A.taps if not (c.module and k == "loss_values")]
    for k in names:
        w = written(run, k)
        a, u = A.taps[k], U.taps[k]
        if w is not None:
            a, u = a[..., :w], u[..., :w]
        rows = torch.isnan(a.float()).any(-1)
        assert not rows.any(), f"{int(rows.sum())} rows of the {k} tap not written, first {torch.nonzero(rows)[0].tolist()}"
        itype = torch.int32 if a.dtype == torch.float32 else torch.int16
        differ = (a.contiguous().view(itype) != u.contiguous().view(itype)).any(-1)
        assert not differ.any(), f"{k}: {int(differ.sum())} rows differ between the binned and the unbinned step, first {torch.nonzero(differ)[0].tolist()}"
    if c.module:
        assert torch.isnan(A.taps["loss_values"]).all(), "a step on the caller's dL/dy writes no loss values"

    t = {k: v.double() for k, v in A.taps.items()}
    width, nh, in_w = c.width, c.nh, run.in_w
    P = run.p16.double()
    W0 = P[: width * in_w].view(width, in_w)
    off = width * in_w
    Ws = [W0]
    for _ in range(1, nh):
        Ws.append(P[off : off + width * width].view(width, width))
        off += width * width
    Wout = P[off : off + 16 * width].view(16, width)
    assert off + 16 * width == run.n_mlp

    # 4. the encoding
    enc = torch.zeros(B, in_w, dtype=torch.float64, device="cuda")
    enc[:, : run.n_feat] = t["encoded"][:, : run.n_feat]
    indexed = counts = None
    if run.grid:
        orc = ob.OracleModel(c.D, N_OUT, run.cfg, scales=run.model.grid_levels()["scales"])
        assert orc.grid.padded_width == in_w and orc.n_mlp == run.n_mlp
        orc.params_fp16 = run.p16.cpu().numpy().view(np.uint16).copy()
        L = orc.grid.n_levels
        offsets = np.asarray(orc.grid.offsets[: L + 1], np.int64)
        counts = np.zeros(offsets[-1], np.int64)
        enc_dev = A.taps["encoded"][:, : run.n_feat].cpu().numpy().view(np.uint16)
        step = 1 << 15
        for lo in range(0, B, step):
            hi = min(B, lo + step)
            ref, idx = orc.encode(np.ascontiguousarray(run.x[lo:hi]), want_indices=True)
            bad = (enc_dev[lo:hi].T != ref[: run.n_feat]).any(axis=0)
            assert not bad.any(), f"{bad.sum()} samples encoded differently from the oracle, first {lo + np.flatnonzero(bad)[:8]}"
            counts += np.bincount((idx.astype(np.int64) + offsets[None, :L, None]).ravel(), minlength=offsets[-1])
        counts = np.repeat(counts, 2)  # two features per entry
        indexed = counts > 0
    else:
        # Identity: fp16(fp32(x * 0.5 + 0.25)) (exact in float64, then rounded once to fp32 and once to fp16), padding ONE
        ref = np.ones((B, in_w), np.float16)
        ref[:, : c.D] = (run.x.astype(np.float64) * 0.5 + 0.25).astype(np.float32).astype(np.float16)
        dev = A.taps["encoded"][:, :in_w].cpu().numpy()
        bad = (dev.view(np.uint16) != ref.view(np.uint16)).any(axis=1)
        assert not bad.any(), f"{bad.sum()} samples encoded differently, first {np.flatnonzero(bad)[:8]}"

    # 5. forward, layer by layer, from the device's input to each layer
    h_prev = enc
    for l in range(nh):
        check_forward(f"hidden[{l}]", c.act, h_prev, pad_rows(Ws[l]), t["hidden"][l])
        h_prev = t["hidden"][l][:, :width]
    check_forward("output", c.out_act, h_prev, Wout, t["output"])
    y = t["output"]

    # 6. loss and dL/d(output)
    dy = t["dL_doutput"]
    assert not dy[:, N_OUT:].any(), "padding columns of dL/d(output) not zero"
    if c.module:
        s, e = run.dy_in.double(), torch.zeros_like(y)
    else:
        n_total = float(B * N_OUT)
        pdf = run.pdf.double() if run.pdf is not None else torch.ones(B, N_OUT, dtype=torch.float64, device="cuda")
        value, grad, mag = loss_reference(c.loss, y[:, :N_OUT], run.yd.double(), pdf, n_total)
        dev_v = t["loss_values"]
        bad = (dev_v - value).abs() > 2.0 ** -18 * mag + 1e-30
        assert not bad.any(), f"{int(bad.sum())} loss values off the formula, first {torch.nonzero(bad)[0].tolist()}"
        lsum = float(dev_v.sum())
        assert abs(A.loss - lsum) <= 1e-4 * float(dev_v.abs().sum()), (A.loss, lsum)
        for other in (U.loss, N.loss):
            assert abs(A.loss - other) <= 1e-4 * abs(other), (A.loss, other)
        s = pad_cols(LOSS_SCALE * grad / n_total, 16)
        e = 2.0 ** -19 * s.abs()
    lo, hi, mid, p = backward_bounds(c.out_act, s[:, :N_OUT], e[:, :N_OUT], y[:, :N_OUT])
    check_interval("dL/d(output)", dy[:, :N_OUT], lo, hi, mid, p)

    # 7. backward, layer by layer
    g = dy
    for l in range(nh, 0, -1):
        W = pad_cols(Wout if l == nh else Ws[l], 64)  # [outputs of the layer][64 inputs]
        check_backward(f"grad_hidden[{l - 1}]", c.act, g[:, : W.shape[0]], W, t["hidden"][l - 1], t["grad_hidden"][l - 1])
        g = t["grad_hidden"][l - 1][:, :width]
    check_backward("dL/d(encoded)", "None", g, pad_cols(W0, 64), None, t["dL_dencoded"])

    # 8. network weight gradients over the whole batch
    g_l = [t["grad_hidden"][l][:, :width] for l in range(nh)]
    h_in = [enc] + [t["hidden"][l][:, :width] for l in range(nh - 1)]
    refs, sums = [], []
    for gl, hl in zip(g_l + [dy], h_in + [t["hidden"][nh - 1][:, :width]]):
        refs.append((gl.T @ hl).flatten())
        sums.append((gl.abs().T @ hl.abs()).flatten())
    ref, S = torch.cat(refs), torch.cat(sums)
    bar = ulp16(ref) + 2.0 ** -20 * S
    for label, st in (("binned", A), ("unbinned", U), ("untapped", N)):
        dev = st.grads[: run.n_mlp].double()
        bad = (dev - ref).abs() > bar
        assert not bad.any(), (f"{label} step: {int(bad.sum())} of {run.n_mlp} network weight gradients off the whole-batch sums, first "
                               f"{torch.nonzero(bad)[0].item()}: dev {dev[bad][0].item()!r} ref {ref[bad][0].item()!r} bar {bar[bad][0].item()!r}")
        if run.grid and run.n_feat < in_w:
            assert not dev[: width * in_w].view(width, in_w)[:, run.n_feat :].any(), f"{label} step: gradients of W_0's padded-feature columns not zero"

    # 9. table gradients
    if run.grid:
        denc = np.ascontiguousarray(A.taps["dL_dencoded"][:, :in_w].cpu().numpy().view(np.uint16).T)
        exact = orc.grid_backward(run.x, denc)
        S_e = orc.grid_backward(run.x, denc & np.uint16(0x7FFF))
        bound = (counts * 2.0 ** -11 + 2.0 ** -10) * S_e + counts * 2.0 ** -24
        res = [int(r) for r in run.model.grid_levels()["resolutions"]]
        T = 1 << run.cfg["encoding"]["log2_hashmap_size"]
        hashed = np.zeros(len(exact), bool)
        for lv in range(L):
            if res[lv] ** c.D > T:
                hashed[2 * offsets[lv] : 2 * offsets[lv + 1]] = True
        assert hashed.any()
        errs = {}
        for label, st in (("binned", A), ("unbinned", U), ("untapped", N)):
            gd = st.grads[run.n_mlp :].double().cpu().numpy()
            assert not gd[~indexed].any(), f"{label} step: gradient written to an entry no sample indexes"
            bad = np.abs(gd - exact) > bound
            assert not bad.any(), (f"{label} step: {bad.sum()} table gradients beyond the fp16-accumulation bound, first {np.flatnonzero(bad)[:4]}: "
                                   f"dev {gd[bad][:4]} exact {exact[bad][:4]} bound {bound[bad][:4]}")
            flips = (gd != 0) != (exact != 0)
            assert flips.sum() <= 1e-4 * indexed.sum(), f"{label} step: {flips.sum()} entries touched in one of the device / the exact sums only"
            errs[label] = rae(gd[hashed], exact[hashed], 99.9)
            assert errs[label] < 1.2e-2, (label, errs)
        assert errs["binned"] <= max(1.2e-2, 1.25 * errs["unbinned"]), errs

    # 10. inference: the TRAIN = false instance against the step's output
    if c.infer:
        import tcnn_b200

        n0 = tcnn_b200.kernel_launch_count()
        out = run.model.network.inference(run.xd)
        assert tcnn_b200.kernel_launch_count() - n0 == 1
        torch.cuda.synchronize()
        want = A.taps["output"][:, :N_OUT].float()
        differ = (out.view(torch.int32) != want.view(torch.int32)).any(1)
        assert not differ.any(), f"inference differs from the training step's output in {int(differ.sum())} rows, first {torch.nonzero(differ)[0].tolist()}"

    # 11. the grid's input gradient on the module tier
    if c.module:
        table = run.p16.cpu().numpy().view(np.uint16)[run.n_mlp :]
        want = orc.grid_input_gradient(run.x, denc, table)
        assert rae(N.dinput.cpu().numpy(), want, 99.0) < 1e-2


@gpu
@pytest.mark.parametrize("name", list(CASES))
def test_fused_instance_stage_by_stage(torch_cuda, name):
    torch = torch_cuda
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert B // TILE >= 4 * n_sms, "premise: every CTA trains at least four tiles"
    run = Run(torch, case(name))
    try:
        check_case(torch, run)
    finally:
        run.close()
