"""The Adam step, element by element, against a float64 restatement of the reference's `adam_step` (optimizers/adam.h:48-129) with
`weight_decay` (common_device.h:1045-1048), the host-side AdaBound bounds (adam.h:161-168) and the ExponentialDecay schedule
(exponential_decay.h:60-70); the Ema wrapper's full-precision average against ema.h:46-75; and snapshots that restore
ExponentialDecay's learning-rate factor.

Each case runs ONE optimizer step from a state the test sets itself, through public entry points only: fp32 masters through
set_params_full_precision, moments and per-parameter step counters (random in 0..200, so that every element evaluates its own powf)
through tcnnb_optimizer_state's arrays, the step count and base learning rate through tcnnb_set_optimizer_progress, and gradients
written into the fp16 table and fp32 network accumulator of gradient_buffers() after a training step without the optimizer -- or,
for the fp16 matrix-gradient path, into param_gradients() after it has materialised them. Errors therefore never compound.

Gradient patterns planted in every case, in groups of eight parameters (the 8-wide kernel's unit):
  * network weights: the first and the last group all zero (+0 / -0), an fp16 subnormal lane, +-65504 (and +-inf under gradient
    clipping) -- a zero-gradient network group must still step;
  * grid table: the first group all +0, a group of mixed +0 / -0 (both must be skipped whole), one non-zero lane among zeros (the
    other seven are skipped but written back), fp16 subnormals, +-65504 (and +-inf under gradient clipping), 30 % all-zero groups.
  * weights of +-0 (absolute decay takes its sign from them) and, under weight clipping, about half beyond the clipping magnitude.

Exact bars: which elements are updated, every step counter, every skipped element's fp32 weight, fp16 weight, both moments and
counter bit-identical to before, and every fp16 weight equal to (half) of the device's own fp32 weight. On the accumulator path
the accumulator is zero afterwards and the fp16 network gradients equal (half) of what was accumulated.

Relative bars, derived from the fast-math lowering (misc_kernels.cu is compiled with --use_fast_math):
  * first moment: |m - m_ref| <= 8 u * (|b1 m0| + (1 - b1) (|g| + |l2 w0|)), u = 2^-24: g carries one rounding (the l2 term), the
    two products and the sum one each -- 4 u, doubled.
  * second moment: the same form with (1 - b2) (|g| + |l2 w0|)^2 and 10 u (5 u derived: two for g^2, three for the update).
  * weight: the bar applies to the update dw = w - w0, |dw - dw_ref| <= 2 (e_lr(t) + 2^-20) * (|rd lr w0| + |ad lr| + |eff m|)
    + |eff| * (the first moment's bar) + 4 ulp(w). e_lr(t) is the relative error of the bias-corrected rate: powf(b, t) =
    ex2.approx(t * lg2.approx(b)) with lg2.approx's absolute error 2^-22.6 and ex2.approx's relative error 2^-22.5, so 1 - b^t is
    off by b^t (ln2 (2^-22.6 t + 2^-24 |t lg2 b|) + 2^-22.5) / (1 - b^t) relative -- largest at t = 1, where 1 - b is small -- plus
    sqrt.approx and div.approx (2^-22 each). 2^-20 covers the second moment's error inside sqrt(v) and the remaining roundings; that
    part is doubled. The first moment enters linearly: when b1 m0 and (1 - b1) g cancel, its absolute error (not a relative one)
    is what reaches the weight. The ulp floor covers the final roundings of w.

Measured on one H100 80GB HBM3 (700 W power limit), as the largest error over every case of this file divided by its bar:
first moment 0.26 (2.1 u of its scale), second moment 0.39 (3.9 u), weight update 0.24. The bars are therefore 2.5-4x above the
largest error seen. MEASURED holds the same ratios for the session that ran, to re-measure them.
"""
import ctypes
import json
import math
import os

import numpy as np
import pytest

import tcnn_b200

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B = 1 << 14
U = 2.0 ** -24
LOSS_SCALE = 128.0  # default_loss_scale<__half>() (common.h:243)
STATIC_DEFAULTS = dict(learning_rate=1e-2, beta1=0.9, beta2=0.99, epsilon=1e-15, l2_reg=1e-6, relative_decay=0.0, absolute_decay=0.0,
                       clipping_magnitude=0.0, gradient_clipping_magnitude=0.0, non_matrix_learning_rate_factor=1.0, non_matrix_l2_reg=0.0,
                       adabound=False, optimize_matrix_params=True, optimize_non_matrix_params=True, skip_zero_grad_non_matrix_params=True)
W_SIGMA = 0.1          # weights ~ N(0, 0.1): median |w| = 0.0674
G_SIGMA = 1e-2         # gradients after the loss scale ~ N(0, 1e-2): median |g| = 6.7e-3

# One hyper-parameter at a time, at a value where its term dominates, and all of them at once.
CASES = {
    "defaults": {},
    "relative_decay": {"relative_decay": 20.0},
    "absolute_decay": {"absolute_decay": 5.0},
    "weight_clipping": {"clipping_magnitude": 0.0674},
    "gradient_clipping": {"gradient_clipping_magnitude": 3e-3},
    "non_matrix": {"non_matrix_learning_rate_factor": 0.25, "non_matrix_l2_reg": 0.5},
    "l2": {"l2_reg": 0.5},
    "epsilon": {"epsilon": 1e-2},
    "betas": {"beta1": 0.5, "beta2": 0.75},
    "no_matrix_params": {"optimize_matrix_params": False},
    "no_non_matrix_params": {"optimize_non_matrix_params": False},
    "no_zero_skip": {"skip_zero_grad_non_matrix_params": False},
    "everything": {"relative_decay": 3.0, "absolute_decay": 0.5, "clipping_magnitude": 0.09, "gradient_clipping_magnitude": 5e-3,
                   "non_matrix_learning_rate_factor": 0.25, "non_matrix_l2_reg": 0.3, "l2_reg": 0.2, "epsilon": 1e-3, "beta1": 0.5,
                   "beta2": 0.75, "adabound": True, "skip_zero_grad_non_matrix_params": False},
}
# whole vector through the 8-wide kernel (network gradients from the fp32 accumulator / from the fp16 buffer), the one-parameter
# kernel through ranges, and 32-bit counters
PATHS = ["vec8", "vec8_fp16", "scalar", "steps32"]


def config(hp, wrappers=()):
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", "configs", "hash3d_tiny.json")))
    opt = {"otype": "Adam", **STATIC_DEFAULTS, **hp}
    for w in wrappers:
        opt = {**w, "nested": opt}
    cfg["optimizer"] = opt
    return cfg


def f32(x):
    return float(np.float32(x))


# ---------------------------------------------------------------- the reference, in float64
def adabound_bounds(hp, step_count):
    """adam.h:161-168 in float, `step_count` = the optimizer's count after this step."""
    if not hp["adabound"]:
        return 0.0, float(np.finfo(np.float32).max)
    one, b2, t = np.float32(1), np.float32(hp["beta2"]), np.float32(step_count)
    lo = np.float32(0.1) - np.float32(0.1) / ((one - b2) * t + one)
    hi = np.float32(0.1) + np.float32(0.1) / ((one - b2) * t)
    return float(lo), float(hi)


def decay_factor_after(n_steps, start, interval, end, base):
    """ExponentialDecayOptimizer::step (exponential_decay.h:60-70) run `n_steps` times: the factor the last of them used."""
    f = np.float32(1)
    for s in range(n_steps):
        if s == 0:
            f = np.float32(1)
        if s >= start and (s - start) % interval == 0 and s <= end:
            f = np.float32(f * np.float32(base))
    return f


def adam_reference(hp, lr, g16, w, m, v, steps, n_matrix, bounds):
    """adam_step (adam.h:48-129) for every element: (updated mask, w, m, v, steps, scales for the bars)."""
    d = lambda x: np.float64(np.float32(x))
    b1, b2, eps = d(hp["beta1"]), d(hp["beta2"]), d(hp["epsilon"])
    n = len(w)
    matrix = np.arange(n) < n_matrix
    g = g16.astype(np.float64) / LOSS_SCALE
    w0, m0, v0 = w.astype(np.float64), m.astype(np.float64), v.astype(np.float64)
    upd = np.where(matrix, bool(hp["optimize_matrix_params"]), bool(hp["optimize_non_matrix_params"]) & ~((g == 0) & bool(hp["skip_zero_grad_non_matrix_params"])))
    with np.errstate(invalid="ignore", over="ignore"):
        l2w = np.where(matrix, d(hp["l2_reg"]), d(hp["non_matrix_l2_reg"])) * w0
        gr = g + l2w
        if hp["gradient_clipping_magnitude"] != 0:
            gr = np.copysign(np.minimum(np.abs(gr), d(hp["gradient_clipping_magnitude"])), gr)
        m1 = b1 * m0 + (1 - b1) * gr
        v1 = b2 * v0 + (1 - b2) * gr * gr
        lr_e = np.where(matrix, np.float64(lr), np.float64(lr) * d(hp["non_matrix_learning_rate_factor"]))
        t = steps.astype(np.float64) + 1
        lr_e = lr_e * np.sqrt(1 - b2 ** t) / (1 - b1 ** t)
        eff = np.minimum(np.maximum(lr_e / (np.sqrt(v1) + eps), bounds[0]), bounds[1])
        rd, ad = d(hp["relative_decay"]), d(hp["absolute_decay"])
        decayed = (1 - rd * lr_e) * w0 - np.copysign(ad * lr_e, w0)
        w1 = decayed - eff * m1
        if hp["clipping_magnitude"] != 0:
            c = d(hp["clipping_magnitude"])
            w1 = np.clip(w1, -c, c)
        gmag = np.abs(g) + np.abs(l2w)
        if hp["gradient_clipping_magnitude"] != 0:
            gmag = np.minimum(gmag, d(hp["gradient_clipping_magnitude"]))
        scale_m = np.abs(b1 * m0) + (1 - b1) * gmag
        scale_v = b2 * v0 + (1 - b2) * gmag * gmag
        scale_w = np.abs(rd * lr_e * w0) + np.abs(ad * lr_e) + np.abs(eff * m1)
    return dict(updated=upd, w=w1, m=m1, v=v1, steps=steps + 1, t=t, eff=eff, scale_m=scale_m, scale_v=scale_v, scale_w=scale_w)


def bias_correction_rel_err(hp, t):
    """Relative error bound of sqrt(1 - b2^t) / (1 - b1^t) under the fast-math powf / sqrtf / '/' (see the module docstring)."""
    out = np.zeros_like(t)
    for beta, weight in ((f32(hp["beta2"]), 0.5), (f32(hp["beta1"]), 1.0)):
        p = beta ** t
        rel_p = math.log(2) * (2.0 ** -22.6 * t + U * np.abs(t * math.log2(beta))) + 2.0 ** -22.5
        out += weight * (p * rel_p / (1 - p) + U)
    return out + 2 * 2.0 ** -22


# ---------------------------------------------------------------- states and the device driver
def make_state(n, n_matrix, seed, hp):
    """fp32 weights, moments, counters and a float32 'raw' gradient (x loss scale) with the patterns of the module docstring."""
    assert n_matrix % 8 == 0, "the network / table boundary must fall on a group of eight"
    rng = np.random.default_rng(seed)
    w = (rng.standard_normal(n) * W_SIGMA).astype(np.float32)
    w[rng.random(n) < 0.02] = 0.0
    w[rng.random(n) < 0.02] = -0.0
    m = (rng.standard_normal(n) * G_SIGMA).astype(np.float32)
    v = (10.0 ** rng.uniform(-8, 4, n)).astype(np.float32)  # sqrt(v) from 1e-4 to 1e2: AdaBound's clamp is hit on both sides
    steps = rng.integers(0, 201, n).astype(np.uint32)
    raw = (rng.standard_normal(n) * G_SIGMA * LOSS_SCALE).astype(np.float32)
    raw[rng.random(n) < 0.05] = -0.0
    table_groups = np.arange(n_matrix // 8, n // 8)
    for gi in table_groups[rng.random(len(table_groups)) < 0.3]:
        raw[8 * gi : 8 * gi + 8] = 0.0
    clip = hp["gradient_clipping_magnitude"] != 0
    big = np.float32(np.inf) if clip else np.float32(65504)
    sub = np.float32(2.0 ** -24)  # the smallest fp16 subnormal
    # network weights (groups from parameter 0)
    raw[0:8] = 0.0
    raw[n_matrix - 8 : n_matrix] = [0.0, -0.0, 0.0, -0.0, -0.0, 0.0, 0.0, -0.0]
    raw[8:16] = [sub, 0.0, -sub, 3 * sub, 0.0, -0.0, 1023 * sub, 0.0]
    raw[16:24] = [65504, -65504, 65519, -65519, big, -big, 1.0, -1.0]  # 65519 rounds to 65504 in the conversion
    # grid table, from the boundary on
    t0 = n_matrix
    raw[t0 : t0 + 8] = 0.0
    raw[t0 + 8 : t0 + 16] = [0.0, -0.0, -0.0, 0.0, -0.0, -0.0, 0.0, -0.0]
    raw[t0 + 16 : t0 + 24] = [0.0, -0.0, 0.0, 0.0, 0.0, 0.5, -0.0, 0.0]
    raw[t0 + 24 : t0 + 32] = [sub, -sub, 0.0, 5 * sub, -1023 * sub, -0.0, sub, 0.0]
    raw[t0 + 32 : t0 + 40] = [65504, -65504, 0.0, -0.0, 65504, 0.25, -65504, 0.0]
    raw[t0 + 40 : t0 + 48] = [big, 0.0, -big, 0.5, -0.0, big, 0.0, -0.25]
    w[t0 + 16 : t0 + 24] = [0.0, -0.0, 0.1, -0.1, 0.0, -0.0, 0.2, -0.2]  # the updated lane and its skipped neighbours
    w[t0 + 32 : t0 + 40] = [0.0, -0.0, 0.0, -0.0, -0.0, 0.0, 0.3, -0.3]
    w[0:8] = [0.0, -0.0, 0.05, -0.05, 0.0, -0.0, 0.5, -0.5]
    return dict(w=w, m=m, v=v, steps=steps, raw=raw)


def optimizer_state(torch, model):
    m1, m2, st = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
    rc = tcnn_b200.load().tcnnb_optimizer_state(model._h, ctypes.byref(m1), ctypes.byref(m2), ctypes.byref(st), None, None)
    assert rc == 0, tcnn_b200.load().tcnnb_last_error().decode()
    n, view = model.trainer.n_params(), model.trainer._view
    return view(m1.value, n, torch.float32), view(m2.value, n, torch.float32), view(st.value, n, torch.int32)


def set_progress(model, step_count, learning_rate):
    lib = tcnn_b200.load()
    assert lib.tcnnb_set_optimizer_progress(model._h, step_count, learning_rate) == 0, lib.tcnnb_last_error().decode()


def new_model(torch, hp, path, wrappers=()):
    model = tcnn_b200.create_from_config(3, 3, config(hp, wrappers))
    if path == "steps32":
        model.debug_set("adam_steps32", 1)
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.rand(B, 3, device="cuda", generator=g)
    y = torch.rand(B, 3, device="cuda", generator=g)
    model.trainer.training_step(x, y, run_optimizer=False)  # arms the fp32 network-gradient accumulator
    torch.cuda.synchronize()
    return model


def device_step(torch, model, state, step_count, path):
    """Writes `state` into the model, runs one optimizer step at the optimizer's step count `step_count` and reads everything back."""
    tr = model.trainer
    n, n_mlp = tr.n_params(), tr._m.n_mlp_params
    tr.set_params_full_precision(torch.from_numpy(state["w"]).cuda())
    m1, m2, st = optimizer_state(torch, model)
    m1.copy_(torch.from_numpy(state["m"]))
    m2.copy_(torch.from_numpy(state["v"]))
    st.copy_(torch.from_numpy(state["steps"].view(np.int32)))
    torch.cuda.synchronize()
    set_progress(model, step_count, state["lr"])
    raw = torch.from_numpy(state["raw"]).cuda()
    if path == "vec8_fp16":
        tr.param_gradients().copy_(raw.half())  # materialises the network part first: the step then reads the fp16 buffer
    else:
        grid, acc = tr.gradient_buffers()
        grid.copy_(raw[n_mlp:].half())
        acc.copy_(raw[:n_mlp])
    torch.cuda.synchronize()
    if path == "scalar":
        # [0, n_mlp + 1021): a length that is not a multiple of 8, network weights from the accumulator; [n_mlp + 1027, n): an unaligned
        # start. Both run through the one-parameter kernel; the six parameters in between are not stepped at all.
        tr.optimizer_step(ranges=[(0, n_mlp + 1021), (n_mlp + 1027, n - n_mlp - 1027)])
    else:
        tr.optimizer_step()
    torch.cuda.synchronize()
    m1, m2, st = optimizer_state(torch, model)
    out = dict(w=tr.params_full_precision().cpu().numpy(), w16=tr.params().cpu().numpy(), m=m1.cpu().numpy(), v=m2.cpu().numpy(),
               steps=st.cpu().numpy().view(np.uint32), acc=tr.mlp_gradient_accumulator().cpu().numpy(), grads=tr.param_gradients().cpu().numpy())
    return out


MEASURED = {"m": 0.0, "v": 0.0, "w": 0.0}  # largest error / bar of each quantity in this session (the docstring's numbers)


def check_step(state, dev, ref, n_matrix, path):
    """The exact and relative bars of the module docstring; returns the largest error / bar of each moment and the weight."""
    n = len(state["w"])
    stepped = np.ones(n, bool)
    if path == "scalar":
        stepped[n_matrix + 1021 : n_matrix + 1027] = False
    upd = ref["updated"] & stepped
    # which elements were updated, and their counters
    assert np.array_equal(dev["steps"], np.where(upd, ref["steps"], state["steps"])), "step counters / updated elements"
    # skipped elements: bit-identical
    w16_before = state["w"].astype(np.float16)
    for name, before in (("w", state["w"]), ("m", state["m"]), ("v", state["v"])):
        assert np.array_equal(dev[name][~upd].view(np.uint32), before[~upd].view(np.uint32)), f"skipped elements changed: {name}"
    assert np.array_equal(dev["w16"][~upd].view(np.uint16), w16_before[~upd].view(np.uint16)), "skipped elements changed: fp16 weights"
    # fp16 weight = (half) fp32 weight, everywhere
    assert np.array_equal(dev["w16"].view(np.uint16), dev["w"].astype(np.float16).view(np.uint16)), "fp16 weights != (half) fp32 weights"
    # network gradients: the accumulator is re-armed; the fp16 buffer holds (half) of what was accumulated (or what was written)
    assert not np.any(dev["acc"]), "the fp32 network-gradient accumulator was not re-armed"
    assert np.array_equal(dev["grads"][:n_matrix].view(np.uint16), state["raw"][:n_matrix].astype(np.float16).view(np.uint16)), "fp16 network gradients"
    ratios = {}
    for name, scale, k in (("m", ref["scale_m"], 8 * U), ("v", ref["scale_v"], 10 * U)):
        err = np.abs(dev[name][upd].astype(np.float64) - ref[name][upd])
        bar = k * scale[upd]
        ratios[name] = float(np.max(err / bar, initial=0.0))
        assert np.all(err <= bar), f"{name}: {np.max(err / bar)} x the bar"
    w0 = state["w"][upd].astype(np.float64)
    dw_dev = dev["w"][upd].astype(np.float64) - w0
    dw_ref = ref["w"][upd] - w0
    ulp = np.spacing(np.maximum(np.abs(state["w"][upd]), np.abs(ref["w"][upd]).astype(np.float32))).astype(np.float64)
    bar = 2 * (bias_correction_rel_err(ref["hp"], ref["t"][upd]) + 2.0 ** -20) * ref["scale_w"][upd] + np.abs(ref["eff"][upd]) * 8 * U * ref["scale_m"][upd] + 4 * ulp
    err = np.abs(dw_dev - dw_ref)
    ratios["w"] = float(np.max(err / bar, initial=0.0))
    worst = np.flatnonzero(upd)[np.argmax(err / bar)] if upd.any() else -1
    assert np.all(err <= bar), f"weight update: {ratios['w']} x the bar at parameter {worst}"
    for k, r in ratios.items():
        MEASURED[k] = max(MEASURED[k], r)
    return upd


def run_case(torch, hp_over, path, step_count=0, seed=0, wrappers=(), lr_factor=None):
    hp = {**STATIC_DEFAULTS, **hp_over}
    model = new_model(torch, hp, path, wrappers)
    n, n_mlp = model.trainer.n_params(), model.n_mlp_params
    state = make_state(n, n_mlp, seed, hp)
    state["lr"] = hp["learning_rate"]
    dev = device_step(torch, model, state, step_count, path)
    lr = np.float32(hp["learning_rate"]) * (np.float32(1) if lr_factor is None else lr_factor)
    ref = adam_reference(hp, float(np.float32(lr)), state["raw"].astype(np.float16), state["w"], state["m"], state["v"], state["steps"], n_mlp,
                         adabound_bounds(hp, step_count + 1))
    ref["hp"] = hp
    upd = check_step(state, dev, ref, n_mlp, path)
    return model, state, dev, ref, upd


# ---------------------------------------------------------------- tests
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("case", list(CASES))
def test_adam_step_matches_the_reference_elementwise(torch_cuda, case, path):
    torch = torch_cuda
    model, state, dev, ref, upd = run_case(torch, CASES[case], path, step_count=3, seed=list(CASES).index(case))
    n_mlp = model.n_mlp_params
    hp = {**STATIC_DEFAULTS, **CASES[case]}
    # premises of the planted patterns
    if hp["optimize_matrix_params"]:
        assert upd[:8].all() and upd[n_mlp - 8 : n_mlp].all(), "zero-gradient network groups must step"
    else:
        assert not upd[:n_mlp].any()
    if hp["optimize_non_matrix_params"]:
        skip_zero = hp["skip_zero_grad_non_matrix_params"]
        assert upd[n_mlp : n_mlp + 16].all() != skip_zero, "zero-gradient table groups (+0, and mixed +0 / -0)"
        assert upd[n_mlp + 21] and upd[n_mlp + 16 : n_mlp + 24].sum() == (8 if not skip_zero else 1)
    else:
        assert not upd[n_mlp:].any()
    if hp["clipping_magnitude"]:
        c = f32(hp["clipping_magnitude"])
        beyond = np.abs(state["w"]) > c
        assert 0.3 < beyond.mean() < 0.7 and np.all(np.abs(dev["w"][upd]) <= c)
    if hp["gradient_clipping_magnitude"]:
        g = np.abs(state["raw"].astype(np.float16).astype(np.float64) / LOSS_SCALE)
        assert hp["gradient_clipping_magnitude"] < np.median(g[g > 0])
    if hp["absolute_decay"]:
        zero = upd & (state["w"] == 0)
        assert zero.sum() > 100 and np.signbit(state["w"][zero]).any() and (~np.signbit(state["w"][zero])).any()


@pytest.mark.parametrize("path", ["vec8", "scalar"])
@pytest.mark.parametrize("step_count", [0, 1, 2, 3, 4])
def test_adabound_clamps_on_both_sides(torch_cuda, step_count, path):
    """AdaBound over the optimizer's steps 1-5: the bounds move with the step count and clamp the effective rate from below and above."""
    torch = torch_cuda
    hp = {"adabound": True}
    _, _, _, ref, upd = run_case(torch, hp, path, step_count=step_count, seed=10 + step_count)
    lo, hi = adabound_bounds({**STATIC_DEFAULTS, **hp}, step_count + 1)
    eff = ref["eff"][upd]
    assert (eff == lo).sum() > 100 and (eff == hi).sum() > 100 and ((eff > lo) & (eff < hi)).sum() > 100


DECAY = {"otype": "ExponentialDecay", "decay_start": 10, "decay_interval": 5, "decay_end": 30, "decay_base": 0.5}


@pytest.mark.parametrize("step_count", [0, 9, 10, 11, 14, 15, 30, 31, 35, 40])
def test_exponential_decay_schedule(torch_cuda, step_count):
    """The learning rate of the step taken at the optimizer's step count `step_count` (set with tcnnb_set_optimizer_progress): before
    and at decay_start, at and between interval boundaries, at and after decay_end."""
    torch = torch_cuda
    factor = decay_factor_after(step_count + 1, DECAY["decay_start"], DECAY["decay_interval"], DECAY["decay_end"], DECAY["decay_base"])
    model, *_ = run_case(torch, {}, "vec8", step_count=step_count, seed=20, wrappers=(DECAY,), lr_factor=factor)
    assert tcnn_b200.load().tcnnb_learning_rate_factor(model._h) == factor
    expected = {0: 1, 9: 1, 10: 0.5, 11: 0.5, 14: 0.5, 15: 0.25, 30: 2.0 ** -5, 31: 2.0 ** -5, 35: 2.0 ** -5, 40: 2.0 ** -5}[step_count]
    assert factor == expected


def test_ema_full_precision_average(torch_cuda):
    """Ema with "full_precision": true (ema.h:46-60): the average is kept in fp32 (`tmp`) and only its fp16 copy is what inference
    reads. Three optimizer steps on injected gradients; the average restated in float64 from the device's own fp16 working weights."""
    torch = torch_cuda
    decay = 0.75
    cfg = config({}, ({"otype": "Ema", "decay": decay, "full_precision": True},))
    model = tcnn_b200.create_from_config(3, 3, cfg)
    tr = model.trainer
    n = tr.n_params()
    rng = np.random.default_rng(3)
    tmp = np.zeros(n)
    half = np.zeros(n, np.float16)  # the same average kept in fp16 (ema.h:62-75), which the fp32 one must not be
    d = float(np.float32(decay))
    for t in range(1, 4):
        tr.param_gradients().copy_(torch.from_numpy((rng.standard_normal(n) * G_SIGMA * LOSS_SCALE).astype(np.float16)).cuda())
        torch.cuda.synchronize()
        tr.optimizer_step()
        torch.cuda.synchronize()
        w16 = tr.params().cpu().numpy().astype(np.float64)
        # the debiasing factors as the host computes them: std::pow of floats promotes to double, the result is rounded to float
        old = f32(1.0 - d ** (t - 1))
        new = f32(1.0 / (1.0 - d ** t))
        tmp = (tmp * d * old + w16 * (1 - d)) * new
        half = ((half.astype(np.float64) * d * old + w16 * (1 - d)) * new).astype(np.float32).astype(np.float16)
        ema = tr.params_inference().cpu().numpy()
        ulps = np.abs(ema.view(np.int16).astype(np.int64) - tmp.astype(np.float32).astype(np.float16).view(np.int16).astype(np.int64))
        # the kernel's fp32 roundings move a value across an fp16 rounding boundary only rarely
        assert ulps.max() <= 1 and (ulps == 0).mean() > 0.999, (t, ulps.max(), (ulps == 0).mean())
    assert (ema.view(np.int16) != half.view(np.int16)).mean() > 0.01, "the fp16 average is indistinguishable here"


# ---------------------------------------------------------------- ExponentialDecay across snapshots
SNAP_DECAY = {"otype": "ExponentialDecay", "decay_start": 2, "decay_interval": 2, "decay_end": 100, "decay_base": 0.5}


def snapshot_model(torch):
    return tcnn_b200.create_from_config(3, 3, config({}, (SNAP_DECAY,)))


def inject_and_step(torch, model, k):
    """One optimizer step on gradients that depend only on k (written into the fp16 gradient buffer: no training step, no atomics)."""
    n = model.trainer.n_params()
    g = np.random.default_rng(1000 + k).standard_normal(n) * G_SIGMA * LOSS_SCALE
    model.trainer.param_gradients().copy_(torch.from_numpy(g.astype(np.float16)).cuda())
    torch.cuda.synchronize()
    model.trainer.optimizer_step()
    torch.cuda.synchronize()


def settle(torch, model):
    """Makes the fp32 masters equal (float) of the fp16 weights, as a snapshot restores them, without touching the optimizer."""
    model.trainer.set_params(model.trainer.params().clone())
    torch.cuda.synchronize()


def weights(model):
    return model.trainer.params_full_precision().cpu().numpy().view(np.uint32).copy()


def test_mid_schedule_snapshot_continues_in_a_fresh_trainer(torch_cuda):
    """A snapshot taken after 5 steps (factor 0.25) loaded into a new trainer: the next 5 steps are bit-identical to the trainer that
    went on. Before the factor followed the restored step count, the new trainer ran them at factor 1, then 0.5."""
    torch = torch_cuda
    a = snapshot_model(torch)
    for k in range(5):
        inject_and_step(torch, a, k)
    settle(torch, a)
    blob = a.trainer.serialize(with_optimizer=True)
    b = snapshot_model(torch)
    b.trainer.deserialize(blob)
    for k in range(5, 10):
        inject_and_step(torch, a, k)
        inject_and_step(torch, b, k)
        assert np.array_equal(weights(a), weights(b)), f"step {k}"
    lib = tcnn_b200.load()
    assert lib.tcnnb_learning_rate_factor(b._h) == lib.tcnnb_learning_rate_factor(a._h) == decay_factor_after(10, 2, 2, 100, 0.5) == 0.0625


def test_earlier_snapshot_rewinds_the_schedule(torch_cuda):
    """A snapshot of step 3 loaded back into the same trainer after it reached step 9: the replayed steps are bit-identical to the
    ones it took the first time. Before, it kept step 9's factor (0.0625 instead of 0.5)."""
    torch = torch_cuda
    a = snapshot_model(torch)
    for k in range(3):
        inject_and_step(torch, a, k)
    settle(torch, a)
    blob = a.trainer.serialize(with_optimizer=True)
    first = []
    for k in range(3, 9):
        inject_and_step(torch, a, k)
        first.append(weights(a))
    a.trainer.deserialize(blob)
    for i, k in enumerate(range(3, 9)):
        inject_and_step(torch, a, k)
        assert np.array_equal(weights(a), first[i]), f"step {k}"
    a.trainer.deserialize(blob)
    assert tcnn_b200.load().tcnnb_learning_rate_factor(a._h) == decay_factor_after(3, 2, 2, 100, 0.5) == 0.5

