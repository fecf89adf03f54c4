"""Trainer::training_step with all of its arguments (trainer.h:254-357) through tcnnb_training_step_ex: data_pdf in the loss, the
application's own dL/dy (external_dL_dy), the gradient modes Ignore / Overwrite / Accumulate, dL_dinput and use_inference_params --
on the fused kernel (HashGrid 3-D F=2 + FullyFusedMLP 64x2) and on the general path (128 neurons)."""
import json
import os
import subprocess

import numpy as np
import pytest

import oracle_binding as ob
from golden_util import rae

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOSSES = ["L2", "RelativeL2", "L1", "RelativeL1", "Mape", "Smape", "RelativeL2Luminance", "CrossEntropy", "Variance"]
PATHS = {"fused": 64, "general": 128}
LOSS_SCALE = 128.0


def config(loss="RelativeL2", neurons=64, output_activation="None", ema=False):
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", "configs", "hash3d_small.json")))
    cfg["loss"] = {"otype": loss}
    cfg["network"]["n_neurons"] = neurons
    cfg["network"]["output_activation"] = output_activation
    if ema:
        cfg["optimizer"] = {"otype": "Ema", "decay": 0.9, "nested": cfg["optimizer"]}
    return cfg


def f16(t):
    return t.cpu().numpy().view(np.uint16)


def grads(model):
    return model.trainer.param_gradients().clone()


def batch(torch, B, seed, n_out=3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand(B, 3, device="cuda", generator=g)
    y = 0.2 + 0.8 * torch.rand(B, n_out, device="cuda", generator=g)
    return x.contiguous(), y.contiguous()


def random_dy(torch, B, seed, n_out=3, pad=16):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dy = torch.zeros(B, pad, device="cuda")
    dy[:, :n_out] = (torch.rand(B, n_out, device="cuda", generator=g) * 2 - 1) * 4
    return dy.to(torch.float16).contiguous()


def np_loss(name, pred, tgt, pdf, n_total):
    """losses/*.h restated with data_pdf: per-element value and d(value)/d(pred) x n_total."""
    d = pred - tgt
    if name in ("RelativeL2", "RelativeL2Luminance"):
        base = pred if name == "RelativeL2" else (0.299 * pred[:, 0] + 0.587 * pred[:, 1] + 0.114 * pred[:, 2])[:, None]
        psq = base * base + 0.01
        return d * d / psq / pdf / n_total, 2 * d / psq / pdf
    if name == "L2":
        return d * d / pdf / n_total, 2 * d / pdf
    if name == "L1":
        return np.abs(d) / pdf / n_total, np.copysign(1.0, d) / pdf
    if name in ("RelativeL1", "Mape", "Smape"):
        denom = {"RelativeL1": np.abs(pred), "Mape": np.abs(tgt), "Smape": 0.5 * (np.abs(tgt) + np.abs(pred))}[name]
        scale = 1.0 / (denom + 1e-2) / pdf
        return np.abs(d) * scale / n_total, np.copysign(scale, d)
    if name == "CrossEntropy":
        factor = -tgt / pdf / n_total
        return factor * np.log(pred), factor / pred * n_total
    assert name == "Variance"
    factor = tgt * tgt / pdf / n_total  # variance_is.h:69-76: the value's second term is factor / pdf
    return factor / pred - factor / pdf, -factor / (pred * pred) * n_total


def touched(g):
    return set(np.flatnonzero(f16(g) & 0x7FFF))


def same_touched(a, b, tol=2e-3):
    """The nonzero entries of two gradient vectors agree up to fp16 atomics that landed on exactly zero in one order only."""
    ta, tb = touched(a), touched(b)
    return len(ta ^ tb) <= tol * max(1, len(ta | tb))


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("loss", LOSSES)
def test_pdf_loss_matches_the_loss_formulas(torch_cuda, path, loss):
    """Per-element loss values and the fp16 dL/d(output) of a step with data_pdf against losses/*.h restated in numpy; pdf == 1
    reproduces the plain step."""
    torch = torch_cuda
    import tcnn_b200

    B, n_out = 4096, 3
    # Exponential output: positive predictions, which CrossEntropy and Variance need
    model = tcnn_b200.create_from_config(3, n_out, config(loss, PATHS[path], "Exponential"))
    x, y = batch(torch, B, 1)
    g = torch.Generator(device="cuda").manual_seed(2)
    pdf = (0.2 + 4.8 * torch.rand(B, n_out, device="cuda", generator=g)).contiguous()
    out_tap = torch.zeros(B, 16, dtype=torch.float16, device="cuda")
    dy_tap = torch.zeros(B, 16, dtype=torch.float16, device="cuda")
    lv_tap = torch.zeros(B, n_out, device="cuda")
    model.set_debug_taps(output=out_tap, dL_doutput=dy_tap, loss_values=lv_tap)

    model.trainer.training_step(x, y, run_optimizer=False, data_pdf=pdf)
    loss_pdf = model.trainer.loss()
    torch.cuda.synchronize()
    pred = out_tap[:, :n_out].float().cpu().numpy().astype(np.float64)
    tgt, p = y.cpu().numpy().astype(np.float64), pdf.cpu().numpy().astype(np.float64)
    value, grad = np_loss(loss, pred, tgt, p, B * n_out)
    assert rae(lv_tap.cpu().numpy(), value) < 1e-3
    assert abs(loss_pdf - value.sum()) <= 1e-3 * abs(value.sum())
    # activation_backward_output of Exponential: fp16(dL/dy) x forward output, in fp16
    want = (np.float16(LOSS_SCALE * grad / (B * n_out)).astype(np.float64) * pred).astype(np.float16)
    got = dy_tap[:, :n_out].cpu().numpy()
    ulp = np.abs(got.view(np.int16).astype(np.int32) - want.view(np.int16).astype(np.int32))
    assert ulp.max() <= 1, (ulp.max(), np.argmax(ulp))

    model.trainer.training_step(x, y, run_optimizer=False)
    loss_plain = model.trainer.loss()
    g_plain = grads(model)
    model.trainer.training_step(x, y, run_optimizer=False, data_pdf=torch.ones_like(pdf))
    loss_one = model.trainer.loss()
    g_one = grads(model)
    assert abs(loss_one - loss_plain) <= 1e-6 * abs(loss_plain)
    assert same_touched(g_one, g_plain)
    assert rae(g_one.float().cpu().numpy(), g_plain.float().cpu().numpy(), 99.9) < 5e-3


@pytest.mark.parametrize("path", list(PATHS))
def test_pdf_enters_through_dL_doutput_only(torch_cuda, path):
    """The gradients of a pdf-weighted step equal those of a step on its own dL/d(output) handed back as external_dL_dy."""
    torch = torch_cuda
    import tcnn_b200

    B = 4096
    model = tcnn_b200.create_from_config(3, 3, config("RelativeL2", PATHS[path]))
    x, y = batch(torch, B, 3)
    pdf = (0.2 + 4.8 * torch.rand(B, 3, device="cuda")).contiguous()
    dy_tap = torch.zeros(B, 16, dtype=torch.float16, device="cuda")
    model.set_debug_taps(dL_doutput=dy_tap)
    model.trainer.training_step(x, y, run_optimizer=False, data_pdf=pdf)
    g_pdf = grads(model)
    model.set_debug_taps()
    model.trainer.training_step(x, None, run_optimizer=False, external_dL_dy=dy_tap.clone())
    g_ext = grads(model)
    assert same_touched(g_pdf, g_ext)
    n_mlp = model.n_mlp_params
    a, b = g_pdf.float().cpu().numpy(), g_ext.float().cpu().numpy()
    assert rae(a[:n_mlp], b[:n_mlp], 99.9) < 1e-3 and rae(a[n_mlp:], b[n_mlp:], 99.9) < 5e-3


@pytest.mark.parametrize("path", list(PATHS))
def test_external_dL_dy_matches_module_backward(torch_cuda, path):
    torch = torch_cuda
    import tcnn_b200

    B = 8192
    cfg = config("L2", PATHS[path], "Tanh")
    model = tcnn_b200.create_from_config(3, 3, cfg)
    mod = tcnn_b200.Module(3, 3, cfg["encoding"], cfg["network"])
    x, _ = batch(torch, B, 4)
    dy = random_dy(torch, B, 5)
    p16 = model.trainer.params().clone()
    dL_dinput = torch.empty(B, 3, device="cuda")
    model.trainer.training_step(x, None, run_optimizer=False, external_dL_dy=dy, dL_dinput=dL_dinput)
    assert model.trainer.loss() == 0.0  # the reference leaves L unfilled
    g_tr = grads(model)
    g_mod, dx_mod = mod.bwd(x, p16, dy, want_input_grad=True)
    g_mod2 = mod.bwd(x, p16, dy)
    torch.cuda.synchronize()
    n_mlp = model.n_mlp_params
    a, b, c = g_tr.float().cpu().numpy(), g_mod.float().cpu().numpy(), g_mod2.float().cpu().numpy()
    # touched sets: a table entry whose fp16 sum cancels to exactly zero in one reduction order only may differ (a handful in 10^5),
    # and only where the gradient is at the bottom of its range
    flips = np.flatnonzero((a != 0) != (b != 0))
    assert len(flips) <= 1e-4 * len(touched(g_mod)), len(flips)
    assert np.all(np.maximum(np.abs(a[flips]), np.abs(b[flips])) <= 1e-3 * np.abs(b).max())
    assert rae(a[:n_mlp], b[:n_mlp], 99.9) < 1e-3
    # The table gradients are sums of fp16 reductions whose order the hardware picks, so two module calls on the same inputs differ
    # by about 1e-3 already: the trainer must be no further from the module than the module is from itself.
    noise = rae(b[n_mlp:], c[n_mlp:], 99.9)
    assert rae(a[n_mlp:], b[n_mlp:], 99.9) < max(1e-3, 2 * noise), noise
    assert rae(dL_dinput.cpu().numpy(), dx_mod.cpu().numpy(), 99.9) < 1e-3


def test_dL_dinput_matches_the_oracle(torch_cuda):
    """dL/d(position) of a trainer step (fused kernel) against the oracle's grid input gradient on the module tier's dL/d(encoded)."""
    torch = torch_cuda
    import tcnn_b200

    B = 1024
    cfg = config("L2", 64)
    model = tcnn_b200.create_from_config(3, 3, cfg)
    x, _ = batch(torch, B, 6)
    dy = random_dy(torch, B, 7)
    denc_tap = torch.zeros(B, 64, dtype=torch.float16, device="cuda")
    model.set_debug_taps(dL_dencoded=denc_tap)  # (a step with dL_dinput hands these rows to the input-gradient kernel instead)
    model.trainer.training_step(x, None, run_optimizer=False, external_dL_dy=dy)
    model.set_debug_taps()
    dL_dinput = torch.empty(B, 3, device="cuda")
    model.trainer.training_step(x, None, run_optimizer=False, external_dL_dy=dy, dL_dinput=dL_dinput)
    torch.cuda.synchronize()
    orc = ob.OracleModel(3, 3, cfg, scales=model.grid_levels()["scales"])
    table = f16(model.trainer.params())[model.n_mlp_params:]
    denc_soa = f16(denc_tap)[:, : model.encoded_width].T
    want = orc.grid_input_gradient(np.ascontiguousarray(x.cpu().numpy()), denc_soa, table)
    assert rae(dL_dinput.cpu().numpy(), want, 99.9) < 2e-3


def test_external_dL_dy_of_the_loss_reproduces_the_plain_step(torch_cuda):
    """Output activation None: the plain step's dL/d(output) fed back reproduces its gradients, and ten steps of (inference, own L2
    dL/dy, external step with Adam) follow the plain trainer's trajectory."""
    torch = torch_cuda
    import tcnn_b200

    B, n_out = 16384, 3
    cfg = config("L2", 64)
    a = tcnn_b200.create_from_config(3, n_out, cfg)
    b = tcnn_b200.create_from_config(3, n_out, cfg)
    x, y = batch(torch, B, 8)
    dy_tap = torch.zeros(B, 16, dtype=torch.float16, device="cuda")
    a.set_debug_taps(dL_doutput=dy_tap)
    a.trainer.training_step(x, y, run_optimizer=False)
    g_plain = grads(a)
    a.set_debug_taps()
    a.trainer.training_step(x, None, run_optimizer=False, external_dL_dy=dy_tap.clone())
    g_ext = grads(a)
    assert same_touched(g_plain, g_ext)
    n_mlp = a.n_mlp_params
    p, q = g_plain.float().cpu().numpy(), g_ext.float().cpu().numpy()
    assert rae(p[:n_mlp], q[:n_mlp], 99.9) < 1e-3 and rae(p[n_mlp:], q[n_mlp:], 99.9) < 5e-3

    for step in range(10):
        xs, ys = batch(torch, B, 100 + step)
        a.trainer.training_step(xs, ys, run_optimizer=True)
        out = b.network.inference(xs)
        dy = torch.zeros(B, 16, device="cuda")
        dy[:, :n_out] = LOSS_SCALE * 2 * (out - ys) / (B * n_out)
        b.trainer.training_step(xs, None, run_optimizer=True, external_dL_dy=dy.to(torch.float16).contiguous())
    torch.cuda.synchronize()
    pa, pb = a.trainer.params().float().cpu().numpy(), b.trainer.params().float().cpu().numpy()
    assert rae(pa, pb) < 0.03


@pytest.mark.parametrize("path,B,read_between", [("fused", 4096, False), ("fused", 4096, True), ("fused", 16384, False), ("fused", 16384, True),
                                                  ("general", 4096, False), ("general", 4096, True)])
def test_overwrite_then_accumulate_sums_the_gradients(torch_cuda, path, B, read_between):
    torch = torch_cuda
    import tcnn_b200

    model = tcnn_b200.create_from_config(3, 3, config("RelativeL2", PATHS[path]))
    xa, ya = batch(torch, B, 10)
    xb, yb = batch(torch, B, 11)
    model.trainer.training_step(xa, ya, run_optimizer=False)
    ga = grads(model).float()
    model.trainer.training_step(xb, yb, run_optimizer=False)
    gb = grads(model).float()
    model.trainer.training_step(xa, ya, run_optimizer=False, gradient_mode="Overwrite")
    if read_between:
        model.trainer.param_gradients()
    model.trainer.training_step(xb, yb, run_optimizer=False, gradient_mode="Accumulate")
    loss_b = model.trainer.loss()
    gc = grads(model).float()
    model.trainer.training_step(xb, yb, run_optimizer=False)
    assert loss_b == pytest.approx(model.trainer.loss(), rel=1e-5)  # the loss accumulator is still zeroed
    n_mlp = model.n_mlp_params
    want, got = (ga + gb).cpu().numpy(), gc.cpu().numpy()
    assert rae(got[:n_mlp], want[:n_mlp], 99.9) < 2e-3
    assert rae(got[n_mlp:], want[n_mlp:], 99.9) < 5e-3
    assert touched(gc.half()) <= touched(ga.half()) | touched(gb.half())


@pytest.mark.parametrize("path", list(PATHS))
def test_ignore_leaves_the_gradient_buffer_alone(torch_cuda, path):
    torch = torch_cuda
    import tcnn_b200

    B = 16384
    model = tcnn_b200.create_from_config(3, 3, config("RelativeL2", PATHS[path]))
    xa, ya = batch(torch, B, 12)
    xb, yb = batch(torch, B, 13)
    model.trainer.training_step(xa, ya, run_optimizer=False)
    grid, accum = model.trainer.gradient_buffers()  # the fp32 network sums are still pending: not materialised
    torch.cuda.synchronize()
    before = (grid.clone(), accum.clone())
    dL_dinput = torch.zeros(B, 3, device="cuda")
    model.trainer.training_step(xb, yb, run_optimizer=False, gradient_mode="Ignore", dL_dinput=dL_dinput)
    loss = model.trainer.loss()
    torch.cuda.synchronize()
    assert torch.equal(grid.view(torch.int16), before[0].view(torch.int16))
    assert torch.equal(accum.view(torch.int32), before[1].view(torch.int32))
    assert loss > 0 and np.isfinite(loss)
    assert torch.isfinite(dL_dinput).all() and dL_dinput.abs().sum() > 0
    # and the buffer is still step A's
    g_after = grads(model)
    model.trainer.training_step(xa, ya, run_optimizer=False)
    assert rae(g_after.float().cpu().numpy(), grads(model).float().cpu().numpy(), 99.9) < 5e-3


def test_use_inference_params_reads_the_ema_weights(torch_cuda):
    torch = torch_cuda
    import tcnn_b200

    B = 8192
    cfg = config("L2", 64, ema=True)
    model = tcnn_b200.create_from_config(3, 3, cfg)
    mod = tcnn_b200.Module(3, 3, cfg["encoding"], cfg["network"])
    for step in range(5):
        model.trainer.training_step(*batch(torch, B, 20 + step), run_optimizer=True)
    ema = model.trainer.params_inference().clone()
    assert not torch.equal(ema, model.trainer.params())
    x, _ = batch(torch, B, 30)
    dy = random_dy(torch, B, 31)
    model.trainer.training_step(x, None, run_optimizer=False, external_dL_dy=dy, use_inference_params=True)
    g_inf = grads(model)
    g_mod = mod.bwd(x, ema, dy)
    model.trainer.training_step(x, None, run_optimizer=False, external_dL_dy=dy)
    g_work = grads(model)
    torch.cuda.synchronize()
    assert same_touched(g_inf, g_mod)
    n_mlp = model.n_mlp_params
    a, b = g_inf.float().cpu().numpy(), g_mod.float().cpu().numpy()
    assert rae(a[:n_mlp], b[:n_mlp], 99.9) < 1e-3 and rae(a[n_mlp:], b[n_mlp:], 99.9) < 5e-3
    assert rae(g_inf.float().cpu().numpy(), g_work.float().cpu().numpy(), 99.9) > 1e-2


def test_header_shim_trains_on_its_own_loss_in_micro_batches(torch_cuda):
    binary = os.path.join(ROOT, "tests", "cpp", "shim_trainer_ext")
    if not os.path.exists(binary):
        pytest.skip("tests/cpp/shim_trainer_ext has not been built (python __graft_entry__.py build)")
    env = dict(os.environ, LD_LIBRARY_PATH=os.path.join(ROOT, "tiny-cuda-nn_b200") + ":" + os.environ.get("LD_LIBRARY_PATH", ""))
    out = subprocess.run([binary, "50"], capture_output=True, text=True, timeout=300, env=env)
    assert out.returncode == 0, out.stderr
    r = json.loads(out.stdout.strip().splitlines()[-1])
    assert r["last_loss"] < 0.5 * r["first_loss"], r
    assert r["ext_step_loss"] == 0.0 and r["pdf_loss"] > 0 and r["dL_dinput_norm"] > 0, r
    assert "check failed: external_dL_dy->m() == m_model->padded_output_width()" in r["shape_error"], r


def test_rejections(torch_cuda):
    torch = torch_cuda
    import tcnn_b200

    lib = tcnn_b200.load()
    B = 4096
    x, y = batch(torch, B, 40)
    cfg = config("L2", 64)

    def call(handle, n, target, mode=1):
        return lib.tcnnb_training_step_ex(handle, None, n, x.data_ptr(), target, None, 0, None, 0, mode, None)

    mod = tcnn_b200.Module(3, 3, cfg["encoding"], cfg["network"])
    assert call(mod._h, B, y.data_ptr()) != 0 and b"tcnnb_module_create" in lib.tcnnb_last_error()
    model = tcnn_b200.create_from_config(3, 3, cfg)
    assert call(model._h, B, None) != 0 and b"target is null" in lib.tcnnb_last_error()
    assert call(model._h, 1000, y.data_ptr()) != 0 and b"multiple of 256" in lib.tcnnb_last_error()
    assert call(model._h, B, y.data_ptr(), mode=3) != 0 and b"param_gradients_mode" in lib.tcnnb_last_error()
    assert lib.tcnnb_dp_init(model._h, None, None, 1, 0, 1) == 0
    assert call(model._h, B, y.data_ptr()) != 0 and b"data-parallel" in lib.tcnnb_last_error()
    assert lib.tcnnb_dp_finish(model._h) == 0
    assert call(model._h, B, y.data_ptr()) == 0
    with pytest.raises(ValueError):
        model.trainer.training_step(x, y, gradient_mode="Sum")


# tests/golden/make_golden_pdf.sh: one step of the unmodified reference's Trainer::training_step with a data_pdf
PDF_GOLDEN = ["pdf_relative_l2_w64", "pdf_variance_w64", "pdf_relative_l2_w128", "pdf_variance_w128"]


@pytest.mark.parametrize("case", PDF_GOLDEN)
def test_pdf_step_matches_the_reference(torch_cuda, case):
    """Loss and step-0 gradients of a pdf-weighted step against the reference's, from the same parameters and batch (64 neurons: the
    fused kernel, 128: the general path)."""
    torch = torch_cuda
    import tcnn_b200
    from golden_util import load_case

    z = load_case(case)
    meta = z["meta"]
    B, n_in, n_out = meta["batch"], meta["n_input_dims"], meta["n_output_dims"]
    model = tcnn_b200.create_from_config(n_in, n_out, meta["config"])
    assert model.n_params == meta["n_params"]
    model.trainer.set_params(torch.from_numpy(z["params_f16"].view(np.float16)).cuda())
    x = torch.from_numpy(z["x_f32"].reshape(B, n_in)).cuda()
    y = torch.from_numpy(z["y_f32"].reshape(B, n_out)).cuda()
    pdf = torch.from_numpy(z["pdf_f32"].reshape(B, n_out)).cuda()
    model.trainer.training_step(x, y, run_optimizer=False, data_pdf=pdf)
    loss = model.trainer.loss()
    want_loss = float(z["loss_f32"][0])
    assert abs(loss - want_loss) <= 2e-3 * abs(want_loss), (loss, want_loss)
    got = grads(model).float().cpu().numpy()
    want = z["grads_f16"].view(np.float16).astype(np.float32)
    n_mlp = model.n_mlp_params
    # The reference sums in fp16 (split-K weight gradients, table atomics) and with pdf-weighted gradients lies 1.2e-2 .. 4e-2 from the
    # exact sums (tests/golden/add_exact_pdf_grads.py): the bars of the plain step (2e-2 network, 1.2e-2 table at p99.9) hold against
    # the reference where its own error allows, and this library must be no further from the exact sums than the reference is.
    exact = z["grads_exact_f32"].astype(np.float64)
    for part, bar in ((slice(0, n_mlp), 2e-2), (slice(n_mlp, None), 1.2e-2)):
        ref_err = rae(want[part], exact[part], 99.9)
        assert rae(got[part], exact[part], 99.9) <= max(bar, 1.25 * ref_err), (rae(got[part], exact[part], 99.9), ref_err)
        assert rae(got[part], want[part], 99.9) <= max(bar, 2.5 * ref_err)
