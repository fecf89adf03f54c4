"""Trainer::forward / Trainer::backward (trainer.h:89-157) through tcnnb_forward / tcnnb_backward / tcnnb_reduce_sum: the context's
predictions, per-element losses and loss gradient, and a backward pass that reproduces training_step -- on the fused kernel (HashGrid
3-D F=2 + FullyFusedMLP 64x2) and on the general path (128 neurons)."""
import json
import os
import subprocess

import numpy as np
import pytest

import oracle_binding as ob
from golden_util import load_case, rae
from test_gpu_trainer_ext import LOSS_SCALE, LOSSES, PATHS, batch, config, f16, grads, np_loss, same_touched

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def close_grads(a, b, n_mlp, mlp_bar=1e-3, table_bar=5e-3):
    """Two gradient vectors of the same step: the bars of test_external_dL_dy_of_the_loss_reproduces_the_plain_step."""
    assert same_touched(a, b)
    p, q = a.float().cpu().numpy(), b.float().cpu().numpy()
    assert rae(p[:n_mlp], q[:n_mlp], 99.9) < mlp_bar, rae(p[:n_mlp], q[:n_mlp], 99.9)
    assert rae(p[n_mlp:], q[n_mlp:], 99.9) < table_bar, rae(p[n_mlp:], q[n_mlp:], 99.9)


def pdf_for(torch, B, n_out, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (0.2 + 4.8 * torch.rand(B, n_out, device="cuda", generator=g)).contiguous()


@pytest.mark.parametrize("path", list(PATHS))
def test_output_is_the_inference_output(torch_cuda, path):
    torch = torch_cuda
    import tcnn_b200

    B, n_out = 8192, 3
    model = tcnn_b200.create_from_config(3, n_out, config("RelativeL2", PATHS[path], "Exponential"))
    x, y = batch(torch, B, 1)
    ctx = model.trainer.forward(x, y)
    inf = model.network.inference(x)
    torch.cuda.synchronize()
    assert ctx.output.shape == (B, model.network.padded_output_width()) and ctx.output.dtype == torch.float16
    assert np.array_equal(ctx.output[:, :n_out].float().cpu().numpy().view(np.uint32), inf.cpu().numpy().view(np.uint32))


@pytest.mark.parametrize("with_pdf", [False, True])
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("loss", LOSSES)
def test_context_matches_the_loss_formulas_and_the_step(torch_cuda, loss, path, with_pdf):
    """ctx.L and ctx.dL_doutput against losses/*.h restated in numpy on ctx.output, and against the debug taps of a training step on
    the same parameters and batch: the fused kernel evaluates the loss with the same expressions in its epilogue, so on that path
    the values agree bit for bit, and its dL/d(output) tap is ctx.dL_doutput through the output activation (Exponential:
    fp16(dL_doutput x output))."""
    torch = torch_cuda
    import tcnn_b200

    B, n_out = 4096, 3
    model = tcnn_b200.create_from_config(3, n_out, config(loss, PATHS[path], "Exponential"))
    pad = model.network.padded_output_width()
    x, y = batch(torch, B, 2)
    pdf = pdf_for(torch, B, n_out, 3) if with_pdf else None
    ctx = model.trainer.forward(x, y, data_pdf=pdf)
    out_tap = torch.zeros(B, 16, dtype=torch.float16, device="cuda")
    dy_tap = torch.zeros(B, 16, dtype=torch.float16, device="cuda")
    lv_tap = torch.zeros(B, n_out, device="cuda")
    model.set_debug_taps(output=out_tap, dL_doutput=dy_tap, loss_values=lv_tap)
    model.trainer.training_step(x, y, run_optimizer=False, data_pdf=pdf)
    model.set_debug_taps()
    torch.cuda.synchronize()

    pred16 = ctx.output[:, :n_out].cpu().numpy()
    pred = pred16.astype(np.float64)
    tgt = y.cpu().numpy().astype(np.float64)
    p = pdf.cpu().numpy().astype(np.float64) if with_pdf else np.ones_like(tgt)
    value, grad = np_loss(loss, pred, tgt, p, B * n_out)
    L, dy = ctx.L.cpu().numpy(), ctx.dL_doutput.cpu().numpy()
    assert L.shape == (B, pad) and not L[:, n_out:].any()
    assert not dy[:, n_out:].view(np.uint16).any()
    assert rae(L[:, :n_out], value) < 1e-3
    want = np.float16(LOSS_SCALE * grad / (B * n_out))
    ulp = np.abs(dy[:, :n_out].view(np.int16).astype(np.int32) - want.view(np.int16).astype(np.int32))
    assert ulp.max() <= 1, (ulp.max(), np.argmax(ulp))

    step_dy = (dy[:, :n_out] * pred16).astype(np.float16)  # activation_backward_output of Exponential, in fp16
    if path == "fused":
        assert np.array_equal(f16(out_tap)[:, :n_out], pred16.view(np.uint16))
        assert np.array_equal(lv_tap.cpu().numpy().view(np.uint32), L[:, :n_out].view(np.uint32))
        assert np.array_equal(f16(dy_tap)[:, :n_out], step_dy.view(np.uint16))
    else:
        assert rae(out_tap[:, :n_out].float().cpu().numpy(), pred) < 1e-3
        assert rae(lv_tap.cpu().numpy(), L[:, :n_out]) < 1e-3
        assert rae(dy_tap[:, :n_out].float().cpu().numpy(), step_dy.astype(np.float32)) < 1e-3


@pytest.mark.parametrize("path", list(PATHS))
def test_forward_backward_reproduces_the_training_step(torch_cuda, path):
    """forward + backward(Overwrite) gives the gradients of training_step(run_optimizer=False); with optimizer_step after each, five
    steps follow the plain trainer's trajectory."""
    torch = torch_cuda
    import tcnn_b200

    B, n_out = 16384, 3  # the fused path bins a batch this large: the step and the split visit the samples in different orders
    cfg = config("L2", PATHS[path])
    a = tcnn_b200.create_from_config(3, n_out, cfg)
    b = tcnn_b200.create_from_config(3, n_out, cfg)
    x, y = batch(torch, B, 4)
    ctx = a.trainer.forward(x, y)
    a.trainer.backward(ctx, x)
    g_split = grads(a)
    a.trainer.training_step(x, y, run_optimizer=False)
    close_grads(g_split, grads(a), a.n_mlp_params)

    for step in range(5):
        xs, ys = batch(torch, B, 200 + step)
        ctx = a.trainer.forward(xs, ys)
        a.trainer.backward(ctx, xs)
        a.trainer.optimizer_step()
        b.trainer.training_step(xs, ys, run_optimizer=True)
    torch.cuda.synchronize()
    pa, pb = a.trainer.params().float().cpu().numpy(), b.trainer.params().float().cpu().numpy()
    assert rae(pa, pb) < 0.03


@pytest.mark.parametrize("path", list(PATHS))
def test_own_loss_through_the_context(torch_cuda, path):
    """forward(external_dL_dy=buf), buf written from ctx.output, backward: the step training_step_ex takes with that buf."""
    torch = torch_cuda
    import tcnn_b200

    B, n_out = 8192, 3
    model = tcnn_b200.create_from_config(3, n_out, config("L2", PATHS[path], "Tanh"))
    pad = model.network.padded_output_width()
    x, y = batch(torch, B, 5)
    buf = torch.zeros(B, pad, dtype=torch.float16, device="cuda")
    ctx = model.trainer.forward(x, None, external_dL_dy=buf)
    assert ctx.dL_doutput is buf
    buf[:, :n_out] = (LOSS_SCALE * 2 * (ctx.output[:, :n_out].float() - y) / (B * n_out)).half()
    dL_dinput = torch.empty(B, 3, device="cuda")
    model.trainer.backward(ctx, x, dL_dinput=dL_dinput)
    assert model.trainer.loss(ctx) == 0.0  # no loss was evaluated
    g_split = grads(model)
    dx_split = dL_dinput.clone()
    model.trainer.training_step(x, None, run_optimizer=False, external_dL_dy=buf, dL_dinput=dL_dinput)
    close_grads(g_split, grads(model), model.n_mlp_params)
    assert rae(dx_split.cpu().numpy(), dL_dinput.cpu().numpy(), 99.9) < 1e-3


@pytest.mark.parametrize("path", list(PATHS))
def test_gradient_modes_and_input_gradients_match_training_step_ex(torch_cuda, path):
    torch = torch_cuda
    import tcnn_b200

    B, n_out = 16384, 3
    model = tcnn_b200.create_from_config(3, n_out, config("RelativeL2", PATHS[path]))
    n_mlp = model.n_mlp_params
    xa, ya = batch(torch, B, 6)
    xb, yb = batch(torch, B, 7)

    # Ignore: the buffer keeps step A's gradients, dL/d(input) is still computed
    model.trainer.training_step(xa, ya, run_optimizer=False)
    grid, accum = model.trainer.gradient_buffers()
    torch.cuda.synchronize()
    before = (grid.clone(), accum.clone())
    dx_split, dx_step = torch.zeros(B, 3, device="cuda"), torch.zeros(B, 3, device="cuda")
    ctx = model.trainer.forward(xb, yb)
    model.trainer.backward(ctx, xb, dL_dinput=dx_split, gradient_mode="Ignore")
    torch.cuda.synchronize()
    assert torch.equal(grid.view(torch.int16), before[0].view(torch.int16))
    assert torch.equal(accum.view(torch.int32), before[1].view(torch.int32))
    model.trainer.training_step(xb, yb, run_optimizer=False, gradient_mode="Ignore", dL_dinput=dx_step)
    torch.cuda.synchronize()
    assert dx_split.abs().sum() > 0
    assert rae(dx_split.cpu().numpy(), dx_step.cpu().numpy(), 99.9) < 1e-3

    # Accumulate onto step A's gradients
    model.trainer.training_step(xa, ya, run_optimizer=False)
    ctx = model.trainer.forward(xb, yb)
    model.trainer.backward(ctx, xb, gradient_mode="Accumulate")
    g_split = grads(model)
    model.trainer.training_step(xa, ya, run_optimizer=False)
    model.trainer.training_step(xb, yb, run_optimizer=False, gradient_mode="Accumulate")
    close_grads(g_split, grads(model), n_mlp, 2e-3, 5e-3)


@pytest.mark.parametrize("path", list(PATHS))
def test_use_inference_params_reads_the_ema_weights(torch_cuda, path):
    torch = torch_cuda
    import tcnn_b200

    B, n_out = 8192, 3
    model = tcnn_b200.create_from_config(3, n_out, config("L2", PATHS[path], ema=True))
    for step in range(5):
        model.trainer.training_step(*batch(torch, B, 20 + step), run_optimizer=True)
    assert not torch.equal(model.trainer.params_inference(), model.trainer.params())
    x, y = batch(torch, B, 30)
    ctx = model.trainer.forward(x, y, use_inference_params=True)
    inf = model.network.inference(x)  # the Ema weights
    dx_split, dx_step = torch.empty(B, 3, device="cuda"), torch.empty(B, 3, device="cuda")
    model.trainer.backward(ctx, x, dL_dinput=dx_split, use_inference_params=True)
    g_split = grads(model)
    model.trainer.training_step(x, y, run_optimizer=False, use_inference_params=True, dL_dinput=dx_step)
    g_step = grads(model)
    work = model.trainer.forward(x, y)
    torch.cuda.synchronize()
    assert np.array_equal(ctx.output[:, :n_out].float().cpu().numpy().view(np.uint32), inf.cpu().numpy().view(np.uint32))
    assert not torch.equal(work.output, ctx.output)
    close_grads(g_split, g_step, model.n_mlp_params)
    assert rae(dx_split.cpu().numpy(), dx_step.cpu().numpy(), 99.9) < 1e-3


@pytest.mark.parametrize("path", list(PATHS))
def test_loss_of_a_context(torch_cuda, path):
    """loss(ctx) sums ctx.L as it is when called; loss() keeps reporting the last training step."""
    torch = torch_cuda
    import tcnn_b200

    B, n_out = 16384, 3
    model = tcnn_b200.create_from_config(3, n_out, config("RelativeL2", PATHS[path]))
    x, y = batch(torch, B, 8)
    model.trainer.training_step(x, y, run_optimizer=False)
    step_loss = model.trainer.loss()
    ctx = model.trainer.forward(x, y)
    assert model.trainer.loss() == step_loss
    assert model.trainer.loss(None) == step_loss
    got = model.trainer.loss(ctx)
    want = ctx.L.double().sum().item()
    assert abs(got - want) <= 1e-5 * abs(want), (got, want)
    assert abs(step_loss - want) <= 1e-5 * abs(want), (step_loss, want)
    ctx.L[:, 0] = 0  # what an application edits counts
    want = ctx.L.double().sum().item()
    assert abs(model.trainer.loss(ctx) - want) <= 1e-5 * abs(want)
    lib = tcnn_b200.load()
    import ctypes

    v = ctypes.c_float(-1)
    assert lib.tcnnb_reduce_sum(None, None, 0, ctypes.byref(v)) == 0 and v.value == 0.0


def test_rejections(torch_cuda):
    torch = torch_cuda
    import tcnn_b200

    lib = tcnn_b200.load()
    B = 4096
    x, y = batch(torch, B, 40)
    cfg = config("L2", 64)
    out = torch.empty(B, 16, dtype=torch.float16, device="cuda")
    L = torch.empty(B, 16, device="cuda")
    dy = torch.zeros(B, 16, dtype=torch.float16, device="cuda")
    ext = torch.zeros(B, 16, dtype=torch.float16, device="cuda")

    def fwd(handle, n, target, external=None, dL_doutput=dy.data_ptr()):
        return lib.tcnnb_forward(handle, None, n, x.data_ptr(), target, None, 0, 0, external, out.data_ptr(), L.data_ptr(), dL_doutput)

    def bwd(handle, n, mode=1):
        return lib.tcnnb_backward(handle, None, n, x.data_ptr(), out.data_ptr(), dy.data_ptr(), None, 0, mode)

    def error():
        return lib.tcnnb_last_error()

    mod = tcnn_b200.Module(3, 3, cfg["encoding"], cfg["network"])
    assert fwd(mod._h, B, y.data_ptr()) != 0 and b"tcnnb_module_create" in error()
    assert bwd(mod._h, B) != 0 and b"tcnnb_module_create" in error()
    model = tcnn_b200.create_from_config(3, 3, cfg)
    assert fwd(model._h, B, None) != 0 and b"target is null" in error()
    assert fwd(model._h, 1000, y.data_ptr()) != 0 and b"multiple of 256" in error()
    assert bwd(model._h, 1000) != 0 and b"multiple of 256" in error()
    assert fwd(model._h, B, None, ext.data_ptr()) != 0 and b"dL_doutput_dev must be null" in error()
    assert bwd(model._h, B, mode=3) != 0 and b"param_gradients_mode" in error()
    assert bwd(model._h, B, mode=-1) != 0 and b"param_gradients_mode" in error()
    assert lib.tcnnb_dp_init(model._h, None, None, 1, 0, 1) == 0
    assert fwd(model._h, B, y.data_ptr()) != 0 and b"data-parallel" in error()
    assert bwd(model._h, B) != 0 and b"data-parallel" in error()
    assert lib.tcnnb_dp_finish(model._h) == 0
    assert fwd(model._h, B, y.data_ptr()) == 0
    assert fwd(model._h, B, None, ext.data_ptr(), None) == 0
    assert bwd(model._h, B) == 0
    with pytest.raises(ValueError):
        model.trainer.backward(model.trainer.forward(x, y), x, gradient_mode="Sum")


def test_header_shim_trains_through_forward_and_backward(torch_cuda):
    binary = os.path.join(ROOT, "tests", "cpp", "shim_trainer_split")
    if not os.path.exists(binary):
        pytest.skip("tests/cpp/shim_trainer_split has not been built (python __graft_entry__.py build)")
    env = dict(os.environ, LD_LIBRARY_PATH=os.path.join(ROOT, "tiny-cuda-nn_b200") + ":" + os.environ.get("LD_LIBRARY_PATH", ""))
    out = subprocess.run([binary, "50"], capture_output=True, text=True, timeout=300, env=env)
    assert out.returncode == 0, out.stderr
    r = json.loads(out.stdout.strip().splitlines()[-1])
    assert r["last_loss"] < 0.5 * r["first_loss"], r
    assert r["max_rel_sum_error"] < 1e-5, r
    assert r["view"] is True and r["ext_loss"] == 0.0 and r["dL_dinput_norm"] > 0, r


# tests/golden/make_golden_split.sh: Trainer::forward + Trainer::backward of the unmodified reference
SPLIT_GOLDEN = ["split_relative_l2_pdf_w64", "split_l2_w128"]


@pytest.mark.parametrize("case", SPLIT_GOLDEN)
def test_split_matches_the_reference(torch_cuda, case):
    """The context and the gradients of a forward / backward pair against the reference's, from the same parameters and batch (64
    neurons: the fused kernel, 128: the general path)."""
    torch = torch_cuda
    import tcnn_b200

    z = load_case(case)
    meta = z["meta"]
    B, n_in, n_out, pad = meta["batch"], meta["n_input_dims"], meta["n_output_dims"], meta["padded_output_width"]
    model = tcnn_b200.create_from_config(n_in, n_out, meta["config"])
    assert model.n_params == meta["n_params"] and model.network.padded_output_width() == pad
    params16 = z["params_f16"].view(np.float16)
    model.trainer.set_params(torch.from_numpy(params16).cuda())
    x = torch.from_numpy(z["x_f32"].reshape(B, n_in)).cuda()
    y = torch.from_numpy(z["y_f32"].reshape(B, n_out)).cuda()
    pdf = torch.from_numpy(z["pdf_f32"].reshape(B, n_out)).cuda() if meta["with_pdf"] else None
    ctx = model.trainer.forward(x, y, data_pdf=pdf)
    model.trainer.backward(ctx, x)
    loss = model.trainer.loss(ctx)
    got = grads(model).float().cpu().numpy()
    want_loss = float(z["loss_f32"][0])
    assert abs(loss - want_loss) <= 2e-3 * abs(want_loss), (loss, want_loss)
    # the context, element by element. The initial network's outputs are ~1e-5: fp16 subnormals, whose steps (2^-24) are 1 % of the
    # values, so the outputs are held to 1 % of their largest magnitude and the loss values and gradients (dominated by the targets) to
    # the reference's bar on network outputs (tests/test_common.h:177)
    ref_out = z["output_f16"].view(np.float16).reshape(B, pad)[:, :n_out].astype(np.float32)
    ref_L = z["L_f32"].reshape(B, pad)
    ref_dy = z["dL_doutput_f16"].view(np.float16).reshape(B, pad)
    out = ctx.output[:, :n_out].float().cpu().numpy()
    assert np.abs(out - ref_out).max() <= 1e-2 * np.abs(ref_out).max(), (np.abs(out - ref_out).max(), np.abs(ref_out).max())
    assert rae(ctx.L[:, :n_out].cpu().numpy(), ref_L[:, :n_out], 99.0) < 1e-2 and not ctx.L[:, n_out:].any()
    assert rae(ctx.dL_doutput[:, :n_out].float().cpu().numpy(), ref_dy[:, :n_out].astype(np.float32), 99.0) < 1e-2
    # gradients: the bars of test_pdf_step_matches_the_reference, against the exact (double-accumulated) sums of the CPU oracle on the
    # reference's own dL/d(output)
    orc = ob.OracleModel(n_in, n_out, meta["config"])
    orc.params_fp16[:] = z["params_f16"]
    xs = np.ascontiguousarray(z["x_f32"].reshape(B, n_in))
    enc = orc.encode(xs)
    hidden, _ = orc.mlp_forward(enc)
    dW, d_enc = orc.mlp_backward(enc, hidden, np.ascontiguousarray(z["dL_doutput_f16"].reshape(B, pad)))
    exact = np.concatenate([dW, orc.grid_backward(xs, d_enc)]).astype(np.float64)
    want = z["grads_f16"].view(np.float16).astype(np.float32)
    n_mlp = model.n_mlp_params
    for part, bar in ((slice(0, n_mlp), 2e-2), (slice(n_mlp, None), 1.2e-2)):
        ref_err = rae(want[part], exact[part], 99.9)
        assert rae(got[part], exact[part], 99.9) <= max(bar, 1.25 * ref_err), (rae(got[part], exact[part], 99.9), ref_err)
        assert rae(got[part], want[part], 99.9) <= max(bar, 2.5 * ref_err)
