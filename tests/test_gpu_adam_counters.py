"""Adam's per-parameter step counters are 16 bits wide (saturating at 65535) when the trainer can prove that this changes no update,
else 32 bits. These tests run the two layouts side by side (the debug switch "adam_steps32" forces 32 bits) and require every
updated fp32 weight, fp16 weight and moment to be bit-identical: after 1 and 50 steps, across the 65535 boundary, through the
8-wide and the one-parameter kernels, with and without the zero-gradient skip."""
import ctypes
import json
import os
import struct

import numpy as np
import pytest

import tcnn_b200

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B = 1 << 14
SATURATED = 65535


def config(skip_zero=True, beta2=0.99):
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", "configs", "hash3d_small.json")))
    cfg["optimizer"]["beta2"] = beta2
    cfg["optimizer"]["skip_zero_grad_non_matrix_params"] = skip_zero
    return cfg


def batch(torch, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand(B, 3, device="cuda", generator=g)
    y = 0.2 + 0.8 * torch.rand(B, 3, device="cuda", generator=g)
    return x.contiguous(), y.contiguous()


def optimizer_state(torch, model):
    """(first moments, second moments, step counters) as device tensors over the arrays tcnnb_optimizer_state hands out."""
    m1, m2, st = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
    rc = tcnn_b200.load().tcnnb_optimizer_state(model._h, ctypes.byref(m1), ctypes.byref(m2), ctypes.byref(st), None, None)
    assert rc == 0, tcnn_b200.load().tcnnb_last_error().decode()
    n, view = model.trainer.n_params(), model.trainer._view
    return view(m1.value, n, torch.float32), view(m2.value, n, torch.float32), view(st.value, n, torch.int32)


def snapshot_steps(model):
    """The step counters a snapshot stores (uint32 whatever the width in use)."""
    blob = model.trainer.serialize(with_optimizer=True)
    n = struct.unpack_from("<Q", blob)[0]
    return np.frombuffer(blob, dtype=np.uint32, count=n, offset=16 + 2 * n + 8 * n)


def with_snapshot_steps(model, value):
    """The model's own snapshot with every step counter replaced by `value`."""
    blob = bytearray(model.trainer.serialize(with_optimizer=True))
    n = struct.unpack_from("<Q", blob)[0]
    np.frombuffer(blob, dtype=np.uint32, count=n, offset=16 + 2 * n + 8 * n)[:] = value
    return bytes(blob)


def step(torch, a, b, x, y, scalar_tail):
    """One training step of both models on the SAME gradients: the fused kernel's fp16 scatter atomics make two runs differ in the
    last bits, so b takes a's gradient table and network-weight accumulator before the optimizer runs."""
    for model in (a, b):
        model.trainer.training_step(x, y, run_optimizer=False)
    torch.cuda.synchronize()
    for dst, src in zip(b.trainer.gradient_buffers(), a.trainer.gradient_buffers()):
        dst.copy_(src)
    torch.cuda.synchronize()
    for model in (a, b):
        if not scalar_tail:
            model.trainer.optimizer_step()
            continue
        # The second range starts 3 parameters past a multiple of 8: its arrays are not 16-byte aligned, so it runs through the
        # one-parameter kernel; the first (from parameter 0, network weights included) through the 8-wide kernel.
        n, n_mlp = model.trainer.n_params(), model.trainer._m.n_mlp_params
        model.trainer.optimizer_step(ranges=[(0, n_mlp + 1024), (n_mlp + 1027, n - n_mlp - 1027)])


def pair(torch, cfg):
    a = tcnn_b200.create_from_config(3, 3, cfg)
    b = tcnn_b200.create_from_config(3, 3, cfg)
    b.debug_set("adam_steps32", 1)
    return a, b


def assert_identical(torch, a, b):
    torch.cuda.synchronize()
    for name in ("params_full_precision", "params"):
        pa, pb = getattr(a.trainer, name)(), getattr(b.trainer, name)()
        assert torch.equal(pa.view(torch.int16 if pa.dtype == torch.float16 else torch.int32), pb.view(torch.int16 if pb.dtype == torch.float16 else torch.int32)), name
    sa, sb = optimizer_state(torch, a), optimizer_state(torch, b)
    for k, name in enumerate(("first moments", "second moments")):
        assert torch.equal(sa[k].view(torch.int32), sb[k].view(torch.int32)), name
    assert torch.equal(sa[2], torch.clamp(sb[2], max=SATURATED)), "step counters"
    return sa[2], sb[2]


@pytest.mark.parametrize("scalar_tail", [False, True])
@pytest.mark.parametrize("skip_zero", [True, False])
@pytest.mark.parametrize("n_steps", [1, 50])
def test_16bit_counters_update_exactly_like_32bit(torch_cuda, n_steps, skip_zero, scalar_tail):
    torch = torch_cuda
    a, b = pair(torch, config(skip_zero))
    for i in range(n_steps):
        x, y = batch(torch, 100 + i)
        step(torch, a, b, x, y, scalar_tail)
    st, _ = assert_identical(torch, a, b)
    assert int(st.max()) == n_steps


@pytest.mark.parametrize("scalar_tail", [False, True])
@pytest.mark.parametrize("skip_zero", [True, False])
def test_counters_cross_65535_exactly(torch_cuda, skip_zero, scalar_tail):
    """Counters restored through the snapshot API just below the 16-bit limit: steps across it and past it."""
    torch = torch_cuda
    a, b = pair(torch, config(skip_zero))
    x, y = batch(torch, 7)
    step(torch, a, b, x, y, scalar_tail)
    blob = with_snapshot_steps(b, SATURATED - 4)
    a.trainer.deserialize(blob)
    b.trainer.deserialize(blob)
    for i in range(12):
        x, y = batch(torch, 200 + i)
        step(torch, a, b, x, y, scalar_tail)
    st_a, st_b = assert_identical(torch, a, b)
    assert int(st_b.max()) == SATURATED - 4 + 12 and int(st_a.max()) == SATURATED


def test_counters_written_through_the_state_pointer_reach_the_next_step(torch_cuda):
    """A caller that writes the counters through tcnnb_optimizer_state's array and then steps (without
    tcnnb_set_optimizer_progress) trains exactly as with 32-bit counters."""
    torch = torch_cuda
    a, b = pair(torch, config())
    for model in (a, b):
        optimizer_state(torch, model)[2].fill_(SATURATED - 2)
        torch.cuda.synchronize()
    for i in range(5):
        x, y = batch(torch, 300 + i)
        step(torch, a, b, x, y, False)
    st_a, st_b = assert_identical(torch, a, b)
    assert int(st_b.max()) == SATURATED + 3 and int(st_a.max()) == SATURATED


@pytest.mark.parametrize("beta2, width", [(0.99, 16), (0.999, 16), (0.9999, 32)])
def test_counter_width_follows_the_betas(torch_cuda, beta2, width):
    """A restored count above 65535 survives in a snapshot only with 32-bit counters; 16-bit ones saturate (exactly, for these betas)."""
    model = tcnn_b200.create_from_config(3, 3, config(beta2=beta2))
    model.trainer.deserialize(with_snapshot_steps(model, 70000))
    assert int(snapshot_steps(model).max()) == (SATURATED if width == 16 else 70000)
    model.debug_set("adam_steps32", 1)
    model.trainer.deserialize(with_snapshot_steps(model, 70000))
    assert int(snapshot_steps(model).max()) == 70000
