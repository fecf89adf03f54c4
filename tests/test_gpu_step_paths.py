"""The backward calls of the trainer and module tiers -- tcnnb_training_step, tcnnb_training_step_ex in every gradient mode and with
each of its optional arrays, tcnnb_module_backward with both gradients, parameters only and input only -- and the forward calls, on
the fused kernel (HashGrid 3-D F=2 + 64 neurons) and on the general path (128 neurons), at a batch without (4096) and with (16384)
the binning pass. Pinned here: how many kernels each call launches, that an input-only module call leaves nothing behind for the
next call, and that every backward call records one profile quadruple with the optimizer inside it."""
import ctypes
import json
import os

import numpy as np
import pytest

from golden_util import rae

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PATHS = {"fused": 64, "general": 128}
BATCHES = [4096, 16384]
GRADIENT_MODES = {"Ignore": 0, "Overwrite": 1, "Accumulate": 2}


def config(neurons, log2_hashmap_size=12):
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", "configs", "hash3d_small.json")))
    cfg["loss"] = {"otype": "L2"}
    cfg["network"]["n_neurons"] = neurons
    cfg["encoding"]["log2_hashmap_size"] = log2_hashmap_size
    return cfg


def ex(model, x, y, mode="Overwrite", run_optimizer=False, data_pdf=None, dL_dinput=None, dL_dy=None):
    """tcnnb_training_step_ex itself: the Python trainer sends a plain Overwrite step to tcnnb_training_step."""
    import tcnn_b200

    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    lib = tcnn_b200.load()
    tcnn_b200._check(lib.tcnnb_training_step_ex(model._h, None, x.shape[0], x.data_ptr(), ptr(y), ptr(data_pdf), int(run_optimizer), ptr(dL_dinput), 0,
                                                GRADIENT_MODES[mode], ptr(dL_dy)))


class Setup:
    """A trainer and a module of one configuration, with a batch, a dL/d(output), a data_pdf and the module's parameters."""

    def __init__(self, torch, path, B, log2_hashmap_size=12):
        import tcnn_b200

        cfg = config(PATHS[path], log2_hashmap_size)
        self.model = tcnn_b200.create_from_config(3, 3, cfg)
        self.module = tcnn_b200.Module(3, 3, cfg["encoding"], cfg["network"])
        g = torch.Generator(device="cuda").manual_seed(B + PATHS[path])
        self.x = torch.rand(B, 3, device="cuda", generator=g).contiguous()
        self.y = (0.2 + 0.8 * torch.rand(B, 3, device="cuda", generator=g)).contiguous()
        self.pdf = (0.2 + 4.8 * torch.rand(B, 3, device="cuda", generator=g)).contiguous()
        dy = torch.zeros(B, 16, device="cuda")
        dy[:, :3] = (torch.rand(B, 3, device="cuda", generator=g) * 2 - 1) * 4
        self.dy = dy.to(torch.float16).contiguous()
        self.dinput = torch.empty(B, 3, device="cuda")
        self.p16 = self.module.initial_params(seed=7).to(torch.float16).contiguous()

    def calls(self):
        """name -> (preparation, call). The preparation leaves the state the call's launch count depends on: Accumulate continues
        the fp32 network sums a step left pending, or first reads them back from the fp16 buffer when param_gradients() consumed them."""
        m, x, y = self.model, self.x, self.y
        pending = lambda: m.trainer.training_step(x, y, run_optimizer=False)  # noqa: E731
        consumed = lambda: (pending(), m.trainer.param_gradients())  # noqa: E731
        nothing = lambda: None  # noqa: E731
        return {
            "train": (nothing, lambda: m.trainer.training_step(x, y)),
            "train_no_optimizer": (nothing, pending),
            "ex_overwrite": (nothing, lambda: ex(m, x, y)),
            "ex_overwrite_optimizer": (nothing, lambda: ex(m, x, y, run_optimizer=True)),
            "ex_accumulate": (pending, lambda: ex(m, x, y, "Accumulate")),
            "ex_accumulate_after_read": (consumed, lambda: ex(m, x, y, "Accumulate")),
            "ex_accumulate_optimizer": (pending, lambda: ex(m, x, y, "Accumulate", run_optimizer=True)),
            "ex_ignore": (pending, lambda: ex(m, x, y, "Ignore")),
            "ex_dL_dinput": (nothing, lambda: ex(m, x, y, dL_dinput=self.dinput)),
            "ex_external_dL_dy": (nothing, lambda: ex(m, x, None, dL_dy=self.dy)),
            "ex_data_pdf": (nothing, lambda: ex(m, x, y, data_pdf=self.pdf)),
            "module_fwd": (nothing, lambda: self.module.fwd(x, self.p16)),
            "module_bwd": (nothing, lambda: self.module.bwd(x, self.p16, self.dy, want_input_grad=True)),
            "module_bwd_params": (nothing, lambda: self.module.bwd(x, self.p16, self.dy)),
            "module_bwd_input": (nothing, lambda: self.module.bwd(x, self.p16, self.dy, want_input_grad=True, want_param_grad=False)),
            "inference": (nothing, lambda: m.network.inference(x)),
        }


def expected_launches(path, B):
    """Kernel launches per call. Fused path: [3 binning kernels (B >= 16384)] + the fused kernel, then Adam, the fp32 -> fp16 network
    gradient finalize of the module tier and the grid input gradient as asked; Accumulate after a read first seeds the fp32 sums from
    the fp16 buffer. General path: grid forward, network forward, loss, dgrad, weight gradients, table scatter, then the same
    extras; Accumulate adds the overwritten table gradients onto the buffer; Ignore computes no parameter gradients."""
    adam = finalize = input_grad = seed = 1
    if path == "fused":
        bwd = (3 if B >= 16384 else 0) + 1
        forward = 1
        accumulate = 0
        no_params = bwd
    else:
        forward = 2
        bwd = forward + 1 + 2 + 1
        accumulate = 1
        no_params = forward + 1 + 1
    module_bwd = bwd - (0 if path == "fused" else 1)  # (no loss)
    module_no_params = no_params - (0 if path == "fused" else 1)
    return {
        "train": bwd + adam,
        "train_no_optimizer": bwd,
        "ex_overwrite": bwd,
        "ex_overwrite_optimizer": bwd + adam,
        "ex_accumulate": bwd + accumulate,
        "ex_accumulate_after_read": seed + bwd + accumulate,
        "ex_accumulate_optimizer": bwd + accumulate + adam,
        "ex_ignore": no_params,
        "ex_dL_dinput": bwd + input_grad,
        "ex_external_dL_dy": bwd - (0 if path == "fused" else 1),
        "ex_data_pdf": bwd,
        "module_fwd": forward,
        "module_bwd": module_bwd + finalize + input_grad,
        "module_bwd_params": module_bwd + finalize,
        "module_bwd_input": module_no_params + input_grad,
        "inference": forward,
    }


CASES = sorted(expected_launches("fused", 4096))


@pytest.fixture(scope="module")
def setups(torch_cuda):
    cache = {}

    def get(path, B):
        if (path, B) not in cache:
            cache[path, B] = Setup(torch_cuda, path, B)
        return cache[path, B]

    return get


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("path", list(PATHS))
def test_launches_per_call(torch_cuda, setups, path, B, case):
    import tcnn_b200

    prepare, call = setups(path, B).calls()[case]
    call()  # first call: scratch allocations
    prepare()
    before = tcnn_b200.kernel_launch_count()
    call()
    launches = tcnn_b200.kernel_launch_count() - before
    torch_cuda.cuda.synchronize()
    assert launches == expected_launches(path, B)[case], launches


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("path", list(PATHS))
def test_module_input_only_call_leaves_nothing_behind(torch_cuda, path, B):
    """Full, input-only, full module backward on the same inputs: the two full calls agree up to the order of the fp16 atomics, and
    the input-only call's dL/d(input) is theirs."""
    torch = torch_cuda
    s = Setup(torch, path, B)
    mod, x, p, dy = s.module, s.x, s.p16, s.dy
    g1, dx1 = mod.bwd(x, p, dy, want_input_grad=True)
    g1 = g1.clone()
    _, dx_only = mod.bwd(x, p, dy, want_input_grad=True, want_param_grad=False)
    g2, dx2 = mod.bwd(x, p, dy, want_input_grad=True)
    torch.cuda.synchronize()
    n_mlp = s.model.n_mlp_params
    a, b = g1.float().cpu().numpy(), g2.float().cpu().numpy()
    assert np.abs(a[:n_mlp]).max() > 0 and np.abs(a[n_mlp:]).max() > 0
    assert rae(a[:n_mlp], b[:n_mlp], 99.9) < 1e-3
    assert rae(a[n_mlp:], b[n_mlp:], 99.9) < 5e-3
    flips = np.flatnonzero((a != 0) != (b != 0))
    assert len(flips) <= 2e-3 * max(1, np.count_nonzero(a)), len(flips)
    for dx in (dx_only, dx2):
        assert rae(dx.cpu().numpy(), dx1.cpu().numpy(), 99.9) < 1e-3


def read_profile(handle):
    import tcnn_b200

    f, o, b, n = ctypes.c_float(0), ctypes.c_float(0), ctypes.c_float(0), ctypes.c_uint32(0)
    tcnn_b200._check(tcnn_b200.load().tcnnb_read_profile(handle, ctypes.byref(f), ctypes.byref(o), ctypes.byref(b), ctypes.byref(n)))
    return {"fused_ms_total": f.value, "optimizer_ms_total": o.value, "binning_ms_total": b.value, "n_steps": n.value}


BACKWARD_CASES = [c for c in CASES if c not in ("module_fwd", "inference")]
OPTIMIZER_CASES = ("train", "ex_overwrite_optimizer", "ex_accumulate_optimizer")


@pytest.fixture(scope="module")
def large_setups(torch_cuda):
    """A 2^19-entry table: Adam over 16 M parameters takes long enough to tell apart from two adjacent events."""
    cache = {}

    def get(path, B):
        if (path, B) not in cache:
            cache[path, B] = Setup(torch_cuda, path, B, log2_hashmap_size=19)
        return cache[path, B]

    return get


@pytest.mark.parametrize("case", BACKWARD_CASES)
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("path", list(PATHS))
def test_every_backward_call_records_one_profile_step(torch_cuda, large_setups, path, B, case):
    """tcnnb_read_profile reads its events in fours (start, after binning, after the backward pass, after the optimizer): each
    backward call adds exactly one such step, and the optimizer of a call that runs it lies inside that step."""
    import tcnn_b200

    s = large_setups(path, B)
    lib = tcnn_b200.load()
    handle = s.module._h if case.startswith("module") else s.model._h
    prepare, call = s.calls()[case]
    call()
    prepare()
    tcnn_b200._check(lib.tcnnb_set_profiling(handle, 1))
    call()
    prof = read_profile(handle)
    tcnn_b200._check(lib.tcnnb_set_profiling(handle, 0))
    assert prof["n_steps"] == 1, prof
    if case in OPTIMIZER_CASES:
        assert prof["optimizer_ms_total"] > 0.02, prof
