"""The trainer over a bare network (tcnnb_create_network_trainer, what include/tiny-cuda-nn/trainer.h builds for a Network of
create_network) against the UNMODIFIED reference's Trainer(create_network<__half>(json), optimizer, loss, 1337): tests/golden/net_trainer_*.npz
(tests/golden/make_golden_net_trainer.sh, oracle/_ref/ref_network_trainer). Same fp16 inputs and targets; each step is
training_step(run_optimizer = false), loss, optimizer_step, as the reference's driver does.
  - initial parameters bit-equal (the same pcg32 stream),
  - step-0 loss within 1e-3,
  - step-0 gradients within 2e-2 RAE at p99.9 (every parameter of a network is a weight: DESIGN.md section 4's bar for weight gradients),
  - the ten-step loss trajectory within 3 %."""
import ctypes
import json
import os

import numpy as np
import pytest

from golden_util import load_case, rae

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ["net_trainer_ffmlp_w64_h2", "net_trainer_cutlass_w128_h3"]


@pytest.mark.parametrize("case", CASES)
def test_network_trainer_matches_the_reference(case):
    import torch

    import tcnn_b200

    lib = tcnn_b200.load()
    g = load_case(case)
    meta = g["meta"]
    n_in, n_out, B = meta["n_input_dims"], meta["n_output_dims"], meta["batch"]
    network = {k: v for k, v in meta["network"].items() if k not in ("n_input_dims", "n_output_dims")}
    config = {"loss": meta["loss"], "optimizer": meta["optimizer"], "network": network}
    h = ctypes.c_void_p()
    rc = lib.tcnnb_create_network_trainer(n_in, n_out, json.dumps(config).encode(), meta["trainer_seed"], ctypes.byref(h))
    assert rc == 0, lib.tcnnb_last_error().decode()
    try:
        n = lib.tcnnb_n_params(h)
        assert n == meta["n_params"]
        view = tcnn_b200._Trainer._view
        p0 = view(None, lib.tcnnb_params_full_precision(h), n, torch.float32).cpu().numpy()
        assert np.array_equal(p0.view(np.uint32), g["params_init_f32"].view(np.uint32)), "initial parameters differ from the reference's"

        x = torch.from_numpy(g["x_f16"].view(np.float16).reshape(B, n_in).copy()).cuda()
        y = torch.from_numpy(g["y_f32"].reshape(B, n_out).copy()).cuda()
        losses = []
        for step in range(len(g["losses_f32"])):
            assert lib.tcnnb_training_step(h, None, B, ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(y.data_ptr()), 0) == 0, lib.tcnnb_last_error().decode()
            v = ctypes.c_float()
            assert lib.tcnnb_loss(h, None, ctypes.byref(v)) == 0
            losses.append(v.value)
            if step == 0:
                grads = view(None, lib.tcnnb_param_gradients(h), n, torch.float16).float().cpu().numpy()
                ref_grads = g["grads_f16"].view(np.float16).astype(np.float32)
                err = rae(grads, ref_grads, 99.9)
                assert err < 2e-2, ("gradients", err)
            assert lib.tcnnb_optimizer_step(h, None) == 0, lib.tcnnb_last_error().decode()
        torch.cuda.synchronize()
        ref = g["losses_f32"].astype(np.float64)
        got = np.array(losses, np.float64)
        assert abs(got[0] - ref[0]) <= 1e-3 * abs(ref[0]), ("step-0 loss", got[0], ref[0])
        assert np.all(np.abs(got - ref) <= 0.03 * np.abs(ref)), ("trajectory", got.tolist(), ref.tolist())
    finally:
        lib.tcnnb_destroy(h)
