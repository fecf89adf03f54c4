"""The edges of the trainer's optimizer that the element-wise, counter and parity tests do not reach: what a module handle (which has
no optimizer) answers to the optimizer calls, the optimizer's config errors and the order in which they are reported, the
hyperparams' "optimizer" section, the restrictions of the Ema wrapper (no optimizer snapshots, no data parallelism) and its average
restarting from the weights set_params / set_params_full_precision write, and set_learning_rate_factor without ExponentialDecay."""
import ctypes
import json
import os

import numpy as np
import pytest

import tcnn_b200

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B = 1 << 14
NO_OPTIMIZER = "this handle was created with tcnnb_module_create: it has no optimizer."


def config(optimizer=None):
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", "configs", "hash3d_small.json")))
    if optimizer is not None:
        cfg["optimizer"] = optimizer
    return cfg


def adam():
    return config()["optimizer"]


def ema(nested, decay=0.9):
    return {"otype": "Ema", "decay": decay, "nested": nested}


def decay(nested, interval=2):
    return {"otype": "ExponentialDecay", "decay_start": 2, "decay_interval": interval, "decay_base": 0.5, "nested": nested}


def error(rc):
    assert rc != 0
    return tcnn_b200.load().tcnnb_last_error().decode()


def batch(torch):
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.rand(B, 3, device="cuda", generator=g).contiguous()
    y = (0.2 + 0.8 * torch.rand(B, 3, device="cuda", generator=g)).contiguous()
    return x, y


def bits(t):
    return t.contiguous().view(-1).cpu().numpy().view(np.uint16)


def test_module_handle_has_no_optimizer(torch_cuda):
    lib = tcnn_b200.load()
    cfg = config()
    module = tcnn_b200.Module(3, 3, cfg["encoding"], cfg["network"])
    h = module._h
    # the default Adam of an optimizer-less handle, as cpp::Module::hyperparams() hands it out
    opt = json.loads(lib.tcnnb_hyperparams(h).decode())["optimizer"]
    assert opt["otype"] == "Adam"
    for key, value in {"learning_rate": 1e-3, "beta1": 0.9, "beta2": 0.999, "epsilon": 1e-8, "l2_reg": 1e-8}.items():
        assert np.float32(opt[key]) == np.float32(value), key
    assert error(lib.tcnnb_optimizer_step(h, None)) == NO_OPTIMIZER
    assert error(lib.tcnnb_optimizer_step_ranges(h, None, 0, None, None)) == NO_OPTIMIZER
    assert error(lib.tcnnb_optimizer_state(h, None, None, None, None, None)) == NO_OPTIMIZER
    assert error(lib.tcnnb_debug_set(h, b"adam_steps32", 1)) == "tcnnb_debug_set(adam_steps32): this handle has no optimizer."
    assert lib.tcnnb_set_optimizer_progress(h, 5, ctypes.c_float(0.01)) == 0
    assert lib.tcnnb_learning_rate_factor(h) == 1.0
    assert error(lib.tcnnb_set_learning_rate_factor(h, ctypes.c_float(0.5))) == "set_learning_rate_factor: the optimizer has no ExponentialDecay wrapper."
    module.close()


@pytest.mark.parametrize("optimizer,message", [
    (decay(decay(adam())), "tcnn_b200: one ExponentialDecay wrapper per optimizer"),
    (ema(ema(adam())), "tcnn_b200: one Ema wrapper per optimizer"),
    (decay(adam(), interval=0), "ExponentialDecay: decay_interval must be positive."),
    (ema(decay({"otype": "SGD"})), "Optimizer 'SGD' is outside the tcnn_b200 hot path (Adam, optionally inside ExponentialDecay and / or Ema, is built)"),
], ids=["two_decays", "two_emas", "decay_interval_0", "not_adam"])
def test_config_errors(torch_cuda, optimizer, message):
    with pytest.raises(tcnn_b200.TcnnError) as e:
        tcnn_b200.create_from_config(3, 3, config(optimizer))
    assert str(e.value) == message


def test_config_errors_are_reported_in_section_order(torch_cuda):
    """The loss is checked before the optimizer, the optimizer before the encoding."""
    bad_optimizer = config({"otype": "SGD"})
    bad_loss = json.loads(json.dumps(bad_optimizer))
    bad_loss["loss"] = {"otype": "Huber"}
    with pytest.raises(tcnn_b200.TcnnError, match="^Loss 'Huber' not found$"):
        tcnn_b200.create_from_config(3, 3, bad_loss)
    bad_optimizer["encoding"]["otype"] = "NoSuchEncoding"
    with pytest.raises(tcnn_b200.TcnnError, match="^Optimizer 'SGD' is outside"):
        tcnn_b200.create_from_config(3, 3, bad_optimizer)


@pytest.mark.parametrize("wrap", [lambda a: a, lambda a: ema(decay(a)), lambda a: decay(ema(a))], ids=["adam", "ema_decay_adam", "decay_ema_adam"])
def test_hyperparams_optimizer_section(torch_cuda, wrap):
    inner = dict(adam(), learning_rate=3e-3, beta1=0.8, beta2=0.95, epsilon=1e-10, l2_reg=2e-6)
    model = tcnn_b200.create_from_config(3, 3, config(wrap(inner)))
    opt = model.hyperparams()["optimizer"]
    assert sorted(opt) == ["beta1", "beta2", "epsilon", "l2_reg", "learning_rate", "otype"]
    assert opt["otype"] == "Adam"
    for key in ("learning_rate", "beta1", "beta2", "epsilon", "l2_reg"):
        assert np.float32(opt[key]) == np.float32(inner[key]), key
    model.close()


def test_ema_restrictions_and_average_reset(torch_cuda):
    torch = torch_cuda
    lib = tcnn_b200.load()
    model = tcnn_b200.create_from_config(3, 3, config(ema(adam())))
    x, y = batch(torch)
    for _ in range(3):
        model.trainer.training_step(x, y)
    torch.cuda.synchronize()
    assert not torch.equal(model.trainer.params_inference(), model.trainer.params())

    assert error(lib.tcnnb_optimizer_state(model._h, None, None, None, None, None)) == \
        "tcnn_b200: snapshots of the Ema wrapper's state are not built (serialize the parameters only)"
    with pytest.raises(tcnn_b200.TcnnError) as e:
        model.trainer.serialize(with_optimizer=True)
    assert str(e.value) == "tcnn_b200: snapshots of the Ema wrapper's state are not built (serialize with_optimizer = 0)"
    blob = model.trainer.serialize(with_optimizer=False)
    n = model.n_params
    assert len(blob) == 16 + 2 * n
    assert np.array_equal(np.frombuffer(blob, dtype=np.uint16, count=n, offset=16), bits(model.trainer.params()))

    # set_params: the average restarts from the new working weights
    new16 = (model.trainer.params().float() * 0.5 + 0.01).to(torch.float16)
    model.trainer.set_params(new16)
    assert np.array_equal(bits(model.trainer.params_inference()), bits(new16))
    assert np.array_equal(bits(model.trainer.params_inference()), bits(model.trainer.params()))
    model.trainer.training_step(x, y)
    torch.cuda.synchronize()
    assert not torch.equal(model.trainer.params_inference(), model.trainer.params())
    # set_params_full_precision: likewise, from the working weights cast from the new masters
    before = bits(model.trainer.params())
    model.trainer.set_params_full_precision(model.trainer.params_full_precision().clone() * 0.75 - 0.002)
    assert not np.array_equal(bits(model.trainer.params()), before)
    assert np.array_equal(bits(model.trainer.params_inference()), bits(model.trainer.params()))

    # no data parallelism: refused before any communicator is created (the ids are null)
    assert error(lib.tcnnb_dp_init(model._h, None, None, 2, 0, 1)) == "tcnn_b200: the Ema optimizer wrapper is not built for the data-parallel engines"
    assert lib.tcnnb_dp_engine(model._h) == 0
    model.close()


def test_set_learning_rate_factor_needs_exponential_decay(torch_cuda):
    lib = tcnn_b200.load()
    plain = tcnn_b200.create_from_config(3, 3, config())
    assert error(lib.tcnnb_set_learning_rate_factor(plain._h, ctypes.c_float(0.5))) == "set_learning_rate_factor: the optimizer has no ExponentialDecay wrapper."
    assert lib.tcnnb_learning_rate_factor(plain._h) == 1.0
    decayed = tcnn_b200.create_from_config(3, 3, config(decay(adam())))
    assert lib.tcnnb_set_learning_rate_factor(decayed._h, ctypes.c_float(0.25)) == 0
    assert lib.tcnnb_learning_rate_factor(decayed._h) == 0.25
    plain.close()
    decayed.close()
