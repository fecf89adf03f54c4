"""Snapshots of the C++ compatibility headers (include/tiny-cuda-nn/config.h) under an ExponentialDecay optimizer: trainer->serialize()
nests the Adam state as the reference does (optimizers/exponential_decay.h:136-148) and deserialize() restores the learning-rate
factor. tests/cpp/snapshot_decay is built by `__graft_entry__.build()`."""
import json
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "snapshot_decay")


@pytest.mark.gpu
def test_exponential_decay_snapshots_use_the_reference_schema(torch_cuda, tmp_path):
    """{"nested": Adam's keys with the DECAYED base_learning_rate, "learning_rate": the undecayed rate, "learning_rate_factor"}. The
    snapshot loads back into a new trainer with the same factor and serializes back unchanged; a document in that schema built by
    hand loads with the factor it stores, and one without a factor gets the factor of its step count."""
    if not os.path.exists(EXE):
        pytest.skip("tests/cpp/snapshot_decay has not been built (python __graft_entry__.py build)")
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", "configs", "hash3d_tiny.json")))
    cfg["optimizer"] = {"otype": "ExponentialDecay", "decay_start": 2, "decay_interval": 2, "decay_end": 100, "decay_base": 0.5, "nested": cfg["optimizer"]}
    cfg_path = str(tmp_path / "decay.json")
    json.dump(cfg, open(cfg_path, "w"))
    B = 1 << 12
    rng = np.random.default_rng(0)
    rng.random((B, 3), dtype=np.float32).tofile(str(tmp_path / "x.f32"))
    rng.random((B, 3), dtype=np.float32).tofile(str(tmp_path / "y.f32"))
    env = dict(os.environ, LD_LIBRARY_PATH=os.path.join(ROOT, "tiny-cuda-nn_b200") + ":" + os.environ.get("LD_LIBRARY_PATH", ""))
    out = subprocess.run([EXE, cfg_path, "3", "3", str(B), str(tmp_path), "7", "0.375"], capture_output=True, text=True, timeout=600, env=env)
    assert out.returncode == 0, out.stdout[-1500:] + out.stderr[-1500:]
    r = json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][-1])
    assert sorted(r["top_keys"]) == ["learning_rate", "learning_rate_factor", "nested"], r
    assert sorted(r["nested_keys"]) == ["base_learning_rate", "current_step", "first_moments_binary", "param_steps_binary", "second_moments_binary"], r
    # 7 steps: decays at steps 2, 4 and 6
    assert r["current_step"] == 7 and r["learning_rate_factor"] == 0.125 and r["trainer_factor"] == 0.125, r
    assert r["learning_rate"] == np.float32(1e-2) and r["nested_base_learning_rate"] == np.float32(np.float32(1e-2) * np.float32(0.125)), r
    assert r["loaded_factor"] == 0.125 and r["reserialized_identical"], r
    assert r["hand_factor"] == 0.375 and r["hand_learning_rate"] == np.float32(1e-2), r
    assert r["no_factor_factor"] == 0.125, r
