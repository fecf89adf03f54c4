"""The C++ source-compatibility headers (include/tiny-cuda-nn/*.h): an application written against tiny-cuda-nn's names
(tests/cpp/shim_sample.cu, modelled on the reference's samples/mlp_learning_an_image.cu) compiles against them, links
libtcnn_b200.so and trains. The binary is built by `__graft_entry__.build()` (nvcc cross-compiles without a GPU)."""
import json
import os
import subprocess

import numpy as np
import pytest

import oracle_binding as ob

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "cpp", "shim_sample")


def test_shim_headers_exist_and_cite_the_reference():
    inc = os.path.join(ROOT, "include", "tiny-cuda-nn")
    for h in ("common.h", "common_device.h", "config.h", "gpu_matrix.h", "gpu_memory.h", "random.h", "trainer.h", "network_with_input_encoding.h", "loss.h", "optimizer.h", "network.h", "encoding.h"):
        text = open(os.path.join(inc, h)).read()
        assert "#pragma once" in text
    assert "trainer.h:254-357" in open(os.path.join(inc, "config.h")).read()


@pytest.mark.gpu
def test_shim_sample_trains(torch_cuda):
    if not os.path.exists(BIN):
        pytest.skip("tests/cpp/shim_sample has not been built (python __graft_entry__.py build)")
    env = dict(os.environ, LD_LIBRARY_PATH=os.path.join(ROOT, "tiny-cuda-nn_b200") + ":" + os.environ.get("LD_LIBRARY_PATH", ""))
    out = subprocess.run([BIN, "300"], capture_output=True, text=True, timeout=300, env=env)
    assert out.returncode == 0, out.stderr
    r = json.loads(out.stdout.strip().splitlines()[-1])
    # HashGrid(2-D, L=16, F=2, T=2^15, base 16, s=1.5): 6 dense + 10 hashed levels = 354 184 entries (SURVEY.md appendix B) + 64x32+64x64+16x64 weights
    assert r["n_params"] == 354184 * 2 + 7168 and r["padded_output_width"] == 16
    assert r["last_loss"] < 0.05 * r["first_loss"], r
    assert r["inference_mse"] < 5e-3, r
    assert np.isfinite(r["create_from_config_loss"]) and abs(r["create_from_config_loss"] - r["first_loss"]) / r["first_loss"] < 0.5
    # default_rng_t{1337} + generate_random_uniform == the reference's generator (random.h:40-69), via the oracle restatement
    expect = ob.generate_random_uniform(ob.default_rng(1337), 8)
    assert np.array_equal(np.array(r["first_uniform"], np.float32), expect)


def test_shim_sample_compiles_without_a_gpu():
    """nvcc cross-compiles the application against the compatibility headers (compile only, no link, no GPU)."""
    import shutil
    import sys
    import tempfile

    sys.path.insert(0, ROOT)
    from __graft_entry__ import json_include_dir

    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    inc = json_include_dir()
    if not os.path.exists(nvcc) or inc is None:
        pytest.skip("nvcc or nlohmann/json.hpp not available")
    with tempfile.TemporaryDirectory() as tmp:
        out = subprocess.run([nvcc, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-I", os.path.join(ROOT, "include"), "-I", inc, "-c",
                              os.path.join(ROOT, "tests", "cpp", "shim_sample.cu"), "-o", os.path.join(tmp, "shim_sample.o")], capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr[-2000:]


# ------------------------------------------------------------------------------------------------------------------
# SURVEY.md section 8(b) acceptance test: the reference's OWN application sources, unmodified, against this library's headers.
# build() compiles them into oracle/_ref/ where the reference's source tree is present; without it there is nothing to check.
# ------------------------------------------------------------------------------------------------------------------
REF_OUT = os.path.join(ROOT, "oracle", "_ref")
HARNESS = os.path.join(REF_OUT, "ref_harness")


def _require_reference_build():
    if not os.path.exists(HARNESS):
        pytest.skip("oracle/_ref/ has not been built: build() had no reference source tree")


@pytest.mark.parametrize("src", ["samples/mlp_learning_an_image.cu", "benchmarks/image/bench_ours.cu"])
def test_unmodified_reference_sources_compile_against_the_shim(src):
    """build() compiled and linked the reference's source file UNCHANGED against include/tiny-cuda-nn/ (a failed compile fails build())."""
    import sys

    _require_reference_build()
    sys.path.insert(0, ROOT)
    from __graft_entry__ import REFERENCE_SAMPLES

    name = {v: k for k, v in REFERENCE_SAMPLES.items()}[src]
    exe = os.path.join(REF_OUT, name)
    assert os.path.isfile(exe) and os.access(exe, os.X_OK) and os.path.getsize(exe) > 0, exe


@pytest.mark.gpu
def test_unmodified_reference_sample_trains(torch_cuda, tmp_path):
    """oracle/_ref/ref_mlp_learning_an_image = the reference's samples/mlp_learning_an_image.cu, byte for byte, linked against
    libtcnn_b200: 300 training steps on a synthetic image with the reference's data/config_hash.json settings."""
    import re

    _require_reference_build()
    exe = os.path.join(REF_OUT, "ref_mlp_learning_an_image")
    assert os.path.exists(exe), "build() built the reference harness but not the sample"
    # a smooth 256 x 256 RGB test image as binary PPM (stb_image reads PNM)
    h = w = 256
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32) / h
    img = np.stack([0.5 + 0.5 * np.sin(9 * xx + 3 * yy), 0.5 + 0.5 * np.cos(7 * yy), xx * yy], -1)
    with open(tmp_path / "img.ppm", "wb") as f:
        f.write(b"P6\n%d %d\n255\n" % (w, h))
        f.write((np.clip(img, 0, 1) * 255).astype(np.uint8).tobytes())
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", "configs", "image2d.json")))
    json.dump(cfg, open(tmp_path / "config.json", "w"))
    env = dict(os.environ, LD_LIBRARY_PATH=os.path.join(ROOT, "tiny-cuda-nn_b200") + ":" + os.environ.get("LD_LIBRARY_PATH", ""))
    out = subprocess.run([exe, str(tmp_path / "img.ppm"), str(tmp_path / "config.json"), "300", str(tmp_path / "learned.jpg")], capture_output=True, text=True, timeout=600, env=env,
                         cwd=str(tmp_path))
    assert out.returncode == 0 and "Uncaught exception" not in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
    losses = [float(m) for m in re.findall(r"Step#\d+: loss=([0-9.eE+-]+)", out.stdout)]
    assert len(losses) >= 3 and losses[-1] < 0.2 * losses[0], out.stdout[-1500:]
    assert os.path.getsize(tmp_path / "learned.jpg") > 1000 and os.path.exists(tmp_path / "reference.jpg")


def _snapshot_env():
    exe = os.path.join(ROOT, "tests", "cpp", "snapshot_interop")
    if not os.path.exists(exe):
        pytest.skip("tests/cpp/snapshot_interop has not been built (python __graft_entry__.py build)")
    env = dict(os.environ, LD_LIBRARY_PATH=os.path.join(ROOT, "tiny-cuda-nn_b200") + ":" + os.environ.get("LD_LIBRARY_PATH", ""))

    def run(cmd):
        out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
        assert out.returncode == 0, out.stdout[-1500:] + out.stderr[-1500:]
        return json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][-1])

    return exe, run


@pytest.mark.gpu
@pytest.mark.parametrize("with_optimizer", [0, 1])
def test_snapshots_interoperate_with_the_reference(torch_cuda, tmp_path, with_optimizer):
    """trainer->serialize() / deserialize() (trainer.h:442-482, optimizers/adam.h:303-325) exchange the reference's JSON schema: a
    snapshot written by the UNMODIFIED reference (msgpack as instant-ngp stores it; stored under tests/golden/snapshot_ref_opt*/ with
    the reference's inputs and inference) loads into this library and reproduces the reference's inference. The other direction:
    test_library_snapshots_load_into_the_reference."""
    import shutil

    from golden_util import rae

    exe, run = _snapshot_env()
    # the reference trained `steps` steps on x.f32 / y.f32, saved the snapshot and its inference on x.f32
    golden = os.path.join(ROOT, "tests", "golden", f"snapshot_ref_opt{with_optimizer}")
    saved = json.load(open(os.path.join(golden, "saved.json")))
    d = str(tmp_path / "from_reference")
    shutil.copytree(golden, d)
    cfg = os.path.join(ROOT, "tests", "golden", saved["config"])
    loaded = run([exe, "load", cfg, str(saved["n_in"]), str(saved["n_out"]), str(saved["batch"]), d, os.path.join(d, "snapshot.msgpack")])
    ref = np.fromfile(os.path.join(d, "inference.f32"), np.float32)
    ours = np.fromfile(os.path.join(d, "inference_loaded.f32"), np.float32)
    assert rae(ours, ref, 99.0) < 1e-2  # same parameters, the two forward kernels (tests/test_common.h:177)
    assert loaded["has_optimizer"] == bool(with_optimizer)
    # the step after loading continues the reference's trajectory (with its optimizer state: moments + per-parameter step counters)
    assert loaded["next_step_loss"] < 1.5 * saved["last_loss"] + 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize("with_optimizer", [0, 1])
def test_library_snapshots_load_into_the_reference(torch_cuda, tmp_path, with_optimizer):
    """A snapshot written by this library loads into the UNMODIFIED reference (oracle/_ref/ref_harness) and reproduces our inference."""
    from golden_util import rae

    _require_reference_build()
    exe, run = _snapshot_env()
    cfg = os.path.join(ROOT, "tests", "golden", "configs", "hash3d_small.json")
    d = str(tmp_path)
    B = 1024
    run([HARNESS, "snapshot", "save", cfg, "3", "3", str(B), "20", d, str(with_optimizer)])  # writes the inputs x.f32 / y.f32
    run([exe, "save", cfg, "3", "3", str(B), d, "20", str(with_optimizer)])
    back = run([HARNESS, "snapshot", "load", cfg, "3", "3", str(B), d, os.path.join(d, "snapshot_b200.msgpack")])
    ours = np.fromfile(os.path.join(d, "inference_b200.f32"), np.float32)
    ref = np.fromfile(os.path.join(d, "inference_loaded.f32"), np.float32)
    assert rae(ours, ref, 99.0) < 1e-2
    assert np.isfinite(back["next_step_loss"])


def test_unmodified_reference_torch_bindings_compile_against_cpp_api_h():
    """bindings/torch/tinycudann/bindings.cpp (the PyTorch extension's C++ half, which includes only <tiny-cuda-nn/cpp_api.h>) compiled
    UNCHANGED against this repo's include/tiny-cuda-nn/cpp_api.h in build() (oracle/_ref/bindings.o; a failed compile fails build()):
    same tcnn::cpp::Module interface, factories and free functions."""
    _require_reference_build()
    obj = os.path.join(REF_OUT, "bindings.o")
    assert os.path.isfile(obj) and os.path.getsize(obj) > 0, obj
