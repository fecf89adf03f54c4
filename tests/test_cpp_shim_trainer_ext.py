"""Trainer::training_step's full signature in the C++ compatibility headers: an application that passes every argument
(data_pdf, run_optimizer, dL_dinput, use_inference_params, GradientMode, external_dL_dy) compiles against include/tiny-cuda-nn/
without a GPU. tests/test_gpu_trainer_ext.py runs the same program."""
import os
import shutil
import subprocess
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_full_training_step_signature_compiles_against_the_shim():
    sys.path.insert(0, ROOT)
    from __graft_entry__ import json_include_dir

    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    inc = json_include_dir()
    if not os.path.exists(nvcc) or inc is None:
        pytest.skip("nvcc or nlohmann/json.hpp not available")
    src = os.path.join(ROOT, "tests", "cpp", "shim_trainer_ext.cu")
    text = open(src).read()
    assert "GradientMode::Accumulate" in text and "&dL_dinput, true, GradientMode::Overwrite" in text
    with tempfile.TemporaryDirectory() as tmp:
        out = subprocess.run([nvcc, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-I", os.path.join(ROOT, "include"), "-I", inc, "-c", src, "-o",
                              os.path.join(tmp, "shim_trainer_ext.o")], capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr[-2000:]


def test_gradient_mode_enum_matches_the_c_abi():
    """GradientMode's values are what tcnnb_training_step_ex takes as param_gradients_mode (0 Ignore, 1 Overwrite, 2 Accumulate)."""
    obj = open(os.path.join(ROOT, "include", "tiny-cuda-nn", "object.h")).read()
    body = obj[obj.index("enum class GradientMode") :].split("}")[0]
    assert [w.strip() for w in body.split("{")[1].split(",") if w.strip()] == ["Ignore", "Overwrite", "Accumulate"]
    header = open(os.path.join(ROOT, "include", "tcnn_b200.h")).read()
    assert all(k in header for k in ("0 Ignore", "1 Overwrite", "2 Accumulate"))
