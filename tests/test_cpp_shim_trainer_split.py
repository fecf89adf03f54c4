"""Trainer::forward / Trainer::backward / Trainer::loss(ctx) in the C++ compatibility headers: applications written against the
reference's declarations (trainer.h:89-157, 372-378) compile against include/tiny-cuda-nn/ without a GPU, and the library exports the
C ABI they call. tests/test_gpu_trainer_split.py runs tests/cpp/shim_trainer_split."""
import ctypes
import os
import shutil
import subprocess
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Every overload with every argument, spelled as the reference declares them, and every member of the reference's ForwardContext.
FULL_SIGNATURES = r"""
#include <tiny-cuda-nn/config.h>
using namespace tcnn;
using precision_t = network_precision_t;

float split_step(Trainer<float, precision_t, precision_t>& trainer, cudaStream_t stream, const GPUMatrix<float>& x, const GPUMatrix<float>& y,
                 const GPUMatrix<float>& pdf, GPUMatrix<float>& dL_dinput, const GPUMatrix<precision_t>& external) {
	std::unique_ptr<Trainer<float, precision_t, precision_t>::ForwardContext> ctx =
		trainer.forward(stream, LOSS_SCALE, x, y, &pdf, false, false, nullptr);
	GPUMatrix<precision_t>& output = ctx->output;
	GPUMatrix<precision_t>& dL_doutput = ctx->dL_doutput;
	GPUMatrix<float>& L = ctx->L;
	GPUMatrix<precision_t>& perturbed = ctx->perturbed_output;
	std::unique_ptr<Context>& model_ctx = ctx->model_ctx;
	(void)output; (void)dL_doutput; (void)L; (void)perturbed; (void)model_ctx;
	trainer.backward(stream, *ctx, x, &dL_dinput, false, GradientMode::Accumulate);
	float loss = trainer.loss(stream, *ctx);
	auto ctx2 = trainer.forward(LOSS_SCALE, x, y, nullptr, true, true, &external);
	trainer.backward(*ctx2, x, nullptr, true, GradientMode::Ignore);
	trainer.backward(*ctx2, x);
	loss += trainer.loss(*ctx2);
	auto ctx3 = trainer.training_step(stream, x, y);
	return loss + trainer.loss(stream, *ctx3) + trainer.loss(*ctx3);
}
"""


def _compile(path, tmp):
    sys.path.insert(0, ROOT)
    from __graft_entry__ import json_include_dir

    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    inc = json_include_dir()
    if not os.path.exists(nvcc) or inc is None:
        pytest.skip("nvcc or nlohmann/json.hpp not available")
    return subprocess.run([nvcc, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-I", os.path.join(ROOT, "include"), "-I", inc, "-c", path, "-o",
                           os.path.join(tmp, "out.o")], capture_output=True, text=True, timeout=600)


def test_reference_declarations_compile_against_the_shim():
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "split.cu")
        with open(src, "w") as f:
            f.write(FULL_SIGNATURES)
        out = _compile(src, tmp)
        assert out.returncode == 0, out.stderr[-2000:]


def test_split_sample_compiles_against_the_shim():
    with tempfile.TemporaryDirectory() as tmp:
        out = _compile(os.path.join(ROOT, "tests", "cpp", "shim_trainer_split.cu"), tmp)
        assert out.returncode == 0, out.stderr[-2000:]


def test_library_exports_the_split():
    import tcnn_b200

    lib = ctypes.CDLL(tcnn_b200.lib_path())
    for name in ("tcnnb_forward", "tcnnb_backward", "tcnnb_reduce_sum"):
        assert hasattr(lib, name), name
    bound = {name for name, _, _ in tcnn_b200.ABI}
    assert {"tcnnb_forward", "tcnnb_backward", "tcnnb_reduce_sum"} <= bound
