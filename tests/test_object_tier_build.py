"""The C++ object tier compiles without a GPU: tests/cpp/object_tier.cu against include/tiny-cuda-nn/ for sm_90a, and -- where build()
found the reference's source tree -- the reference's own tests/test_networks.cu and benchmarks/mlp/bench_mlp_ours.cu, unmodified, against
these headers (and the benchmark once more against the reference library). tests/test_gpu_object_tier.py runs them."""
import os
import shutil
import subprocess
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_OUT = os.path.join(ROOT, "oracle", "_ref")
NVCC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")


def test_object_tier_program_compiles_for_sm90a():
    sys.path.insert(0, ROOT)
    from __graft_entry__ import json_include_dir

    inc = json_include_dir()
    if inc is None or not os.path.exists(NVCC):
        pytest.skip("nvcc or nlohmann/json.hpp not available")
    with tempfile.TemporaryDirectory() as tmp:
        obj = os.path.join(tmp, "object_tier.o")
        subprocess.run([NVCC, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-I", os.path.join(ROOT, "include"), "-I", inc, "-c",
                        os.path.join(ROOT, "tests", "cpp", "object_tier.cu"), "-o", obj], check=True, capture_output=True)
        assert os.path.getsize(obj) > 0


@pytest.mark.parametrize("name", ["ref_test_networks", "ref_bench_mlp_ours", "ref_bench_mlp_ours_tcnn"])
def test_reference_object_programs_were_built(name):
    path = os.path.join(REF_OUT, name)
    if not os.path.isdir(REF_OUT) or not os.path.exists(os.path.join(REF_OUT, "ref_harness")):
        pytest.skip("oracle/_ref/ was not built (no reference source tree)")
    assert os.path.isfile(path) and os.access(path, os.X_OK), path
    with open(path, "rb") as f:
        assert f.read(4) == b"\x7fELF"
