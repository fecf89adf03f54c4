"""The C++ object tier on the H100: create_network / create_encoding objects, NetworkWithInputEncoding composed from them, a Trainer over
a bare Network (tcnnb_create_network_trainer), row-major matrices (tcnnb_transpose) and generate_random_uniform<__half>.
tests/cpp/object_tier checks the objects against the C ABI tiers they sit on; oracle/_ref/ref_test_networks is the reference's own
tests/test_networks.cu compiled unchanged against include/tiny-cuda-nn/."""
import ctypes
import json
import os
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run(path, timeout=1200):
    if not os.path.exists(path):
        pytest.skip(f"{os.path.relpath(path, ROOT)} is not built (python __graft_entry__.py build)")
    return subprocess.run([path], capture_output=True, text=True, timeout=timeout, cwd=ROOT)


def test_object_tier_matches_the_tiers_below():
    r = run(os.path.join(ROOT, "tests", "cpp", "object_tier"))
    lines = [l for l in r.stdout.splitlines() if l.startswith(("ok ", "FAIL "))]
    failed = [l for l in lines if l.startswith("FAIL")]
    assert r.returncode == 0 and not failed and len(lines) >= 30, r.stdout + r.stderr


# The stand-alone network kernels take inputs up to 64 wide below 128 neurons, so the reference's sections with 128 inputs into 32 or 64
# neurons do not pass: an unmet part of the reference's test, marked as such (a build that takes them turns these into failures to
# remove the mark).
NARROW_WIDE_INPUT = pytest.mark.xfail(strict=True, reason="not built: 128-wide network inputs below 128 neurons")
SECTIONS = [
    pytest.param(n_in, n_hidden, n_out, marks=[NARROW_WIDE_INPUT] if n_in > max(64, n_hidden) else [])
    for n_in in (16, 32, 48, 64, 128) for n_hidden in (32, 64, 128) for n_out in (16, 32)
]


@pytest.mark.parametrize("n_in,n_hidden,n_out", SECTIONS)
def test_reference_test_networks_section(n_in, n_hidden, n_out):
    """One section of the reference's invariance test (CutlassMLP and FullyFusedMLP, depth 2): inference vs inference_mixed_precision
    and inference_mixed_precision vs forward. Its JIT sections are skipped by the test itself: supports_jit_fusion() is false, there is
    no run-time compiler here."""
    path = os.path.join(ROOT, "oracle", "_ref", "ref_test_networks")
    if not os.path.exists(path):
        pytest.skip("oracle/_ref/ref_test_networks is not built (no reference source tree)")
    r = subprocess.run([path, "-c", f"MLP testing {n_in}->{n_hidden}x2->{n_out}"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "All tests passed" in r.stdout, r.stdout[-3000:] + r.stderr[-1000:]


def half_uniform_host(state, inc, n, lower, upper):
    """random.h:40-69 with T = __half, restated: thread i of ceil(n / 4) jumps ahead 4 i draws and writes i, i + n_thr, ...; each draw is
    next_float() rounded to half, then draw * (upper - lower) + lower in half arithmetic. The device contracts the product and the sum
    into one fused multiply-add (one rounding), so this computes them exactly in float64 and rounds once."""
    import tcnn_b200

    n_thr = -(-n // 4)
    n_thr = -(-n_thr // 128) * 128  # whole blocks of 128 threads, as launched
    out = np.zeros(n, dtype=np.float16)
    lo, hi = np.float16(lower), np.float16(upper)
    span = np.float16(hi - lo)
    for i in range(n_thr):
        if i >= n:
            break
        rng = tcnn_b200.Pcg32()
        rng.state, rng.inc = state, inc
        rng.advance(4 * i)
        for j in range(4):
            idx = i + n_thr * j
            if idx >= n:
                break
            old = rng.state
            rng.state = (old * rng.MULT + rng.inc) & rng.MASK
            xorshifted = (((old >> 18) ^ old) >> 27) & 0xFFFFFFFF
            rot = old >> 59
            u = ((xorshifted >> rot) | (xorshifted << ((-rot) & 31))) & 0xFFFFFFFF
            f = np.array([(u >> 9) | 0x3F800000], dtype=np.uint32).view(np.float32)[0] - np.float32(1.0)
            out[idx] = np.float16(float(np.float16(f)) * float(span) + float(lo))
    return out


@pytest.mark.parametrize("lower,upper", [(0.0, 1.0), (-0.75, 2.5)])
def test_generate_random_uniform_half_is_the_reference_stream(lower, upper):
    import torch

    import tcnn_b200

    lib = tcnn_b200.load()
    n = 3000
    rng = tcnn_b200.Pcg32(1337)
    rng.advance(12345)
    out = torch.empty(n, dtype=torch.float16, device="cuda")
    assert lib.tcnnb_generate_random_uniform_half(None, ctypes.c_uint64(rng.state), ctypes.c_uint64(rng.inc), ctypes.c_uint64(n), ctypes.c_void_p(out.data_ptr()),
                                                  ctypes.c_float(lower), ctypes.c_float(upper)) == 0
    torch.cuda.synchronize()
    ref = half_uniform_host(rng.state, rng.inc, n, lower, upper)
    assert np.array_equal(out.cpu().numpy().view(np.uint16), ref.view(np.uint16))


@pytest.mark.parametrize("dtype,rows,cols", [("float16", 1000, 48), ("float32", 1000, 48), ("float16", (1 << 21) + 4128, 16)])
def test_transpose_kernel(dtype, rows, cols):
    """Tails in both dimensions, and more row tiles than one grid dimension holds (the row loop)."""
    import torch

    import tcnn_b200

    t = getattr(torch, dtype)
    src = torch.randn(rows, cols, device="cuda").to(t)
    dst = torch.empty(cols, rows, device="cuda", dtype=t)
    assert tcnn_b200.load().tcnnb_transpose(None, rows, cols, src.element_size(), ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(dst.data_ptr())) == 0
    torch.cuda.synchronize()
    assert torch.equal(dst, src.t().contiguous())


def test_network_trainer_rejects_misaligned_rows():
    """A network trainer's fp16 rows go to the network kernels as they are: a misaligned view is an error, not a fault."""
    import torch

    import tcnn_b200

    lib = tcnn_b200.load()
    config = {"loss": {"otype": "L2"}, "optimizer": {"otype": "Adam"}, "network": {"otype": "FullyFusedMLP", "n_neurons": 64, "n_hidden_layers": 2}}
    h = ctypes.c_void_p()
    assert lib.tcnnb_create_network_trainer(32, 16, json.dumps(config).encode(), 1337, ctypes.byref(h)) == 0, lib.tcnnb_last_error().decode()
    try:
        x = torch.zeros(256 * 32 + 8, dtype=torch.float16, device="cuda")
        y = torch.zeros(256, 16, device="cuda")
        rc = lib.tcnnb_training_step(h, None, 256, ctypes.c_void_p(x.data_ptr() + 2), ctypes.c_void_p(y.data_ptr()), 1)
        assert rc != 0 and "16-byte aligned" in lib.tcnnb_last_error().decode()
        assert lib.tcnnb_training_step(h, None, 256, ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(y.data_ptr()), 1) == 0, lib.tcnnb_last_error().decode()
        torch.cuda.synchronize()
    finally:
        lib.tcnnb_destroy(h)
