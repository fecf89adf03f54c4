"""ctypes binding of tests/cpp/grid_bwd_bwd_oracle.cpp: the reference's second-order derivatives of the grid encoding
(grid.h:910-1042) restated in double on the CPU. TEST INFRASTRUCTURE ONLY; the grid description is oracle_binding's."""
import ctypes
import os
import subprocess

import numpy as np

import oracle_binding as ob

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "grid_bwd_bwd_oracle.cpp")
LIB = os.path.join(ROOT, "tests", "cpp", "libgrid_bwd_bwd_oracle.so")


def build():
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-o", LIB, SRC])


_lib = None


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            build()
        _lib = ctypes.CDLL(LIB)
    return _lib


def grid_backward_backward_input(grid, x, table16, dL_denc_soa, dL_ddLdx, max_level=1.0, want=("params", "doutput", "input")):
    """-> (dL_dparams double [n_params] | None, dL_ddLdoutput double [B][L*F] | None, dL_dinput double [B][D] | None).
    grid: oracle_binding.Grid; x, dL_ddLdx fp32 [B][D]; table16 fp16 bits [n_params]; dL_denc_soa fp16 bits [>= L*F][B]."""
    B, D = x.shape
    L, F = grid.n_levels, grid.n_features_per_level
    gp = np.zeros(grid.n_params, np.float64) if "params" in want else None
    gd = np.zeros((B, L * F), np.float64) if "doutput" in want else None
    gx = np.zeros((B, D), np.float64) if "input" in want else None
    keep = [np.ascontiguousarray(a) for a in (x.astype(np.float32), table16.astype(np.uint16), dL_denc_soa.astype(np.uint16), dL_ddLdx.astype(np.float32))]
    load().orc_grid_backward_backward_input(ctypes.byref(grid), ctypes.c_uint32(B), *[ob._p(a) for a in keep], ctypes.c_float(max_level), ob._p(gp), ob._p(gd), ob._p(gx))
    return gp, gd, gx
