"""CPU pins of the second-order grid oracle (tests/cpp/grid_bwd_bwd_oracle.cpp) by identities that need no GPU.

dL/dx = sum_{l,f} u_{l,f} dy_{l,f}/dx (orc_grid_input_gradient) is linear in the table theta and in u, so the parameter result and the
dL_ddLdoutput result of backward_backward_input are its exact adjoints:
    <dL_dparams, theta> = <v, dL_dx(theta, u)> = <dL_ddLdoutput, u>.
The input result is the derivative of <v, dL_dx(x)> in x, checked against central differences away from cell faces."""
import ctypes

import numpy as np
import pytest

import grid_bwd_bwd_oracle as bb
import oracle_binding as ob

GRID_TYPES = {"hash": ob.GRID_HASH, "dense": ob.GRID_DENSE, "tiled": ob.GRID_TILED}
INTERP = {"Linear": ob.INTERP_LINEAR, "Smoothstep": ob.INTERP_SMOOTHSTEP}

# (D, F, n_levels, log2_hashmap_size, base_resolution, per_level_scale, grid type)
GRIDS = [
    (2, 2, 4, 8, 4, 1.5, "hash"),
    (3, 1, 4, 8, 3, 1.5, "hash"),
    (3, 4, 3, 10, 4, 1.5, "dense"),
    (3, 2, 3, 6, 3, 1.5, "tiled"),
    (4, 2, 3, 8, 2, 1.5, "hash"),
    (4, 8, 2, 6, 2, 2.0, "dense"),
]
CASES = [(g, i) for g in GRIDS for i in INTERP]


def make_grid(D, F, L, log2_T, base, pls, gtype, interp):
    g = ob.Grid(D, L, F, log2_T, base, pls, GRID_TYPES[gtype], INTERP[interp], 0)
    assert ob.load().orc_grid_setup(ctypes.byref(g)) == 0
    return g


def make_inputs(g, B, seed):
    rng = np.random.default_rng(seed)
    D, L, F = g.n_pos_dims, g.n_levels, g.n_features_per_level
    x = rng.uniform(0.0, 1.0, (B, D)).astype(np.float32)
    table = rng.uniform(-1.0, 1.0, g.n_params).astype(np.float16)
    u = np.zeros((g.padded_width, B), np.float16)
    u[: L * F] = rng.uniform(-1.0, 1.0, (L * F, B)).astype(np.float16)
    v = rng.uniform(-1.0, 1.0, (B, D)).astype(np.float32)
    return x, table.view(np.uint16), u.view(np.uint16), v


def input_gradient(g, x, table, u):
    out = np.zeros(x.shape, np.float32)
    ob.load().orc_grid_input_gradient(ctypes.byref(g), x.shape[0], ob._p(np.ascontiguousarray(x)), ob._p(table), ob._p(u), ob._p(out))
    return out


def case_id(c):
    (D, F, L, _, _, _, gtype), interp = c
    return f"D{D}_F{F}_{gtype}_{interp}"


@pytest.mark.parametrize("grid,interp", CASES, ids=[case_id(c) for c in CASES])
def test_params_and_doutput_results_are_adjoints_of_the_input_gradient(grid, interp):
    g = make_grid(*grid, interp)
    B = 256
    x, table, u, v = make_inputs(g, B, seed=1)
    L, F = g.n_levels, g.n_features_per_level
    dx = input_gradient(g, x, table, u).astype(np.float64)
    terms = v.astype(np.float64) * dx
    rhs, scale = terms.sum(), np.abs(terms).sum()
    gp, gd, _ = bb.grid_backward_backward_input(g, x, table, u, v, want=("params", "doutput"))
    theta = table.view(np.float16).astype(np.float64)
    uf = u.view(np.float16).astype(np.float64)[: L * F].T  # [B][L*F]
    assert abs((gp * theta).sum() - rhs) <= 1e-5 * scale, ((gp * theta).sum(), rhs)
    assert abs((gd * uf).sum() - rhs) <= 1e-5 * scale, ((gd * uf).sum(), rhs)
    assert np.abs(gp).max() > 0 and np.abs(gd).max() > 0


@pytest.mark.parametrize("grid,interp", CASES, ids=[case_id(c) for c in CASES])
def test_input_result_matches_central_differences(grid, interp):
    g = make_grid(*grid, interp)
    B, D, L = 256, g.n_pos_dims, g.n_levels
    x, table, u, v = make_inputs(g, B, seed=2)
    h = np.float32(1e-4)
    scales = np.array(g.scales[:L], np.float64)
    # samples whose every coordinate stays at least 2 h scale_l away from a cell face at every level: the encoding is smooth there
    p = scales[None, None, :] * x[:, :, None].astype(np.float64) + 0.5
    frac = p - np.floor(p)
    keep = (np.minimum(frac, 1.0 - frac) > 2.0 * float(h) * scales[None, None, :]).all(axis=(1, 2))
    assert keep.sum() > B // 2
    _, _, gx = bb.grid_backward_backward_input(g, x, table, u, v, want=("input",))
    fd = np.zeros((B, D))
    for e in range(D):
        xp, xm = x.copy(), x.copy()
        xp[:, e] += h
        xm[:, e] -= h
        fp = (v.astype(np.float64) * input_gradient(g, xp, table, u)).sum(axis=1)
        fm = (v.astype(np.float64) * input_gradient(g, xm, table, u)).sum(axis=1)
        fd[:, e] = (fp - fm) / (xp[:, e].astype(np.float64) - xm[:, e].astype(np.float64))
    ref, got = fd[keep], gx[keep]
    assert np.abs(got).max() > 0
    assert np.abs(got - ref).max() <= 2e-3 * np.abs(ref).max(), (np.abs(got - ref).max(), np.abs(ref).max())


def test_masked_levels_and_nearest_contribute_nothing():
    g = make_grid(3, 2, 4, 8, 4, 1.5, "hash", "Linear")
    x, table, u, v = make_inputs(g, 256, seed=3)
    gp, gd, gx = bb.grid_backward_backward_input(g, x, table, u, v, max_level=0.5)
    n_active = 3  # level l takes part while l < 0.5 * 4 + 1e-3
    assert (gp[g.offsets[n_active] * 2 :] == 0).all() and np.abs(gp[: g.offsets[n_active] * 2]).max() > 0
    assert (gd[:, n_active * 2 :] == 0).all() and np.abs(gd[:, : n_active * 2]).max() > 0
    # the masked levels' share of dL_dx is gone: the result equals that of the active levels with u zero on the others
    u_masked = u.copy()
    u_masked[n_active * 2 :] = 0
    _, _, gx_ref = bb.grid_backward_backward_input(g, x, table, u_masked, v)
    assert np.array_equal(gx, gx_ref)
    g.interpolation = ob.INTERP_NEAREST
    for r in bb.grid_backward_backward_input(g, x, table, u, v):
        assert (r == 0).all()
