"""The spatial binning pass of the fused training step (csrc/binning.cu) beyond one scan chunk, on crowded, empty and clamped bins
and across changing batch sizes.

A fused step of at least 16 384 samples first sorts the batch by the (y, z) column of each sample: bin_count_kernel ranks every
sample inside its bin (and zeroes the table gradients), bin_scan_kernel turns the bin counters into first output slots,
SCAN_CHUNK bins per pass with the running total carried from chunk to chunk, and bin_scatter_kernel writes the permutation the
fused kernel reads the batch through. A wrong permutation trains some samples twice and others never while the loss and the
gradients still look plausible. So every batch here is trained three times on the same device and the same weights: binned,
unbinned (debug_set("binning", 0)) and on the general path (debug_set("general", 1)), which never bins. Then:

  1. no row of the debug taps, NaN-filled before each step, is left unwritten: every sample was trained;
  2. every binned row is bit-identical to the unbinned row of the same sample. The taps are written in caller order and a row's
     forward and backward depend only on that row and the weights, so a misrouted sample cannot hide. The encoded features also
     equal the CPU oracle's bit for bit;
  3. the binned loss equals the sum of its own loss values, the unbinned loss (another fp32 summation order) and the general
     path's loss (whose MLP kernels may round an output differently by one fp16 ulp);
  4. the network weight gradients agree (fp32 sums in another order);
  5. the table gradients are no further from the exact sums of the device's own dL/d(encoded) (the oracle's grid scatter, in
     double) than the unbinned step's, nothing outside the entries the batch indexes is written, and both orders touch the same
     entries.

Which batches reach the scan's later chunks follows from the sizing rule of binning.cu, restated below. The premise test (no GPU
needed, so the GPU tests carry their own mark instead of a module-wide one) pins that restatement and the bins each batch fills,
so that a change of the rule cannot silently turn the multi-chunk cases into single-chunk ones.
"""
import json
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest

import oracle_binding as ob
from golden_util import GOLDEN, rae

gpu = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_OUT = 3
SCAN_CHUNK = 16384  # counters bin_scan_kernel stages per pass
MIN_BINNED_BATCH = 16384  # model.cu: smaller batches are trained in caller order


def binning_log2_resolution(n, n_pos_dims):
    """binning.cu: about 16 samples per bin; R bins in 2-D, R^2 Morton-ordered (y, z) bins in 3-D with at most 2^8 cells per axis."""
    log2_bins = 0
    while (1 << (log2_bins + 1)) * 16 <= n:
        log2_bins += 1
    log2_r = log2_bins if n_pos_dims == 2 else min(log2_bins // 2, 8)
    return min(log2_r, 16)


def binning_n_bins(log2_r, n_pos_dims):
    return 1 << log2_r if n_pos_dims == 2 else 1 << (2 * log2_r)


def scan_chunks(n, n_pos_dims):
    """Passes bin_scan_kernel makes over this batch's bin counters; 0 when the batch is not binned."""
    if n < MIN_BINNED_BATCH:
        return 0
    return -(-binning_n_bins(binning_log2_resolution(n, n_pos_dims), n_pos_dims) // SCAN_CHUNK)


def part1by1(v):
    v = v.astype(np.uint32) & 0xFF
    v = (v | (v << 4)) & 0x0F0F
    v = (v | (v << 2)) & 0x3333
    return (v | (v << 1)) & 0x5555


def compact1by1(k):
    """Inverse of part1by1 on the even bits of k."""
    return sum(((k >> (2 * b)) & 1) << b for b in range(8))


def bin_keys(x, log2_r):
    """bin_key of binning.cu: the cell of y (and z), clamped to [0, R - 1] per axis, Morton-interleaved in 3-D."""
    R = 1 << log2_r

    def cell(v):
        return np.clip((v * np.float32(R)).astype(np.int64), 0, R - 1).astype(np.uint32)  # (int) truncates like the kernel's cast

    if x.shape[1] == 2:
        return cell(x[:, 1])
    return part1by1(cell(x[:, 1])) | (part1by1(cell(x[:, 2])) << 1)


# bins either side of every chunk boundary of the 3-D (65 536 bins) and 2-D (32 768 bins) batches below
STRADDLE_KEYS = {3: [16383, 16384, 32767, 32768, 49151, 49152], 2: [16383, 16384]}
ONE_BIN_KEY = 40000  # in the third chunk: the first two chunks are empty and the fourth starts at B


def one_bin_key(D, B):
    return ONE_BIN_KEY % binning_n_bins(binning_log2_resolution(B, D), D)

# name: (config, D, batch, positions, scan chunks)
CASES = {
    "uniform_4chunks": ("headline", 3, 1 << 20, "uniform", 4),
    "uniform_2chunks_2d": ("image2d", 2, 1 << 19, "uniform", 2),
    "odd_batch": ("headline", 3, (1 << 20) + 256 * 37, "uniform", 4),  # partial last tile, uneven tiles per CTA
    "straddle_3d": ("headline", 3, 1 << 20, "straddle", 4),
    "straddle_2d": ("image2d", 2, 1 << 19, "straddle", 2),
    "one_bin": ("headline", 3, 1 << 20, "one_bin", 4),
    "clamped": ("headline", 3, 1 << 20, "clamped", 4),
    "threshold_off": ("headline", 3, 16128, "uniform", 0),
    "threshold_on": ("headline", 3, 16384, "uniform", 1),
}
CASE_SEED = 2024
# bin counts 65 536, 65 536, 4 096, 16 384, 16 384, 65 536 on one model (test_changing_batch_sizes_on_one_model)
CHANGING_BATCHES = [1 << 20, 1 << 20, 1 << 16, 1 << 19, 1 << 18, 1 << 20]


def load_cfg(name):
    with open(os.path.join(GOLDEN, "configs", name + ".json")) as f:
        return json.load(f)


def cell_positions(rng, cells, log2_r):
    """A position inside the middle half of each given cell index (away from its faces) along one axis."""
    u = ob.generate_random_uniform(rng, len(cells), 0.25, 0.75).astype(np.float64)
    return ((cells + u) / (1 << log2_r)).astype(np.float32)


def make_positions(kind, D, B, seed):
    rng = ob.default_rng(seed)
    x = ob.generate_random_uniform(rng, B * D).reshape(B, D)
    if kind == "uniform":
        return x
    log2_r = binning_log2_resolution(B, D)
    if kind == "clamped":
        # y and z both below the unit cube or both above it (x stays inside): bins 0 and R^2 - 1 only
        low = ob.generate_random_uniform(rng, B) < 0.5
        for d in (1, 2):
            x[:, d] = np.where(low, ob.generate_random_uniform(rng, B, -0.5, 0.0), ob.generate_random_uniform(rng, B, 1.0, 1.5))
        return x
    if kind == "straddle":
        keys = np.asarray(STRADDLE_KEYS[D], np.int64)
        keys = keys[np.minimum((ob.generate_random_uniform(rng, B) * len(keys)).astype(np.int64), len(keys) - 1)]
    else:
        assert kind == "one_bin"
        keys = np.full(B, one_bin_key(D, B), np.int64)
    if D == 2:
        x[:, 1] = cell_positions(rng, keys, log2_r)
    else:
        x[:, 1] = cell_positions(rng, compact1by1(keys), log2_r)
        x[:, 2] = cell_positions(rng, compact1by1(keys >> 1), log2_r)
    return x


def expected_keys(kind, D, B):
    """The bins a batch of this kind fills (None: not pinned)."""
    if kind == "straddle":
        return set(STRADDLE_KEYS[D])
    if kind == "one_bin":
        return {one_bin_key(D, B)}
    if kind == "clamped":
        return {0, binning_n_bins(binning_log2_resolution(B, D), D) - 1}
    return None


def make_batch(kind, D, B, seed):
    x = make_positions(kind, D, B, seed)
    return np.ascontiguousarray(x), ob.make_targets(x, N_OUT)


@pytest.mark.parametrize("name", list(CASES))
def test_premise_scan_chunks_and_bins(name):
    """The sizing rule restated here matches binning.cu's scan chunk, gives the chunk counts the cases below are named for, and
    every batch fills exactly the bins it is built for."""
    with open(os.path.join(ROOT, "tiny-cuda-nn_b200", "csrc", "binning.cu")) as f:
        src = f.read()
    assert re.search(r"constexpr uint32_t SCAN_CHUNK = (\d+);", src).group(1) == str(SCAN_CHUNK)
    assert binning_n_bins(binning_log2_resolution(1 << 20, 3), 3) == 65536 and scan_chunks(1 << 20, 3) == 4
    assert binning_n_bins(binning_log2_resolution(1 << 19, 2), 2) == 32768 and scan_chunks(1 << 19, 2) == 2
    assert [binning_n_bins(binning_log2_resolution(n, 3), 3) for n in CHANGING_BATCHES] == [65536, 65536, 4096, 16384, 16384, 65536]

    _, D, B, kind, chunks = CASES[name]
    assert scan_chunks(B, D) == chunks
    want = expected_keys(kind, D, B)
    if want is not None:
        x, _ = make_batch(kind, D, B, seed=CASE_SEED)
        keys, counts = np.unique(bin_keys(x, binning_log2_resolution(B, D)), return_counts=True)
        assert set(keys.tolist()) == want and counts.min() > B // (4 * len(want)), (keys, counts)
        if kind == "clamped":
            assert ((x[:, 0] >= 0) & (x[:, 0] < 1)).all() and not ((x[:, 1:] > 0) & (x[:, 1:] < 1)).any()


# ---- GPU side


def f16_bits(a):
    return a.view(np.uint16)


class Setup:
    """One model of a configuration and the CPU oracle of its grid (same initial parameters)."""

    def __init__(self, cfg_name, D):
        import tcnn_b200

        self.cfg = load_cfg(cfg_name)
        self.D = D
        self.model = tcnn_b200.create_from_config(D, N_OUT, self.cfg)
        self.orc = ob.OracleModel(D, N_OUT, self.cfg, scales=self.model.grid_levels()["scales"])
        self.n_mlp = self.model.n_mlp_params
        self.W = self.orc.grid.padded_width
        assert self.W == 32 and self.n_mlp == self.orc.n_mlp

    def close(self):
        self.model.set_debug_taps()
        self.model.close()


def train_step(torch, s, xd, yd, path):
    """One step without the optimizer on `path` ("binned", "unbinned", "general"), every tap NaN-filled first."""
    import tcnn_b200

    B = xd.shape[0]
    nan = float("nan")
    taps = {
        "encoded": torch.full((B, 64), nan, dtype=torch.float16, device="cuda"),
        "output": torch.full((B, 16), nan, dtype=torch.float16, device="cuda"),
        "loss_values": torch.full((B, N_OUT), nan, dtype=torch.float32, device="cuda"),
        "dL_dencoded": torch.full((B, 64), nan, dtype=torch.float16, device="cuda"),
    }
    m = s.model
    m.debug_set("binning", int(path == "binned"))
    m.debug_set("general", int(path == "general"))
    m.set_debug_taps(**taps)
    try:
        n0 = tcnn_b200.kernel_launch_count()
        m.trainer.training_step(xd, yd, run_optimizer=False)
        loss = m.trainer.loss()
        launches = tcnn_b200.kernel_launch_count() - n0
    finally:
        m.set_debug_taps()
        m.debug_set("binning", 1)
        m.debug_set("general", 0)
    grads = m.trainer.param_gradients().cpu().numpy()
    taps = {k: v.cpu().numpy() for k, v in taps.items()}
    return SimpleNamespace(loss=loss, launches=launches, grads=grads, taps=taps)


def oracle_encode_check(s, x, enc_dev, want_indexed):
    """orc.encode(x) == the device's encoded features bit for bit, for every sample; optionally the set of table parameters any
    sample indexes (from the oracle's integer indices). In chunks, to bound the index array."""
    orc = s.orc
    L, F = orc.grid.n_levels, orc.grid.n_features_per_level
    offsets = np.asarray(orc.grid.offsets[:L], np.int64)
    indexed = np.zeros(orc.grid.n_params // F, bool) if want_indexed else None
    step = 1 << 17
    for lo in range(0, x.shape[0], step):
        hi = min(x.shape[0], lo + step)
        enc_ref, idx = orc.encode(np.ascontiguousarray(x[lo:hi]), want_indices=True) if want_indexed else (orc.encode(np.ascontiguousarray(x[lo:hi])), None)
        bad = (f16_bits(enc_dev[lo:hi, : s.W]).T != enc_ref).any(axis=0)
        assert not bad.any(), f"{bad.sum()} samples encoded differently from the oracle, first {lo + np.flatnonzero(bad)[:8]}"
        if want_indexed:
            indexed[(idx.astype(np.int64) + offsets[None, :, None]).ravel()] = True
    return np.repeat(indexed, F) if want_indexed else None


# set of table parameters a batch indexes, by (configuration, positions, batch, seed): the oracle's indices cost as much as its
# encoding, about 12 s per 2^20 samples of the headline grid on 8 CPU cores
_INDEXED = {}


def check_batch(torch, s, x, y, full_oracle=True, exact_sums=True, key=None):
    """Checks 1-5 of the module docstring on one batch. The CPU oracle bounds the cost: without `full_oracle`, checks 1-4 with
    the oracle's encoding of the first 2^15 samples only; without `exact_sums`, check 5 without the oracle's grid scatter (as
    long again as its encoding). `key` caches the indexed set for a later test on the same batch."""
    B, D = x.shape
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    binned = train_step(torch, s, xd, yd, "binned")
    unbinned = train_step(torch, s, xd, yd, "unbinned")
    general = train_step(torch, s, xd, yd, "general")
    # premise: the binning pass (three kernels) ran in the binned step exactly when the batch is large enough
    assert binned.launches - unbinned.launches == (3 if scan_chunks(B, D) else 0), (binned.launches, unbinned.launches)

    # 1. every sample trained: no tap row still holds the sentinel
    width = {"encoded": s.W, "output": 16, "loss_values": N_OUT, "dL_dencoded": s.W}
    for path, st, names in (("binned", binned, width), ("unbinned", unbinned, width), ("general", general, ("output", "loss_values"))):
        for tap in names:
            missed = np.isnan(st.taps[tap][:, : width[tap]]).any(axis=1)
            assert not missed.any(), f"{path} step: {missed.sum()} of {B} rows of the {tap} tap not written, first {np.flatnonzero(missed)[:8]}"

    # 2. per-sample values bit for bit, in caller order
    for tap, w in width.items():
        a, b = binned.taps[tap][:, :w], unbinned.taps[tap][:, :w]
        itype = np.uint32 if a.dtype == np.float32 else np.uint16
        differ = (a.view(itype) != b.view(itype)).any(axis=1)
        assert not differ.any(), f"{tap}: {differ.sum()} rows differ between the binned and the unbinned step, first {np.flatnonzero(differ)[:8]}"
    n_orc = B if full_oracle else min(B, 1 << 15)
    indexed = oracle_encode_check(s, x[:n_orc], binned.taps["encoded"][:n_orc], full_oracle)
    if key is not None:
        _INDEXED[key] = indexed

    # 3. the loss
    lsum = binned.taps["loss_values"].sum(dtype=np.float64)
    assert abs(binned.loss - lsum) <= 1e-4 * abs(lsum), (binned.loss, lsum)
    assert abs(binned.loss - unbinned.loss) <= 1e-4 * abs(unbinned.loss), (binned.loss, unbinned.loss)
    assert abs(binned.loss - general.loss) <= 1e-3 * abs(general.loss), (binned.loss, general.loss)

    # 4. network weight gradients: the same fp32 sums in another order; the general path's bar of test_gpu_general.py
    n_mlp = s.n_mlp
    assert rae(binned.grads[:n_mlp], unbinned.grads[:n_mlp], 99.9) < 1e-3
    assert rae(binned.grads[:n_mlp], general.grads[:n_mlp], 99.9) < 5e-3

    # 5. table gradients: only entries some sample indexes, the same touched sets in both orders (up to sums that cancel to
    #    exactly zero in one order only), and against the exact sums of the device's own dL/d(encoded) (bit-identical in both
    #    orders, check 2) as in test_gpu_parity_large.py's test_benchmarked_size_against_reference
    if full_oracle:
        gb, gu = binned.grads[n_mlp:].astype(np.float64), unbinned.grads[n_mlp:].astype(np.float64)
        assert not gb[~indexed].any() and not gu[~indexed].any(), "gradient written to an entry no sample indexes"
        assert ((gb != 0) != (gu != 0)).sum() <= 1e-4 * indexed.sum()
        if exact_sums:
            exact = s.orc.grid_backward(x, np.ascontiguousarray(f16_bits(binned.taps["dL_dencoded"][:, : s.W]).T))
            own_err = rae(gb[indexed], exact[indexed], 99.9)
            ref_err = rae(gu[indexed], exact[indexed], 99.9)
            assert own_err <= max(1.2e-2, 1.25 * ref_err), (own_err, ref_err)


@gpu
@pytest.mark.parametrize("name", list(CASES))
def test_binned_step_matches_unbinned_and_general(torch_cuda, name):
    cfg_name, D, B, kind, _ = CASES[name]
    s = Setup(cfg_name, D)
    try:
        x, y = make_batch(kind, D, B, seed=CASE_SEED)
        # odd_batch: the uniform_4chunks scatter with 2.5 % more samples; its exact sums would add 13 s of CPU time
        check_batch(torch_cuda, s, x, y, exact_sums=name != "odd_batch", key=(cfg_name, kind, B, CASE_SEED) if kind == "one_bin" else None)
    finally:
        s.close()


@gpu
def test_changing_batch_sizes_on_one_model(torch_cuda):
    """65 536 bins, again 65 536 (the scan must have re-armed the counters it read), 4 096 and 16 384 (bin_hist reallocated and
    zeroed), 16 384 from another batch size (no reallocation), and 65 536 again; every step on a batch of its own. The table
    gradients of these sizes are checked against the exact sums by test_binned_step_matches_unbinned_and_general."""
    s = Setup("headline", 3)
    try:
        for i, B in enumerate(CHANGING_BATCHES):
            x, y = make_batch("uniform", 3, B, seed=300 + i)
            check_batch(torch_cuda, s, x, y, full_oracle=False)
    finally:
        s.close()


@gpu
@pytest.mark.parametrize("binning,B", [(1, 1 << 20), (0, 1 << 20), (1, 1 << 14)], ids=["binned", "unbinned", "binned_2^14"])
def test_overwrite_clears_previous_gradients(torch_cuda, binning, B):
    """GradientMode::Overwrite: after a uniform step, a step on one (y, z) column leaves every entry it does not index at exactly
    zero. Binned, the table is zeroed by bin_count_kernel's grid-stride loop, whose stride is set by the batch (several passes
    over the 26 MB table at 2^14 samples); unbinned, by a memset."""
    torch = torch_cuda
    s = Setup("headline", 3)
    try:
        xa, ya = make_batch("uniform", 3, B, seed=11)
        xb, yb = make_batch("one_bin", 3, B, seed=CASE_SEED)  # at 2^20 the one_bin case's batch: its indexed set is known
        first = train_step(torch, s, torch.from_numpy(xa).cuda(), torch.from_numpy(ya).cuda(), "binned" if binning else "unbinned")
        second = train_step(torch, s, torch.from_numpy(xb).cuda(), torch.from_numpy(yb).cuda(), "binned" if binning else "unbinned")
        key = ("headline", "one_bin", B, CASE_SEED)
        if key not in _INDEXED:
            _INDEXED[key] = oracle_encode_check(s, xb, second.taps["encoded"], True)
        indexed = _INDEXED[key]
        ga, gb = first.grads[s.n_mlp :], second.grads[s.n_mlp :]
        stale = (ga != 0) & ~indexed
        assert stale.sum() > 0.5 * (ga != 0).sum(), "premise: most entries the first step wrote are not indexed by the second"
        left = (gb != 0) & ~indexed
        assert not left.any(), f"{left.sum()} gradients of the previous step survived, first {np.flatnonzero(left)[:8]}"
        if binning:
            other = train_step(torch, s, torch.from_numpy(xb).cuda(), torch.from_numpy(yb).cuda(), "unbinned")
            assert second.launches - other.launches == 3, "premise: the binning pass ran"
    finally:
        s.close()


@gpu
def test_binned_and_unbinned_trajectories_agree(torch_cuda):
    """Five Adam steps on a 2^20-sample batch (four scan chunks), binned and unbinned, on two models of the same seed."""
    torch = torch_cuda
    x, y = make_batch("uniform", 3, 1 << 20, seed=21)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    losses = {}
    for binning in (1, 0):
        s = Setup("headline", 3)
        try:
            s.model.debug_set("binning", binning)
            losses[binning] = []
            for _ in range(5):
                s.model.trainer.training_step(xd, yd)
                losses[binning].append(s.model.trainer.loss())
        finally:
            s.close()
    assert losses[1][-1] < losses[1][0]
    for a, b in zip(losses[1], losses[0]):
        assert abs(a - b) <= 1e-3 * abs(b), losses
