"""The fused commit transforms (csrc/fft_fused.cu) at every size, blow-up and output they are built for, and the generic FFT pass
kernel (csrc/fft.cu) on columns that are not 16-byte aligned (run on an H100: `pytest -m gpu`).  Bar: bit-exact, against the oracle or
against the single-GPU proof bytes.

  * every fused size 2^16..2^22 at blow-up 2 and 4 (the A/C kernels <12, 4, 3> and <13, 2, 2>, the six mid kernels, 2 and 4 forward heads),
    and both edges of the fused plan (2^15 and 2^23 take the per-pass route);
  * the same transforms on a context whose twiddle bank was prepared for a larger domain first (the kernels index the bank from its end);
  * the two D2 heads of the mid kernel (the half-coset extension of a sharded commit), through whole proofs on a one-rank communicator;
  * columns at a 4-byte offset, which only fft_pass_kernel / fft_small_kernel can transform.

Every batch holds 5 columns, so the last column group of the CB = 4 and CB = 2 kernels is partly filled (4 + 1, 2 + 2 + 1); every column
mixes structured rows (zeros, P - 1, an impulse, bytes) with uniform values in [0, P)."""
import gc
import os

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200.prover import CudaBackend
from oracle import pyoracle as orc

pytestmark = pytest.mark.gpu
P = (1 << 31) - 1
N_COLS = 5
SLOW_LOG = 21      # the oracle takes seconds per column from here on


@pytest.fixture(scope="module", autouse=True)
def _oracle_threads():
    before = orc.num_threads()
    orc.set_num_threads(os.cpu_count())
    yield
    orc.set_num_threads(before)


@pytest.fixture(scope="module")
def ctx():
    c = nb.Context(0)
    yield c
    gc.collect()
    c.close()


def _param(log, *rest):
    return pytest.param(log, *rest, marks=[pytest.mark.slow] if log >= SLOW_LOG else [])


def _columns(n_cols, log, seed):
    """Each column is cut into five row ranges (in an order that rotates with the column): all zero, all P - 1, zero but one row,
    byte-valued, uniform in [0, P)."""
    rng = np.random.default_rng(seed)
    n = 1 << log
    out = np.empty((n_cols, n), np.uint32)
    for c in range(n_cols):
        for k, rows in enumerate(np.array_split(np.arange(n), 5)):
            kind = (k + c) % 5
            if kind == 0:
                out[c, rows] = 0
            elif kind == 1:
                out[c, rows] = P - 1
            elif kind == 2:
                out[c, rows] = 0
                out[c, rows[rng.integers(0, rows.size)]] = 1 + rng.integers(0, P - 1)
            elif kind == 3:
                out[c, rows] = rng.integers(0, 256, rows.size)
            else:
                out[c, rows] = rng.integers(0, P, rows.size)
    return out


def _same(got, exp, what):
    assert got.shape == exp.shape, f"{what}: shape {got.shape} != {exp.shape}"
    bad = np.nonzero(got != exp)
    if bad[0].size:
        c, r = int(bad[0][0]), int(bad[1][0])
        pytest.fail(f"{what}: {bad[0].size} words differ, the first in column {c} row {r}: {got[c, r]} != {exp[c, r]}")


def _check_interpolate_evaluate(ctx, log, log_blowup, n_cols, seed):
    host = _columns(n_cols, log, seed)
    oco, olde = orc.interpolate_evaluate_batch(host, log_blowup, want_coeffs=True)
    ev = ctx.upload(host)
    co, lde = ctx.interpolate_evaluate(ev, log_blowup)
    _same(co.download(), oco, "coefficients")
    _same(lde.download(), olde, "LDE")
    _same(ev.download(), host, "evaluations after interpolate_evaluate")
    # the header's promise: the same words as interpolate followed by evaluate
    ctx.interpolate(ev)
    _same(ev.download(), oco, "interpolate")
    _same(ctx.evaluate(ev, log_blowup).download(), olde, "evaluate")


# ---- 1. the fused pipeline on its own -------------------------------------------------------------------------------------------

FUSED = [_param(log, bl, N_COLS) for log in range(16, 23) for bl in (1, 2)]
EDGES = [_param(15, 1, N_COLS), _param(23, 1, N_COLS)]          # one below and one above fused_plan's range
ONE_COLUMN = [_param(16, 2, 1), _param(22, 1, 1)]


@pytest.mark.parametrize("log,log_blowup,n_cols", FUSED + EDGES + ONE_COLUMN)
def test_interpolate_evaluate_matches_oracle(ctx, log, log_blowup, n_cols):
    _check_interpolate_evaluate(ctx, log, log_blowup, n_cols, seed=1000 * log + 10 * log_blowup + n_cols)


@pytest.mark.slow
def test_commit_evals_at_2p22_matches_oracle_root(ctx):
    # 17 columns: 8 full column pairs of the <13, 2, 2> A/C kernels and a lone one; the small batch is committed into the same tree
    big = _columns(17, 22, seed=22)
    small = _columns(3, 6, seed=6)
    batches = [ctx.upload(big), ctx.upload(small)]
    coeffs, ldes, tree = ctx.commit_evals(batches, 1)
    flat = []
    for h, ev, co, lde in zip((big, small), batches, coeffs, ldes):
        oco, olde = orc.interpolate_evaluate_batch(h, 1, want_coeffs=True)
        _same(ev.download(), h, "evaluations after commit_evals")
        _same(co.download(), oco, "coefficients")
        _same(lde.download(), olde, "LDE")
        flat += list(olde)
    assert tree.root == orc.merkle_commit(flat)


# ---- 2. a twiddle bank prepared for a larger domain than the transform -----------------------------------------------------------

@pytest.fixture(scope="module")
def big_bank_ctx():
    c = nb.Context(0)
    c.precompute_twiddles(24)
    yield c
    gc.collect()
    c.close()


@pytest.mark.parametrize("log,log_blowup,n_cols", [_param(14, 1, N_COLS), _param(16, 1, N_COLS), _param(20, 1, N_COLS), _param(22, 1, N_COLS)])
def test_interpolate_evaluate_with_a_larger_twiddle_bank(big_bank_ctx, log, log_blowup, n_cols):
    assert nb.lib().nb200_twiddles_domain_log(big_bank_ctx._h) == 24
    _check_interpolate_evaluate(big_bank_ctx, log, log_blowup, n_cols, seed=1000 * log + 10 * log_blowup + n_cols)
    assert nb.lib().nb200_twiddles_domain_log(big_bank_ctx._h) == 24


# ---- 3. the fused D2 heads, on one GPU -----------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def one_rank_ctx():
    c = nb.Context(0)
    c.comm_init(0, 1, nb.Context.comm_unique_id())
    yield c
    gc.collect()
    c.close()


def _sharded_matches_single(one_rank_ctx, ctx, m, cols, mult, verify):
    proof, claimed, aux = M.prove_sharded(m, CudaBackend(one_rank_ctx), cols, mult, 0, 1, associated_data=b"d2")
    single, claimed1, aux1 = M.prove(m, CudaBackend(ctx), cols, mult, associated_data=b"d2")
    assert aux["roots"] == aux1["roots"]
    assert claimed == claimed1
    assert proof == single
    if verify:
        from tests.oracle_backend import verify_with_replayed_transcript
        verify_with_replayed_transcript(m, proof, claimed, aux)      # raises on a rejected proof


@pytest.mark.parametrize("log", [_param(log) for log in range(16, 23)])
def test_sharded_proof_with_fused_d2_heads_matches_single_gpu(one_rank_ctx, ctx, log):
    """AddMachine has log_expand 2 and degree-3 constraints, so the sharded commit asks commit_transforms for the half-coset extension D2:
    at these sizes the fused mid kernel computes it with two extra forward heads (ftn = n + 2, fhi = 0 and 1).  The ordinary proof on another
    context takes its D2 from fft.cu's half-domain transform; a wrong D2 word in a column a degree-3 constraint reads changes the composition
    polynomial and hence the proof bytes.  The row scatter of the last pass is NOT reached: a one-rank communicator has no peer heap, so the
    commit re-shards by copies; only the multi-GPU tests (tests/test_gpu_multi.py) cover it."""
    m = M.AddMachine(log_size=log, n_lanes=1)
    cols, mult = m.fill_main_trace(seed=log, n_padding=37)
    _sharded_matches_single(one_rank_ctx, ctx, m, cols, mult, verify=log in (17, 22))


def test_sharded_v1_proof_with_fused_d2_heads_matches_single_gpu(one_rank_ctx, ctx):
    # 347 main columns: the last column group of the mid kernel (CB = 2 at 2^16) is partly filled.  On the padding witness every degree-3 and
    # degree-4 constraint is gated by a selector that is the constant 0 (the opcode flags are all zero, 1 - IsPadding too), so a wrong D2 word
    # does not change these bytes: this case pins the LDE heads of that group, not its D2 heads (the AddMachine cases pin those, on full groups)
    from nexus_zkvm_b200.nexus_v1 import NexusV1Machine
    m = NexusV1Machine(16)
    _sharded_matches_single(one_rank_ctx, ctx, m, m.fill_main_trace(seed=16), None, verify=False)


# ---- 4. columns that are not 16-byte aligned -----------------------------------------------------------------------------------

class _Unaligned:
    """n_cols x 2^log words at a 4-byte offset into a device buffer of one word more: only the 32-bit FFT kernels can read them."""

    def __init__(self, ctx, n_cols, log):
        import torch
        self.buf = torch.zeros((n_cols << log) + 1, dtype=torch.int32, device="cuda:0")
        torch.cuda.synchronize()
        self.cols = ctx.wrap_device(self.buf.data_ptr() + 4, n_cols, log)
        assert self.cols.device_ptr % 16 == 4


@pytest.mark.parametrize("log", [_param(log) for log in (9, 13, 14, 17, 21, 22)])
def test_unaligned_columns_match_aligned(ctx, log):
    host = _columns(N_COLS, log, seed=7000 + log)
    aligned = {}
    for bl in (1, 2):
        co, lde = ctx.interpolate_evaluate(ctx.upload(host), bl)
        aligned[bl] = (co.download(), lde.download())
    if log < SLOW_LOG:   # the aligned results of the larger sizes are pinned to the oracle by test_interpolate_evaluate_matches_oracle
        for bl in (1, 2):
            oco, olde = orc.interpolate_evaluate_batch(host, bl, want_coeffs=True)
            _same(aligned[bl][0], oco, "aligned coefficients")
            _same(aligned[bl][1], olde, "aligned LDE")
    coeffs = aligned[1][0]
    # interpolate in place: every pass reads and writes unaligned columns
    u = _Unaligned(ctx, N_COLS, log)
    u.cols.upload(host)
    ctx.interpolate(u.cols)
    _same(u.cols.download(), coeffs, "interpolate (unaligned)")
    # evaluate from unaligned coefficients into an aligned LDE
    for bl in (1, 2):
        _same(ctx.evaluate(u.cols, bl).download(), aligned[bl][1], f"evaluate (unaligned coefficients, blow-up {1 << bl})")
    # interpolate_evaluate with unaligned evaluations, coefficients and LDE
    for bl in (1, 2):
        ev, co, lde = _Unaligned(ctx, N_COLS, log), _Unaligned(ctx, N_COLS, log), _Unaligned(ctx, N_COLS, log + bl)
        ev.cols.upload(host)
        ctx.interpolate_evaluate(ev.cols, bl, coeffs=co.cols, lde=lde.cols)
        _same(co.cols.download(), coeffs, f"interpolate_evaluate coefficients (unaligned, blow-up {1 << bl})")
        _same(lde.cols.download(), aligned[bl][1], f"interpolate_evaluate LDE (unaligned, blow-up {1 << bl})")
        _same(ev.cols.download(), host, "evaluations after interpolate_evaluate (unaligned)")
