"""GPU parity AT THE BENCHMARKED SIZE (run on an H100: `pytest -m gpu`).

bench.py's configuration (BASELINE.json configs[1]: 2^20 rows, trees of 27 / 347 / 1012 columns, blow-up 2) runs kernel
instantiations that the small-size parity tests never reach: the 2^20 iFFT is `fft_tile_kernel<1,12,0,4,0>` +
`fft_tile_kernel<1,12,4,4,0>`, the 2^20 -> 2^21 LDE is the zero-extension pass `fft_tile_kernel<0,13,4,2,1>` (NZ = 1, FUSE_TOP,
two columns per CTA) followed by `fft_tile_kernel<0,12,0,4,0>`, and since round 2 the fused iFFT-tail + LDE-head kernel
`fft_fused_mid_kernel`.  Every one of them is compared here with the oracle, bit for bit, on real 2^20 / 2^21-point columns;
the whole commit (what bench.py times) is compared through both public entry points; and the 21-lane machine whose
generated 45 k-instruction constraint kernel bench.py's full proof runs is compared on proof BYTES.
Reference call sites: nexus-zkvm prover/src/machine.rs:208-263 (extend_evals / commit), :286-290 (prove)."""
import os

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200.prover import CudaBackend
from oracle import pyoracle as orc
from tests.oracle_backend import OracleBackend, verify

pytestmark = pytest.mark.gpu
P = (1 << 31) - 1


@pytest.fixture(scope="module")
def ctx():
    orc.set_num_threads(os.cpu_count() or 1)
    c = nb.Context(0)
    yield c
    c.close()


def _cols(rng, n_cols, log, structured=True):
    v = rng.integers(0, P, (n_cols, 1 << log), dtype=np.uint32)
    if structured and n_cols >= 3:
        v[1, :] = P - 1                                  # all P-1
        v[2, :] = rng.integers(0, 256, 1 << log)         # byte-valued like the reference's main trace
    return v


@pytest.mark.parametrize("log", [21, 22])
def test_twiddle_bank_matches_oracle_at_bench_size(log):
    """(d) the bank every butterfly of the 2^20 / 2^21 transforms reads (PolyOps::precompute_twiddles, machine.rs:186-194)."""
    c = nb.Context(0)
    tw, itw = c.twiddles(log)
    otw, oitw = orc.twiddles(log)
    assert np.array_equal(tw, otw)
    assert np.array_equal(itw, oitw)
    c.close()


@pytest.mark.parametrize("log", [20, 21])
def test_interpolate_bit_exact_at_bench_size(ctx, log):
    """2^20: fft_tile_kernel<1,12,0,4,0> + <1,12,4,4,0>; 2^21: <1,12,0,4,0> + <1,13,4,2,0>.  Five columns so that a partly
    filled column group (ncb < CB) is exercised too."""
    rng = np.random.default_rng(1000 + log)
    v = _cols(rng, 5, log)
    cols = ctx.upload(v)
    ctx.interpolate(cols)
    got = cols.download()
    for c in range(5):
        assert np.array_equal(got[c], orc.interpolate(v[c])), f"log={log} col={c}"


@pytest.mark.parametrize("log,blow", [(20, 1), (21, 1), (19, 2), (20, 2)])
def test_evaluate_lde_bit_exact_at_bench_size(ctx, log, blow):
    """(a) the zero-extended forward transforms bench.py launches: 2^20 -> 2^21 = fft_tile_kernel<0,13,4,2,1> (NZ=1, FUSE_TOP)
    + <0,12,0,4,0>; 2^21 -> 2^22 = <0,12,7,4,1>-family two-strided-pass plan; blow-up 4 exercises NZ = 2."""
    rng = np.random.default_rng(2000 + log + blow)
    coeffs = _cols(rng, 3, log)
    cols = ctx.upload(coeffs)
    got = ctx.evaluate(cols, blow).download()
    for c in range(3):
        assert np.array_equal(got[c], orc.evaluate(coeffs[c], log + blow)), f"log={log} col={c}"


def _oracle_tree(evals_by_batch, blow):
    flat, coeffs, ldes = [], [], []
    for ev in evals_by_batch:
        co, ld = orc.interpolate_evaluate_batch(ev, blow, want_coeffs=True)
        coeffs.append(co); ldes.append(ld); flat += list(ld)
    return coeffs, ldes, orc.merkle_commit(flat)


@pytest.mark.parametrize("n_cols", [27, 68, 80])
def test_commit_evals_at_bench_size(ctx, n_cols):
    """(b) nb200_commit_evals (the call bench.py's `value` times) on 2^20-row trees: 27 columns = the reference's tree 0; 68 and 80
    columns = slices of trees 1 / 2 (347 / 1012 columns; the oracle hashes 64+ real columns per tree in seconds, not 1012) —
    68 is not a multiple of the 16-column Blake2s block, 80 is."""
    rng = np.random.default_rng(3000 + n_cols)
    ev = _cols(rng, n_cols, 20)
    batch = ctx.upload(ev)
    coeffs, ldes, tree = ctx.commit_evals([batch], 1)
    oco, old, oroot = _oracle_tree([ev], 1)
    assert np.array_equal(coeffs[0].download(), oco[0])
    assert np.array_equal(ldes[0].download(), old[0])
    assert tree.root == oroot
    assert np.array_equal(batch.download(), ev)   # the evaluations are left untouched


@pytest.mark.parametrize("coset_order", [False, True])
def test_commit_host_at_bench_size(ctx, coset_order):
    """(b) nb200_commit_host (the e2e leg: pinned host columns -> chunked H2D -> transforms -> incremental leaf hashing)."""
    rng = np.random.default_rng(4000)
    n_cols = 72
    host = ctx.host_alloc(n_cols, 20)
    host[:] = _cols(rng, n_cols, 20)
    small = rng.integers(0, P, (3, 1 << 8), dtype=np.uint32)     # an extension-sized batch in the same tree (mixed sizes)
    evals, coeffs, ldes, tree = ctx.commit_host([host, small], 1, coset_order=coset_order)
    ref = [np.stack([orc.finalize_column(c) for c in b]) if coset_order else np.array(b) for b in (host, small)]
    oco, old, oroot = _oracle_tree(ref, 1)
    for k in range(2):
        assert np.array_equal(evals[k].download(), ref[k])
        assert np.array_equal(coeffs[k].download(), oco[k])
        assert np.array_equal(ldes[k].download(), old[k])
    assert tree.root == oroot


def test_commit_host_packed_bytes_at_bench_size(ctx):
    """The packed host format (u8 words for byte-valued columns, nb200_commit_host_packed) commits to the same root."""
    rng = np.random.default_rng(4100)
    n_cols = 40
    v = rng.integers(0, 256, (n_cols, 1 << 20), dtype=np.uint32)
    host8 = ctx.host_alloc_bytes(n_cols << 20).reshape(n_cols, 1 << 20)
    host8[:] = v.astype(np.uint8)
    evals, coeffs, ldes, tree = ctx.commit_host_packed([host8], [20], 1, coset_order=True)
    ref = np.stack([orc.finalize_column(c) for c in v])
    oco, old, oroot = _oracle_tree([ref], 1)
    assert np.array_equal(evals[0].download(), ref)
    assert np.array_equal(ldes[0].download(), old[0])
    assert tree.root == oroot


def test_proof_bytes_of_the_bench_machine(ctx):
    """(c) AddMachine(n_lanes=21) — 3 / 339 / 1012 columns, the machine of `bench.py --machine add21`, with its shipped generated
    constraint and logup kernels (jit_cache) — proof bytes equal the oracle's at 2^16 rows (the oracle needs ~30 s here).  bench.py's
    default machine, NexusV1Machine, is compared on proof bytes in tests/test_gpu_opening_at_scale.py."""
    be = CudaBackend(ctx)
    m = M.AddMachine(log_size=16, n_lanes=21)
    cols, mult = m.fill_main_trace(seed=21, n_padding=1000)
    g_proof, g_claimed, g_aux = M.prove(m, be, cols, mult, associated_data=b"bench")
    o_proof, o_claimed, o_aux = M.prove(m, OracleBackend(), cols, mult, associated_data=b"bench")
    assert g_aux["roots"] == o_aux["roots"]
    assert g_claimed == o_claimed
    assert g_proof == o_proof, f"proof bytes differ (len {len(g_proof)} vs {len(o_proof)})"
    verify(m, g_proof, o_aux)
