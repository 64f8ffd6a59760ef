"""Device-memory ownership of the prover (run on an H100: `pytest -m gpu`).

A proof that fails must give back every byte it took from the device's memory pool, and the row-sharded code path
(sharded commits, interaction trace, constraint rows, DEEP quotients, decommitments) must reproduce the single-GPU bytes
on a one-rank communicator.  The library allocates columns, trees and temporaries from the device's default memory pool;
twiddles and FFT tables come from cudaMalloc and are not counted."""
import ctypes as C
import gc

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200.air import Air
from nexus_zkvm_b200.prover import CommitmentSchemeProver, CudaBackend

pytestmark = pytest.mark.gpu
P = (1 << 31) - 1
CU_MEMPOOL_ATTR_USED_MEM_CURRENT = 7
CFG = dict(pow_bits=5, log_blowup=1, log_last=0, n_queries=3)


def _pool_used_bytes(device=0):
    cu = C.CDLL("libcuda.so.1")
    assert cu.cuInit(0) == 0
    dev, pool, used = C.c_int(), C.c_void_p(), C.c_uint64()
    assert cu.cuDeviceGet(C.byref(dev), device) == 0
    assert cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    assert cu.cuMemPoolGetAttribute(pool, CU_MEMPOOL_ATTR_USED_MEM_CURRENT, C.byref(used)) == 0
    return used.value


def _settled_pool_bytes(ctx):
    gc.collect()
    ctx.sync()
    return _pool_used_bytes()


@pytest.fixture
def ctx():
    c = nb.Context(0)
    yield c
    gc.collect()
    c.close()


def _tampered_add_proof(ctx):
    m = M.AddMachine(log_size=8, n_lanes=1)
    cols, mult = m.fill_main_trace(seed=4)
    cols[2 + 8][17] = (int(cols[2 + 8][17]) + 1) % 256
    with pytest.raises(nb.Nb200Error, match="status 5"):
        M.prove(m, CudaBackend(ctx), cols, mult)


def _zero_constraint_proof(ctx):
    air = Air()
    air.component(10, 2).next_trace_mask()
    p = CommitmentSchemeProver(ctx, air.serialize(), CFG)
    ch = CudaBackend(ctx).channel()
    rng = np.random.default_rng(3)
    for _ in range(3):
        p.commit([rng.integers(0, P, 1 << 10, dtype=np.uint32)], ch)
    with pytest.raises(nb.Nb200Error, match="status 2"):
        p.prove(ch, [])


def test_failed_proof_releases_device_memory(ctx):
    m = M.AddMachine(log_size=8, n_lanes=1)
    cols, mult = m.fill_main_trace(seed=4)
    M.prove(m, CudaBackend(ctx), cols, mult)   # warm-up: every lazily created buffer of this machine exists
    base = _settled_pool_bytes(ctx)
    _tampered_add_proof(ctx)
    assert _settled_pool_bytes(ctx) == base


def test_rejected_air_releases_device_memory(ctx):
    # an AIR without constraints is rejected with NB200_ERR_ARG before anything is drawn or allocated for the proof
    _zero_constraint_proof(ctx)
    base = _settled_pool_bytes(ctx)
    _zero_constraint_proof(ctx)
    assert _settled_pool_bytes(ctx) == base


@pytest.fixture
def one_rank_ctx():
    c = nb.Context(0)
    c.comm_init(0, 1, nb.Context.comm_unique_id())
    yield c
    gc.collect()
    c.close()


def _machine(kind):
    if kind == "nexus_v1":
        from nexus_zkvm_b200.nexus_v1 import NexusV1Machine
        m = NexusV1Machine(12)
        return m, m.fill_main_trace(seed=12), None
    m = M.AddMachine(log_size=12, n_lanes=21)
    cols, mult = m.fill_main_trace(seed=12, n_padding=37)
    return m, cols, mult


@pytest.mark.parametrize("kind", ["add", "nexus_v1"])
def test_sharded_proof_on_one_rank_matches_single_gpu_bytes(one_rank_ctx, kind):
    m, cols, mult = _machine(kind)
    proof, claimed, aux = M.prove_sharded(m, CudaBackend(one_rank_ctx), cols, mult, 0, 1, associated_data=b"ng")
    single_ctx = nb.Context(0)
    try:
        single, claimed1, aux1 = M.prove(m, CudaBackend(single_ctx), cols, mult, associated_data=b"ng")
        assert aux1["roots"] == aux["roots"]
        assert claimed1 == claimed
        assert proof == single
    finally:
        gc.collect()
        single_ctx.close()


def test_library_sharded_commit_on_one_rank_matches_commit_root(one_rank_ctx):
    rng = np.random.default_rng(5)
    big = rng.integers(0, P, (48, 1 << 12), dtype=np.uint32)
    small = rng.integers(0, P, (3, 1 << 6), dtype=np.uint32)
    ctx = one_rank_ctx
    _, _, _, caps, root = ctx.commit_sharded(ctx.upload(big), 48, 12, 1, [ctx.upload(small)])
    _, _, tree = ctx.commit_evals([ctx.upload(big), ctx.upload(small)], 1)
    assert caps == [root]
    assert root == tree.root
