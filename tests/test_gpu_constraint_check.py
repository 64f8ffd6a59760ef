"""The constraint check on the GPU (run on an H100: `pytest -m gpu`): nb200_check_constraints, reached through machine.check_constraints /
CommitmentSchemeProver.check_constraints, reports what the oracle's check (tests/oracle_check.py) reports on valid and broken witnesses,
at the benchmark size too, and gives back every byte it takes from the device's memory pool."""
import gc

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200.air import Air
from nexus_zkvm_b200.prover import CommitmentSchemeProver, CudaBackend
from tests import constraint_ref as ref
from tests import oracle_check
from tests.test_gpu_prove_ownership import _settled_pool_bytes

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = nb.Context(0)
    yield c
    gc.collect()
    c.close()


def _committed(ctx, m, t1):
    """prove's sequence up to the tree-2 commit on the GPU: (prover, params, host copies of the three trees' committed columns)."""
    _ch, prover, params, claimed, _roots, _ls = M._commit_trees(m, CudaBackend(ctx), t1, None, None, b"", None)
    assert M.verify_claimed_sums(claimed)
    host = [[c for b in batches for c in b.download()] for batches in prover.tree_evals]
    return prover, params, host


def _write_back(prover, host, touched):
    """Upload the batches that hold a changed column (committed order, as they are)."""
    for t in {t for t, _c in touched}:
        g = 0
        for b in prover.tree_evals[t]:
            if any(t == tt and g <= c < g + b.n_cols for tt, c in touched):
                b.upload(np.stack(host[t][g:g + b.n_cols]))
            g += b.n_cols


def _report(prover, m, params):
    return {k: [(i, a, r) for (i, _d, a, r) in prover.check_constraints(k, params)] for k in range(len(m.air.components))}


def _want(m, host, params):
    out = {}
    for k in range(len(m.air.components)):
        out[k] = [(i, a, r) for i, (a, r) in enumerate(oracle_check.check(m.words, k, host, params)) if a]
    return out


@pytest.mark.parametrize("log_size", [8, 12])
@pytest.mark.parametrize("kind", ref.KINDS, ids=ref.KIND_IDS)
def test_gpu_check_matches_the_reference(ctx, kind, log_size):
    m, t1 = ref.make_machine(kind, log_size)
    for case in ref.cases(kind):
        prover, params, host = _committed(ctx, m, t1)
        _write_back(prover, host, ref.apply_case(m, host, params, case))
        got, want = _report(prover, m, params), _want(m, host, params)
        assert got == want, case
        if case == "valid":
            assert not any(got.values())
        else:
            assert got[0], case


def test_degrees_in_the_report(ctx):
    m, t1 = ref.make_machine((1, False))
    prover, params, host = _committed(ctx, m, t1)
    ref.apply_case(m, host, params, "cumsum_shift")
    (k, deg, n_rows, first), = prover.check_constraints(0, params)
    assert (k, n_rows, first) == (len(m.air.components[0].constraints) - 1, 1 << m.log_size, 0) and deg >= 1


def test_machine_check_constraints(ctx):
    m, t1 = ref.make_machine("multi")
    report, balanced = M.check_constraints(m, CudaBackend(ctx), t1, None)
    assert balanced and set(report) == set(range(len(m.air.components))) and not any(report.values())
    t1 = [c.copy() for c in t1]
    t1[3][5] = (int(t1[3][5]) + 1) % 256                          # an ADD limb of the 2^4-row component, before the interaction trace
    report, balanced = M.check_constraints(m, CudaBackend(ctx), t1, None)
    assert report[0] and not balanced
    assert (report, balanced) == M.check_constraints(m, oracle_check.OracleCheckBackend(), t1, None)   # degrees included


def test_component_without_constraints(ctx):
    """A component with no constraint gives an empty report, not an error."""
    air = Air()
    air.component(10, 2).next_trace_mask()
    p = CommitmentSchemeProver(ctx, air.serialize(), dict(pow_bits=5, log_blowup=1, log_last=0, n_queries=3))
    ch = CudaBackend(ctx).channel()
    rng = np.random.default_rng(3)
    for _ in range(3):
        p.commit([rng.integers(0, ref.P, 1 << 10, dtype=np.uint32)], ch)
    assert p.check_constraints(0, []) == []


def test_benchmark_size_v1(ctx):
    """NexusV1Machine(20): the padding witness holds; one changed cell at coset row 100 (IsPadding cleared) is reported exactly as the same
    change at 2^12."""
    from nexus_zkvm_b200.nexus_v1 import MAIN_COLUMNS, NexusV1Machine
    ip = sum(s for name, s in MAIN_COLUMNS[:[x for x, _ in MAIN_COLUMNS].index("IsPadding")])
    reports = {}
    for log_size in (12, 20):
        m = NexusV1Machine(log_size)
        t1 = ref.flat(m.fill_main_trace(seed=1))
        backend = CudaBackend(ctx)
        valid, balanced = M.check_constraints(m, backend, t1, None)
        assert balanced and not any(valid.values()), log_size
        t1[ip][100] = 0
        reports[log_size], _ = M.check_constraints(m, backend, t1, None)
        del t1
        gc.collect()
    assert reports[20][0] and reports[20] == reports[12]


def test_check_releases_device_memory(ctx):
    m, t1 = ref.make_machine("nexus_v1")
    prover, params, host = _committed(ctx, m, t1)
    ref.apply_case(m, host, params, "cumsum_shift")
    prover.check_constraints(0, params)                       # warm-up: the check kernel is loaded
    base = _settled_pool_bytes(ctx)
    assert prover.check_constraints(0, params)
    assert _settled_pool_bytes(ctx) == base
