"""The constraint, half-domain, LogUp and check kernels on the GPU against the oracle, on witnesses where every constraint matters
(tests/random_witness.py: `full`, `main_random`, `sparse`), bit-exact.  The trees go through the ordinary commits on both sides.

The padding witness makes 42 of the 45 constraints of the v1 D2 kernel identically zero; here nb200_constraint_quotients_half reaches the D2
kernel, the D2 column gather and the q_high side sum with data on which each of them matters, at 2^12 rows and once at 2^16, where the grid
has many CTAs and waves.  (At 2^8 rows the LDE is smaller than the generated kernels' CTA, and the half route runs the bytecode interpreter,
which these tests also compare.)"""
import gc

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200.prover import CudaBackend
from tests import oracle_check
from tests import random_witness as rw
from tests.oracle_backend import OracleBackend
from tests.test_d2_high_degree_cpu import _walk_degrees
from tests.test_gpu_backend_ops import component_headers

pytestmark = pytest.mark.gpu
P = (1 << 31) - 1


@pytest.fixture(scope="module")
def ctx():
    c = nb.Context(0)
    yield c
    gc.collect()
    c.close()


def machine(name, log_size):
    if name == "nexus_v1":
        from nexus_zkvm_b200.nexus_v1 import NexusV1Machine
        return NexusV1Machine(log_size)
    if name == "add":
        return M.AddMachine(log_size=log_size, n_lanes=1 if log_size == 8 else 3)
    assert name == "multi"
    return M.MultiMachine(list(range(4, 12)))


def committed(ctx, m, w):
    """The witness committed on the GPU and on the oracle: (GPU prover, oracle prover, params); both sides agree on the parameters."""
    gpu, g_params = rw.commit(CudaBackend(ctx), m, w)
    orc_p, o_params = rw.commit(OracleBackend(), m, w)
    assert g_params == o_params
    return gpu, orc_p, g_params


CONFIG_BLOWUP = rw.CONFIG["log_blowup"]


def half_route(m, k):
    """Whether nb200_prove evaluates component k on the two half domains (prove.cu, quotient_mode)."""
    lg, expand, _n = component_headers(m.words)[k]
    return expand == CONFIG_BLOWUP + 1 and lg + CONFIG_BLOWUP > 8


def check_full_route(ctx, m, gpu, orc_p, params, seed, components=None):
    """nb200_constraint_quotients against the oracle for every component (or those listed in `components`), added to a random accumulator."""
    rng = np.random.default_rng(seed)
    for k, (lg, expand, n) in enumerate(component_headers(m.words)):
        if components is not None and k not in components:
            continue
        elog = lg + expand
        coeffs = rw.mixed(rng, 4 * n).reshape(n, 4)
        acc0 = rw.mixed(rng, 4 << elog).reshape(4, -1)
        g_acc = ctx.upload(acc0)
        gpu.constraint_quotients(k, params, coeffs, g_acc)
        want = orc_p.p.constraint_quotients(k, elog, np.array(params, dtype=np.uint32), coeffs, acc0)
        assert np.array_equal(g_acc.download(), want), f"component {k}"


# the generated constraint kernels run on at least this many rows (csrc/jit.h, JIT_BLOCK); below, the bytecode interpreter evaluates
JIT_MIN_LOG_ROWS = 10


def check_half_route(ctx, m, gpu, orc_p, params, seed, jit=True):
    """nb200_constraint_quotients_half against the oracle, for every component prove evaluates on the half domains: q on D1, the high
    constraints' q on D2 (the first half of the next larger canonic domain) and on D1, each added to a random accumulator.  Returns the number
    of components compared.  Where the bytecode interpreter evaluates (NB200_JIT=0, or an LDE smaller than the generated kernels' CTA) every
    constraint counts as a high one."""
    rng = np.random.default_rng(seed)
    prm = np.array(params, dtype=np.uint32)
    done = 0
    for k, (lg, expand, n) in enumerate(component_headers(m.words)):
        if not half_route(m, k):
            continue
        lde = lg + CONFIG_BLOWUP
        coeffs = rw.mixed(rng, 4 * n).reshape(n, 4)
        high = np.array([d > 2 for d in _walk_degrees(m.air.components[k])])
        c_high = np.where(high[:, None], coeffs, 0).astype(np.uint32)
        acc0 = [rw.mixed(rng, 4 << lde).reshape(4, -1) for _ in range(3)]
        g = [ctx.upload(a) for a in acc0]
        gpu.constraint_quotients_half(k, params, coeffs, *g)
        q_d1, q_high_d2, q_high_d1 = (x.download() for x in g)
        if not (jit and lde >= JIT_MIN_LOG_ROWS):
            c_high = coeffs
        assert np.array_equal(q_d1, orc_p.p.constraint_quotients(k, lde, prm, coeffs, acc0[0])), f"component {k}: q on D1"
        assert np.array_equal(q_high_d1, orc_p.p.constraint_quotients(k, lde, prm, c_high, acc0[2])), f"component {k}: q_high on D1"
        d2 = orc_p.p.constraint_quotients(k, lde + 1, prm, c_high)[:, :1 << lde]
        assert np.array_equal(q_high_d2, ((d2.astype(np.uint64) + acc0[1]) % P).astype(np.uint32)), f"component {k}: q_high on D2"
        done += 1
    return done


def check_report(m, gpu, orc_p, params):
    trees = [[c for b in batches for c in b.download()] for batches in gpu.tree_evals]
    for k in range(len(m.air.components)):
        want = [(i, a, r) for i, (a, r) in enumerate(oracle_check.check(m.words, k, trees, params)) if a]
        assert [(i, a, r) for (i, _d, a, r) in gpu.check_constraints(k, params)] == want, f"component {k}"
    return trees


@pytest.mark.parametrize("log_size", [8, 12])
@pytest.mark.parametrize("kind", ["full", "main_random"])
def test_v1_quotients(ctx, kind, log_size):
    m = machine("nexus_v1", log_size)
    gpu, orc_p, params = committed(ctx, m, rw.random_trees(m, 100 + log_size, kind))
    check_full_route(ctx, m, gpu, orc_p, params, 1)
    assert check_half_route(ctx, m, gpu, orc_p, params, 2) == 1


@pytest.mark.parametrize("log_size", [8, 12])
def test_v1_half_route_with_the_interpreter(ctx, monkeypatch, log_size):
    monkeypatch.setenv("NB200_JIT", "0")
    m = machine("nexus_v1", log_size)
    gpu, orc_p, params = committed(ctx, m, rw.random_trees(m, 200 + log_size, "full"))
    assert check_half_route(ctx, m, gpu, orc_p, params, 3, jit=False) == 1


def test_half_route_rejects_a_full_route_component(ctx):
    """The v1 machine's 2^8-row table component is evaluated on its own domain (Q_FULL): the half-domain entry point refuses it."""
    m = machine("nexus_v1", 8)
    gpu, _orc, params = committed(ctx, m, rw.random_trees(m, 5, "full"))
    lg, _e, n = component_headers(m.words)[1]
    assert not half_route(m, 1)
    acc = [ctx.upload(np.zeros((4, 1 << (lg + CONFIG_BLOWUP)), np.uint32)) for _ in range(3)]
    with pytest.raises(nb.Nb200Error):
        gpu.constraint_quotients_half(1, params, np.zeros((n, 4), np.uint32), *acc)


@pytest.mark.parametrize("log_size", [8, 12])
def test_v1_interaction_trace(ctx, log_size):
    """nb200_gen_interaction_trace on random trees 0 and 1 with random lookup elements: every column and the claimed sum equal the
    oracle's (the sums do not cancel)."""
    m = machine("nexus_v1", log_size)
    w = rw.random_trees(m, 300 + log_size, "full")
    sides = []
    for be in (CudaBackend(ctx), OracleBackend()):
        ch = be.channel()
        p = be.prover(m.words, rw.CONFIG)
        p.commit(w.tree0, ch, coset_order=True)
        p.commit(w.tree1, ch, coset_order=True)
        sides.append([p.gen_interaction(k, comp.log_size, max(comp.batching) + 1, w.params) for k, comp in enumerate(m.air.components)])
    for k, ((g_cols, g_sum), (o_cols, o_sum)) in enumerate(zip(*sides)):
        assert g_sum == o_sum, k
        assert np.array_equal(g_cols.download(), o_cols), k
    assert not M.verify_claimed_sums([s for _c, s in sides[0]])


@pytest.mark.parametrize("log_size", [8, 12])
@pytest.mark.parametrize("kind", ["sparse", "full"])
def test_v1_check(ctx, kind, log_size):
    m = machine("nexus_v1", log_size)
    gpu, orc_p, params = committed(ctx, m, rw.random_trees(m, 400 + log_size, kind))
    check_report(m, gpu, orc_p, params)


@pytest.mark.parametrize("name,log_size", [("add", 8), ("add", 12), ("multi", 11)])
def test_other_machines_on_full_trees(ctx, name, log_size):
    """AddMachine (log_expand 2) and MultiMachine (components of 2^4 to 2^11 rows), whose LogUp constraints hold in every other test, with
    random trees and parameters."""
    m = machine(name, log_size)
    gpu, orc_p, params = committed(ctx, m, rw.random_trees(m, 500 + log_size, "full"))
    check_full_route(ctx, m, gpu, orc_p, params, 4)
    assert check_half_route(ctx, m, gpu, orc_p, params, 5) >= 1


@pytest.mark.slow
def test_v1_at_2p16(ctx):
    """Once at 2^16 rows: many CTAs and waves in every kernel."""
    m = machine("nexus_v1", 16)
    gpu, orc_p, params = committed(ctx, m, rw.random_trees(m, 16, "full"))
    check_full_route(ctx, m, gpu, orc_p, params, 6)
    assert check_half_route(ctx, m, gpu, orc_p, params, 7) == 1
    check_report(m, gpu, orc_p, params)
    del gpu, orc_p
    gc.collect()
    gpu, orc_p, params = committed(ctx, m, rw.random_trees(m, 17, "sparse"))
    check_report(m, gpu, orc_p, params)
