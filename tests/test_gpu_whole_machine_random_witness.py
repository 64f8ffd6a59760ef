"""The whole machine's fifteen components (whole_machine.NexusV1KeccakMachine) on the GPU against the oracle, on witnesses where every
constraint matters (tests/random_witness.py: `full`, `main_random`, `sparse`), bit-exact: the constraint quotients (the main component's
on the half domains too), the interaction trace and the constraint check.

The machine's own witness leaves 146 of the main component's constraints and 200 of the keccak memory check's identically zero, so the proof
comparisons of test_gpu_whole_machine.py cannot see a wrong operand inside them.  Which kernel evaluates a program depends on its size
(csrc/jit.h): the generated kernel runs on 2^10 rows or more, the bytecode interpreter below that, on programs under 64 instructions, and
everywhere under NB200_JIT=0.  Two machines and the interpreter-only run cover both paths of every component (test_every_program_runs_on_
both_paths lists the exceptions):
  small  main 2^8, 15 permutations: the keccak round components run through the interpreter, in blocks of 32 threads (a 3.2 KB register
         file per thread);
  wide   main 2^10, 64 permutations: the main component is evaluated on the half domains by the generated kernels, the round components,
         RamInitFinal and the keccak tables get generated kernels with many CTAs; with NB200_JIT=0 every program runs through the
         interpreter, the round components on 2^9 to 2^11 rows.
The machines are built once per module.  On an H100 80GB HBM3 the module takes about a minute with every generated kernel in the cubin
cache; NVRTC dominates a cold run (the wide machine's four largest check kernels alone, the keccak rounds', the memory check's and the main
component's, took six minutes there)."""
import gc
import os

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200 import whole_machine as W
from nexus_zkvm_b200.prover import CudaBackend
from tests import random_witness as rw
from tests.oracle_backend import OracleBackend
from tests.test_constraint_check_cpu import kernel_source
from tests.test_gpu_backend_ops import component_headers
from tests.test_gpu_v1_random_witness import CONFIG_BLOWUP, JIT_MIN_LOG_ROWS, check_full_route, check_half_route, check_report, committed
from tests.test_gpu_v1_random_witness import half_route

pytestmark = pytest.mark.gpu
N_COMPONENTS = 15
# (main log size, permutations, seed) of each machine
MACHINES = {"small": (8, 15, 1), "wide": (10, 64, 0)}
# the runs of the constraint and LogUp programs in this module: (machine, generated kernels enabled)
RUNS = [("small", True), ("wide", True), ("wide", False)]
# programs whose generated kernel no run here reaches; tests/test_whole_machine_random_witness_cpu.py compares their generated sources on the
# host.  FinalReg (2^5 rows) and BitOpMultiplicity (2^8) have fixed sizes below 2^10 rows: a proof never runs their generated kernels.  The
# keccak memory check (2^4 and 2^6 rows here) and KeccakRound 1's LogUp (2^7 and 2^9) reach 2^10 rows only from 512 and 1024 permutations on.
NOT_GENERATED = {(1, "constraints"), (1, "logup"), (2, "constraints"), (9, "constraints"), (9, "logup"), (11, "logup")}


@pytest.fixture(scope="module")
def ctx():
    """A context with NB200_TRACE on: a generated kernel that cannot be compiled or loaded leaves its program to the interpreter with no
    more than a line on stderr, which the tests look for (no_fallback)."""
    old = os.environ.get("NB200_TRACE")
    os.environ["NB200_TRACE"] = "1"
    try:
        c = nb.Context(0)
    finally:
        if old is None:
            del os.environ["NB200_TRACE"]
        else:
            os.environ["NB200_TRACE"] = old
    yield c
    gc.collect()
    c.close()


@pytest.fixture(scope="module")
def machines():
    return {name: W.NexusV1KeccakMachine(ls, n, seed=s) for name, (ls, n, s) in MACHINES.items()}


def no_fallback(capfd):
    """Every generated constraint, D2 and LogUp kernel the calls since the last capture asked for was there (prove.cu ensure_jit): the trace
    shows the attempts and no failure."""
    err = capfd.readouterr().err
    assert "jit: compile" in err
    assert "jit unavailable" not in err, err[err.index("jit unavailable"):][:2000]


def n_half(m):
    return sum(half_route(m, k) for k in range(N_COMPONENTS))


@pytest.mark.parametrize("name", ["small", "wide"])
@pytest.mark.parametrize("kind", ["full", "main_random"])
def test_quotients(ctx, machines, capfd, kind, name):
    """constraint_quotients of every component on its full domain and constraint_quotients_half of the main component: q on D1, q_high on
    D2 and q_high on D1, each added to a random accumulator."""
    m = machines[name]
    gpu, orc_p, params = committed(ctx, m, rw.random_trees(m, 100 + MACHINES[name][0], kind))
    check_full_route(ctx, m, gpu, orc_p, params, 1)
    assert n_half(m) == 1 and half_route(m, 0)
    assert check_half_route(ctx, m, gpu, orc_p, params, 2) == 1
    no_fallback(capfd)


def check_interaction(ctx, m, w):
    """nb200_gen_interaction_trace on the trees of `w` with its lookup elements: every column, the last secure one after the prefix sum
    included, and the claimed sum equal the oracle's (the sums do not cancel)."""
    sides = []
    for be in (CudaBackend(ctx), OracleBackend()):
        ch = be.channel()
        p = be.prover(m.words, rw.CONFIG)
        p.commit(w.tree0, ch, coset_order=True)
        p.commit(w.tree1, ch, coset_order=True)
        sides.append([p.gen_interaction(k, comp.log_size, max(comp.batching) + 1, w.params) for k, comp in enumerate(m.air.components)])
    assert len(sides[0]) == N_COMPONENTS
    for k, ((g_cols, g_sum), (o_cols, o_sum)) in enumerate(zip(*sides)):
        assert g_sum == o_sum, k
        assert np.array_equal(g_cols.download(), o_cols), k
    assert not M.verify_claimed_sums([s for _c, s in sides[0]])


def test_quotients_and_interaction_with_the_interpreter(ctx, machines, monkeypatch):
    """NB200_JIT=0 on the wide machine: every constraint and LogUp program runs through the bytecode interpreter, the keccak round
    components' on 2^9 to 2^11 rows, and on D2 every constraint counts as a high one."""
    monkeypatch.setenv("NB200_JIT", "0")
    m = machines["wide"]
    w = rw.random_trees(m, 200, "full")
    gpu, orc_p, params = committed(ctx, m, w)
    check_full_route(ctx, m, gpu, orc_p, params, 3)
    assert check_half_route(ctx, m, gpu, orc_p, params, 4, jit=False) == 1
    del gpu, orc_p
    gc.collect()
    check_interaction(ctx, m, w)


@pytest.mark.parametrize("name", ["small", "wide"])
def test_interaction_trace(ctx, machines, capfd, name):
    m = machines[name]
    check_interaction(ctx, m, rw.random_trees(m, 300 + MACHINES[name][0], "full"))
    no_fallback(capfd)


@pytest.mark.parametrize("kind", ["sparse", "full"])
def test_check(ctx, machines, kind):
    """check_constraints of every component of the wide machine against the oracle's check: on `full` every constraint fails, on `sparse`
    each on its own rows.  The check has no interpreter: every component's generated check kernel runs, the 2^4-row tables' with threads
    past the end of their domain."""
    m = machines["wide"]
    gpu, orc_p, params = committed(ctx, m, rw.random_trees(m, 400, kind))
    check_report(m, gpu, orc_p, params)
    failing = [len(gpu.check_constraints(k, params)) for k in range(N_COMPONENTS)]
    if kind == "full":
        assert failing == [n for _lg, _e, n in component_headers(m.words)]
    else:
        assert all(failing[k] for k in (0, 9, 10, 11))


def routes(m, jit):
    """{(component, "constraints" / "logup"): set of "generated" / "interpreter"} for one machine, as the library picks them (csrc/jit.h
    jit_usable, prove.cu ensure_jit): a generated kernel where the library generates one for the program (nb200_air_kernel_source: a
    program of at least 64 instructions), generation is enabled and the rows number at least 2^10.  The constraint program runs on the
    component's full domain (check_full_route) and, for the main component, on the half domains; the LogUp program on the trace domain."""
    out = {}
    for k, (lg, expand, _n) in enumerate(component_headers(m.words)):
        for prog, which, row_logs in (("constraints", 0, [lg + expand] + ([lg + CONFIG_BLOWUP] if half_route(m, k) else [])),
                                      ("logup", 1, [lg])):
            has_source = kernel_source(m.words, k, which)[0] == 0
            out[(k, prog)] = {"generated" if jit and has_source and r >= JIT_MIN_LOG_ROWS else "interpreter" for r in row_logs}
    return out


def test_every_program_runs_on_both_paths(machines):
    """Across the runs of this module every component's constraint and LogUp program went through the interpreter at least once, and
    through its generated kernel wherever the library generates one, but for NOT_GENERATED: a change of sizes that drops a path fails here.
    (no_fallback checks that the generated kernels the runs ask for are there, so a derived route is the route taken.)"""
    seen, generated = {}, set()
    for name, jit in RUNS:
        m = machines[name]
        assert len(m.air.components) == N_COMPONENTS
        for key, paths in routes(m, jit).items():
            seen.setdefault(key, set()).update(paths)
        generated |= {(k, prog) for k in range(N_COMPONENTS) for prog, which in (("constraints", 0), ("logup", 1))
                      if kernel_source(m.words, k, which)[0] == 0}
    assert len(seen) == 2 * N_COMPONENTS
    assert [key for key, paths in sorted(seen.items()) if "interpreter" not in paths] == []
    assert {key for key in generated if "generated" not in seen[key]} == NOT_GENERATED
    # the keccak round components run through the interpreter on the small machine, through generated kernels on the wide one
    small, wide = routes(machines["small"], True), routes(machines["wide"], True)
    for k in (10, 11):
        assert small[(k, "constraints")] == {"interpreter"} and wide[(k, "constraints")] == {"generated"}
    assert small[(0, "constraints")] == {"generated", "interpreter"} and wide[(0, "constraints")] == {"generated"}
