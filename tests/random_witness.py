"""Witnesses that are not valid traces, for testing the constraint, LogUp and check kernels where the padding witness says nothing.

The v1 padding witness (NexusV1Machine.fill_main_trace) leaves most of tree 1 zero or constant: a third of the v1 constraints, and 42 of
the 45 that the half-coset D2 kernel evaluates, are identically zero under it, so a kernel could compute anything for them and still match
the oracle.  The constraint quotients, the interaction trace and the check report are defined for any trees and parameters, so the tests
compare them on these witnesses instead:

  full         every cell of trees 0 and 1 random, tree 2 and every parameter (lookup elements, cumsum shifts) random as well: the chip
               constraints and the LogUp constraints fail;
  main_random  trees 0 and 1 random, tree 2 from the interaction-trace generator and the cumsum shifts set as machine._commit_trees sets
               them: the chip constraints fail, the LogUp constraints hold;
  sparse       the valid (padding) witness with about 1 % of the cells of every tree-1 column replaced, rows 0 and N - 1 among them (the
               masks at a row offset wrap around there): each constraint fails on its own subset of rows.

Random cells are drawn from a mix that brings the field's edges into every constraint: uniform in [0, P), P - 1, 0, 1, bytes and 16-bit
values.  Everything is seeded."""
from dataclasses import dataclass

import numpy as np

from nexus_zkvm_b200 import air as A
from nexus_zkvm_b200 import machine as M
from oracle import pyoracle as orc
from tests import constraint_ref as ref

P = (1 << 31) - 1
KINDS = ("full", "main_random", "sparse")
CONFIG = dict(pow_bits=5, log_blowup=1, log_last=0, n_queries=3)


@dataclass
class Witness:
    tree0: list            # host columns in trace (coset) order
    tree1: list
    tree2: list = None     # committed (bit-reversed circle-domain) order, component by component; None: the interaction-trace generator's
    params: list = None    # the parameter table; None: drawn from the channel, cumsum shifts from the generated interaction trace


def mixed(rng, n):
    """n field elements from the mix: half uniform in [0, P), the rest P - 1, 0, 1, bytes and 16-bit values in equal parts."""
    pick = rng.integers(0, 10, n)
    out = rng.integers(0, P, n, dtype=np.uint32)
    out[pick == 5] = P - 1
    out[pick == 6] = 0
    out[pick == 7] = 1
    out[pick == 8] = rng.integers(0, 1 << 8, int((pick == 8).sum()), dtype=np.uint32)
    out[pick == 9] = rng.integers(0, 1 << 16, int((pick == 9).sum()), dtype=np.uint32)
    return out


def valid_tree1(m, seed=1):
    """The machine's own witness (the padding witness for v1), tree-1 host columns in trace order."""
    if isinstance(m, M.AddMachine):
        cols, mult = m.fill_main_trace(seed=seed, n_padding=2)
        return ref.flat(list(cols) + [mult])
    return ref.flat(m.fill_main_trace(seed=seed))


def random_trees(m, seed, kind):
    """A Witness of `kind` (module docstring) for machine m."""
    assert kind in KINDS, kind
    rng = np.random.default_rng(seed)
    pre = ref.flat(m.preprocessed_columns())
    if kind == "sparse":
        t1 = [c.copy() for c in valid_tree1(m, seed)]
        for c in t1:
            n = len(c)
            rows = np.union1d(rng.choice(n, max(1, n // 100), replace=False), [0, n - 1])
            c[rows] = rng.integers(1, P, rows.size, dtype=np.uint32)
        return Witness(pre, t1)
    t0 = [mixed(rng, len(c)) for c in pre]
    t1 = [mixed(rng, len(c)) for c in valid_tree1(m, seed)]
    if kind == "main_random":
        return Witness(t0, t1)
    t2 = [mixed(rng, 1 << comp.log_size) for comp in m.air.components for _ in range(4 * (max(comp.batching) + 1))]
    params = [tuple(int(x) for x in mixed(rng, 4)) for _ in range(m.air.n_params)]
    return Witness(t0, t1, t2, params)


def commit(backend, m, w):
    """Machine::prove's commit sequence on `backend` with the witness's trees: (prover, params).  Without a tree 2 of its own the witness
    gets the interaction trace the backend generates, with the cumsum shifts machine._commit_trees sets."""
    ch = backend.channel()
    p = backend.prover(m.words, CONFIG)
    p.commit(w.tree0, ch, coset_order=True)
    p.commit(w.tree1, ch, coset_order=True)
    if w.tree2 is not None:
        p.commit(w.tree2, ch)
        return p, list(w.params)
    params = [(0, 0, 0, 0)] * m.air.n_params
    for rel in (getattr(m, "relations", None) or [m.range256]):
        rel.draw(ch, params)
    inter = []
    for k, comp in enumerate(m.air.components):
        c, cs = p.gen_interaction(k, comp.log_size, max(comp.batching) + 1, params)
        inter.append(c)
        params[comp.cumsum_shift_param] = M.F.qm31_mul_m31(cs, M.F.m31_inv((1 << comp.log_size) % P))
    p.commit_interaction(inter, ch)
    p.interaction = inter
    return p, params


def padding(m, seed=1):
    """The machine's valid witness as a Witness (for v1: the padding witness)."""
    return Witness(ref.flat(m.preprocessed_columns()), valid_tree1(m, seed))


def on_oracle(m, w):
    """commit() on the oracle: (oracle prover, params, trees[t][col] as committed, in bit-reversed circle-domain order)."""
    from tests.oracle_backend import OracleBackend
    p, params = commit(OracleBackend(), m, w)
    t2 = w.tree2 if w.tree2 is not None else [c for block in p.interaction for c in block]
    trees = [[orc.finalize_column(np.ascontiguousarray(c, dtype=np.uint32)) for c in w.tree0],
             [orc.finalize_column(np.ascontiguousarray(c, dtype=np.uint32)) for c in w.tree1],
             [np.ascontiguousarray(c, dtype=np.uint32) for c in t2]]
    return p, params, trees


def identically_zero(words, comp, trees):
    """One flag per constraint of component `comp`: True when the constraint is zero on every domain whatever the parameters, because of
    the columns of `trees` (trees[t][col], any order) that are zero in every row; the columns of a tree left out of `trees` count as
    non-zero.  A zero column has a zero extension; a load of one is zero, a product with a zero factor is zero, a sum or difference of
    zeros is zero, a negation of zero is zero."""
    _ls, masks, prog = ref.parse_component(words, comp)
    zcol = [t < len(trees) and not np.any(np.asarray(trees[t][c])) for (t, c, _o) in masks]
    zb, ze, out = {}, {}, []
    for (op, dst, a, b) in prog:
        if op == A.OP_LOADM:
            zb[dst] = zcol[a]
        elif op == A.OP_CONSTB:
            zb[dst] = a == 0
        elif op in (A.OP_ADDB, A.OP_SUBB):
            zb[dst] = zb[a] and zb[b]
        elif op == A.OP_MULB:
            zb[dst] = zb[a] or zb[b]
        elif op == A.OP_NEGB:
            zb[dst] = zb[a]
        elif op == A.OP_PARAME:
            ze[dst] = False
        elif op in (A.OP_ADDE, A.OP_SUBE):
            ze[dst] = ze[a] and ze[b]
        elif op == A.OP_MULE:
            ze[dst] = ze[a] or ze[b]
        elif op == A.OP_NEGE:
            ze[dst] = ze[a]
        elif op in (A.OP_ADDEB, A.OP_SUBEB):
            ze[dst] = ze[a] and zb[b]
        elif op == A.OP_MULEB:
            ze[dst] = ze[a] or zb[b]
        elif op == A.OP_BTOE:
            ze[dst] = zb[a]
        elif op == A.OP_LOADME:
            ze[dst] = all(zcol[a:a + 4])
        elif op == A.OP_CONSTRB:
            out.append(zb[a])
        elif op == A.OP_CONSTRE:
            out.append(ze[a])
        else:
            raise ValueError(f"opcode {op}")
    return out
