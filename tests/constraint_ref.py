"""The machines and broken witnesses the constraint check (nb200_check_constraints) is tested on, and a second, vectorised restatement of
stwo's assert_constraints_on_polys in numpy (`check`) that the tests hold against the oracle's check (tests/oracle_check.py) as a
cross-check: the component's constraint program runs on every row of its trace domain at once, each mask reading its column at the coset
(trace) row r + offset modulo the domain size.  A constraint fails on a row when its value is not zero.  Columns are given as committed:
evaluations in bit-reversed circle-domain order (finalize_column of the host trace)."""
import numpy as np

from nexus_zkvm_b200 import air as A
from oracle import pyoracle as orc

P = (1 << 31) - 1


def parse_component(words, k):
    """(log_size, masks [(tree, col, offset)], constraint program [(op, dst, a, b)]) of component k (layout: nexus_zkvm_b200/air.py)."""
    w = [int(x) for x in words]
    i = 4
    for c in range(w[3]):
        log_size = w[i]
        i += 3
        n_masks = w[i]
        masks = [(w[i + 1 + 3 * m], w[i + 2 + 3 * m], np.int32(np.uint32(w[i + 3 + 3 * m])).item()) for m in range(n_masks)]
        i += 1 + 3 * n_masks + 2
        n_instr = w[i]
        prog = [tuple(w[i + 1 + 4 * j: i + 5 + 4 * j]) for j in range(n_instr)]
        i += 1 + 4 * n_instr
        n_fracs = w[i]
        i += 3
        i += 1 + 4 * w[i]
        i += n_fracs + 2
        if c == k:
            return log_size, masks, prog
    raise IndexError(k)


def flat(cols):
    out = []
    for c in cols:
        a = np.asarray(c)
        out += list(a.astype(np.uint32)) if a.ndim == 2 else [np.ascontiguousarray(a, dtype=np.uint32)]
    return out


# ---- the machines and broken witnesses the check is tested on (CPU: host-compiled kernel, GPU: nb200_check_constraints)
KINDS = [(1, False), (2, True), "multi", "nexus_v1"]
KIND_IDS = ["add1", "add2_pairs", "multi", "nexus_v1"]


def make_machine(kind, log_size=8):
    """(machine, tree-1 host columns in trace order)"""
    from nexus_zkvm_b200 import machine as M
    if kind == "nexus_v1":
        from nexus_zkvm_b200.nexus_v1 import NexusV1Machine
        m = NexusV1Machine(log_size)
        return m, flat(m.fill_main_trace(seed=1))
    if kind == "multi":
        m = M.MultiMachine([4, 5, log_size])           # 2^4 and 2^5 rows: smaller than a warp / a CTA
        return m, flat(m.fill_main_trace(seed=2))
    lanes, pairs = kind
    m = M.AddMachine(log_size=log_size, n_lanes=lanes, logup_in_pairs=pairs)
    cols, mult = m.fill_main_trace(seed=3 + lanes, n_padding=2)
    return m, flat(list(cols) + [mult])


def cases(kind):
    return ["valid", "main_cell"] + (["unpadded"] if kind == "nexus_v1" else []) + ["interaction_cell", "cumsum_shift", "edges"]


def position(row, log_size):
    """Index of coset (trace) row `row` in a committed column."""
    return orc.bit_reverse_index(orc.coset_index_to_circle_domain_index(row, log_size), log_size)


def apply_case(m, trees, params, case, row=37):
    """Break the committed witness (trees[t][col], params; in place) the way `case` names; returns the (tree, column) pairs changed."""
    main = m.air.components[0]
    n = 1 << main.log_size
    col = next(c for (t, c, off) in main.masks if t == 1 and off == 0 and len(trees[1][c]) == n and c > 1)   # a plain main-trace cell
    touched = set()

    def bump(t, c, r):
        a = trees[t][c]
        i = position(r, main.log_size)
        a[i] = (int(a[i]) + 1) % P
        touched.add((t, c))

    if case == "main_cell":                       # after the interaction trace was generated from the valid trace
        bump(1, col, row % n)
    elif case == "unpadded":                      # v1: one padding row turned into a (non-)instruction row
        from nexus_zkvm_b200.nexus_v1 import MAIN_COLUMNS
        ip = sum(s for name, s in MAIN_COLUMNS[:[x for x, _ in MAIN_COLUMNS].index("IsPadding")])
        trees[1][ip][position(11, main.log_size)] = 0
        touched.add((1, ip))
    elif case == "interaction_cell":
        bump(2, main.interaction_col0, 21 % n)
    elif case == "cumsum_shift":
        s = list(params[main.cumsum_shift_param])
        s[0] = (int(s[0]) + 1) % P
        params[main.cumsum_shift_param] = tuple(s)
    elif case == "edges":                         # rows 0 and N - 1: the masks at a row offset wrap around there
        for r in (0, n - 1):
            bump(1, col, r)
            bump(2, main.interaction_col0 + 4 * max(main.batching), r)   # the cumulative-sum column
    else:
        assert case == "valid", case
    return touched


def _qmul(x, y):
    # (a + b u)(c + d u) = (ac + (2 + i) bd) + (ad + bc) u over CM31 = M31[i] / (i^2 + 1)
    def cmul(p, q):
        return ((p[0] * q[0] - p[1] * q[1]) % P, (p[0] * q[1] + p[1] * q[0]) % P)

    a, b, c, d = (x[0], x[1]), (x[2], x[3]), (y[0], y[1]), (y[2], y[3])
    ac, bd, ad, bc = cmul(a, c), cmul(b, d), cmul(a, d), cmul(b, c)
    rbd = ((2 * bd[0] - bd[1]) % P, (2 * bd[1] + bd[0]) % P)
    return ((ac[0] + rbd[0]) % P, (ac[1] + rbd[1]) % P, (ad[0] + bc[0]) % P, (ad[1] + bc[1]) % P)


def check(words, comp, trees, params):
    """[(failing rows, first failing coset row or None)] per constraint of component `comp`; trees[t][col] = committed evaluations."""
    log_size, masks, prog = parse_component(words, comp)
    n = 1 << log_size
    # position of coset row r in a committed column
    pos = np.array([orc.bit_reverse_index(orc.coset_index_to_circle_domain_index(r, log_size), log_size) for r in range(n)], dtype=np.int64)
    rows = np.arange(n)
    mval = [np.asarray(trees[t][c], dtype=np.int64)[pos[(rows + off) % n]] for (t, c, off) in masks]
    prm = [tuple(np.int64(int(v)) for v in q) for q in params]
    b, e, out = {}, {}, []
    zero = np.zeros(n, np.int64)
    for (op, dst, a, bb) in prog:
        if op == A.OP_LOADM:
            b[dst] = mval[a]
        elif op == A.OP_CONSTB:
            b[dst] = np.full(n, a, np.int64)
        elif op == A.OP_ADDB:
            b[dst] = (b[a] + b[bb]) % P
        elif op == A.OP_SUBB:
            b[dst] = (b[a] - b[bb]) % P
        elif op == A.OP_MULB:
            b[dst] = (b[a] * b[bb]) % P
        elif op == A.OP_NEGB:
            b[dst] = (-b[a]) % P
        elif op == A.OP_PARAME:
            e[dst] = tuple(np.full(n, v, np.int64) for v in prm[a])
        elif op == A.OP_ADDE:
            e[dst] = tuple((x + y) % P for x, y in zip(e[a], e[bb]))
        elif op == A.OP_SUBE:
            e[dst] = tuple((x - y) % P for x, y in zip(e[a], e[bb]))
        elif op == A.OP_MULE:
            e[dst] = _qmul(e[a], e[bb])
        elif op == A.OP_NEGE:
            e[dst] = tuple((-x) % P for x in e[a])
        elif op == A.OP_ADDEB:
            e[dst] = ((e[a][0] + b[bb]) % P,) + e[a][1:]
        elif op == A.OP_SUBEB:
            e[dst] = ((e[a][0] - b[bb]) % P,) + e[a][1:]
        elif op == A.OP_MULEB:
            e[dst] = tuple((x * b[bb]) % P for x in e[a])
        elif op == A.OP_BTOE:
            e[dst] = (b[a], zero, zero, zero)
        elif op == A.OP_LOADME:
            e[dst] = tuple(mval[a + j] % P for j in range(4))
        elif op in (A.OP_CONSTRB, A.OP_CONSTRE):
            v = (b[a] % P) if op == A.OP_CONSTRB else (e[a][0] % P) | (e[a][1] % P) | (e[a][2] % P) | (e[a][3] % P)
            bad = np.flatnonzero(v != 0)
            out.append((int(bad.size), int(bad[0]) if bad.size else None))
        else:
            raise ValueError(f"opcode {op}")
    return out
