"""A numpy restatement of the table multiplicities (nb200_table_multiplicities) from what air.py records per fraction
(ComponentBuilder.lookups: relation, numerator, values), independent of the bytecode and of csrc/air.h's parser.

A table fraction has the numerator -m for one tree-1 mask m and values that read tree 0 and constants only; a lookup is any other fraction
into a relation that has a table fraction.  A table row's multiplicity is the sum of the numerators of the lookups whose values equal the
row's, over every row of every component; a lookup with a nonzero numerator whose values are in no table row is unmatched."""
import numpy as np

from nexus_zkvm_b200.air import Expr

P = (1 << 31) - 1


def flat(cols):
    """1-D columns and 2-D blocks (commitment order) -> a list of 1-D uint32 columns."""
    out = []
    for c in cols:
        a = np.asarray(c)
        out += [np.asarray(r, dtype=np.uint32) for r in a] if a.ndim == 2 else [a.astype(np.uint32)]
    return out


def _leaves(comp, e, seen=None):
    """{(tree, col, off)} of the masks a base expression reads."""
    if not isinstance(e, Expr):
        return set()
    op, a, b, _k = comp.nodes[e.id]
    if op == "mask":
        return {comp.masks[a]}
    out = set()
    for x in comp._operands(e.id):
        out |= _leaves(comp, Expr(comp, x, comp.nodes[x][3]))
    return out


def _table_mask(comp, num):
    """The tree-1 mask (tree, col, off) when num = -mask, else None."""
    op, a, _b, _k = comp.nodes[num.id]
    if op != "neg":
        return None
    op2, a2, _b2, _k2 = comp.nodes[a]
    if op2 != "mask" or comp.masks[a2][0] != 1:
        return None
    return comp.masks[a2]


def classify(air):
    """Per component, per fraction: ("table", relation, tree-1 column) | ("lookup", relation, tuple length) | ("ignored", relation, None)."""
    kinds = []
    for comp in air.components:
        row = []
        for rel, num, vals in comp.lookups:
            tm = _table_mask(comp, num)
            if tm is not None and all(t == 0 for v in vals for (t, _c, _o) in _leaves(comp, v)):
                row.append(("table", rel, tm[1]))
            else:
                row.append(("other", rel, len(vals)))
        kinds.append(row)
    tables = {id(rel) for row in kinds for (k, rel, _x) in row if k == "table"}
    return [[(k if k == "table" else ("lookup" if id(rel) in tables else "ignored"), rel, x) for (k, rel, x) in row] for row in kinds]


def evaluate(comp, e, trees):
    """A base expression on every row of the component (trace order); trees[t][col] = trace-order columns."""
    n = 1 << comp.log_size
    if not isinstance(e, Expr):
        return np.full(n, int(e) % P, np.int64)
    op, a, b, _k = comp.nodes[e.id]
    ev = lambda x: evaluate(comp, Expr(comp, x, comp.nodes[x][3]), trees)
    if op == "mask":
        t, col, off = comp.masks[a]
        assert off == 0
        return np.asarray(trees[t][col], dtype=np.int64) % P
    if op == "const":
        return np.full(n, a % P, np.int64)
    if op == "add":
        return (ev(a) + ev(b)) % P
    if op == "sub":
        return (ev(a) - ev(b)) % P
    if op == "mul":
        return (ev(a) * ev(b)) % P
    if op == "neg":
        return (-ev(a)) % P
    raise ValueError(op)


def _rows_key(a):
    a = np.ascontiguousarray(a, dtype=np.int64)
    return a.view(np.dtype((np.void, a.dtype.itemsize * a.shape[1]))).ravel()


def multiplicities(air, tree0, tree1):
    """({tree-1 column of a table fraction: multiplicities mod P, trace order}, n_unmatched, first unmatched (component, fraction, row) or None).
    tree0 / tree1: the host columns in trace order (1-D columns and 2-D blocks, commitment order)."""
    trees = [flat(tree0), flat(tree1)]
    kinds = classify(air)
    tables = {}   # id(relation) -> [(values (rows, len), column)]
    for k, comp in enumerate(air.components):
        for i, (kind, rel, col) in enumerate(kinds[k]):
            if kind == "table":
                vals = np.stack([evaluate(comp, v, trees) for v in comp.lookups[i][2]], axis=1)
                tables.setdefault(id(rel), []).append((vals, col))
    out = {col: np.zeros(len(v), np.int64) for ts in tables.values() for (v, col) in ts}
    n_unmatched, first = 0, None
    for k, comp in enumerate(air.components):
        for i, (kind, rel, _x) in enumerate(kinds[k]):
            if kind != "lookup":
                continue
            _rel, num, vals = comp.lookups[i]
            nv = evaluate(comp, num, trees)
            lv = np.stack([evaluate(comp, v, trees) for v in vals], axis=1)
            matched = np.zeros(len(nv), bool)
            for tv, col in tables[id(rel)]:
                if tv.shape[1] != lv.shape[1]:
                    continue
                tk, lk = _rows_key(tv), _rows_key(lv)
                order = np.argsort(tk)
                pos = np.searchsorted(tk[order], lk)
                pos = np.minimum(pos, len(tk) - 1)
                hit = tk[order][pos] == lk
                rows = order[pos[hit]]
                np.add.at(out[col], rows, nv[hit])
                matched |= hit
            bad = np.nonzero(~matched & (nv != 0))[0]
            if len(bad):
                n_unmatched += len(bad)
                if first is None:
                    first = (k, i, int(bad[0]))
    return {c: (v % P).astype(np.uint32) for c, v in out.items()}, n_unmatched, first
