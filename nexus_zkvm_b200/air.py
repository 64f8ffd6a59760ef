"""AIR builder: the host-side mirror of stwo-constraint-framework's `EvalAtRow` / `FrameworkComponent` /
`relation!` / `TraceLocationAllocator`, emitting the SSA bytecode that `nb200_air_load` consumes.

In the reference every chip declares its constraints as Rust generic code over `EvalAtRow`
(nexus-zkvm prover/src/traits.rs:45-50, prover/src/components/mod.rs:39-57, prover/src/trace/eval.rs:22-50);
a GPU needs that as data.  The Rust shim (INTEGRATION.md) does it with a recording evaluator; this module is the
same recorder for the Python harness: same call names (`next_trace_mask`, `next_interaction_mask`,
`get_preprocessed_column`, `add_constraint`, `add_to_relation`, `finalize_logup[_in_pairs]`), same mask/column
allocation order, same logup constraint shapes.

Bytecode (little-endian u32 words):
  'NBAR', version=1, n_params, n_components, then per component:
    log_size, log_expand, n_constraints,
    n_masks, n_masks x (tree, column index inside the tree, signed row offset),
    n_base_regs, n_ext_regs, n_instr, n_instr x (op, dst, a, b),              -- constraint program
    n_fracs, lg_base_regs, lg_ext_regs, n_lg_instr, n_lg_instr x (op,dst,a,b), -- logup trace program (OP_FRAC num, den)
    n_fracs x batch id, cumsum_shift_param, first interaction column
"""
import numpy as np

P = (1 << 31) - 1
PREPROCESSED_TRACE_IDX, ORIGINAL_TRACE_IDX, INTERACTION_TRACE_IDX = 0, 1, 2

(OP_LOADM, OP_CONSTB, OP_ADDB, OP_SUBB, OP_MULB, OP_NEGB, OP_PARAME, _, OP_ADDE, OP_SUBE, OP_MULE, OP_NEGE,
 OP_ADDEB, OP_SUBEB, OP_MULEB, OP_BTOE, OP_LOADME, OP_CONSTRB, OP_CONSTRE, OP_FRAC) = range(20)
NO_PARAM = 0xFFFFFFFF


class Expr:
    """A value of the row evaluation: kind 'B' (base field) or 'E' (secure field)."""
    __slots__ = ("c", "id", "kind")

    def __init__(self, comp, nid, kind):
        self.c, self.id, self.kind = comp, nid, kind

    def _lift(self, o):
        if isinstance(o, Expr):
            return o
        return self.c.const(int(o))

    def __add__(self, o):
        return self.c._bin("add", self, self._lift(o))

    __radd__ = __add__

    def __sub__(self, o):
        return self.c._bin("sub", self, self._lift(o))

    def __rsub__(self, o):
        return self.c._bin("sub", self._lift(o), self)

    def __mul__(self, o):
        return self.c._bin("mul", self, self._lift(o))

    __rmul__ = __mul__

    def __neg__(self):
        return self.c._neg(self)


class Relation:
    """`relation!(Name, N)`: lookup elements z, alpha^0..alpha^(N-1) living in the proof-wide parameter table."""

    def __init__(self, air, name, size):
        self.name, self.size = name, size
        self.z = air.alloc_param(f"{name}.z")
        self.alpha_powers = [air.alloc_param(f"{name}.alpha^{i}") for i in range(size)]

    def draw(self, channel, params):
        """LookupElements::draw: [z, alpha] = channel.draw_felts(2)."""
        from . import field as F
        z, alpha = [tuple(int(x) for x in q) for q in channel.draw_felts(2)]
        params[self.z] = z
        cur = (1, 0, 0, 0)
        for i in range(self.size):
            params[self.alpha_powers[i]] = cur
            cur = F.qm31_mul(cur, alpha)


class Air:
    def __init__(self):
        self.param_names = []
        self.components = []
        self.next_col = [0, 0, 0]           # TraceLocationAllocator: next free column per tree
        self.preprocessed_ids = {}           # PreProcessedColumnId -> column index in tree 0

    def alloc_param(self, name):
        self.param_names.append(name)
        return len(self.param_names) - 1

    @property
    def n_params(self):
        return len(self.param_names)

    def relation(self, name, size):
        return Relation(self, name, size)

    def preprocessed_column(self, col_id):
        if col_id not in self.preprocessed_ids:
            self.preprocessed_ids[col_id] = self.next_col[0]
            self.next_col[0] += 1
        return self.preprocessed_ids[col_id]

    def component(self, log_size, log_expand=1):
        c = ComponentBuilder(self, log_size, log_expand)
        self.components.append(c)
        return c

    def n_columns(self):
        return list(self.next_col)

    def column_log_sizes(self):
        """log size of every column per tree (commitment order)."""
        out = [[None] * n for n in self.next_col]
        for c in self.components:
            for (t, col, _o) in c.masks:
                out[t][col] = c.log_size
        for t in range(3):
            assert all(v is not None for v in out[t]), f"tree {t} has unreferenced columns"
        return out

    def serialize(self):
        w = [0x5241424E, 1, self.n_params, len(self.components)]
        for c in self.components:
            w += c._serialize()
        return np.array(w, dtype=np.uint32)


class ComponentBuilder:
    def __init__(self, air, log_size, log_expand):
        self.air, self.log_size, self.log_expand = air, log_size, log_expand
        self.nodes = []       # (op, a, b, kind)  with op in {"mask","maske","const","param","add","sub","mul","neg","btoe"}
        self.masks = []       # (tree, col, offset)
        self.mask_slot = {}
        self.constraints = []  # node ids
        self.fracs = []        # (num node id (E), den node id (E))
        self.lookups = []      # per fraction: (relation, numerator Expr, values: Exprs or ints) — kept on the Python side only (not serialized)
        self.batching = None
        self.cumsum_shift_param = NO_PARAM
        self.interaction_col0 = None
        self._cse = {}

    # -- nodes
    def _node(self, op, a, b, kind):
        key = (op, a, b, kind)
        if key in self._cse:
            return Expr(self, self._cse[key], kind)
        self.nodes.append(key)
        self._cse[key] = len(self.nodes) - 1
        return Expr(self, len(self.nodes) - 1, kind)

    def const(self, v):
        return self._node("const", v % P, 0, "B")

    def param(self, idx):
        return self._node("param", idx, 0, "E")

    def _to_e(self, x):
        return x if x.kind == "E" else self._node("btoe", x.id, 0, "E")

    def _bin(self, op, x, y):
        if x.kind == "B" and y.kind == "B":
            return self._node(op, x.id, y.id, "B")
        if x.kind == "E" and y.kind == "E":
            return self._node(op, x.id, y.id, "E")
        if x.kind == "E":  # E op B
            return self._node(op + "_eb", x.id, y.id, "E")
        # B op E
        if op == "sub":
            return self._node("sub", self._to_e(x).id, y.id, "E")
        return self._node(op + "_eb", y.id, x.id, "E")

    def _neg(self, x):
        return self._node("neg", x.id, 0, x.kind)

    # -- EvalAtRow surface
    def _slot(self, tree, col, off):
        k = (tree, col, off)
        if k not in self.mask_slot:
            self.mask_slot[k] = len(self.masks)
            self.masks.append(k)
        return self.mask_slot[k]

    def get_preprocessed_column(self, col_id):
        col = self.air.preprocessed_column(col_id)
        return self._node("mask", self._slot(0, col, 0), 0, "B")

    def next_interaction_mask(self, tree, offsets):
        col = self.air.next_col[tree]
        self.air.next_col[tree] += 1
        if tree == INTERACTION_TRACE_IDX and self.interaction_col0 is None:
            self.interaction_col0 = col
        return [self._node("mask", self._slot(tree, col, o), 0, "B") for o in offsets]

    def next_trace_mask(self):
        return self.next_interaction_mask(ORIGINAL_TRACE_IDX, [0])[0]

    def next_extension_interaction_mask(self, tree, offsets):
        cols = []
        for _ in range(4):
            cols.append(self.air.next_col[tree])
            self.air.next_col[tree] += 1
        if tree == INTERACTION_TRACE_IDX and self.interaction_col0 is None:
            self.interaction_col0 = cols[0]
        out = []
        for o in offsets:
            slots = [self._slot(tree, c, o) for c in cols]
            # the 4 coordinate slots of one offset must be consecutive for OP_LOADME
            assert slots == list(range(slots[0], slots[0] + 4)), "extension mask slots must be contiguous"
            out.append(self._node("maske", slots[0], 0, "E"))
        return out

    def add_constraint(self, e):
        if not isinstance(e, Expr):
            e = self.const(e)
        self.constraints.append(e.id)

    def combine(self, relation, values):
        """Relation::combine: sum_i alpha^i * v_i - z."""
        acc = None
        for i, v in enumerate(values):
            if not isinstance(v, Expr):
                v = self.const(v)
            term = self.param(relation.alpha_powers[i]) * v
            acc = term if acc is None else acc + term
        return acc - self.param(relation.z)

    def add_to_relation(self, relation, multiplicity, values):
        assert len(values) <= relation.size
        if not isinstance(multiplicity, Expr):
            multiplicity = self.const(multiplicity)
        self.lookups.append((relation, multiplicity, list(values)))
        self.fracs.append((self._to_e(multiplicity).id, self.combine(relation, values).id))

    def _frac_sum(self, ids):
        num, den = Expr(self, self.fracs[ids[0]][0], "E"), Expr(self, self.fracs[ids[0]][1], "E")
        for k in ids[1:]:
            n2, d2 = Expr(self, self.fracs[k][0], "E"), Expr(self, self.fracs[k][1], "E")
            num, den = d2 * num + den * n2, den * d2
        return num, den

    def finalize_logup_batched(self, batching):
        assert self.batching is None and len(batching) == len(self.fracs) and self.fracs
        self.batching = list(batching)
        last = max(batching)
        assert set(batching) == set(range(last + 1))
        self.cumsum_shift_param = self.air.alloc_param(f"component{len(self.air.components) - 1}.cumsum_shift")
        prev_col = None
        for b in range(last):
            num, den = self._frac_sum([k for k, x in enumerate(batching) if x == b])
            (cur,) = self.next_extension_interaction_mask(INTERACTION_TRACE_IDX, [0])
            diff = cur if prev_col is None else cur - prev_col
            prev_col = cur
            self.add_constraint(diff * den - num)
        num, den = self._frac_sum([k for k, x in enumerate(batching) if x == last])
        prev_row, cur = self.next_extension_interaction_mask(INTERACTION_TRACE_IDX, [-1, 0])
        diff = cur - prev_row
        if prev_col is not None:
            diff = diff - prev_col
        fixed = diff + self.param(self.cumsum_shift_param)
        self.add_constraint(fixed * den - num)

    def finalize_logup(self):
        self.finalize_logup_batched(list(range(len(self.fracs))))

    def finalize_logup_in_pairs(self):
        self.finalize_logup_batched([k // 2 for k in range(len(self.fracs))])

    # -- code generation
    _OPS = {("add", "B"): OP_ADDB, ("sub", "B"): OP_SUBB, ("mul", "B"): OP_MULB, ("neg", "B"): OP_NEGB,
            ("add", "E"): OP_ADDE, ("sub", "E"): OP_SUBE, ("mul", "E"): OP_MULE, ("neg", "E"): OP_NEGE,
            ("add_eb", "E"): OP_ADDEB, ("sub_eb", "E"): OP_SUBEB, ("mul_eb", "E"): OP_MULEB}

    _BIN = ("add", "sub", "mul", "add_eb", "sub_eb", "mul_eb")

    def _operands(self, n):
        op, a, b, _k = self.nodes[n]
        if op in self._BIN:
            return [a, b]
        if op in ("neg", "btoe"):
            return [a]
        return []

    def _emit(self, sinks):
        """Emit code for `sinks` = [(sink_op, node, node|None)] in declaration order: before each sink, the not yet
        computed part of its expression DAG (post-order), then the sink itself.  Leaves (mask loads, constants,
        parameters) are rematerialised per sink instead of being kept alive — a reload is one instruction, a long live
        range is a virtual register held for thousands of instructions (the interpreter keeps registers in shared
        memory, so the register count sets the occupancy).  Registers are reused as soon as an instance's last
        consumer has been emitted (the interpreters read all operands before writing the result)."""
        LEAVES = ("mask", "maske", "const", "param")
        seq = []          # ("n", node) | ("s", sink index)
        done = set()
        for idx, s in enumerate(sinks):
            fresh = set()  # leaves already emitted for this sink
            for root in s[1:]:
                if root is None or root in done or root in fresh:
                    continue
                stack = [(root, False)]
                while stack:
                    n, expanded = stack.pop()
                    if n in done or n in fresh:
                        continue
                    if expanded:
                        (fresh if self.nodes[n][0] in LEAVES else done).add(n)
                        seq.append(("n", n))
                        continue
                    stack.append((n, True))
                    for x in reversed(self._operands(n)):
                        if x not in done and x not in fresh:
                            stack.append((x, False))
            seq.append(("s", idx))
        # a shared non-leaf value computed under an earlier sink may read a leaf that is re-emitted later: that is fine,
        # each emission is its own instance.  Instance liveness: backward scan.
        last = {}          # node -> position of the last use of the instance currently being scanned
        inst_last = {}     # definition position -> last use position (or None)
        for pos in range(len(seq) - 1, -1, -1):
            kind, v = seq[pos]
            if kind == "n":
                inst_last[pos] = last.pop(v, None)
                for x in self._operands(v):
                    last.setdefault(x, pos)
            else:
                for x in sinks[v][1:]:
                    if x is not None:
                        last.setdefault(x, pos)
        free_at = {}
        for dpos, lpos in inst_last.items():
            if lpos is not None:
                free_at.setdefault(lpos, []).append(dpos)
        reg, reg_of_def, out = {}, {}, []
        free = {"B": [], "E": []}
        nreg = {"B": 0, "E": 0}
        for pos, (kind, v) in enumerate(seq):
            if kind == "s":
                sop, n1, n2 = sinks[v]
                out.append((sop, 0, reg[n1], reg[n2] if n2 is not None else 0))
            else:
                op, a, b, k = self.nodes[v]
                ops = self._operands(v)
                ra = reg[a] if ops else None
                rb = reg[b] if len(ops) == 2 else None
            # release every instance whose last use is this position (operands are read before the result is written)
            for dpos in free_at.get(pos, []):
                free[self.nodes[seq[dpos][1]][3]].append(reg_of_def[dpos])
            if kind == "s":
                continue
            if free[k]:
                r = free[k].pop()
            else:
                r = nreg[k]
                nreg[k] += 1
            reg[v] = r
            reg_of_def[pos] = r
            if op == "mask":
                out.append((OP_LOADM, r, a, 0))
            elif op == "maske":
                out.append((OP_LOADME, r, a, 0))
            elif op == "const":
                out.append((OP_CONSTB, r, a, 0))
            elif op == "param":
                out.append((OP_PARAME, r, a, 0))
            elif op == "btoe":
                out.append((OP_BTOE, r, ra, 0))
            elif op == "neg":
                out.append((self._OPS[("neg", k)], r, ra, 0))
            else:
                out.append((self._OPS[(op, k)], r, ra, rb))
            if inst_last[pos] is None:
                free[k].append(r)
        return out, nreg["B"], nreg["E"]

    def _serialize(self):
        if self.fracs and self.batching is None:
            raise ValueError("logup fractions were added but finalize_logup was not called")
        sinks = [((OP_CONSTRB if self.nodes[n][3] == "B" else OP_CONSTRE), n, None) for n in self.constraints]
        prog, nb, ne = self._emit(sinks)
        lprog, lb, le = self._emit([(OP_FRAC, n, d) for (n, d) in self.fracs]) if self.fracs else ([], 0, 0)
        w = [self.log_size, self.log_expand, len(self.constraints), len(self.masks)]
        for (t, c, o) in self.masks:
            w += [t, c, o & 0xFFFFFFFF]
        w += [nb, ne, len(prog)]
        for ins in prog:
            w += list(ins)
        w += [len(self.fracs), lb, le, len(lprog)]
        for ins in lprog:
            w += list(ins)
        w += list(self.batching or [])
        w += [self.cumsum_shift_param, self.interaction_col0 if self.interaction_col0 is not None else 0]
        return w
