"""A Nexus-shaped synthetic machine driven through the drop-in boundary.

The reference's `Machine::<C>::prove_with_extensions` (nexus-zkvm prover/src/machine.rs:130-297) fills the trace
with Rust chips and then drives Stwo: channel prefix -> tree 0 (preprocessed) -> tree 1 (main) -> draw lookup
elements -> interaction trace -> mix claimed sums -> tree 2 -> stwo::prover::prove.  The chips themselves cannot be
executed here (Rust, no toolchain), so this module provides a machine of the same *shape* that exercises every part
of the backend surface: a wide ADD chip (byte limbs + carries, the core of prover/src/chips/instructions/i/add.rs:98-139),
a next-row constraint on a program counter (mask offset +1, like `Pc`, prover/src/column.rs:17-19), boolean-ity
constraints (range_bool.rs), one LogUp fraction per range-checked byte with one secure column per fraction
(`finalize_logup`, components/mod.rs:52-54), and a second, small component (a 2^8 multiplicity table with a
preprocessed column addressed by id, like prover/src/extensions/multiplicity.rs) so that trees hold mixed-size columns.
With 21 lanes the column counts are 3 / 339 / 1012 — the reference's 27 / 347 / 1012 (SURVEY.md §8).

`prove(backend, ...)` is written against a small backend protocol (channel / prover.commit / gen_interaction /
commit_interaction / prove); the product backend is nexus_zkvm_b200.prover.CudaBackend, and the parity tests plug
their CPU checker into the same driver.
"""
import numpy as np

from . import air as A
from . import field as F

P = (1 << 31) - 1


class AddMachine:
    def __init__(self, log_size, n_lanes=1, log_expand=2, logup_in_pairs=False):
        """logup_in_pairs: batch the fractions two per secure column (`finalize_logup_in_pairs`, the prover2 style —
        nexus-zkvm prover2/machine/src/lookups/logup_trace_builder.rs:88-101) instead of one per column (v1)."""
        assert log_size >= 8
        self.log_size, self.n_lanes, self.log_expand = log_size, n_lanes, log_expand
        air = A.Air()
        self.range256 = air.relation("Range256", 1)
        main = air.component(log_size, log_expand)
        is_first = main.get_preprocessed_column("IsFirst")
        is_last = main.get_preprocessed_column("IsLast")
        # main trace (tree 1), column order = declaration order (trace/eval.rs:31-44)
        pc = main.next_interaction_mask(A.ORIGINAL_TRACE_IDX, [0, 1])  # like Column::Pc: [cur, next]
        is_pad = main.next_trace_mask()
        lanes = []
        for _ in range(n_lanes):
            a = [main.next_trace_mask() for _ in range(4)]
            b = [main.next_trace_mask() for _ in range(4)]
            c = [main.next_trace_mask() for _ in range(4)]
            carry = [main.next_trace_mask() for _ in range(4)]
            lanes.append((a, b, c, carry))
        # constraints
        main.add_constraint(is_pad * (1 - is_pad))
        main.add_constraint(is_first * pc[0])                          # pc starts at 0
        main.add_constraint((1 - is_last) * (pc[1] - pc[0] - 4))       # pc advances by WORD_SIZE
        for (a, b, c, carry) in lanes:
            for i in range(4):
                main.add_constraint((1 - is_pad) * carry[i] * (1 - carry[i]))
                prev = carry[i - 1] if i else 0
                main.add_constraint((1 - is_pad) * (a[i] + b[i] + prev - c[i] - carry[i] * 256))
        for (a, b, c, carry) in lanes:
            for x in a + b + c:
                main.add_to_relation(self.range256, 1, [x])
        if logup_in_pairs:
            main.finalize_logup_in_pairs()
        else:
            main.finalize_logup()
        table = air.component(8, 1)
        val = table.get_preprocessed_column("Range256Values")
        mult = table.next_trace_mask()
        table.add_to_relation(self.range256, -mult, [val])
        table.finalize_logup()
        self.air = air
        self.main, self.table = main, table
        self.words = air.serialize()

    # ---- trace filling (host side; trace/coset order, finalized by the backend on upload)
    def preprocessed_columns(self):
        n = 1 << self.log_size
        cols = [None] * self.air.n_columns()[0]
        is_first = np.zeros(n, np.uint32); is_first[0] = 1
        is_last = np.zeros(n, np.uint32); is_last[n - 1] = 1
        cols[self.air.preprocessed_ids["IsFirst"]] = is_first
        cols[self.air.preprocessed_ids["IsLast"]] = is_last
        cols[self.air.preprocessed_ids["Range256Values"]] = np.arange(256, dtype=np.uint32)
        return cols

    def n_main_columns(self):
        """Columns of the main component in tree 1 (the multiplicity column of the table component comes after them)."""
        return 2 + 16 * self.n_lanes

    def fill_main_trace(self, seed=0, n_padding=0, out=None, packed_out=None):
        """ADD chain: every lane adds two pseudo-random 32-bit words per row.  With `out` (an (n_main_columns, 2^log_size)
        uint32 array, e.g. pinned memory from Context.host_alloc) the columns are written in place and `out` is returned.
        With `packed_out` = (pc_block: (1, n) uint32, byte_block: (n_main_columns - 1, n) uint8) the trace is written in the
        packed host format (nb200_scheme_commit_host_packed): every column but `pc` holds byte limbs / flags; the list
        [pc_block, byte_block] is returned (commitment order is unchanged: 2-D blocks are consecutive columns)."""
        n = 1 << self.log_size
        rng = np.random.default_rng(seed)

        class _Sink(list):
            def append(self_inner, col):
                k = len(self_inner)
                if packed_out is not None:
                    dst = packed_out[0][0] if k == 0 else packed_out[1][k - 1]
                    dst[:] = col
                    col = dst
                elif out is not None:
                    out[k] = col
                    col = out[k]
                list.append(self_inner, col)

            def __iadd__(self_inner, more):
                for c in more:
                    self_inner.append(c)
                return self_inner

        cols = _Sink()
        cols.append((4 * np.arange(n, dtype=np.uint64) % P).astype(np.uint32))  # pc
        pad = np.zeros(n, np.uint32)
        if n_padding:
            pad[n - n_padding:] = 1
        cols.append(pad)
        hist = np.zeros(256, np.int64)
        for _ in range(self.n_lanes):
            a = rng.integers(0, 1 << 32, n, dtype=np.uint64)
            b = rng.integers(0, 1 << 32, n, dtype=np.uint64)
            c = (a + b) & 0xFFFFFFFF
            al = [((a >> (8 * i)) & 0xFF).astype(np.uint32) for i in range(4)]
            bl = [((b >> (8 * i)) & 0xFF).astype(np.uint32) for i in range(4)]
            cl = [((c >> (8 * i)) & 0xFF).astype(np.uint32) for i in range(4)]
            carry, prev = [], np.zeros(n, np.uint32)
            for i in range(4):
                s = al[i] + bl[i] + prev
                prev = (s >> 8).astype(np.uint32)
                carry.append(prev)
            cols += al + bl + cl + carry
            for x in al + bl + cl:
                hist += np.bincount(x, minlength=256)
        assert len(cols) == self.air.n_columns()[1] - 1
        mult = (hist % P).astype(np.uint32)
        if packed_out is not None:
            return [packed_out[0], packed_out[1]], mult
        return (out if out is not None else list(cols)), mult

    def column_log_sizes(self):
        return self.air.column_log_sizes()


def prove(machine, backend, main_cols, mult, config=None, associated_data=b"", resident=None):
    """The Machine::prove sequence (machine.rs:130-297) over `backend`.  Returns (proof_bytes, claimed_sums, aux).
    `resident` = (tree0 device batches, tree1 device batches) commits evaluations that are already on the device (finalized
    order) instead of uploading `main_cols` — the HBM-resident variant bench.py's `value` times."""
    ch, prover, params, claimed, roots, log_sizes = _commit_trees(machine, backend, main_cols, mult, config, associated_data, resident)
    aux = {"channel_at_prove": ch.clone(), "params": params, "roots": roots, "log_sizes": log_sizes,
           "associated_data": bytes(associated_data)}
    proof = prover.prove(ch, params)
    return proof, claimed, aux


def check_constraints(machine, backend, main_cols, mult, associated_data=b"", resident=None):
    """assert_constraints_on_polys for every component (the reference's `assert_chip` / `assert_component`) on the GPU: the trees are committed
    as `prove` commits them, then each component's constraints are evaluated on every row of its trace domain.  Returns
    ({component: [(constraint, degree, failing rows, first failing row in trace order)]}, whether the claimed LogUp sums cancel).
    `resident` as in `prove`: trees 0 and 1 already on the device (e.g. a keccak trace filled there)."""
    _ch, prover, params, claimed, _roots, _ls = _commit_trees(machine, backend, main_cols, mult, None, associated_data, resident)
    report = {k: prover.check_constraints(k, params) for k in range(len(machine.air.components))}
    return report, verify_claimed_sums(claimed)


def fill_table_multiplicities(machine, ctx, tree0, tree1, air=None, first_row=False):
    """Overwrite the multiplicity columns of `tree1` (device batches, finalized order, before tree 1 is committed) with the counts of the
    machine's own lookups, on the GPU (nb200_table_multiplicities): what each machine's fill_main_trace counts on the host.  Raises
    Nb200Error naming the first lookup whose tuple is in no table row.  `air`: the machine's loaded AIR (prover.Air) on `ctx`; by default
    one is loaded on the first call per context and kept on the machine, so the count kernels are compiled or loaded once, not per call.
    `first_row`: a tuple that several table rows list is credited to the first of them (nb200_table_multiplicities_first_row), and the
    number of rows written as 0 is returned."""
    from . import Nb200Error
    from .prover import Air
    if air is None:
        cache = machine.__dict__.setdefault("_count_air", {})
        air = cache.get(id(ctx))
        if air is None or air.ctx is not ctx:
            air = cache[id(ctx)] = Air(ctx, machine.words)
    n, first, *repeated = ctx.table_multiplicities(air, list(tree0), list(tree1), first_row=first_row)
    if n:
        comp, frac, row = first
        raise Nb200Error(f"{n} lookup(s) match no table row; the first: component {comp}, fraction {frac}, trace row {row}")
    return repeated[0] if first_row else None


def _commit_trees(machine, backend, main_cols, mult, config, associated_data, resident):
    """Machine::prove up to and including the tree-2 commit: (channel, prover, params, claimed sums, roots, log sizes)."""
    config = config or dict(pow_bits=5, log_blowup=1, log_last=0, n_queries=3)
    air = machine.air
    ch = backend.channel()
    for byte in associated_data:                      # machine.rs:197-200
        ch.mix_u64(int(byte))
    log_sizes = list(getattr(machine, "log_sizes", None) or [machine.log_size, 8])
    for ls in log_sizes:                              # machine.rs:204-206
        ch.mix_u64(ls)
    prover = backend.prover(machine.words, config)
    # tree 0: preprocessed (machine.rs:208-228)
    if resident is not None:
        roots = [prover.commit_batches(list(resident[0]), ch), prover.commit_batches(list(resident[1]), ch)]
    else:
        roots = [prover.commit(machine.preprocessed_columns(), ch, coset_order=True)]
        # tree 1: main trace + extension main columns (machine.rs:230-237)
        main_part = [main_cols] if getattr(main_cols, "ndim", 1) == 2 else list(main_cols)  # a 2-D block or a list of columns / blocks
        roots.append(prover.commit(main_part + ([mult] if mult is not None else []), ch, coset_order=True))
    # lookup elements (machine.rs:239-240)
    params = [(0, 0, 0, 0)] * air.n_params
    for rel in (getattr(machine, "relations", None) or [machine.range256]):
        rel.draw(ch, params)
    # interaction trace per component (machine.rs:242-260); claimed sums mixed before the commit (machine.rs:262-263)
    inter, claimed = [], []
    for k, comp in enumerate(air.components):
        cols, cs = prover.gen_interaction(k, comp.log_size, max(comp.batching) + 1, params)
        inter.append(cols)
        claimed.append(cs)
        inv_n = F.m31_inv((1 << comp.log_size) % P)
        params[comp.cumsum_shift_param] = F.qm31_mul_m31(cs, inv_n)
    ch.mix_felts(claimed)
    roots.append(prover.commit_interaction(inter, ch))
    return ch, prover, params, claimed, roots, log_sizes


def shard_host_tree(machine, prover, host_cols, rank, world, coset_order=True):
    """Upload this rank's part of one tree's host columns: (column shard of the leading 2^log_size-row batch or None, its total column count,
    replicated device batches of the smaller columns).  coset_order=False: the columns are already in finalized order (an interaction trace)."""
    from . import Context
    n, cols = machine.log_size, []
    for c_ in host_cols:
        a_ = np.asarray(c_)
        cols += list(a_) if a_.ndim == 2 else [a_]
    total_big = 0
    while total_big < len(cols) and len(cols[total_big]) == 1 << n:
        total_big += 1
    assert all(len(c_) < 1 << n for c_ in cols[total_big:]), "the sharded columns must be the leading, largest batch of the tree"
    first, count = Context.shard_range(total_big, world, rank)
    shard = prover.ctx.upload(np.stack([np.ascontiguousarray(c_, dtype=np.uint32) for c_ in cols[first:first + count]]), coset_order=coset_order) if count else None
    small = prover._batches_from_host(cols[total_big:], coset_order) if len(cols) > total_big else []
    return shard, total_big, small


def commit_sharded_tree(machine, prover, t, part, keep_eval_rows, ch):
    """Commit tree t of a sharded proof from `part` = (column shard or None, total sharded columns, replicated batches), as shard_host_tree returns
    it.  Every rank keeps a full copy of the sharded columns that the main component reads at a row offset."""
    shard, total_big, small = part
    replicate = sorted({c for (tt, c, off) in machine.air.components[0].masks if tt == t and off != 0 and c < total_big})
    return prover.commit_sharded(shard, total_big, machine.log_size, small, replicate, keep_eval_rows, ch)


def interaction_traces_sharded(machine, prover, parts, params):
    """The interaction traces of a sharded proof, trees 0 and 1 committed from `parts` (their shard_host_tree results) with keep_eval_rows: the
    main component's column shard, the other components' batches and every component's claimed sum.  Each cumsum shift is set in `params` as
    its trace is made."""
    air, ctx, n = machine.air, prover.ctx, machine.log_size
    # the replicated components read trees 0 and 1 as batch lists in commitment order: a placeholder batch stands for the sharded columns they never read
    ph = [shard for shard, _total, _small in parts if shard is not None][0]
    t0_list, t1_list = ([ctx.wrap_device(ph.device_ptr, total, 0)] + small for _shard, total, small in parts)
    shard2, cs = prover.gen_interaction_sharded(0, params)
    inter_small, claimed = [], [cs]
    params[air.components[0].cumsum_shift_param] = F.qm31_mul_m31(cs, F.m31_inv((1 << n) % P))
    for k_, comp in enumerate(air.components[1:], start=1):
        cols_k, cs = prover.gen_interaction_replicated(k_, comp.log_size, max(comp.batching) + 1, params, t0_list, t1_list)
        inter_small.append(cols_k)
        claimed.append(cs)
        params[comp.cumsum_shift_param] = F.qm31_mul_m31(cs, F.m31_inv((1 << comp.log_size) % P))
    return shard2, inter_small, claimed


def _commit_trees_sharded(machine, backend, main_cols, mult, rank, world, config, associated_data, resident):
    """prove_sharded up to and including the tree-2 commit: (channel, prover, params, claimed sums, roots)."""
    config = config or dict(pow_bits=5, log_blowup=1, log_last=0, n_queries=3)
    air = machine.air
    ch = backend.channel()
    for byte in associated_data:
        ch.mix_u64(int(byte))
    for ls in (getattr(machine, "log_sizes", None) or [machine.log_size, 8]):
        ch.mix_u64(ls)
    prover = backend.prover(machine.words, config)
    parts, roots = [], []
    for t in (0, 1):
        if resident is not None:
            parts.append(resident[t])
        elif t == 0:
            parts.append(shard_host_tree(machine, prover, machine.preprocessed_columns(), rank, world))
        else:
            main_part = [main_cols] if getattr(main_cols, "ndim", 1) == 2 else list(main_cols)
            parts.append(shard_host_tree(machine, prover, main_part + ([mult] if mult is not None else []), rank, world))
        roots.append(commit_sharded_tree(machine, prover, t, parts[t], True, ch))
    params = [(0, 0, 0, 0)] * air.n_params
    for rel in (getattr(machine, "relations", None) or [machine.range256]):
        rel.draw(ch, params)
    # interaction traces: the main component sharded, the others replicated
    shard2, inter_small, claimed = interaction_traces_sharded(machine, prover, parts, params)
    ch.mix_felts(claimed)
    big2 = 4 * (max(air.components[0].batching) + 1)
    roots.append(commit_sharded_tree(machine, prover, 2, (shard2 if shard2.n_cols else None, big2, inter_small), False, ch))
    return ch, prover, params, claimed, roots


def prove_sharded(machine, backend, main_cols, mult, rank, world, config=None, associated_data=b"", resident=None):
    """ONE proof by `world` GPUs (one process per GPU; `backend.ctx` holds an initialised communicator: Context.comm_init*).  Every rank calls this
    with the same arguments and gets the same proof bytes — the bytes `prove` returns on one GPU.  The Machine::prove order (machine.rs:197-290):
    the main component's columns (the first, largest batch of every tree) are column-sharded over the ranks for the transforms and row-sharded for
    hashing, constraint rows and DEEP quotients; the other components' small columns are replicated.  For the harness every rank is handed the full host
    trace and uploads only its nb200_shard_range of it (a real host would fill only that range); `resident` = the two shard_host_tree results of
    trees 0 and 1 when they are already on the device."""
    ch, prover, params, claimed, roots = _commit_trees_sharded(machine, backend, main_cols, mult, rank, world, config, associated_data, resident)
    log_sizes = list(getattr(machine, "log_sizes", None) or [machine.log_size, 8])
    aux = {"params": params, "roots": roots, "log_sizes": log_sizes, "associated_data": bytes(associated_data)}
    proof = prover.prove(ch, params)
    return proof, claimed, aux


class MultiMachine:
    """A prover2-shaped machine (SURVEY §8 row f4): MANY components of DISTINCT log sizes instead of one wide component — the
    reference's prover2 builds one component per opcode family, each with its own log size (nexus-zkvm
    prover2/machine/src/lib.rs:9-65) — with constraint degree bounds 1 and 2 mixed (`log_expand`), LogUp fractions batched in
    pairs where the degree bound allows (prover2/machine/src/lookups/logup_trace_builder.rs:88-101), two shared lookup relations
    and two table components with preprocessed columns addressed by id:
      * `Range256` (arity 1) against a 2^8-row table, like prover/src/extensions/multiplicity.rs;
      * `BitOp` (arity 3: a, b, a XOR b) against a 2^16-row preprocessed table — the shape of the v1 bit-op extension
        (prover/src/extensions/bit_op.rs) and of the keccak extension's XorTable / BitNotAndTable / BitRotateTable
        (prover/src/extensions/keccak/mod.rs:12-33: tuple lookups into preprocessed truth tables).
    Component kinds alternate: `add` (byte-limb ADD with carries, range-checked through Range256; degree 2, fractions one per
    column) and `xor` (a XOR b = c proven by a BitOp lookup per byte, Range256 on nothing; degree bound 3, fractions in pairs).
    Every tree therefore holds columns of len(log_sizes) + 2 different sizes, and FRI's first layer has as many column sizes."""

    def __init__(self, log_sizes, lanes=1):
        assert all(4 <= ls <= 24 for ls in log_sizes)
        self.comp_log_sizes, self.lanes = list(log_sizes), lanes
        air = A.Air()
        self.range256 = air.relation("Range256", 1)
        self.bitop = air.relation("BitOp", 3)
        self.relations = [self.range256, self.bitop]
        self.kinds = []
        for i, ls in enumerate(log_sizes):
            kind = "add" if i % 2 == 0 else "xor"
            self.kinds.append(kind)
            c = air.component(ls, 1 if kind == "add" else 2)
            for _ in range(lanes):
                a = [c.next_trace_mask() for _ in range(4)]
                b = [c.next_trace_mask() for _ in range(4)]
                r = [c.next_trace_mask() for _ in range(4)]
                if kind == "add":
                    carry = [c.next_trace_mask() for _ in range(4)]
                    for k in range(4):
                        c.add_constraint(carry[k] * (1 - carry[k]))
                        prev = carry[k - 1] if k else 0
                        c.add_constraint(a[k] + b[k] + prev - r[k] - carry[k] * 256)
                    for x in a + b + r:
                        c.add_to_relation(self.range256, 1, [x])
                else:
                    for k in range(4):
                        c.add_to_relation(self.bitop, 1, [a[k], b[k], r[k]])
            if kind == "add":
                c.finalize_logup()
            else:
                c.finalize_logup_in_pairs()
        t8 = air.component(8, 1)
        v8 = t8.get_preprocessed_column("Range256Values")
        m8 = t8.next_trace_mask()
        t8.add_to_relation(self.range256, -m8, [v8])
        t8.finalize_logup()
        t16 = air.component(16, 1)
        ta, tb, tc = (t16.get_preprocessed_column(n) for n in ("BitOpA", "BitOpB", "BitOpXor"))
        m16 = t16.next_trace_mask()
        t16.add_to_relation(self.bitop, -m16, [ta, tb, tc])
        t16.finalize_logup()
        self.air = air
        self.log_sizes = list(log_sizes) + [8, 16]
        self.log_size = max(self.log_sizes)
        self.words = air.serialize()

    def preprocessed_columns(self):
        cols = [None] * self.air.n_columns()[0]
        i = np.arange(1 << 16, dtype=np.uint32)
        cols[self.air.preprocessed_ids["Range256Values"]] = np.arange(256, dtype=np.uint32)
        cols[self.air.preprocessed_ids["BitOpA"]] = i >> 8
        cols[self.air.preprocessed_ids["BitOpB"]] = i & 0xFF
        cols[self.air.preprocessed_ids["BitOpXor"]] = (i >> 8) ^ (i & 0xFF)
        return cols

    def fill_main_trace(self, seed=0):
        """Returns the list of main-trace columns in commitment order (component by component, the two multiplicity columns last)."""
        rng = np.random.default_rng(seed)
        cols = []
        h8, h16 = np.zeros(256, np.int64), np.zeros(1 << 16, np.int64)
        for ls, kind in zip(self.comp_log_sizes, self.kinds):
            n = 1 << ls
            for _ in range(self.lanes):
                a = rng.integers(0, 1 << 32, n, dtype=np.uint64)
                b = rng.integers(0, 1 << 32, n, dtype=np.uint64)
                al = [((a >> (8 * k)) & 0xFF).astype(np.uint32) for k in range(4)]
                bl = [((b >> (8 * k)) & 0xFF).astype(np.uint32) for k in range(4)]
                if kind == "add":
                    c = (a + b) & 0xFFFFFFFF
                    cl = [((c >> (8 * k)) & 0xFF).astype(np.uint32) for k in range(4)]
                    carry, prev = [], np.zeros(n, np.uint32)
                    for k in range(4):
                        prev = ((al[k] + bl[k] + prev) >> 8).astype(np.uint32)
                        carry.append(prev)
                    cols += al + bl + cl + carry
                    for x in al + bl + cl:
                        h8 += np.bincount(x, minlength=256)
                else:
                    cl = [al[k] ^ bl[k] for k in range(4)]
                    cols += al + bl + cl
                    for k in range(4):
                        h16 += np.bincount((al[k] << 8) | bl[k], minlength=1 << 16)
        cols.append((h8 % P).astype(np.uint32))
        cols.append((h16 % P).astype(np.uint32))
        assert len(cols) == self.air.n_columns()[1]
        return cols

    def column_log_sizes(self):
        return self.air.column_log_sizes()


def verify_claimed_sums(claimed):
    """machine.rs:343-347: the logup sums of all components must cancel."""
    tot = (0, 0, 0, 0)
    for c in claimed:
        tot = F.qm31_add(tot, c)
    return tot == (0, 0, 0, 0)
