"""The v1 main component, its eight base extensions and the keccak precompile extension proven as one machine: the shape of the reference's
`Machine::prove_with_extensions(keccak_extensions())` (nexus-zkvm prover/src/machine.rs:130-297), whose LogUp sums cancel.

Components, in the reference's order (the main component, BASE_EXTENSIONS of machine.rs:82-91, then keccak_extensions(), extensions/keccak/mod.rs:12-33):
   0 main component              nexus_v1.record_main_component, with KeccakChip's constraint (chips/custom.rs:178-196)
   1 FinalReg                    extensions/final_reg.rs:80-116          2^5 rows
   2 BitOpMultiplicity           extensions/bit_op.rs:55-93              2^8 rows
   3 RamInitFinal                extensions/ram_init_final.rs:54-249     max(log2ceil(#addresses), 4) (compute_log_size, :339-343)
   4 Multiplicity8               extensions/multiplicity8.rs:64-88       2^4 rows
   5-8 Multiplicity16/32/128/256 extensions/multiplicity.rs:103-125      2^4, 2^5, 2^7, 2^8 rows
   9-14 the keccak extension     keccak.py (memory check, KeccakRound 0 and 1, XorTable, BitNotAndTable, BitRotateTable)
Relations are drawn in `C::draw_lookup_elements` order over BaseComponent (machine.rs:49-79): BitOpChip, LoadStoreChip, then KeccakChip in
CustomInstructionChip (chips/custom.rs:127-139: Xor, BitNotAnd, State, BitRotate), ProgramMemCheckChip, RegisterMemCheckChip and the range
checks (8, 16, 32, 128, 256).

Witness.  The main component keeps NexusV1Machine's padding-only rows (no register, RAM or bit-op lookup; IsCustomKeccak = 0).  The keccak
side note comes from a byte-memory simulation: K buffers of 200 bytes (some overlapping at offsets that are not multiples of 8, some across
a 2^16 boundary), every touched byte a random initial value given as public initial memory in ascending address order, and permutation i
runs Keccak-f[1600] on buffer b_i: its input is the current memory, its previous timestamps the bytes' access counts, and its output is
written back.  RamInitFinal then holds one row per touched byte in ascending address order (the side note's `last_access` BTreeMap): its
init fractions add (address, initial value, 0), its final fractions subtract (address, final value, final counter), so the memory check's
LoadStore fractions cancel and the 15 claimed sums add up to zero (machine.rs:343-347).  Exit code and public output are empty.

Rows are filled in trace order as in the other machines here: the reference's extension columns are taken as they are, in bit-reversed
order (extensions/trace.rs:18-34 does not permute them), and a row of that order is a row of ours; the device fill writes row r at its
finalized position, as nb200_keccak_main_trace does.

Table multiplicities.  fill_main_trace counts them on the host, as the reference's side note does: Range256 also counts RamInitFinal's nine
lookups per row, whose numerator is 1 on padding rows too (ram_init_final.rs:219-248), and the keccak tables' columns come from the keccak
extension's host fill.  device_trees counts every table column on the device from the filled trace with
nb200_table_multiplicities_first_row: Multiplicity8's preprocessed column is 0..7 then eight zeros (multiplicity8.rs:48), so the Range8 table
lists the tuple (0) nine times; the first of those rows gets the count and the eight padding rows 0, as the reference's
`side_note.range8.multiplicity[checked] += 1` (chips/range_check/range8.rs:298, multiplicity8.rs:194-204) does.  The plain
nb200_table_multiplicities refuses this machine, as it refuses any relation that lists one tuple twice."""
import numpy as np

from . import air as A
from . import keccak as K
from . import nexus_v1 as V

P = (1 << 31) - 1
RAM_COLS = 10
RAM_PREPROCESSED = ["preprocessed_ram_init_final_addr0", "preprocessed_ram_init_final_addr1", "preprocessed_ram_init_final_addr2",
                    "preprocessed_ram_init_final_addr3", "preprocessed_ram_init_final_init_flag", "preprocessed_ram_init_final_init_value",
                    "preprocessed_ram_init_final_output_flag", "preprocessed_ram_init_final_output_value"]
BITOP_PREPROCESSED = ["preprocessed_bitwise_input_b", "preprocessed_bitwise_input_c", "preprocessed_bitwise_output_and",
                      "preprocessed_bitwise_output_or", "preprocessed_bitwise_output_xor"]
FINAL_REG_LOG_SIZE, BIT_OP_LOG_SIZE = 5, 8
# (relation, table length, log size) of Multiplicity8, 16, 32, 128, 256 in BASE_EXTENSIONS order
MULTIPLICITY_TABLES = [("Range8", 8, 4), ("Range16", 16, 4), ("Range32", 32, 5), ("Range128", 128, 7), ("Range256", 256, 8)]


def _le_bytes(x, k=4):
    x = np.asarray(x, dtype=np.uint64)
    return [((x >> np.uint64(8 * i)) & np.uint64(255)).astype(np.uint32) for i in range(k)]


def _log2_ceil(n):
    return max(int(n - 1).bit_length(), 0)


def ram_log_size(n_addresses):
    """RamInitFinal::compute_log_size (ram_init_final.rs:339-343)."""
    return max(_log2_ceil(max(n_addresses, 1)), K.LOG_N_LANES)


def last_access(inputs, addresses, timestamps, init_addresses, init_values):
    """The side note's `rw_mem_check.last_access` after the permutations, rebuilt from the keccak side note and the public initial memory:
    (ascending addresses, final values, final counters), one entry per distinct address.  Permutation p reads the 200 bytes at addresses[p]
    and leaves the bytes of Keccak-f[1600](inputs[p]) with counter timestamps[p][k] + 1; the last permutation (in order) to touch an address
    gives its final state, and an initial-memory entry no permutation touches keeps its value with counter 0."""
    inputs = np.asarray(inputs, dtype=np.uint64).reshape(-1, 25)
    n_perms = inputs.shape[0]
    out_bytes = np.concatenate([K._lane_bytes(l) for l in K.keccak_f(np.ascontiguousarray(inputs.T))]).T     # (n_perms, 200)
    acc_addr = (np.asarray(addresses, dtype=np.uint64)[:, None] + np.arange(K.STATE_SIZE, dtype=np.uint64)[None, :]).ravel()
    acc_seq = np.repeat(np.arange(1, n_perms + 1, dtype=np.uint64), K.STATE_SIZE)
    acc_val = out_bytes.ravel().astype(np.uint64)
    acc_ctr = np.asarray(timestamps, dtype=np.uint64).ravel() + np.uint64(1)
    ia = np.asarray(init_addresses, dtype=np.uint64)
    addr = np.concatenate([acc_addr, ia])
    seq = np.concatenate([acc_seq, np.zeros(ia.size, np.uint64)])
    val = np.concatenate([acc_val, np.asarray(init_values, dtype=np.uint64)])
    ctr = np.concatenate([acc_ctr, np.zeros(ia.size, np.uint64)])
    order = np.lexsort((seq, addr))
    addr, val, ctr = addr[order], val[order], ctr[order]
    last = np.ones(addr.size, bool)
    last[:-1] = addr[1:] != addr[:-1]
    return addr[last], val[last], ctr[last]


def ram_init_final_columns(inputs, addresses, timestamps, init_addresses, init_values, log_size):
    """RamInitFinal::original_columns (ram_init_final.rs:458-511) in trace order: (10, 2^log_size) uint32 — address bytes, flag, final value,
    final counter bytes — one row per distinct address (last_access), zero rows after them."""
    addr, val, ctr = last_access(inputs, addresses, timestamps, init_addresses, init_values)
    n = 1 << log_size
    assert addr.size <= n, "more distinct addresses than rows"
    t = np.zeros((RAM_COLS, n), np.uint32)
    m = addr.size
    t[0:4, :m] = _le_bytes(addr)
    t[4, :m] = 1
    t[5, :m] = val
    t[6:10, :m] = _le_bytes(ctr)
    return t


def memory_simulation(n_perms, n_buffers, seed):
    """The keccak side note of `n_perms` permutations over `n_buffers` 200-byte buffers on a byte memory (module docstring).  Returns
    (inputs (n_perms, 25) uint64, addresses (n_perms,) uint32, timestamps (n_perms, 200) uint32, init addresses (ascending) uint32, init
    values uint8)."""
    rng = np.random.default_rng(seed)
    bases = np.empty(n_buffers, np.uint64)
    for b in range(n_buffers):
        if b % 3 == 1:                                       # overlaps the previous buffer at an offset that is not a multiple of 8
            off = int(rng.integers(1, K.STATE_SIZE))
            off += off % 8 == 0
            bases[b] = bases[b - 1] + np.uint64(off)
        elif b % 3 == 2:                                     # crosses a 2^16 boundary inside its 200 bytes
            bases[b] = np.uint64((int(rng.integers(1, 1 << 15)) << 16) - int(rng.integers(1, K.STATE_SIZE)))
        else:
            bases[b] = np.uint64(int(rng.integers(0, (1 << 31) - K.STATE_SIZE)))
    which = rng.integers(0, n_buffers, n_perms)
    which[:n_buffers] = np.arange(min(n_buffers, n_perms))    # every buffer is used when there are enough permutations
    addresses = bases[which]
    ranges = addresses[:, None] + np.arange(K.STATE_SIZE, dtype=np.uint64)[None, :]
    init_addresses = np.unique(ranges.ravel())
    slot = np.searchsorted(init_addresses, ranges)            # (n_perms, 200) memory slot of each accessed byte
    init_values = rng.integers(0, 256, init_addresses.size, dtype=np.uint64).astype(np.uint8)
    value, count = init_values.astype(np.uint64).copy(), np.zeros(init_addresses.size, np.uint64)
    inputs = np.empty((n_perms, 25), np.uint64)
    timestamps = np.empty((n_perms, K.STATE_SIZE), np.uint64)
    p = 0
    while p < n_perms:                                       # waves of consecutive permutations on disjoint bytes run together
        q, used = p, set()
        while q < n_perms and used.isdisjoint(slot[q].tolist()):
            used.update(slot[q].tolist())
            q += 1
        s = slot[p:q]
        inputs[p:q] = value[s].astype(np.uint8).reshape(q - p, 25, 8).view("<u8")[..., 0]
        timestamps[p:q] = count[s]
        out = K.keccak_f(np.ascontiguousarray(inputs[p:q].T))
        value[s] = np.concatenate([K._lane_bytes(l) for l in out]).T
        count[s] += np.uint64(1)
        p = q
    return inputs, addresses.astype(np.uint32), timestamps.astype(np.uint32), init_addresses.astype(np.uint32), init_values


def _final_reg_component(air, rel_reg):
    """FinalRegEval::evaluate (final_reg.rs:80-116)."""
    c = air.component(FINAL_REG_LOG_SIZE, 1)
    reg_idx = c.get_preprocessed_column(f"preprocessed_register_idx_{FINAL_REG_LOG_SIZE}")
    final_ts = [c.next_trace_mask() for _ in range(4)]
    final_value = [c.next_trace_mask() for _ in range(4)]
    c.add_to_relation(rel_reg, 1, [reg_idx] + [0] * 8)                     # the initial register state
    c.add_to_relation(rel_reg, -1, [reg_idx] + final_ts + final_value)      # the final register state
    c.finalize_logup_in_pairs()
    return c


def _bit_op_component(air, rel_bitop):
    """BitOpMultiplicityEval::evaluate (bit_op.rs:55-93): BitOp::And, Or, Xor are the op codes 1, 2, 3 of BitOpChip's lookups."""
    c = air.component(BIT_OP_LOG_SIZE, 1)
    b, cc, a_and, a_or, a_xor = (c.get_preprocessed_column(n) for n in BITOP_PREPROCESSED)
    mults = [c.next_trace_mask() for _ in range(3)]
    for op, answer, mult in zip((1, 2, 3), (a_and, a_or, a_xor), mults):
        c.add_to_relation(rel_bitop, -mult, [c.const(op), b, cc, answer])
    c.finalize_logup()
    return c


def _ram_init_final_component(air, log_size, rel_ls, rel256):
    """RamInitFinalEval::evaluate (ram_init_final.rs:61-249)."""
    c = air.component(log_size, 1)
    pre_addr = [c.get_preprocessed_column(n) for n in RAM_PREPROCESSED[:4]]
    init_flag, init_value, out_flag, out_value = (c.get_preprocessed_column(n) for n in RAM_PREPROCESSED[4:])
    addr = [c.next_trace_mask() for _ in range(4)]
    flag = c.next_trace_mask()
    final_value = c.next_trace_mask()
    counter = [c.next_trace_mask() for _ in range(4)]
    for i in range(4):                                                       # :93-98
        c.add_constraint((init_flag + out_flag) * (addr[i] - pre_addr[i]))
    c.add_constraint(out_flag * (final_value - out_value))                   # :100-102
    c.add_constraint(flag * (flag - 1))                                      # :104-107
    addr_lo, addr_hi = addr[0] + addr[1] * 256, addr[2] + addr[3] * 256
    c.add_to_relation(rel_ls, flag, [addr_lo, addr_hi, init_flag * init_value, 0, 0])                       # :156-185
    c.add_to_relation(rel_ls, -flag, [addr_lo, addr_hi, final_value, counter[0] + counter[1] * 256,
                                      counter[2] + counter[3] * 256])                                    # :186-218
    for v in addr + [final_value] + counter:                                 # :219-248
        c.add_to_relation(rel256, 1, [v])
    c.finalize_logup()
    return c


def _multiplicity_component(air, rel, length, log_size):
    """MultiplicityEval::evaluate (multiplicity.rs:112-124) and MultiplicityEval8 (multiplicity8.rs:76-87)."""
    c = air.component(log_size, 1)
    value = c.get_preprocessed_column(f"preprocessed_range_values_{length}")
    c.add_to_relation(rel, -c.next_trace_mask(), [value])
    c.finalize_logup()
    return c


class NexusV1KeccakMachine:
    """The whole machine of the module docstring: main component at 2^log_size rows, `n_perms` keccak permutations over `n_buffers` buffers
    (default max(n_perms // 4, 1)).  Same interface as the other machines: `air`, `words`, `relations`, `log_sizes`, `preprocessed_columns()`,
    `fill_main_trace()` (tree 1 in commitment order, the multiplicity columns included), `column_log_sizes()`, and `device_trees(ctx)`.

    Recorded sizes (column counts per tree / constraints including the LogUp ones):
      main            27 / 347 / 1012 columns, 414 constraints (v1's 413 and IsCustomKeccak's booleanity)
      FinalReg         1 /   8 /    4,   1         BitOpMultiplicity   5 / 3 / 12, 3
      RamInitFinal     8 /  10 /   44,  17 (6 + 11 fractions)        Multiplicity8/16/32/128/256  1 / 1 / 4, 1 each
      keccak           as KeccakMachine (27 / 5444 / 5040 over its six components)."""

    def __init__(self, log_size, n_perms, n_buffers=None, seed=0):
        assert log_size >= 8 and n_perms >= 1
        self.n_perms = int(n_perms)
        self.n_buffers = int(n_buffers or max(self.n_perms // 4, 1))
        self.seed = seed
        inputs, addresses, timestamps, self.init_addresses, self.init_values = memory_simulation(self.n_perms, self.n_buffers, seed)
        self.keccak = K.KeccakMachine(inputs=inputs, addresses=addresses, timestamps=timestamps)
        self.ram_log_size = ram_log_size(self.init_addresses.size)
        air = A.Air()
        names = [("BitOp", 4), ("LoadStore", 5), ("KeccakXor", 3), ("KeccakBitNotAnd", 3), ("KeccakState", K.STATE_SIZE), ("KeccakBitRotate", 4),
                 ("ProgramCheck", 8), ("RegisterCheck", 9), ("Range8", 1), ("Range16", 1), ("Range32", 1), ("Range128", 1), ("Range256", 1)]
        self.relations = [air.relation(n, s) for n, s in names]
        rel = {r.name: r for r in self.relations}
        self.log_size_main = log_size
        self.main, _col = V.record_main_component(air, log_size, rel, keccak=True)
        self.final_reg = _final_reg_component(air, rel["RegisterCheck"])
        self.bit_op = _bit_op_component(air, rel["BitOp"])
        self.ram = _ram_init_final_component(air, self.ram_log_size, rel["LoadStore"], rel["Range256"])
        self.tables = [_multiplicity_component(air, rel[r], length, ls) for r, length, ls in MULTIPLICITY_TABLES]
        km = self.keccak
        K._mem_check_component(air, km.mem_log_size, rel["KeccakState"], rel["LoadStore"])
        for (index, _r, _o), ls in zip(K.ROUND_SPLIT, km.round_log_sizes):
            K._round_component(air, ls, index, rel["KeccakState"], rel["KeccakXor"], rel["KeccakBitNotAnd"], rel["KeccakBitRotate"])
        K._bitwise_table_component(air, rel["KeccakXor"], 2)
        K._bitwise_table_component(air, rel["KeccakBitNotAnd"], 3)
        K._bit_rotate_component(air, rel["KeccakBitRotate"])
        self.air = air
        self.log_sizes = ([log_size, FINAL_REG_LOG_SIZE, BIT_OP_LOG_SIZE, self.ram_log_size] + [ls for _r, _l, ls in MULTIPLICITY_TABLES]
                          + km.log_sizes)
        self.log_size = max(self.log_sizes)
        self.words = air.serialize()
        self._main = None

    # ---- side notes
    def side_note(self):
        """The keccak side note: the arguments of nb200_keccak_main_trace."""
        return self.keccak.side_note()

    def initial_memory(self):
        """The public initial memory: (ascending addresses uint32, values uint8)."""
        return self.init_addresses, self.init_values

    def ram_init_final_columns(self):
        """RamInitFinal's 10 main columns in trace order (numpy reference of nb200_ram_init_final_trace)."""
        return ram_init_final_columns(*self.side_note(), self.init_addresses, self.init_values, self.ram_log_size)

    # ---- tree 0
    def _ram_preprocessed(self):
        """RamInitFinal::preprocessed_columns (ram_init_final.rs:347-457): the init-memory rows, then zero rows (no exit code or output)."""
        n, m = 1 << self.ram_log_size, self.init_addresses.size
        cols = {k: np.zeros(n, np.uint32) for k in RAM_PREPROCESSED}
        for i, limb in enumerate(_le_bytes(self.init_addresses)):
            cols[RAM_PREPROCESSED[i]][:m] = limb
        cols["preprocessed_ram_init_final_init_flag"][:m] = 1
        cols["preprocessed_ram_init_final_init_value"][:m] = self.init_values
        return cols

    def preprocessed_columns(self):
        ids = self.air.preprocessed_ids
        by_id = dict(V.main_preprocessed_columns(self.log_size_main))
        by_id[f"preprocessed_register_idx_{FINAL_REG_LOG_SIZE}"] = np.arange(32, dtype=np.uint32)
        r = np.arange(256, dtype=np.uint32)                                  # bit_op.rs:198-210: row 16 b + c
        b, c = r >> 4, r & 15
        for name, v in zip(BITOP_PREPROCESSED, [b, c, b & c, b | c, b ^ c]):
            by_id[name] = v
        by_id.update(self._ram_preprocessed())
        for _r, length, ls in MULTIPLICITY_TABLES:                          # multiplicity8.rs:186-193: 0..7 then eight zeros
            v = np.zeros(1 << ls, np.uint32)
            v[:length] = np.arange(length, dtype=np.uint32)
            by_id[f"preprocessed_range_values_{length}"] = v
        kc = self.keccak.preprocessed_columns()
        for name, i in self.keccak.air.preprocessed_ids.items():
            by_id[name] = kc[i]
        cols = [None] * self.air.n_columns()[0]
        for name, i in ids.items():
            cols[i] = by_id[name]
        return cols

    # ---- tree 1
    def _main_and_hist(self, seed, hist=True):
        t = V.padding_witness(self.log_size_main, seed)
        cols = [limb for name, _ in V.MAIN_COLUMNS for limb in t[name]]
        if not hist:
            return cols, None, None
        # lookups with a nonzero numerator in the padding witness: Range32's five columns and Range256's words, half words and bytes (numerator
        # 1); every other relation's lookups are gated by an opcode flag, all zero here
        h256, h32 = np.zeros(256, np.int64), np.zeros(32, np.int64)
        for w in V.R256_WORDS + V.R256_HALF_WORDS + V.R256_BYTES:
            for limb in t[w]:
                h256 += np.bincount(limb, minlength=256)
        for w in V.R32:
            h32 += np.bincount(t[w][0], minlength=32)
        return cols, h256, h32

    def base_extension_columns(self, h256, h32, ram_cols):
        """Tree 1 of the eight base extensions in commitment order: FinalReg (8 columns), BitOpMultiplicity (3), RamInitFinal (`ram_cols`),
        Multiplicity8, 16, 32, 128, 256 (one column each, counted as the reference's side note counts them)."""
        h256 = np.asarray(h256, np.int64).copy()
        for v in ram_cols[[0, 1, 2, 3, 5, 6, 7, 8, 9]]:                      # ram_init_final.rs:262-272: nine lookups per row, padding included
            h256 += np.bincount(v, minlength=256)
        cols = [np.zeros(1 << FINAL_REG_LOG_SIZE, np.uint32) for _ in range(8)]   # no register is accessed: final state = initial state
        cols += [np.zeros(1 << BIT_OP_LOG_SIZE, np.uint32) for _ in range(3)]     # no bit-op lookup
        cols += list(ram_cols)
        counts = {"Range32": h32, "Range256": h256}
        for r, length, ls in MULTIPLICITY_TABLES:                           # row k of the table counts value k (multiplicity8.rs:194-204)
            v = np.zeros(1 << ls, np.int64)
            if r in counts:
                v[:length] = counts[r]
            cols.append((v % P).astype(np.uint32))
        return cols

    def fill_main_trace(self, seed=0):
        """Tree 1 in commitment order: the 347 main columns, the base extensions' columns, then the keccak extension's blocks and multiplicity
        columns (KeccakMachine.fill_main_trace).  Built once and cached."""
        if self._main is None:
            cols, h256, h32 = self._main_and_hist(seed)
            self._main = cols + self.base_extension_columns(h256, h32, self.ram_init_final_columns()) + self.keccak.fill_main_trace()
        return list(self._main)

    def column_log_sizes(self):
        return self.air.column_log_sizes()

    def device_trees(self, ctx, seed=0):
        """(tree-0 device batches, tree-1 device batches), finalized order, for machine.prove(..., resident=...): tree 0 uploaded; of tree 1
        only the main component's columns and FinalReg's and BitOpMultiplicity's are uploaded.  RamInitFinal is filled on the device
        (nb200_ram_init_final_trace) and the keccak extension too (nb200_keccak_main_trace), both from the side note; then every table's
        multiplicity column (BitOp, Range8 to Range256 and the keccak tables) is counted from that trace (nb200_table_multiplicities_first_row),
        so Range256 picks up RamInitFinal's lookups from the filled batch, after RamInitFinal as the reference orders them (machine.rs:81)."""
        from .machine import fill_table_multiplicities

        def upload_runs(cols):
            out, i = [], 0
            while i < len(cols):
                j = i
                while j < len(cols) and len(cols[j]) == len(cols[i]):
                    j += 1
                out.append(ctx.upload(np.stack(cols[i:j]), coset_order=True))
                i = j
            return out

        tree0 = upload_runs(self.preprocessed_columns())
        main, _h256, _h32 = self._main_and_hist(seed, hist=False)
        tree1 = [ctx.upload(np.stack(main), coset_order=True)]
        del main
        tree1 += upload_runs([np.zeros(1 << FINAL_REG_LOG_SIZE, np.uint32)] * 8)      # no register is accessed: final state = initial state
        tree1 += upload_runs([np.zeros(1 << BIT_OP_LOG_SIZE, np.uint32)] * 3)         # BitOp's multiplicities: counted below
        ram, n_rows = ctx.ram_init_final_trace(*self.side_note(), self.init_addresses, self.init_values, self.ram_log_size)
        assert n_rows == self.init_addresses.size
        tree1.append(ram)
        i = 0                                                                 # Multiplicity8 ... 256: one batch per run of equal sizes
        while i < len(MULTIPLICITY_TABLES):
            j = i
            while j < len(MULTIPLICITY_TABLES) and MULTIPLICITY_TABLES[j][2] == MULTIPLICITY_TABLES[i][2]:
                j += 1
            tree1.append(ctx.alloc(j - i, MULTIPLICITY_TABLES[i][2]))
            i = j
        tree1 += ctx.keccak_main_trace(*self.side_note())
        fill_table_multiplicities(self, ctx, tree0, tree1, first_row=True)
        return tree0, tree1
