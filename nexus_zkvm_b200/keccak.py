"""The reference's keccak precompile extension as data: its six components recorded through air.py, and a witness filled from
Keccak-f[1600] over random input states.

`keccak_extensions()` (nexus-zkvm prover/src/extensions/keccak/mod.rs:12-33) is, in this order:
  PermutationMemoryCheck                          memory_check/constraints.rs:18-128   one row per permutation
  KeccakRound { index 0, rounds 16, offset 0 }    round/constraints.rs:24-193          one row per round: rounds 0..15 of every permutation
  KeccakRound { index 1, rounds 8, offset 16 }                                         rounds 16..23
  XorTable, BitNotAndTable                        bitwise_table/constraints.rs:30-73    2^12 rows, 16 lookups per row (EXPAND_BITS = 2)
  BitRotateTable                                  bit_rotate/mod.rs:69-91               2^11 rows
Relations, in the order KeccakChip / LoadStoreChip draw them (chips/custom.rs:127-139, chips/instructions/i/load_store.rs:70-76):
LoadStore (5 values), Xor (3), BitNotAnd (3), State (25 * 8 = 200, chips/custom.rs:45), BitRotate (4).
Every component has max_constraint_log_degree_bound = log_size + 1 (log_expand 1) and batches its LogUp fractions in pairs, except
BitRotateTable (one fraction, finalize_logup).

The memory check's LoadStore fractions are balanced, in a whole machine, by the main component's RAM accesses (KeccakChip); on their own
the claimed sums of the six components add up to the net LoadStore contribution of the memory-check rows (`net_load_store`), not to zero.

Trace columns are filled in trace (coset) order, like the other machines here: a row of the reference's bit-reversed column order is a row
of ours, and no constraint reads another row, so the assignment of permutations and rounds to rows is only a permutation of the rows."""
import numpy as np

from . import air as A
from . import field as F

P = (1 << 31) - 1
LANE_SIZE = 8                       # field elements (bytes) per 64-bit lane (round/constants.rs:45)
STATE_SIZE = 25 * LANE_SIZE
ROUNDS = 24
WORD_SIZE_HALVED = 2                # 16-bit limbs per address / timestamp (memory_check/constraints.rs:61)
ELEM_BITS, EXPAND_BITS = 8, 2       # bitwise_table/mod.rs:61-62
LIMB_BITS = ELEM_BITS - EXPAND_BITS
BITWISE_LOG_SIZE = 2 * LIMB_BITS    # preprocessed_columns.rs:38-40
ROTATE_LOG_SIZE = 8 + 3             # bit_rotate/mod.rs:57
LOG_N_LANES = 4                     # smallest component (round/component.rs:128, memory_check/mod.rs:124)
ROUND_SPLIT = [(0, 16, 0), (1, 8, 16)]   # (index, rounds, offset) of the two KeccakRound components (mod.rs:15-24)


# ---- FIPS 202 constants, computed ----------------------------------------------------------------------------------------------
def _rc_bit(t):
    """FIPS 202 Algorithm 5: rc(t), the output of the LFSR x^8 + x^6 + x^5 + x^4 + 1 after t steps."""
    if t % 255 == 0:
        return 1
    r = [1, 0, 0, 0, 0, 0, 0, 0]
    for _ in range(t % 255):
        r = [0] + r
        for k in (0, 4, 5, 6):
            r[k] ^= r[8]
        r = r[:8]
    return r[0]


def round_constants():
    """RC[i] of the 24 rounds (FIPS 202 Algorithm 6): bit 2^j - 1 of RC[i] is rc(j + 7 i)."""
    return [sum(_rc_bit(j + 7 * i) << ((1 << j) - 1) for j in range(7)) for i in range(ROUNDS)]


def rotation_offsets():
    """r[x + 5 y] of the rho step (FIPS 202 Algorithm 2): (t + 1)(t + 2) / 2 mod 64 along the walk (x, y) <- (y, 2x + 3y)."""
    r = [0] * 25
    x, y = 1, 0
    for t in range(24):
        r[x + 5 * y] = ((t + 1) * (t + 2) // 2) % 64
        x, y = y, (2 * x + 3 * y) % 5
    return r


RC = round_constants()
ROTATIONS = rotation_offsets()


def _rotl(v, r):
    return v if r == 0 else (v << np.uint64(r)) | (v >> np.uint64(64 - r))


def keccak_round(a, rc):
    """One round on states `a` = (25, n) uint64, lane x + 5 y (round/mod.rs:11-51)."""
    c = [a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20] for x in range(5)]
    d = [c[(x + 4) % 5] ^ _rotl(c[(x + 1) % 5], 1) for x in range(5)]
    a = np.stack([a[i] ^ d[i % 5] for i in range(25)])
    b = [None] * 25
    for x in range(5):
        for y in range(5):
            b[y + ((2 * x + 3 * y) % 5) * 5] = _rotl(a[x + 5 * y], ROTATIONS[x + 5 * y])
    out = np.stack([b[i] ^ (~b[(i % 5 + 1) % 5 + 5 * (i // 5)] & b[(i % 5 + 2) % 5 + 5 * (i // 5)]) for i in range(25)])
    out[0] ^= np.uint64(rc)
    return out


def keccak_f(a):
    """Keccak-f[1600] on (25, n) uint64 states."""
    for rc in RC:
        a = keccak_round(a, rc)
    return a


def _lane_bytes(v):
    """(n,) uint64 lanes -> (8, n) uint8 little-endian bytes."""
    return np.ascontiguousarray(np.ascontiguousarray(v, dtype="<u8").view(np.uint8).reshape(-1, 8).T)


def _log2_ceil(n):
    return max(int(n - 1).bit_length(), 0)


# ---- the recorded AIR ---------------------------------------------------------------------------------------------------------
def _mem_check_component(air, log_size, rel_state, rel_ls):
    """PermutationMemoryCheckEval::eval (memory_check/constraints.rs:18-128)."""
    c = air.component(log_size, 1)
    nxt = lambda k: [c.next_trace_mask() for _ in range(k)]
    input_state, output_state = nxt(STATE_SIZE), nxt(STATE_SIZE)                                # :19-20
    addrs = nxt(STATE_SIZE * WORD_SIZE_HALVED)                                                  # :21
    prev_ts, next_ts = nxt(STATE_SIZE * WORD_SIZE_HALVED), nxt(STATE_SIZE * WORD_SIZE_HALVED)   # :22-23
    addr_carries, ts_carries = nxt(STATE_SIZE), nxt(STATE_SIZE)                                 # :24-25
    is_padding, _next_is_padding = c.next_interaction_mask(A.ORIGINAL_TRACE_IDX, [0, 1])        # :27-45
    c.get_preprocessed_column("keccak_memory_check_is_last_row")
    c.add_constraint(is_padding * (1 - is_padding))
    c.add_to_relation(rel_state, 1 - is_padding, input_state)                                  # :47-56
    c.add_to_relation(rel_state, is_padding - 1, output_state)
    h = WORD_SIZE_HALVED
    for i in range(STATE_SIZE):                                                                 # :58-86 (addr, val, ts)
        j = i * h
        c.add_to_relation(rel_ls, is_padding - 1, addrs[j:j + h] + [input_state[i]] + prev_ts[j:j + h])
        c.add_to_relation(rel_ls, 1 - is_padding, addrs[j:j + h] + [output_state[i]] + next_ts[j:j + h])
    for i in range(0, STATE_SIZE, h):                                                           # :88-105 (as upstream: the first 100 steps)
        addr, next_addr, carry = addrs[i:i + h], addrs[i + h:i + 2 * h], addr_carries[i // h]
        c.add_constraint((1 - is_padding) * (next_addr[0] + carry * (1 << 16) - addr[0] - 1))
        c.add_constraint((1 - is_padding) * (next_addr[1] - addr[1] - carry))
    for i in range(STATE_SIZE):                                                                 # :107-123
        p, q, carry = prev_ts[i * h:(i + 1) * h], next_ts[i * h:(i + 1) * h], ts_carries[i]
        c.add_constraint((1 - is_padding) * (q[0] + carry * (1 << 16) - p[0] - 1))
        c.add_constraint((1 - is_padding) * (q[1] - p[1] - carry))
    c.finalize_logup_in_pairs()                                                                 # :125
    return c


def _round_component(air, log_size, index, rel_state, rel_xor, rel_nand, rel_rot):
    """KeccakRoundEval::eval (round/constraints.rs:24-193)."""
    c = air.component(log_size, 1)
    next_u64 = lambda: [c.next_trace_mask() for _ in range(LANE_SIZE)]

    def xor(a, b):                                                                              # :128-139
        out = next_u64()
        for i in range(LANE_SIZE):
            c.add_to_relation(rel_xor, 1, [a[i], b[i], out[i]])
        return out

    def bitwise_not_and(a, b):                                                                  # :141-156
        out = next_u64()
        for i in range(LANE_SIZE):
            c.add_to_relation(rel_nand, 1, [a[i], b[i], out[i]])
        return out

    def rotate_left(a, r):                                                                      # :158-193
        if r == 0:
            return a
        bit_rotate, limb_rotate = r % 8, r // 8
        bits_low, bits_high, out = next_u64(), next_u64(), next_u64()
        for i in range(LANE_SIZE):
            c.add_to_relation(rel_rot, 1, [a[i], c.const(bit_rotate), bits_high[i], bits_low[i]])
            low, high = (i - limb_rotate) & 7, (i - limb_rotate + 7) & 7
            c.add_constraint(bits_low[low] + bits_high[high] - out[i])
        return out

    a = [next_u64() for _ in range(25)]                                                         # :25-26
    input_state = [v for lane in a for v in lane]
    col = []
    for x in range(5):                                                                          # theta :32-52
        acc = a[x]
        for i in range(1, 5):
            acc = xor(acc, a[x + 5 * i])
        col.append(acc)
    d = [xor(col[(x + 4) % 5], rotate_left(col[(x + 1) % 5], 1)) for x in range(5)]
    for x in range(5):
        for y in range(5):
            a[x + 5 * y] = xor(a[x + 5 * y], d[x])
    b = [None] * 25                                                                             # rho and pi :54-63
    for x in range(5):
        for y in range(5):
            b[y + ((2 * x + 3 * y) % 5) * 5] = rotate_left(a[x + 5 * y], ROTATIONS[x + 5 * y])
    for x in range(5):                                                                          # chi :65-72
        for y in range(5):
            rhs = bitwise_not_and(b[(x + 1) % 5 + 5 * y], b[(x + 2) % 5 + 5 * y])
            a[x + 5 * y] = xor(b[x + 5 * y], rhs)
    rc = [c.get_preprocessed_column(f"keccak_{index}_round_constant_{i}") for i in range(LANE_SIZE)]   # iota :74-81
    a[0] = xor(a[0], rc)
    is_padding, _next_is_padding = c.next_interaction_mask(A.ORIGINAL_TRACE_IDX, [0, 1])        # :83-101
    c.get_preprocessed_column(f"keccak_{index}_is_last_row")
    c.add_constraint(is_padding * (1 - is_padding))
    output_state = [v for lane in a for v in lane]
    c.add_to_relation(rel_state, is_padding - 1, input_state)                                  # :105-114
    c.add_to_relation(rel_state, 1 - is_padding, output_state)
    c.finalize_logup_in_pairs()                                                                 # :116
    return c


def _bitwise_op(c_col, i, j):
    return i ^ j if c_col == 2 else (~i & j) & ((1 << 32) - 1)


def _bitwise_table_component(air, rel, c_col):
    """BitwiseTableEvalAtRow::eval (bitwise_table/constraints.rs:30-73); c_col = B::C_COL_INDEX (2: Xor, 3: BitNotAnd, mod.rs:231,253)."""
    c = air.component(BITWISE_LOG_SIZE, 1)
    name = lambda k: f"keccakf_preprocessed_bit_table_{ELEM_BITS}_{EXPAND_BITS}_{k}"          # preprocessed_columns.rs:25-32
    al, bl, cl = c.get_preprocessed_column(name(0)), c.get_preprocessed_column(name(1)), c.get_preprocessed_column(name(c_col))
    for k in range(1 << (2 * EXPAND_BITS)):
        i, j = k >> EXPAND_BITS, k % (1 << EXPAND_BITS)
        mult = c.next_trace_mask()
        c.add_to_relation(rel, -mult, [al + (i << LIMB_BITS), bl + (j << LIMB_BITS), cl + (_bitwise_op(c_col, i, j) << LIMB_BITS)])
    c.finalize_logup_in_pairs()
    return c


ROTATE_COLUMNS = ["rotate_table_input_byte", "rotate_table_byte_shift", "rotate_table_bits_high", "rotate_table_bits_low"]


def _bit_rotate_component(air, rel):
    """BitRotateTableEval::evaluate (bit_rotate/mod.rs:69-91)."""
    c = air.component(ROTATE_LOG_SIZE, 1)
    pre = [c.get_preprocessed_column(n) for n in ROTATE_COLUMNS]
    mult = c.next_trace_mask()
    c.add_to_relation(rel, -mult, pre)
    c.finalize_logup()
    return c


class KeccakMachine:
    """The six components of `keccak_extensions()` over `n_perms` random input states (default 2^log_n_perms - 1, as the reference's
    prove_keccak test takes (1 << log_n_instances) - 1 inputs: every component then has padding rows).  Sizes (compute_log_size):
    memory check 2^max(log2ceil(n_perms), 4) rows, KeccakRound 0 / 1 16 / 8 rows per permutation rounded up to a power of two, the tables
    fixed.  Same interface as the other machines: `air`, `words`, `relations`, `log_sizes`, `preprocessed_columns()`, `fill_main_trace()`
    (tree 1 in commitment order, the table multiplicities last: `multiplicity_columns()`), `column_log_sizes()`.

    An explicit side note (the layout of KeccakSideNote, prover/src/trace/sidenote/keccak.rs:16-25) proves given permutations instead of
    seeded random ones: `inputs` (n_perms, 25) lanes x + 5 y, `addresses` (n_perms,) base addresses, `timestamps` (n_perms, 200) previous
    timestamps; `log_n_perms`, `seed` and `n_perms` are then ignored.  An address range must not wrap 2^32 and no timestamp may be 2^32 - 1.
    `device_trees(ctx)` fills tree 1 on the device from the side note (nb200_keccak_main_trace) for machine.prove(..., resident=...)."""

    def __init__(self, log_n_perms=None, seed=0, n_perms=None, inputs=None, addresses=None, timestamps=None):
        if inputs is not None:
            inputs = np.array(inputs, dtype=np.uint64)
            n_perms = inputs.shape[0]
            addresses = np.array(addresses, dtype=np.uint64)
            timestamps = np.array(timestamps, dtype=np.uint64)
            assert inputs.shape == (n_perms, 25) and addresses.shape == (n_perms,) and timestamps.shape == (n_perms, STATE_SIZE)
            assert int(addresses.max(initial=0)) <= (1 << 32) - STATE_SIZE, "an address range of 200 bytes wraps 2^32"
            assert int(timestamps.max(initial=0)) < (1 << 32) - 1, "a timestamp of 2^32 - 1 has no successor"
        self.n_perms = (1 << log_n_perms) - 1 if n_perms is None else int(n_perms)
        assert self.n_perms >= 1
        self.seed = seed
        self.mem_log_size = max(_log2_ceil(self.n_perms), LOG_N_LANES)
        self.round_log_sizes = [max(_log2_ceil(self.n_perms * rounds), LOG_N_LANES) for _i, rounds, _o in ROUND_SPLIT]
        air = A.Air()
        self.rel_ls = air.relation("LoadStore", 2 * WORD_SIZE_HALVED + 1)
        self.rel_xor = air.relation("KeccakXor", 3)
        self.rel_nand = air.relation("KeccakBitNotAnd", 3)
        self.rel_state = air.relation("KeccakState", STATE_SIZE)
        self.rel_rot = air.relation("KeccakBitRotate", 4)
        self.relations = [self.rel_ls, self.rel_xor, self.rel_nand, self.rel_state, self.rel_rot]
        self.mem = _mem_check_component(air, self.mem_log_size, self.rel_state, self.rel_ls)
        self.rounds = [_round_component(air, ls, index, self.rel_state, self.rel_xor, self.rel_nand, self.rel_rot)
                       for (index, _r, _o), ls in zip(ROUND_SPLIT, self.round_log_sizes)]
        self.xor_table = _bitwise_table_component(air, self.rel_xor, 2)
        self.nand_table = _bitwise_table_component(air, self.rel_nand, 3)
        self.rot_table = _bit_rotate_component(air, self.rel_rot)
        self.air = air
        self.log_sizes = [self.mem_log_size] + self.round_log_sizes + [BITWISE_LOG_SIZE, BITWISE_LOG_SIZE, ROTATE_LOG_SIZE]
        self.log_size = max(self.log_sizes)
        self.words = air.serialize()
        self._main = None
        if inputs is not None:
            self.inputs, self.addresses, self.timestamps = np.ascontiguousarray(inputs.T), addresses, timestamps
            return
        rng = np.random.default_rng(seed)
        self.inputs = rng.integers(0, 1 << 64, (25, self.n_perms), dtype=np.uint64, endpoint=False)
        # memory side note: one base address per permutation, one previous timestamp per state byte; low 16 bits near 0xffff on
        # every other permutation so that the carry columns are exercised
        lo = np.where(np.arange(self.n_perms) % 2 == 0, rng.integers(0xFF00, 0x10000, self.n_perms), rng.integers(0, 0x10000, self.n_perms))
        self.addresses = (rng.integers(0, 1 << 14, self.n_perms).astype(np.uint64) << np.uint64(16)) | lo.astype(np.uint64)
        ts_lo = np.where(rng.integers(0, 8, (self.n_perms, STATE_SIZE)) == 0, 0xFFFF, rng.integers(0, 0x10000, (self.n_perms, STATE_SIZE)))
        self.timestamps = (rng.integers(0, 1 << 14, (self.n_perms, STATE_SIZE)).astype(np.uint64) << np.uint64(16)) | ts_lo.astype(np.uint64)

    def side_note(self):
        """(inputs (n_perms, 25) uint64, addresses (n_perms,) uint32, timestamps (n_perms, 200) uint32): the arguments of
        nb200_keccak_main_trace."""
        return (np.ascontiguousarray(self.inputs.T), self.addresses.astype(np.uint32), np.ascontiguousarray(self.timestamps, dtype=np.uint32))

    def device_trees(self, ctx):
        """(tree-0 device batches, tree-1 device batches), finalized order, for machine.prove / check_constraints(..., resident=...): tree 0
        uploaded from preprocessed_columns() (27 small columns), tree 1 filled on the device from the side note (nb200_keccak_main_trace:
        the memory check, the two round components, the 32 bitwise and the rotate multiplicity columns, batched as the host columns are)."""
        cols, tree0, i = self.preprocessed_columns(), [], 0
        while i < len(cols):
            j = i
            while j < len(cols) and len(cols[j]) == len(cols[i]):
                j += 1
            tree0.append(ctx.upload(np.stack(cols[i:j]), coset_order=True))
            i = j
        return tree0, ctx.keccak_main_trace(*self.side_note())

    # ---- tree 0
    def preprocessed_columns(self):
        ids = self.air.preprocessed_ids
        cols = [None] * self.air.n_columns()[0]

        def is_last(log_size):
            v = np.zeros(1 << log_size, np.uint32)
            v[-1] = 1
            return v

        cols[ids["keccak_memory_check_is_last_row"]] = is_last(self.mem_log_size)
        for (index, rounds, offset), ls in zip(ROUND_SPLIT, self.round_log_sizes):   # round/trace.rs:209-238: RC[offset + row % rounds]
            rc = np.array(RC[offset:offset + rounds], dtype=np.uint64)[np.arange(1 << ls) % rounds]
            b = _lane_bytes(rc)
            for i in range(LANE_SIZE):
                cols[ids[f"keccak_{index}_round_constant_{i}"]] = b[i].astype(np.uint32)
            cols[ids[f"keccak_{index}_is_last_row"]] = is_last(ls)
        r = np.arange(1 << BITWISE_LOG_SIZE, dtype=np.uint32)                         # preprocessed_columns.rs:43-68
        a, b = r >> LIMB_BITS, r & ((1 << LIMB_BITS) - 1)
        for k, v in enumerate([a, b, a ^ b, ~a & b]):
            cols[ids[f"keccakf_preprocessed_bit_table_{ELEM_BITS}_{EXPAND_BITS}_{k}"]] = v.astype(np.uint32)
        r = np.arange(1 << ROTATE_LOG_SIZE, dtype=np.uint32)                          # bit_rotate/mod.rs:183-207
        byte, shift = r >> 3, r & 7
        for name, v in zip(ROTATE_COLUMNS, [byte, shift, byte >> (8 - shift), (byte << shift) & 255]):
            cols[ids[name]] = v.astype(np.uint32)
        assert all(c is not None for c in cols)
        return cols

    # ---- tree 1
    def _mem_trace(self):
        """generate_keccak_mem_check_trace (memory_check/trace.rs:32-123): (2 * 200 + 3 * 400 + 2 * 200 + 1, 2^log_size) uint16."""
        n, m = 1 << self.mem_log_size, self.n_perms
        h = WORD_SIZE_HALVED
        t = np.zeros((STATE_SIZE * 2 + STATE_SIZE * h * 3 + STATE_SIZE * 2 + 1, n), np.uint16)
        out = keccak_f(self.inputs)
        t[0:STATE_SIZE, :m] = np.concatenate([_lane_bytes(l) for l in self.inputs])
        t[STATE_SIZE:2 * STATE_SIZE, :m] = np.concatenate([_lane_bytes(l) for l in out])
        addr = self.addresses[None, :] + np.arange(STATE_SIZE, dtype=np.uint64)[:, None]          # (200, m)
        ts, ts1 = self.timestamps.T, self.timestamps.T + np.uint64(1)
        o = 2 * STATE_SIZE
        for block in (addr, ts, ts1):
            t[o:o + 2 * STATE_SIZE:2, :m] = block & np.uint64(0xFFFF)
            t[o + 1:o + 2 * STATE_SIZE:2, :m] = block >> np.uint64(16)
            o += 2 * STATE_SIZE
        t[o:o + STATE_SIZE, :m] = (addr & np.uint64(0xFFFF)) == 0xFFFF
        t[o + STATE_SIZE:o + 2 * STATE_SIZE, :m] = (ts & np.uint64(0xFFFF)) == 0xFFFF
        t[-1, m:] = 1                                                                            # is_padding
        return t

    def _round_trace(self, index, rounds, offset, log_size, states, hist):
        """generate_round_component_trace (round/trace.rs:297-366): rows perm * rounds + t hold round offset + t of a permutation (padding rows:
        the zero state), every row a full round.  `states` = (25, n_perms) inputs; returns ((1705, 2^log_size) uint8, the states after the
        component's rounds) and adds the lookups to `hist` (the three tables' multiplicities, counted over every row)."""
        n, m = 1 << log_size, self.n_perms
        rows = np.zeros((25, n), np.uint64)
        s = states
        for k in range(rounds):
            rows[:, k:m * rounds:rounds] = s
            s = keccak_round(s, RC[offset + k])
        rc = np.array(RC[offset:offset + rounds], dtype=np.uint64)[np.arange(n) % rounds]
        n_lanes = 25 + 20 + 5 * 4 + 25 + 24 * 3 + 50 + 1
        t = np.zeros((n_lanes * LANE_SIZE + 1, n), np.uint8)
        top = [0]

        def alloc(lane_bytes):
            k = top[0]
            t[k:k + LANE_SIZE] = lane_bytes
            top[0] += LANE_SIZE
            return t[k:k + LANE_SIZE]

        def count(key, a, b):
            hist[key] += np.bincount(((a.astype(np.uint32) << 8) | b).ravel(), minlength=1 << 16)

        def xor(a, b):
            count("xor", a, b)
            return alloc(a ^ b)

        def bitwise_not_and(a, b):
            count("nand", a, b)
            return alloc(~a & b)

        def rotate_left(a, r):
            if r == 0:
                return a
            bits, limbs = r % 8, r // 8
            hist["rot"] += np.bincount((8 * a.astype(np.uint32) + bits).ravel(), minlength=1 << ROTATE_LOG_SIZE)
            low = alloc((a.astype(np.uint32) << bits) & 255)
            high = alloc(a >> (8 - bits) if bits else np.zeros_like(a))
            return alloc(np.stack([low[(i - limbs) & 7] + high[(i - limbs + 7) & 7] for i in range(LANE_SIZE)]))

        a = [alloc(_lane_bytes(rows[i])) for i in range(25)]
        col = []
        for x in range(5):
            acc = a[x]
            for i in range(1, 5):
                acc = xor(acc, a[x + 5 * i])
            col.append(acc)
        d = [xor(col[(x + 4) % 5], rotate_left(col[(x + 1) % 5], 1)) for x in range(5)]
        for x in range(5):
            for y in range(5):
                a[x + 5 * y] = xor(a[x + 5 * y], d[x])
        b = [None] * 25
        for x in range(5):
            for y in range(5):
                b[y + ((2 * x + 3 * y) % 5) * 5] = rotate_left(a[x + 5 * y], ROTATIONS[x + 5 * y])
        for x in range(5):
            for y in range(5):
                a[x + 5 * y] = xor(b[x + 5 * y], bitwise_not_and(b[(x + 1) % 5 + 5 * y], b[(x + 2) % 5 + 5 * y]))
        a[0] = xor(a[0], _lane_bytes(rc))
        assert top[0] == n_lanes * LANE_SIZE
        t[-1, m * rounds:] = 1                                                                   # is_padding
        return t, s

    def fill_main_trace(self, seed=None):
        """Tree 1 in commitment order: the memory check (uint16 block), the two round components (uint8 blocks), then the 33 multiplicity
        columns of XorTable, BitNotAndTable and BitRotateTable (`multiplicity_columns`).  `seed` is accepted for the common interface; the
        inputs are the constructor's.  Built once and cached."""
        if self._main is None:
            hist = {"xor": np.zeros(1 << 16, np.int64), "nand": np.zeros(1 << 16, np.int64), "rot": np.zeros(1 << ROTATE_LOG_SIZE, np.int64)}
            blocks, s = [self._mem_trace()], self.inputs
            for (index, rounds, offset), ls in zip(ROUND_SPLIT, self.round_log_sizes):
                t, s = self._round_trace(index, rounds, offset, ls, s, hist)
                blocks.append(t)
            self.outputs = s
            self._mults = self._table_multiplicities(hist)
            self._main = blocks
            assert sum(b.shape[0] for b in blocks) + len(self._mults) == self.air.n_columns()[1]
        return list(self._main) + list(self._mults)

    @staticmethod
    def _table_multiplicities(hist):
        """BitwiseAccumulator / BitRotateAccumulator: a lookup (a, b) of a bitwise table is row ((a & 63) << 6) | (b & 63) of multiplicity
        column (a >> 6) * 4 + (b >> 6) (bitwise_table/constraints.rs:46-68); a rotation (byte, r) is row 8 byte + r."""
        out = []
        for key in ("xor", "nand"):
            h = hist[key].reshape(1 << EXPAND_BITS, 1 << LIMB_BITS, 1 << EXPAND_BITS, 1 << LIMB_BITS)   # [a_hi, a_lo, b_hi, b_lo]
            out += [(h[i, :, j, :].reshape(-1) % P).astype(np.uint32) for i in range(1 << EXPAND_BITS) for j in range(1 << EXPAND_BITS)]
        out.append((hist["rot"] % P).astype(np.uint32))
        return out

    def multiplicity_columns(self):
        self.fill_main_trace()
        return list(self._mults)

    def column_log_sizes(self):
        return self.air.column_log_sizes()

    def net_load_store(self, params):
        """The LoadStore part of the memory check's claimed sum, from the side note alone (no trace): per permutation and state byte,
        -1 / combine(addr, prev, ts) + 1 / combine(addr, next, ts + 1), combine = sum_i alpha^i v_i - z (Relation::combine)."""
        rel = self.rel_ls
        z, al = params[rel.z], [params[k] for k in rel.alpha_powers]

        def combine(vals):
            acc = F.qm31_neg(z)
            for a, v in zip(al, vals):
                acc = F.qm31_add(acc, F.qm31_mul_m31(a, int(v) % P))
            return acc

        outs = keccak_f(self.inputs)
        tot = (0, 0, 0, 0)
        for p in range(self.n_perms):
            bi = np.concatenate([_lane_bytes(self.inputs[l, p:p + 1])[:, 0] for l in range(25)])
            bo = np.concatenate([_lane_bytes(outs[l, p:p + 1])[:, 0] for l in range(25)])
            for i in range(STATE_SIZE):
                addr, ts = int(self.addresses[p]) + i, int(self.timestamps[p, i])
                lim = lambda x: [x & 0xFFFF, x >> 16]
                tot = F.qm31_sub(tot, F.qm31_inv(combine(lim(addr) + [bi[i]] + lim(ts))))
                tot = F.qm31_add(tot, F.qm31_inv(combine(lim(addr) + [bo[i]] + lim(ts + 1))))
        return tot
