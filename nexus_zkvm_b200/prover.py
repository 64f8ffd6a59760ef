"""ctypes mirror of the proving half of the C ABI (include/nb200.h): Blake2sChannel, AIR, CommitmentSchemeProver,
interaction-trace generation and stwo::prover::prove — the surface nexus-zkvm prover/src/machine.rs:197-290 drives.
`CudaBackend` plugs into nexus_zkvm_b200.machine.prove()."""
import ctypes as C
import os

import numpy as np

from . import Context, Columns, Nb200Error, lib, u32p, u8p


class Channel:
    """Blake2sChannel (host side of the library)."""

    def __init__(self, ctx=None, _h=None):
        self.ctx = ctx
        if _h is not None:
            self._h = _h
            return
        self._h = C.c_void_p()
        st = lib().nb200_channel_new(ctx._h if ctx is not None else None, C.byref(self._h))
        if st:
            raise Nb200Error(f"nb200_channel_new failed ({st})")

    def __del__(self):
        try:
            lib().nb200_channel_free(self._h)
        except Exception:
            pass

    def clone(self):
        h = C.c_void_p()
        lib().nb200_channel_clone(self._h, C.byref(h))
        return Channel(self.ctx, h)

    def digest(self):
        out = (C.c_uint8 * 32)(); lib().nb200_channel_digest(self._h, out); return bytes(out)

    def mix_u64(self, v):
        lib().nb200_channel_mix_u64(self._h, C.c_uint64(v))

    def mix_u32s(self, words):
        w = np.ascontiguousarray(words, dtype=np.uint32)
        lib().nb200_channel_mix_u32s(self._h, w.ctypes.data_as(u32p), C.c_size_t(w.size))

    def mix_felts(self, felts):
        f = np.ascontiguousarray(np.asarray(felts, dtype=np.uint32).reshape(-1))
        lib().nb200_channel_mix_felts(self._h, f.ctypes.data_as(u32p), C.c_size_t(f.size // 4))

    def mix_root(self, root):
        lib().nb200_channel_mix_root(self._h, (C.c_uint8 * 32).from_buffer_copy(root))

    def draw_felt(self):
        out = np.zeros(4, np.uint32); lib().nb200_channel_draw_felt(self._h, out.ctypes.data_as(u32p)); return out

    def draw_felts(self, n):
        out = np.zeros((n, 4), np.uint32); lib().nb200_channel_draw_felts(self._h, C.c_size_t(n), out.ctypes.data_as(u32p)); return out

    def draw_random_bytes(self):
        out = (C.c_uint8 * 32)(); lib().nb200_channel_draw_random_bytes(self._h, out); return bytes(out)


class Air:
    def __init__(self, ctx, words):
        self.ctx = ctx
        self.words = np.ascontiguousarray(words, dtype=np.uint32)
        self._h = C.c_void_p()
        ctx._chk(lib().nb200_air_load(ctx._h, self.words.ctypes.data_as(u32p), C.c_size_t(self.words.size), C.byref(self._h)))

    def __del__(self):
        try:
            lib().nb200_air_free(self._h)
        except Exception:
            pass


class CommitmentSchemeProver:
    """CommitmentSchemeProver::<CudaBackend, Blake2sMerkleChannel> + the Machine-level steps that need device data."""

    def __init__(self, ctx, air_words, config):
        self.ctx, self.config = ctx, config
        self.air = air_words if isinstance(air_words, Air) else Air(ctx, air_words)
        self._h = C.c_void_p()
        ctx._chk(lib().nb200_scheme_new(ctx._h, C.c_uint32(config["pow_bits"]), C.c_uint32(config["log_blowup"]),
                                        C.c_uint32(config["log_last"]), C.c_uint32(config["n_queries"]), C.byref(self._h)))
        lib().nb200_air_max_log_expand.restype = C.c_uint32
        lib().nb200_air_max_log_expand.argtypes = [C.c_void_p]
        ctx._chk(lib().nb200_scheme_set_constraint_log_degree(self._h, C.c_uint32(lib().nb200_air_max_log_expand(self.air._h))))
        self.tree_evals = []  # per committed tree: list of eval batches (kept alive; read by gen_interaction)

    def __del__(self):
        try:
            if self.ctx._h:
                lib().nb200_scheme_free(self._h)
        except Exception:
            pass

    def _batches_from_host(self, cols, coset_order):
        """Group consecutive equal-length host columns into device batches (commitment order is preserved)."""
        batches, i = [], 0
        while i < len(cols):
            j = i
            while j < len(cols) and len(cols[j]) == len(cols[i]):
                j += 1
            host = np.stack([np.ascontiguousarray(c, dtype=np.uint32) for c in cols[i:j]])
            batches.append(self.ctx.upload(host, coset_order=coset_order))
            i = j
        return batches

    def commit_batches(self, batches, ch):
        arr = (C.c_void_p * len(batches))(*[b._h for b in batches])
        root = (C.c_uint8 * 32)()
        self.ctx._chk(lib().nb200_scheme_commit(self._h, arr, C.c_size_t(len(batches)), ch._h, root))
        self.tree_evals.append(list(batches))
        return bytes(root)

    @staticmethod
    def _host_batches(cols):
        """Normalise `cols` (1-D columns and/or 2-D blocks of columns, commitment order) into contiguous 2-D host batches.
        2-D blocks are used as they are (no copy) — fill the trace straight into `ctx.host_alloc` memory for H2D at link speed."""
        out, run = [], []

        def flush():
            if run:
                out.append(np.stack(run))
                run.clear()

        for c in cols:
            a = np.asarray(c)
            if a.ndim == 2:
                flush()
                # packed host formats: uint8 / uint16 blocks travel at their natural width and are widened on the device
                out.append(np.ascontiguousarray(a) if a.dtype in (np.uint8, np.uint16, np.uint32) else np.ascontiguousarray(a, dtype=np.uint32))
            else:
                a = np.ascontiguousarray(a, dtype=np.uint32)
                if run and run[0].size != a.size:
                    flush()
                run.append(a)
        flush()
        return out

    def commit(self, cols, ch, coset_order=False):
        """tree_builder.extend_evals(host columns); commit(channel) — pipelined H2D + transforms (nb200_scheme_commit_host)."""
        hb = self._host_batches(cols)
        n = len(hb)
        ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in hb])
        widths = (C.c_uint32 * n)(*[b.dtype.itemsize for b in hb])
        ncols = (C.c_size_t * n)(*[b.shape[0] for b in hb])
        logs = (C.c_uint32 * n)(*[int(b.shape[1]).bit_length() - 1 for b in hb])
        evals = (C.c_void_p * n)()
        root = (C.c_uint8 * 32)()
        self.ctx._chk(lib().nb200_scheme_commit_host_packed(self._h, ptrs, widths, ncols, logs, C.c_size_t(n), C.c_int(1 if coset_order else 0), ch._h, root, evals))
        self.h2d_bytes = getattr(self, "h2d_bytes", 0) + sum(b.nbytes for b in hb)
        self.ctx.sync()  # the host batches may be released by the caller after this returns
        self.tree_evals.append([Columns(self.ctx, C.c_void_p(evals[i])) for i in range(n)])
        return bytes(root)

    # ---- one proof over N GPUs (ctx.comm_init first): include/nb200.h "one PROOF over N GPUs"
    def commit_sharded(self, big_shard, total_big, log_size, small, replicate, keep_eval_rows, ch):
        """nb200_scheme_commit_sharded.  big_shard: this rank's column range (device batch, finalized order) or None when the range is empty;
        small: replicated device batches; replicate: indices of big columns read at a row offset."""
        sm = (C.c_void_p * max(len(small), 1))(*[b._h for b in small])
        rep = (C.c_uint32 * max(len(replicate), 1))(*[int(x) for x in replicate])
        root = (C.c_uint8 * 32)()
        self.ctx._chk(lib().nb200_scheme_commit_sharded(self._h, big_shard._h if big_shard is not None else None, C.c_size_t(total_big), C.c_uint32(log_size),
                                                        sm, C.c_size_t(len(small)), rep, C.c_size_t(len(replicate)), C.c_int(1 if keep_eval_rows else 0), ch._h, root))
        self.tree_evals.append(([big_shard] if big_shard is not None else []) + list(small))   # kept alive
        return bytes(root)

    def gen_interaction_sharded(self, comp, params):
        p = np.ascontiguousarray(np.array(params, dtype=np.uint32).reshape(-1, 4))
        out = C.c_void_p()
        claimed = np.zeros(4, np.uint32)
        self.ctx._chk(lib().nb200_gen_interaction_trace_sharded(self._h, self.air._h, C.c_uint32(comp), p.ctypes.data_as(u32p), C.c_size_t(p.shape[0]),
                                                                C.byref(out), claimed.ctypes.data_as(u32p)))
        return Columns(self.ctx, out), tuple(int(x) for x in claimed)

    def gen_interaction_replicated(self, comp, log_size, n_logup_cols, params, tree0, tree1):
        """nb200_gen_interaction_trace for a component whose columns are replicated: tree0 / tree1 are batch lists that cover ALL columns of the trees
        in commitment order (a placeholder batch stands for the sharded columns, which such a component never reads)."""
        p = np.ascontiguousarray(np.array(params, dtype=np.uint32).reshape(-1, 4))
        a0 = (C.c_void_p * len(tree0))(*[b._h for b in tree0])
        a1 = (C.c_void_p * len(tree1))(*[b._h for b in tree1])
        out = C.c_void_p()
        claimed = np.zeros(4, np.uint32)
        self.ctx._chk(lib().nb200_gen_interaction_trace(self.ctx._h, self.air._h, C.c_uint32(comp), a0, C.c_size_t(len(tree0)), a1, C.c_size_t(len(tree1)),
                                                        p.ctypes.data_as(u32p), C.c_size_t(p.shape[0]), C.byref(out), claimed.ctypes.data_as(u32p)))
        cols = Columns(self.ctx, out)
        assert cols.n_cols == 4 * n_logup_cols and cols.log_size == log_size
        return cols, tuple(int(x) for x in claimed)

    def gen_interaction(self, comp, log_size, n_logup_cols, params):
        p = np.ascontiguousarray(np.array(params, dtype=np.uint32).reshape(-1, 4))
        t0, t1 = self.tree_evals[0], self.tree_evals[1]
        a0 = (C.c_void_p * len(t0))(*[b._h for b in t0])
        a1 = (C.c_void_p * len(t1))(*[b._h for b in t1])
        out = C.c_void_p()
        claimed = np.zeros(4, np.uint32)
        self.ctx._chk(lib().nb200_gen_interaction_trace(self.ctx._h, self.air._h, C.c_uint32(comp), a0, C.c_size_t(len(t0)), a1, C.c_size_t(len(t1)),
                                                        p.ctypes.data_as(u32p), C.c_size_t(p.shape[0]), C.byref(out), claimed.ctypes.data_as(u32p)))
        cols = Columns(self.ctx, out)
        assert cols.n_cols == 4 * n_logup_cols and cols.log_size == log_size
        return cols, tuple(int(x) for x in claimed)

    def commit_interaction(self, inter, ch):
        # `inter` holds device batches straight from gen_interaction: no host round trip
        return self.commit_batches(list(inter), ch)

    def constraint_quotients(self, comp, params, coeffs, accum):
        """ComponentProver::evaluate_constraint_quotients_on_domain for one component: accum (4-column batch) += quotients."""
        p = np.ascontiguousarray(np.array(params, dtype=np.uint32).reshape(-1, 4))
        cf = np.ascontiguousarray(np.array(coeffs, dtype=np.uint32).reshape(-1, 4))
        self.ctx._chk(lib().nb200_constraint_quotients(self._h, self.air._h, C.c_uint32(comp), p.ctypes.data_as(u32p), C.c_size_t(p.shape[0]),
                                                       cf.ctypes.data_as(u32p), C.c_size_t(cf.shape[0]), accum._h))

    def constraint_quotients_half(self, comp, params, coeffs, q_d1, q_high_d2, q_high_d1):
        """The half-domain route prove takes for a degree-4 component (nb200_constraint_quotients_half): q_d1 += every constraint's quotient on
        the committed LDE domain, q_high_d2 / q_high_d1 += the degree > 2 constraints' quotient on the first half of the next larger canonic domain
        and on the LDE domain; each a 4-column batch of the LDE size.  Where the bytecode interpreter evaluates the component (NB200_JIT=0, an LDE
        of fewer than 2^10 rows) every constraint counts as a high one."""
        p = np.ascontiguousarray(np.array(params, dtype=np.uint32).reshape(-1, 4))
        cf = np.ascontiguousarray(np.array(coeffs, dtype=np.uint32).reshape(-1, 4))
        self.ctx._chk(lib().nb200_constraint_quotients_half(self._h, self.air._h, C.c_uint32(comp), p.ctypes.data_as(u32p), C.c_size_t(p.shape[0]),
                                                            cf.ctypes.data_as(u32p), C.c_size_t(cf.shape[0]), q_d1._h, q_high_d2._h, q_high_d1._h))

    def check_constraints(self, comp, params):
        """assert_constraints_on_polys for component `comp` on the GPU (nb200_check_constraints), over the three committed trees' batches.
        Returns the failing constraints as [(constraint index, degree, failing rows, first failing row in trace order)]."""
        p = np.ascontiguousarray(np.array(params, dtype=np.uint32).reshape(-1, 4))
        trees = [(C.c_void_p * max(len(t), 1))(*[b._h for b in t]) for t in self.tree_evals[:3]]
        assert len(trees) == 3, "commit the three trees first"
        lib().nb200_air_n_constraints.restype = C.c_uint32
        n_constraints = int(lib().nb200_air_n_constraints(self.air._h, C.c_uint32(comp)))
        deg = np.zeros(max(n_constraints, 1), np.uint32)
        self.ctx._chk(lib().nb200_air_constraint_degrees(self.air._h, C.c_uint32(comp), deg.ctypes.data_as(u32p), C.c_size_t(n_constraints)))
        n_failing = np.zeros(max(n_constraints, 1), np.uint64)
        first_row = np.zeros(max(n_constraints, 1), np.uint64)
        u64p = C.POINTER(C.c_uint64)
        self.ctx._chk(lib().nb200_check_constraints(self.ctx._h, self.air._h, C.c_uint32(comp),
                                                    trees[0], C.c_size_t(len(self.tree_evals[0])), trees[1], C.c_size_t(len(self.tree_evals[1])),
                                                    trees[2], C.c_size_t(len(self.tree_evals[2])), p.ctypes.data_as(u32p), C.c_size_t(p.shape[0]),
                                                    n_failing.ctypes.data_as(u64p), first_row.ctypes.data_as(u64p), C.c_size_t(n_constraints)))
        return [(k, int(deg[k]), int(n_failing[k]), int(first_row[k])) for k in range(n_constraints) if n_failing[k]]

    def prove(self, ch, params):
        p = np.ascontiguousarray(np.array(params, dtype=np.uint32).reshape(-1, 4))
        out = u8p(); ln = C.c_size_t()
        self.ctx._chk(lib().nb200_prove(self._h, self.air._h, p.ctypes.data_as(u32p), C.c_size_t(p.shape[0]), ch._h, C.byref(out), C.byref(ln)))
        data = bytes(np.ctypeslib.as_array(out, shape=(max(ln.value, 1),))[:ln.value])
        lib().nb200_free(C.cast(out, C.c_void_p))
        return data


class SampleBatch(C.Structure):
    _fields_ = [("point", C.c_uint32 * 8), ("first_entry", C.c_size_t), ("n_entries", C.c_size_t)]


class SampleEntry(C.Structure):
    _fields_ = [("column", C.c_uint32), ("value", C.c_uint32 * 4)]


def _q(v):
    return (C.c_uint32 * 4)(*[int(x) for x in np.asarray(v, dtype=np.uint32).reshape(4)])


def fold_line(ctx, src, alpha):
    """FriOps::fold_line on a secure column (4-column batch) -> new batch of half the length."""
    out = C.c_void_p()
    ctx._chk(lib().nb200_fold_line(ctx._h, src._h, _q(alpha), C.byref(out)))
    return Columns(ctx, out)


def fold_circle_into_line(ctx, dst, src, alpha):
    """FriOps::fold_circle_into_line: dst = dst * alpha^2 + fold(src) (in place)."""
    ctx._chk(lib().nb200_fold_circle_into_line(ctx._h, dst._h, src._h, _q(alpha)))


def accumulate(ctx, a, b):
    """AccumulationOps::accumulate: a += b."""
    ctx._chk(lib().nb200_accumulate(ctx._h, a._h, b._h))


def grind(ctx, digest, pow_bits):
    """GrindOps::grind."""
    nonce = C.c_uint64()
    ctx._chk(lib().nb200_grind(ctx._h, (C.c_uint8 * 32).from_buffer_copy(digest), C.c_uint32(pow_bits), C.byref(nonce)))
    return int(nonce.value)


def fri_quotients(ctx, batches, log_size, sample_batches, random_coeff):
    """QuotientOps::accumulate_quotients.  batches: device column batches (columns numbered through them);
    sample_batches: [(point8, [(column, value4), ...]), ...] -> new secure column (4 x 2^log_size)."""
    arr = (C.c_void_p * len(batches))(*[b._h for b in batches])
    n_e = sum(len(e) for _p, e in sample_batches)
    sb = (SampleBatch * max(len(sample_batches), 1))()
    se = (SampleEntry * max(n_e, 1))()
    k = 0
    for i, (pt, ents) in enumerate(sample_batches):
        sb[i].point = (C.c_uint32 * 8)(*[int(x) for x in np.asarray(pt, dtype=np.uint32).reshape(8)])
        sb[i].first_entry, sb[i].n_entries = k, len(ents)
        for ci, v in ents:
            se[k].column = int(ci); se[k].value = _q(v); k += 1
    out = C.c_void_p()
    ctx._chk(lib().nb200_fri_quotients(ctx._h, arr, C.c_size_t(len(batches)), C.c_uint32(log_size), sb, C.c_size_t(len(sample_batches)),
                                       se, C.c_size_t(n_e), _q(random_coeff), C.byref(out)))
    return Columns(ctx, out)


def _sample_tables(sample_batches):
    n_e = sum(len(e) for _p, e in sample_batches)
    sb = (SampleBatch * max(len(sample_batches), 1))()
    se = (SampleEntry * max(n_e, 1))()
    k = 0
    for i, (pt, ents) in enumerate(sample_batches):
        sb[i].point = (C.c_uint32 * 8)(*[int(x) for x in np.asarray(pt, dtype=np.uint32).reshape(8)])
        sb[i].first_entry, sb[i].n_entries = k, len(ents)
        for ci, v in ents:
            se[k].column = int(ci); se[k].value = _q(v); k += 1
    return sb, se, n_e


def fri_quotients_from_coeffs(ctx, coeffs, log_size, log_blowup, sample_batches, random_coeff):
    """fri_quotients over the LDEs (2^log_size rows) of the columns whose coefficients (2^(log_size - log_blowup) words) `coeffs` holds, by
    the prover's route: every sample batch's columns combined on their coefficients, then only the combinations extended."""
    arr = (C.c_void_p * len(coeffs))(*[b._h for b in coeffs])
    sb, se, n_e = _sample_tables(sample_batches)
    out = C.c_void_p()
    ctx._chk(lib().nb200_fri_quotients_from_coeffs(ctx._h, arr, C.c_size_t(len(coeffs)), C.c_uint32(log_size), C.c_uint32(log_blowup), sb,
                                                   C.c_size_t(len(sample_batches)), se, C.c_size_t(n_e), _q(random_coeff), C.byref(out)))
    return Columns(ctx, out)


def deep_plan(sample_batches, random_coeff):
    """The host tables of fri_quotients_from_coeffs (no device): (lines, alphas).  lines: n_batches x 24 words (point parts
    x0 x1 y0 y1 x2 x3 y2 y3, A[4], B[4], random_coeff ^ n_entries [4], c[4]); alphas: one row of 4 words per entry.  Columns are ignored."""
    sb, se, n_e = _sample_tables(sample_batches)
    lines = np.zeros((max(len(sample_batches), 1), 24), np.uint32)
    alphas = np.zeros((max(n_e, 1), 4), np.uint32)
    u32p = C.POINTER(C.c_uint32)
    st = lib().nb200_deep_plan(sb, C.c_size_t(len(sample_batches)), se, C.c_size_t(n_e), _q(random_coeff), lines.ctypes.data_as(u32p),
                               alphas.ctypes.data_as(u32p))
    if st != 0:
        raise RuntimeError(f"nb200_deep_plan failed: status {st}")
    return lines[:len(sample_batches)], alphas[:n_e]


class CudaBackend:
    """Backend protocol used by nexus_zkvm_b200.machine.prove (the stand-in for `SimdBackend`)."""

    def __init__(self, ctx=None, device=0):
        self.ctx = ctx or Context(device)
        self._airs = {}

    def channel(self):
        return Channel(self.ctx)

    def prover(self, words, config):
        # a loaded AIR (and its NVRTC-specialised kernels) is reused across proofs of the same machine
        key = (np.asarray(words, dtype=np.uint32).tobytes(), os.environ.get("NB200_JIT", ""))
        air = self._airs.get(key)
        if air is None:
            air = self._airs[key] = Air(self.ctx, words)
        return CommitmentSchemeProver(self.ctx, air, config)


def smoke(ctx):
    """Tiny full prove on the GPU (used by __graft_entry__.smoke); raises on failure."""
    from . import machine as M
    m = M.AddMachine(log_size=8, n_lanes=1)
    cols, mult = m.fill_main_trace(seed=1)
    proof, claimed, _aux = M.prove(m, CudaBackend(ctx), cols, mult)
    assert M.verify_claimed_sums(claimed) and len(proof) > 1000
    return proof
