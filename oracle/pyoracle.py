"""ORACLE — TEST INFRASTRUCTURE ONLY.

ctypes binding of oracle/liboracle.so (the CPU restatement of the reference's hot path, i.e. of
stwo @0790eba as called from nexus-zkvm prover/src/machine.rs:186-290).  Only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this module.
PARITY UNPINNED for Stwo-internal transcript details (no golden vectors exist in the reference).
"""
import ctypes as C
import os
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)
u8p = C.POINTER(C.c_uint8)


def build(force=False):
    so = os.path.join(_HERE, "liboracle.so")
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith((".h", ".cc"))]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        L = _LIB
        L.orc_m31_mul.restype = C.c_uint32
        L.orc_m31_mul.argtypes = [C.c_uint32, C.c_uint32]
        L.orc_m31_inv.restype = C.c_uint32
        L.orc_m31_inv.argtypes = [C.c_uint32]
        L.orc_bit_reverse_index.restype = C.c_uint64
        L.orc_bit_reverse_index.argtypes = [C.c_uint64, C.c_uint32]
        L.orc_coset_index_to_circle_domain_index.restype = C.c_uint64
        L.orc_coset_index_to_circle_domain_index.argtypes = [C.c_uint64, C.c_uint32]
        L.orc_channel_new.restype = C.c_void_p
        L.orc_num_threads.restype = C.c_int
    return _LIB


def _u32(a):
    a = np.ascontiguousarray(a, dtype=np.uint32)
    return a, a.ctypes.data_as(u32p)


def set_flavor(merkle_hash=0, draw_domain_sep=0, pow_variant=0):
    lib().orc_set_flavor(C.c_int(merkle_hash), C.c_int(draw_domain_sep), C.c_int(pow_variant))


def num_threads():
    return lib().orc_num_threads()


def set_num_threads(n):
    lib().orc_set_num_threads(C.c_int(n))


def m31_mul(a, b):
    return lib().orc_m31_mul(a, b)


def m31_inv(a):
    return lib().orc_m31_inv(a)


def qm31_mul(a, b):
    a, pa = _u32(a); b, pb = _u32(b)
    out = np.zeros(4, np.uint32)
    lib().orc_qm31_mul(pa, pb, out.ctypes.data_as(u32p))
    return out


def qm31_inv(a):
    a, pa = _u32(a)
    out = np.zeros(4, np.uint32)
    lib().orc_qm31_inv(pa, out.ctypes.data_as(u32p))
    return out


def circle_domain_at(log_size, i):
    out = np.zeros(2, np.uint32)
    lib().orc_circle_domain_at(C.c_uint32(log_size), C.c_uint64(i), out.ctypes.data_as(u32p))
    return int(out[0]), int(out[1])


def bit_reverse_index(i, log_size):
    return lib().orc_bit_reverse_index(i, log_size)


def coset_index_to_circle_domain_index(i, log_size):
    return lib().orc_coset_index_to_circle_domain_index(i, log_size)


def finalize_column(col):
    col, p = _u32(col)
    log = int(col.size).bit_length() - 1
    out = np.empty_like(col)
    lib().orc_finalize_column(p, C.c_uint32(log), out.ctypes.data_as(u32p))
    return out


def twiddles(domain_log):
    n = 1 << (domain_log - 1)
    tw = np.empty(n, np.uint32); itw = np.empty(n, np.uint32)
    lib().orc_twiddles(C.c_uint32(domain_log), tw.ctypes.data_as(u32p), itw.ctypes.data_as(u32p))
    return tw, itw


def interpolate(evals):
    evals, p = _u32(evals)
    log = int(evals.size).bit_length() - 1
    out = np.empty_like(evals)
    lib().orc_interpolate(C.c_uint32(log), p, out.ctypes.data_as(u32p))
    return out


def evaluate(coeffs, domain_log):
    coeffs, p = _u32(coeffs)
    log = int(coeffs.size).bit_length() - 1
    out = np.empty(1 << domain_log, np.uint32)
    lib().orc_evaluate(C.c_uint32(log), C.c_uint32(domain_log), p, out.ctypes.data_as(u32p))
    return out


def interpolate_evaluate_batch(evals2d, log_blowup, want_coeffs=False):
    """evals2d: (n_cols, 2^log) uint32.  Returns (coeffs or None, lde (n_cols, 2^(log+blowup)))."""
    evals2d = np.ascontiguousarray(evals2d, dtype=np.uint32)
    n_cols, n = evals2d.shape
    log = int(n).bit_length() - 1
    lde = np.empty((n_cols, n << log_blowup), np.uint32)
    co = np.empty_like(evals2d) if want_coeffs else None
    lib().orc_interpolate_evaluate_batch(C.c_uint32(log), C.c_uint32(log_blowup), C.c_size_t(n_cols),
                                         evals2d.ctypes.data_as(u32p),
                                         co.ctypes.data_as(u32p) if want_coeffs else None,
                                         lde.ctypes.data_as(u32p))
    return co, lde


def eval_at_point(coeffs, px, py):
    coeffs, p = _u32(coeffs)
    log = int(coeffs.size).bit_length() - 1
    px, ppx = _u32(px); py, ppy = _u32(py)
    out = np.zeros(4, np.uint32)
    lib().orc_eval_at_point(C.c_uint32(log), p, ppx, ppy, out.ctypes.data_as(u32p))
    return out


def blake2s(data: bytes) -> bytes:
    out = (C.c_uint8 * 32)()
    buf = (C.c_uint8 * max(1, len(data))).from_buffer_copy(data if data else b"\0")
    lib().orc_blake2s(buf, C.c_size_t(len(data)), out)
    return bytes(out)


def blake2s_compress(h, m, t0=0, t1=0, f0=0, f1=0):
    h = np.array(h, dtype=np.uint32).copy()
    m, pm = _u32(m)
    lib().orc_blake2s_compress(h.ctypes.data_as(u32p), pm, C.c_uint32(t0), C.c_uint32(t1), C.c_uint32(f0), C.c_uint32(f1))
    return h


def _col_ptrs(cols):
    cols = [np.ascontiguousarray(c, dtype=np.uint32) for c in cols]
    arr = (u32p * len(cols))(*[c.ctypes.data_as(u32p) for c in cols])
    logs = np.array([int(c.size).bit_length() - 1 for c in cols], dtype=np.uint32)
    return cols, arr, logs


def merkle_commit(cols, want_layers=False):
    """cols: list of uint32 arrays (power-of-two lengths, any mix).  Returns root bytes (and layers root->leaves)."""
    cols, arr, logs = _col_ptrs(cols)
    root = (C.c_uint8 * 32)()
    layers = None
    if want_layers:
        max_log = int(logs.max()) if len(cols) else 0
        layers = np.zeros(((2 << max_log) - 1) * 32, np.uint8)
    lib().orc_merkle_commit(C.c_size_t(len(cols)), arr, logs.ctypes.data_as(u32p), root,
                            layers.ctypes.data_as(u8p) if want_layers else None)
    if want_layers:
        return bytes(root), layers
    return bytes(root)


def merkle_decommit(cols, queries):
    """queries: dict log_size -> sorted positions.  Returns (queried_values, hash_witness bytes list, column_witness)."""
    cols, arr, logs = _col_ptrs(cols)
    ks = sorted(queries.keys())
    qls = np.array(ks, dtype=np.uint32)
    cnt = np.array([len(queries[k]) for k in ks], dtype=np.uint64)
    pos = np.array([p for k in ks for p in queries[k]], dtype=np.uint64)
    total_cols = len(cols)
    cap = max(1, int(cnt.sum())) * (total_cols + 64) * 64
    qv = np.zeros(cap, np.uint32); hw = np.zeros(cap * 32, np.uint8); cw = np.zeros(cap, np.uint32)
    nq = C.c_size_t(); nh = C.c_size_t(); nc = C.c_size_t()
    lib().orc_merkle_decommit(C.c_size_t(len(cols)), arr, logs.ctypes.data_as(u32p),
                              C.c_size_t(len(ks)), qls.ctypes.data_as(u32p), cnt.ctypes.data_as(u64p), pos.ctypes.data_as(u64p),
                              qv.ctypes.data_as(u32p), C.byref(nq), hw.ctypes.data_as(u8p), C.byref(nh), cw.ctypes.data_as(u32p), C.byref(nc))
    return qv[:nq.value].copy(), [bytes(hw[32 * i:32 * i + 32]) for i in range(nh.value)], cw[:nc.value].copy()


class Channel:
    def __init__(self):
        self._h = C.c_void_p(lib().orc_channel_new())

    def __del__(self):
        try:
            lib().orc_channel_free(self._h)
        except Exception:
            pass

    def digest(self):
        out = (C.c_uint8 * 32)(); lib().orc_channel_digest(self._h, out); return bytes(out)

    def mix_u64(self, v):
        lib().orc_channel_mix_u64(self._h, C.c_uint64(v))

    def mix_u32s(self, words):
        w, p = _u32(words); lib().orc_channel_mix_u32s(self._h, p, C.c_size_t(w.size))

    def mix_felts(self, felts):
        f, p = _u32(np.asarray(felts).reshape(-1)); lib().orc_channel_mix_felts(self._h, p, C.c_size_t(f.size // 4))

    def mix_root(self, root: bytes):
        lib().orc_channel_mix_root(self._h, (C.c_uint8 * 32).from_buffer_copy(root))

    def draw_felt(self):
        out = np.zeros(4, np.uint32); lib().orc_channel_draw_felt(self._h, out.ctypes.data_as(u32p)); return out

    def draw_felts(self, n):
        out = np.zeros((n, 4), np.uint32); lib().orc_channel_draw_felts(self._h, C.c_size_t(n), out.ctypes.data_as(u32p)); return out

    def draw_random_bytes(self):
        out = (C.c_uint8 * 32)(); lib().orc_channel_draw_random_bytes(self._h, out); return bytes(out)


def _clone_channel(ch):
    c = Channel.__new__(Channel)
    lib().orc_channel_clone.restype = C.c_void_p
    c._h = C.c_void_p(lib().orc_channel_clone(ch._h))
    return c


Channel.clone = _clone_channel


def last_error():
    lib().orc_last_error.restype = C.c_char_p
    return lib().orc_last_error().decode()


class OracleError(RuntimeError):
    pass


def _component_eval_log(words, comp):
    """log_size + log_expand of component `comp`, read from the AIR bytecode (layout: nexus_zkvm_b200/air.py)."""
    w = [int(x) for x in words]
    i = 4
    for k in range(w[3]):
        if k == comp:
            return w[i] + w[i + 1]
        i += 3
        i += 1 + 3 * w[i] + 2            # masks, register counts
        i += 1 + 4 * w[i]                # constraint program
        n_fracs = w[i]
        i += 3
        i += 1 + 4 * w[i]                # logup program
        i += n_fracs + 2
    raise IndexError(comp)


class Prover:
    """Oracle restatement of CommitmentSchemeProver + stwo::prover::prove over a bytecode AIR."""

    def __init__(self, air_words):
        self.air_words = np.ascontiguousarray(air_words, dtype=np.uint32)
        lib().orc_prover_new.restype = C.c_void_p
        h = lib().orc_prover_new(self.air_words.ctypes.data_as(u32p), C.c_size_t(self.air_words.size))
        if not h:
            raise OracleError(last_error())
        self._h = C.c_void_p(h)

    def __del__(self):
        try:
            lib().orc_prover_free(self._h)
        except Exception:
            pass

    def commit(self, cols, channel, log_blowup=1):
        cols, arr, logs = _col_ptrs(cols)
        root = (C.c_uint8 * 32)()
        st = lib().orc_prover_commit(self._h, channel._h, C.c_size_t(len(cols)), arr, logs.ctypes.data_as(u32p), C.c_uint32(log_blowup), root)
        if st:
            raise OracleError(last_error())
        return bytes(root)

    def gen_interaction(self, comp, log_size, n_logup_cols, params):
        params = np.ascontiguousarray(params, dtype=np.uint32).reshape(-1, 4)
        out = np.zeros((4 * n_logup_cols, 1 << log_size), np.uint32)
        claimed = np.zeros(4, np.uint32)
        st = lib().orc_prover_gen_interaction(self._h, C.c_uint32(comp), params.ctypes.data_as(u32p), C.c_size_t(params.shape[0]),
                                              out.ctypes.data_as(u32p), claimed.ctypes.data_as(u32p))
        if st:
            raise OracleError(last_error())
        return out, tuple(int(x) for x in claimed)

    def prove(self, channel, params, pow_bits=5, log_blowup=1, log_last=0, n_queries=3):
        params = np.ascontiguousarray(params, dtype=np.uint32).reshape(-1, 4)
        cap = 1 << 26
        buf = (C.c_uint8 * cap)()
        ln = C.c_size_t()
        st = lib().orc_prover_prove(self._h, channel._h, params.ctypes.data_as(u32p), C.c_size_t(params.shape[0]),
                                    C.c_uint32(pow_bits), C.c_uint32(log_blowup), C.c_uint32(log_last), C.c_uint32(n_queries),
                                    buf, C.c_size_t(cap), C.byref(ln))
        if st:
            raise OracleError(f"prove failed ({st}): {last_error()}")
        return bytes(buf[:ln.value])

    def constraint_quotients(self, comp, eval_log, params, coeffs, accum=None):
        """ComponentProver::evaluate_constraint_quotients_on_domain for one component on CanonicCoset(eval_log).circle_domain(); returns
        accum (4 x 2^eval_log) + quotients.  eval_log=None is the component's own domain (log_size + log_expand, where the prover evaluates);
        any eval_log > log_size gives the same quotient polynomial elsewhere, e.g. on the committed LDE domain."""
        params = np.ascontiguousarray(params, dtype=np.uint32).reshape(-1, 4)
        coeffs = np.ascontiguousarray(coeffs, dtype=np.uint32).reshape(-1, 4)
        if eval_log is None:
            eval_log = _component_eval_log(self.air_words, comp)
        acc = np.zeros((4, 1 << eval_log), np.uint32) if accum is None else np.ascontiguousarray(accum, dtype=np.uint32).copy()
        if acc.shape != (4, 1 << eval_log):
            raise OracleError(f"constraint quotients: accumulator shape {acc.shape}, want (4, {1 << eval_log})")
        st = lib().orc_prover_constraint_quotients(self._h, C.c_uint32(comp), C.c_uint32(eval_log), params.ctypes.data_as(u32p),
                                                   C.c_size_t(params.shape[0]), coeffs.ctypes.data_as(u32p), acc.ctypes.data_as(u32p))
        if st:
            raise OracleError(last_error())
        return acc


def fold_line(src, alpha):
    """FriOps::fold_line; src = 4 x 2^k coordinate columns on LineDomain(Coset::half_odds(k))."""
    src = np.ascontiguousarray(src, dtype=np.uint32)
    k = src.shape[1].bit_length() - 1
    out = np.zeros((4, src.shape[1] // 2), np.uint32)
    lib().orc_fold_line(C.c_uint32(k), src.ctypes.data_as(u32p), _u32(alpha)[1], out.ctypes.data_as(u32p))
    return out


def fold_circle_into_line(dst, src, alpha):
    """FriOps::fold_circle_into_line; returns the new dst (dst * alpha^2 + fold(src))."""
    src = np.ascontiguousarray(src, dtype=np.uint32)
    out = np.ascontiguousarray(dst, dtype=np.uint32).copy()
    k = src.shape[1].bit_length() - 1
    lib().orc_fold_circle_into_line(C.c_uint32(k), out.ctypes.data_as(u32p), src.ctypes.data_as(u32p), _u32(alpha)[1])
    return out


def accumulate_quotients(cols, random_coeff, batches):
    """QuotientOps::accumulate_quotients.  cols: equal-length columns; batches: [(point8, [(col_index, value4), ...]), ...]."""
    cols, arr, logs = _col_ptrs(cols)
    log_size = int(logs[0])
    pts = np.ascontiguousarray([b[0] for b in batches], dtype=np.uint32).reshape(-1, 8)
    first, count, ecols, evals = [], [], [], []
    for _pt, ents in batches:
        first.append(len(ecols)); count.append(len(ents))
        for ci, v in ents:
            ecols.append(ci); evals.append(v)
    first = np.array(first, np.uint64); count = np.array(count, np.uint64)
    ecols = np.array(ecols, np.uint32); evals = np.ascontiguousarray(evals, dtype=np.uint32).reshape(-1, 4)
    out = np.zeros((4, 1 << log_size), np.uint32)
    u64p = C.POINTER(C.c_uint64)
    lib().orc_accumulate_quotients(C.c_uint32(log_size), C.c_size_t(len(cols)), arr, _u32(random_coeff)[1],
                                   C.c_size_t(len(batches)), pts.ctypes.data_as(u32p), first.ctypes.data_as(u64p), count.ctypes.data_as(u64p),
                                   ecols.ctypes.data_as(u32p), evals.ctypes.data_as(u32p), out.ctypes.data_as(u32p))
    return out


def grind(digest: bytes, pow_bits):
    lib().orc_grind.restype = C.c_uint64
    return int(lib().orc_grind((C.c_uint8 * 32).from_buffer_copy(digest), C.c_uint32(pow_bits)))


def bit_reverse_column(col):
    out = np.ascontiguousarray(col, dtype=np.uint32).copy()
    lib().orc_bit_reverse_column(out.ctypes.data_as(u32p), C.c_uint32(out.size.bit_length() - 1))
    return out


def verify(air_words, params, proof_bytes, channel, col_logs):
    """col_logs: [tree0 logs, tree1 logs, tree2 logs].  Raises OracleError on rejection."""
    air_words = np.ascontiguousarray(air_words, dtype=np.uint32)
    params = np.ascontiguousarray(params, dtype=np.uint32).reshape(-1, 4)
    ncols = np.array([len(x) for x in col_logs], dtype=np.uint32)
    flat = np.array([l for t in col_logs for l in t], dtype=np.uint32)
    buf = (C.c_uint8 * len(proof_bytes)).from_buffer_copy(proof_bytes)
    st = lib().orc_verify(air_words.ctypes.data_as(u32p), C.c_size_t(air_words.size), params.ctypes.data_as(u32p), C.c_size_t(params.shape[0]),
                          buf, C.c_size_t(len(proof_bytes)), channel._h, ncols.ctypes.data_as(u32p), flat.ctypes.data_as(u32p))
    if st:
        raise OracleError(last_error())
