"""nexus_zkvm_b200 — H100-native (sm_90a) STARK proving backend for the Nexus zkVM hot path.

Python is only the test/bench harness: a ctypes binding of the C ABI in include/nb200.h (libnexus_b200.so,
hand-written CUDA for sm_90a + C++ host library).  The names mirror the Stwo backend surface the reference
calls (PolyOps.interpolate / evaluate / eval_at_point, MerkleProver.commit / decommit, TreeBuilder.extend_evals
+ commit — nexus-zkvm prover/src/machine.rs:186-290).

There is NO CPU fallback: if the library is missing or there is no CUDA device, construction raises.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libnexus_b200.so")
_LIB = None

u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)
u8p = C.POINTER(C.c_uint8)


class Nb200Error(RuntimeError):
    pass


def lib():
    """Load libnexus_b200.so; fail loudly when it has not been built (no fallback path exists)."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise Nb200Error(f"{LIB_PATH} is missing: run `python -m nexus_zkvm_b200.build` "
                             "(the product path has no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        L.nb200_last_error.restype = C.c_char_p
        L.nb200_last_error.argtypes = [C.c_void_p]
        L.nb200_launch_count.restype = C.c_uint64
        L.nb200_launch_count.argtypes = [C.c_void_p]
        L.nb200_cols_count.restype = C.c_size_t
        L.nb200_cols_count.argtypes = [C.c_void_p]
        L.nb200_cols_log_size.restype = C.c_uint32
        L.nb200_cols_log_size.argtypes = [C.c_void_p]
        L.nb200_cols_device_ptr.restype = C.c_void_p
        L.nb200_cols_device_ptr.argtypes = [C.c_void_p]
        L.nb200_twiddles_domain_log.restype = C.c_uint32
        L.nb200_twiddles_domain_log.argtypes = [C.c_void_p]
        L.nb200_tree_log_size.restype = C.c_uint32
        L.nb200_tree_log_size.argtypes = [C.c_void_p]
        L.nb200_free.argtypes = [C.c_void_p]
        L.nb200_cols_free.argtypes = [C.c_void_p, C.c_void_p]
        L.nb200_tree_free.argtypes = [C.c_void_p, C.c_void_p]
        L.nb200_ctx_destroy.argtypes = [C.c_void_p]
        _LIB = L
    return _LIB


def exported_symbols():
    """Every entry point include/nb200.h declares (used by the CPU-side ABI test)."""
    import re
    hdr = open(os.path.join(_HERE, "..", "include", "nb200.h")).read()
    return sorted(set(re.findall(r"\b(nb200_[a-z0-9_]+)\s*\(", hdr)) - {"nb200_status"})


class Context:
    """One GPU.  Mirrors `CommitmentSchemeProver::<B, MC>::new(config, &twiddles)` ownership: twiddles live here."""

    def __init__(self, device=0, stream=None):
        self._h = C.c_void_p()
        st = lib().nb200_ctx_create(C.c_int(device), C.byref(self._h))
        if st != 0:
            raise Nb200Error(f"nb200_ctx_create failed ({st}): {lib().nb200_last_error(None).decode()}")
        self._pinned = []
        if stream is not None:
            self._chk(lib().nb200_ctx_set_stream(self._h, C.c_void_p(stream)))

    def _chk(self, st):
        if st != 0:
            raise Nb200Error(f"nb200 status {st}: {lib().nb200_last_error(self._h).decode()}")

    def close(self):
        if self._h:
            lib().nb200_ctx_destroy(self._h)
            self._h = C.c_void_p()
            for p, _buf in self._pinned:
                lib().nb200_host_free(p)
            self._pinned = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sync(self):
        self._chk(lib().nb200_sync(self._h))

    def set_flavor(self, merkle_hash=0, draw_domain_sep=0, pow_variant=0):
        self._chk(lib().nb200_set_flavor(self._h, C.c_int(merkle_hash), C.c_int(draw_domain_sep), C.c_int(pow_variant)))

    @property
    def launches(self):
        return int(lib().nb200_launch_count(self._h))

    # ---- columns
    def alloc(self, n_cols, log_size):
        h = C.c_void_p()
        self._chk(lib().nb200_cols_alloc(self._h, C.c_size_t(n_cols), C.c_uint32(log_size), C.byref(h)))
        return Columns(self, h)

    def wrap_device(self, device_ptr, n_cols, log_size):
        """Non-owning batch over caller-owned device memory (e.g. a torch tensor's data_ptr())."""
        h = C.c_void_p()
        self._chk(lib().nb200_cols_from_device(self._h, C.c_void_p(device_ptr), C.c_size_t(n_cols), C.c_uint32(log_size), C.byref(h)))
        return Columns(self, h)

    def upload(self, host2d, coset_order=False):
        """host2d: (n_cols, 2^log) uint32, one row per column."""
        a = np.ascontiguousarray(host2d, dtype=np.uint32)
        if a.ndim == 1:
            a = a[None, :]
        log = int(a.shape[1]).bit_length() - 1
        assert a.shape[1] == 1 << log
        cols = self.alloc(a.shape[0], log)
        self._chk(lib().nb200_cols_upload(self._h, cols._h, C.c_size_t(0), C.c_size_t(a.shape[0]),
                                          a.ctypes.data_as(u32p), C.c_int(1 if coset_order else 0)))
        return cols

    # ---- PolyOps
    def precompute_twiddles(self, max_domain_log):
        self._chk(lib().nb200_twiddles_prepare(self._h, C.c_uint32(max_domain_log)))

    def twiddles(self, max_domain_log):
        self.precompute_twiddles(max_domain_log)
        # the cached bank may be larger than requested: every smaller domain's buffer is its suffix
        have = int(lib().nb200_twiddles_domain_log(self._h))
        n = 1 << (have - 1)
        tw = np.empty(n, np.uint32); itw = np.empty(n, np.uint32)
        self._chk(lib().nb200_twiddles_download(self._h, tw.ctypes.data_as(u32p), itw.ctypes.data_as(u32p)))
        want = 1 << (max_domain_log - 1)
        return tw[n - want:], itw[n - want:]

    def interpolate(self, cols):
        """In place: evaluations (bit-reversed circle-domain order) -> coefficients."""
        self._chk(lib().nb200_interpolate(self._h, cols._h))
        return cols

    def evaluate(self, coeffs, log_blowup):
        out = self.alloc(coeffs.n_cols, coeffs.log_size + log_blowup)
        self._chk(lib().nb200_evaluate(self._h, coeffs._h, C.c_uint32(log_blowup), out._h))
        return out

    def interpolate_evaluate(self, evals, log_blowup, coeffs=None, lde=None):
        """evals -> (coeffs, lde) without touching evals (nb200_interpolate_evaluate)."""
        coeffs = coeffs or self.alloc(evals.n_cols, evals.log_size)
        lde = lde or self.alloc(evals.n_cols, evals.log_size + log_blowup)
        self._chk(lib().nb200_interpolate_evaluate(self._h, evals._h, C.c_uint32(log_blowup), coeffs._h, lde._h))
        return coeffs, lde

    def eval_at_points(self, coeffs, points):
        """points: (n_points, 2, 4) uint32 = (x, y) QM31 pairs.  Returns (n_cols, n_points, 4)."""
        pts = np.ascontiguousarray(points, dtype=np.uint32).reshape(-1, 8)
        out = np.zeros((coeffs.n_cols, pts.shape[0], 4), np.uint32)
        self._chk(lib().nb200_eval_at_points(self._h, coeffs._h, pts.ctypes.data_as(u32p), C.c_size_t(pts.shape[0]),
                                             out.ctypes.data_as(u32p)))
        return out

    # ---- MerkleOps
    def merkle_commit(self, batches):
        arr = (C.c_void_p * len(batches))(*[b._h for b in batches])
        t = C.c_void_p()
        root = (C.c_uint8 * 32)()
        self._chk(lib().nb200_merkle_commit(self._h, arr, C.c_size_t(len(batches)), C.byref(t), root))
        return MerkleTree(self, t, bytes(root), list(batches))

    def host_alloc(self, n_cols, log_size):
        """Pinned host memory for a block of trace columns, as an (n_cols, 2^log_size) uint32 numpy array."""
        n = n_cols << log_size
        p = C.c_void_p()
        st = lib().nb200_host_alloc(C.c_size_t(4 * max(n, 1)), C.byref(p))
        if st:
            raise Nb200Error(f"nb200_host_alloc failed ({st})")
        buf = (C.c_uint32 * max(n, 1)).from_address(p.value)
        arr = np.ctypeslib.as_array(buf)[:n].reshape(n_cols, 1 << log_size)
        self._pinned.append((p, buf))
        return arr

    def host_alloc_bytes(self, n_bytes):
        """Pinned host memory as a flat uint8 array (the packed host formats of nb200_commit_host_packed)."""
        p = C.c_void_p()
        if lib().nb200_host_alloc(C.c_size_t(n_bytes), C.byref(p)) != 0:
            raise Nb200Error("nb200_host_alloc failed")
        buf = (C.c_uint8 * n_bytes).from_address(p.value)
        arr = np.frombuffer(buf, dtype=np.uint8)
        self._pinned.append((p, arr))
        return arr

    def commit_host_packed(self, host_batches, log_sizes, log_blowup, coset_order=False):
        """nb200_commit_host_packed: host_batches are 2-D uint8 / uint16 / uint32 arrays (n_cols x 2^log_size)."""
        n = len(host_batches)
        hb = [np.ascontiguousarray(h) if not h.flags["C_CONTIGUOUS"] else h for h in host_batches]
        ptrs = (C.c_void_p * n)(*[h.ctypes.data for h in hb])
        eb = (C.c_uint32 * n)(*[h.dtype.itemsize for h in hb])
        ncols = (C.c_size_t * n)(*[h.shape[0] for h in hb])
        logs = (C.c_uint32 * n)(*[int(x) for x in log_sizes])
        ev, co, ld = (C.c_void_p * n)(), (C.c_void_p * n)(), (C.c_void_p * n)()
        tree = C.c_void_p()
        root = (C.c_uint8 * 32)()
        self._chk(lib().nb200_commit_host_packed(self._h, ptrs, eb, ncols, logs, C.c_size_t(n), C.c_int(1 if coset_order else 0), C.c_uint32(log_blowup),
                                                 ev, co, ld, C.byref(tree), root))
        self.sync()
        evals = [Columns(self, C.c_void_p(ev[i])) for i in range(n)]
        coeffs = [Columns(self, C.c_void_p(co[i])) for i in range(n)]
        ldes = [Columns(self, C.c_void_p(ld[i])) for i in range(n)]
        return evals, coeffs, ldes, MerkleTree(self, tree, bytes(root), ldes)

    def commit_host(self, host_batches, log_blowup, coset_order=False, evals=None, coeffs=None, ldes=None):
        """Commit from HOST batches (2-D uint32 arrays; pinned for copy/compute overlap): returns (evals, coeffs, ldes, tree)."""
        n = len(host_batches)
        hb = [np.ascontiguousarray(b, dtype=np.uint32) for b in host_batches]
        ptrs = (u32p * n)(*[b.ctypes.data_as(u32p) for b in hb])
        ncols = (C.c_size_t * n)(*[b.shape[0] for b in hb])
        logs = (C.c_uint32 * n)(*[int(b.shape[1]).bit_length() - 1 for b in hb])
        ev = (C.c_void_p * n)(*([b._h for b in evals] if evals else [None] * n))
        co = (C.c_void_p * n)(*([b._h for b in coeffs] if coeffs else [None] * n))
        ld = (C.c_void_p * n)(*([b._h for b in ldes] if ldes else [None] * n))
        t = C.c_void_p()
        root = (C.c_uint8 * 32)()
        self._chk(lib().nb200_commit_host(self._h, ptrs, ncols, logs, C.c_size_t(n), C.c_int(1 if coset_order else 0), C.c_uint32(log_blowup),
                                          ev, co, ld, C.byref(t), root))
        if evals is None:
            evals = [Columns(self, C.c_void_p(ev[i])) for i in range(n)]
        if coeffs is None:
            coeffs = [Columns(self, C.c_void_p(co[i])) for i in range(n)]
        if ldes is None:
            ldes = [Columns(self, C.c_void_p(ld[i])) for i in range(n)]
        return evals, coeffs, ldes, MerkleTree(self, t, bytes(root), ldes)

    def keccak_main_trace(self, inputs, addresses, timestamps):
        """nb200_keccak_main_trace: tree 1 of the keccak extension filled on the device from its side note (inputs: (n_perms, 25) uint64
        lanes, addresses: (n_perms,) uint32, timestamps: (n_perms, 200) uint32).  Returns its five device batches in commitment order."""
        inp = np.ascontiguousarray(inputs, dtype=np.uint64)
        addr = np.ascontiguousarray(addresses, dtype=np.uint32)
        ts = np.ascontiguousarray(timestamps, dtype=np.uint32)
        n = inp.shape[0] if inp.ndim == 2 else 0
        assert inp.shape == (n, 25) and addr.shape == (n,) and ts.shape == (n, 200), "side note shapes"
        out = (C.c_void_p * 5)()
        self._chk(lib().nb200_keccak_main_trace(self._h, C.c_size_t(n), inp.ctypes.data_as(u64p), addr.ctypes.data_as(u32p),
                                                ts.ctypes.data_as(u32p), out))
        return [Columns(self, C.c_void_p(out[i])) for i in range(5)]

    def ram_init_final_trace(self, inputs, addresses, timestamps, init_addresses, init_values, log_size, out=None):
        """nb200_ram_init_final_trace: RamInitFinal's 10 main columns in finalized order, filled on the device from the keccak side note (as
        keccak_main_trace takes it) and the public initial memory (init_addresses: (n_init,) uint32, strictly ascending; init_values:
        (n_init,) bytes).  `out`: a batch of 10 columns of 2^log_size rows to overwrite (default: a new one).  Returns (out, number of
        distinct addresses)."""
        inp = np.ascontiguousarray(inputs, dtype=np.uint64)
        addr = np.ascontiguousarray(addresses, dtype=np.uint32)
        ts = np.ascontiguousarray(timestamps, dtype=np.uint32)
        n = inp.shape[0] if inp.ndim == 2 else 0
        assert inp.shape == (n, 25) and addr.shape == (n,) and ts.shape == (n, 200), "side note shapes"
        ia = np.ascontiguousarray(init_addresses, dtype=np.uint32)
        iv = np.ascontiguousarray(init_values, dtype=np.uint8)
        assert ia.shape == iv.shape and ia.ndim == 1, "initial memory shapes"
        if out is None:
            out = self.alloc(10, log_size)
        n_rows = C.c_size_t()
        self._chk(lib().nb200_ram_init_final_trace(self._h, C.c_size_t(n), inp.ctypes.data_as(u64p), addr.ctypes.data_as(u32p), ts.ctypes.data_as(u32p),
                                                   C.c_size_t(ia.size), ia.ctypes.data_as(u32p), iv.ctypes.data_as(u8p), C.c_uint32(log_size),
                                                   out._h, C.byref(n_rows)))
        return out, int(n_rows.value)

    def v1_main_trace(self, steps, final_ctr, log_size, out=None):
        """nb200_v1_main_trace: the v1 main component's 347 columns in finalized order, filled on the device from an ADD / ADDI program's
        step record (steps: (13, n_steps) uint32 in add_chain.STEP_FIELDS order) and the final execution count of each program row
        (final_ctr: (n_prog,) uint32).  `out`: a batch of 347 columns of 2^log_size rows to overwrite (default: a new one).  Returns out."""
        st = np.ascontiguousarray(steps, dtype=np.uint32)
        ctr = np.ascontiguousarray(final_ctr, dtype=np.uint32)
        assert st.ndim == 2 and st.shape[0] == 13 and ctr.ndim == 1, "step record shapes"
        if out is None:
            out = self.alloc(347, log_size)
        self._chk(lib().nb200_v1_main_trace(self._h, C.c_size_t(st.shape[1]), st.ctypes.data_as(u32p), C.c_size_t(ctr.size), ctr.ctypes.data_as(u32p),
                                            C.c_uint32(log_size), out._h))
        return out

    def v1_alu_trace(self, steps, final_ctr, log_size, out=None):
        """nb200_v1_alu_trace: v1_main_trace for a program of the 19 ALU opcodes of add_chain.OPCODES (ADD ... SRAI), same arguments and
        step record.  Returns out."""
        st = np.ascontiguousarray(steps, dtype=np.uint32)
        ctr = np.ascontiguousarray(final_ctr, dtype=np.uint32)
        assert st.ndim == 2 and st.shape[0] == 13 and ctr.ndim == 1, "step record shapes"
        if out is None:
            out = self.alloc(347, log_size)
        self._chk(lib().nb200_v1_alu_trace(self._h, C.c_size_t(st.shape[1]), st.ctypes.data_as(u32p), C.c_size_t(ctr.size), ctr.ctypes.data_as(u32p),
                                           C.c_uint32(log_size), out._h))
        return out

    def v1_control_trace(self, steps, final_ctr, log_size, out=None):
        """nb200_v1_control_trace: v1_alu_trace for a looping program of those 19 opcodes and the branches, JAL, JALR, LUI and AUIPC of
        add_chain.CONTROL_OPCODES (opcodes 19-28), same arguments and step record; final_ctr holds each program row's execution count.
        Returns out."""
        st = np.ascontiguousarray(steps, dtype=np.uint32)
        ctr = np.ascontiguousarray(final_ctr, dtype=np.uint32)
        assert st.ndim == 2 and st.shape[0] == 13 and ctr.ndim == 1, "step record shapes"
        if out is None:
            out = self.alloc(347, log_size)
        self._chk(lib().nb200_v1_control_trace(self._h, C.c_size_t(st.shape[1]), st.ctypes.data_as(u32p), C.c_size_t(ctr.size),
                                               ctr.ctypes.data_as(u32p), C.c_uint32(log_size), out._h))
        return out

    def table_multiplicities(self, air, tree0, tree1, first_row=False):
        """nb200_table_multiplicities: every table fraction's multiplicity column of `tree1` (device batches, finalized order) is overwritten
        with the count of the AIR's lookups into it.  `air` is a loaded AIR (prover.Air).  Returns (n_unmatched, first_unmatched), the latter
        (component, fraction, row in trace order) of the smallest unmatched lookup, or None.  `first_row`: nb200_table_multiplicities_first_row,
        which credits a tuple listed by several table rows of one relation to the first of them and writes 0 into the others, and also
        returns the number of rows written as 0: (n_unmatched, first_unmatched, n_repeated)."""
        t0 = (C.c_void_p * max(len(tree0), 1))(*[b._h for b in tree0])
        t1 = (C.c_void_p * max(len(tree1), 1))(*[b._h for b in tree1])
        n = C.c_uint64()
        first = (C.c_uint32 * 3)()
        if first_row:
            rep = C.c_uint64()
            self._chk(lib().nb200_table_multiplicities_first_row(self._h, air._h, t0, C.c_size_t(len(tree0)), t1, C.c_size_t(len(tree1)), C.byref(n),
                                                                 first, C.byref(rep)))
        else:
            self._chk(lib().nb200_table_multiplicities(self._h, air._h, t0, C.c_size_t(len(tree0)), t1, C.c_size_t(len(tree1)), C.byref(n), first))
        out = int(n.value), (None if n.value == 0 else tuple(int(x) for x in first))
        return out + (int(rep.value),) if first_row else out

    # ---- multi-GPU (one process per GPU): NCCL communicator inside the library
    @staticmethod
    def comm_unique_id():
        n = lib().nb200_comm_unique_id_bytes()
        buf = (C.c_uint8 * n)()
        if lib().nb200_comm_get_unique_id(buf) != 0:
            raise Nb200Error("nb200_comm_get_unique_id failed: " + lib().nb200_last_error(None).decode())
        return bytes(buf)

    def comm_init(self, rank, world, unique_id):
        self._chk(lib().nb200_comm_init(self._h, C.c_int(rank), C.c_int(world), (C.c_uint8 * len(unique_id)).from_buffer_copy(unique_id)))

    def comm_init_from_torch(self, dist, device):
        """Create the library's communicator for the ranks of a torch.distributed group (the id travels over that group)."""
        import torch
        rank, world = dist.get_rank(), dist.get_world_size()
        n = lib().nb200_comm_unique_id_bytes()
        t = torch.zeros(n, dtype=torch.uint8, device=device)
        if rank == 0:
            t.copy_(torch.frombuffer(bytearray(self.comm_unique_id()), dtype=torch.uint8))
        dist.broadcast(t, 0)
        self.comm_init(rank, world, bytes(t.cpu().numpy().tobytes()))

    @staticmethod
    def shard_range(total_cols, world, rank):
        f, c = C.c_size_t(), C.c_size_t()
        assert lib().nb200_shard_range(C.c_size_t(total_cols), C.c_int(world), C.c_int(rank), C.byref(f), C.byref(c)) == 0
        return int(f.value), int(c.value)

    def commit_sharded(self, shard_evals, total_cols, log_size, log_blowup, replicated=()):
        """nb200_commit_sharded: returns (coeffs of this rank's columns, row-slice batch of all columns, sub-tree, caps, root)."""
        rep = (C.c_void_p * max(len(replicated), 1))(*[b._h for b in replicated])
        co, rows, sub = C.c_void_p(), C.c_void_p(), C.c_void_p()
        world = lib().nb200_comm_world(self._h)
        caps = (C.c_uint8 * (32 * world))()
        root = (C.c_uint8 * 32)()
        self._chk(lib().nb200_commit_sharded(self._h, shard_evals._h if shard_evals is not None else None, C.c_size_t(total_cols), C.c_uint32(log_size),
                                             C.c_uint32(log_blowup), rep, C.c_size_t(len(replicated)), C.byref(co), C.byref(rows), C.byref(sub), caps, root))
        rows_b = Columns(self, rows)
        return Columns(self, co), rows_b, MerkleTree(self, sub, None, [rows_b]), [bytes(caps[32 * i:32 * i + 32]) for i in range(world)], bytes(root)

    def commit_evals(self, eval_batches, log_blowup, coeffs=None, ldes=None):
        """TreeBuilder.extend_evals(evals) + commit(): returns (coeff_batches, lde_batches, tree).
        `coeffs` / `ldes` may be batches from a previous call (reused, no allocation)."""
        n = len(eval_batches)
        arr = (C.c_void_p * n)(*[b._h for b in eval_batches])
        co = (C.c_void_p * n)(*([b._h for b in coeffs] if coeffs else [None] * n))
        lde = (C.c_void_p * n)(*([b._h for b in ldes] if ldes else [None] * n))
        t = C.c_void_p()
        root = (C.c_uint8 * 32)()
        self._chk(lib().nb200_commit_evals(self._h, arr, C.c_size_t(n), C.c_uint32(log_blowup), co, lde, C.byref(t), root))
        if coeffs is None:
            coeffs = [Columns(self, C.c_void_p(co[i])) for i in range(n)]
        if ldes is None:
            ldes = [Columns(self, C.c_void_p(lde[i])) for i in range(n)]
        return coeffs, ldes, MerkleTree(self, t, bytes(root), ldes)


class Columns:
    def __init__(self, ctx, h):
        self.ctx = ctx
        self._h = h

    @property
    def n_cols(self):
        return int(lib().nb200_cols_count(self._h))

    @property
    def log_size(self):
        return int(lib().nb200_cols_log_size(self._h))

    @property
    def device_ptr(self):
        return int(lib().nb200_cols_device_ptr(self._h) or 0)

    def download(self):
        out = np.empty((self.n_cols, 1 << self.log_size), np.uint32)
        self.ctx._chk(lib().nb200_cols_download(self.ctx._h, self._h, C.c_size_t(0), C.c_size_t(self.n_cols), out.ctypes.data_as(u32p)))
        return out

    def upload(self, host2d, coset_order=False):
        a = np.ascontiguousarray(host2d, dtype=np.uint32)
        assert a.shape == (self.n_cols, 1 << self.log_size)
        self.ctx._chk(lib().nb200_cols_upload(self.ctx._h, self._h, C.c_size_t(0), C.c_size_t(self.n_cols),
                                              a.ctypes.data_as(u32p), C.c_int(1 if coset_order else 0)))

    def finalize_order(self):
        self.ctx._chk(lib().nb200_cols_finalize_order(self.ctx._h, self._h))

    def free(self):
        if self._h and self.ctx._h:  # a closed ctx already returned its pool to the driver
            lib().nb200_cols_free(self.ctx._h, self._h)
        self._h = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class MerkleTree:
    def __init__(self, ctx, h, root, batches):
        self.ctx = ctx
        self._h = h
        self.root = root
        self.batches = batches  # keeps the committed columns alive

    @property
    def log_size(self):
        return int(lib().nb200_tree_log_size(self._h))

    def layer(self, layer_log):
        out = np.empty(32 << layer_log, np.uint8)
        self.ctx._chk(lib().nb200_tree_layer_download(self.ctx._h, self._h, C.c_uint32(layer_log), out.ctypes.data_as(u8p)))
        return out

    def decommit(self, queries):
        """queries: dict log_size -> sorted positions. Returns (queried_values, [hash_witness bytes], column_witness)."""
        ks = sorted(queries.keys())
        qls = np.array(ks, dtype=np.uint32)
        cnt = np.array([len(queries[k]) for k in ks], dtype=np.uint64)
        pos = np.array([p for k in ks for p in queries[k]], dtype=np.uint64)
        arr = (C.c_void_p * len(self.batches))(*[b._h for b in self.batches])
        qv = u32p(); hw = u8p(); cw = u32p()
        nq = C.c_size_t(); nh = C.c_size_t(); nc = C.c_size_t()
        self.ctx._chk(lib().nb200_merkle_decommit(self.ctx._h, self._h, arr, C.c_size_t(len(self.batches)),
                                                  qls.ctypes.data_as(u32p), cnt.ctypes.data_as(u64p), pos.ctypes.data_as(u64p), C.c_size_t(len(ks)),
                                                  C.byref(qv), C.byref(nq), C.byref(hw), C.byref(nh), C.byref(cw), C.byref(nc)))
        q = np.ctypeslib.as_array(qv, shape=(max(nq.value, 1),))[:nq.value].copy()
        h = bytes(np.ctypeslib.as_array(hw, shape=(max(nh.value * 32, 1),))[:nh.value * 32])
        c = np.ctypeslib.as_array(cw, shape=(max(nc.value, 1),))[:nc.value].copy()
        for p in (qv, hw, cw):
            lib().nb200_free(C.cast(p, C.c_void_p))
        return q, [h[32 * i:32 * i + 32] for i in range(nh.value)], c

    def free(self):
        if self._h and self.ctx._h:
            lib().nb200_tree_free(self.ctx._h, self._h)
        self._h = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass
