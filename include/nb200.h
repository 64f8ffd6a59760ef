/* nb200.h — C ABI of libnexus_b200.so: the H100 (sm_90a) STARK proving backend that stands in for
 * Stwo's `SimdBackend` behind the Nexus zkVM prover.
 *
 * The reference has no FFI: its boundary is the Rust type parameter `SimdBackend` in
 *   CommitmentSchemeProver::<SimdBackend, Blake2sMerkleChannel>::new   prover/src/machine.rs:202-203
 *   tree_builder.extend_evals(..) / commit(..)                         prover/src/machine.rs:208-263
 *   stwo::prover::prove::<SimdBackend, Blake2sMerkleChannel>           prover/src/machine.rs:286-290
 *   (same surface in prover2/machine/src/prove.rs:53-128).
 * Each entry point below names the Stwo backend-trait method (and the reference call site) it replaces.
 * A Rust shim `struct CudaBackend;` implementing ColumnOps/PolyOps/MerkleOps/QuotientOps/FriOps/
 * AccumulationOps/GrindOps by calling these functions is shown in INTEGRATION.md.
 *
 * Conventions: every function returns nb200_status (0 = OK); no exceptions cross the ABI; host buffers are
 * only borrowed for the duration of a call; a ctx is single-threaded (one ctx per host thread / per GPU).
 * All field elements are canonical M31 values as uint32_t in [0, 2^31-1); a QM31 is 4 consecutive uint32_t;
 * hashes are 32 raw bytes.  Columns are column-major: one contiguous uint32_t[2^log_size] per column, in
 * bit-reversed circle-domain order (the order `finalize_columns` produces, prover/src/trace/utils.rs:94-106).
 */
#ifndef NB200_H
#define NB200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef int nb200_status;
enum {
  NB200_OK = 0,
  NB200_ERR_CUDA = 1,      /* a CUDA runtime call failed (see nb200_last_error) */
  NB200_ERR_ARG = 2,       /* invalid argument */
  NB200_ERR_NO_DEVICE = 3, /* no CUDA device: the product path never falls back to the CPU */
  NB200_ERR_OOM = 4,
  NB200_ERR_CONSTRAINTS = 5, /* ProvingError::ConstraintsNotSatisfied (prover/src/lib.rs:24-31) */
  NB200_ERR_STATE = 6
};

typedef struct nb200_ctx nb200_ctx;   /* one GPU: device, stream, twiddle cache, transcript flavour   */
typedef struct nb200_cols nb200_cols; /* a batch of n_cols device columns of one log_size, contiguous */
typedef struct nb200_tree nb200_tree; /* a device Merkle tree (all layers)                            */

/* ---- context -------------------------------------------------------------------------------------- */
nb200_status nb200_ctx_create(int device, nb200_ctx** out);
void nb200_ctx_destroy(nb200_ctx*);
const char* nb200_last_error(nb200_ctx*); /* also valid with ctx == NULL for create failures */
/* run all work of this ctx on an externally owned cudaStream_t (e.g. torch's current stream) */
nb200_status nb200_ctx_set_stream(nb200_ctx*, void* cuda_stream);
nb200_status nb200_sync(nb200_ctx*);
/* transcript-affecting variants (see DESIGN.md "parity risk switches"); defaults 0,0,0 */
nb200_status nb200_set_flavor(nb200_ctx*, int merkle_hash, int draw_domain_sep, int pow_variant);
/* number of kernel launches issued by this ctx since creation (bench.py's gpu_launches) */
uint64_t nb200_launch_count(nb200_ctx*);

/* ---- columns: ColumnOps / BaseColumn (prover/src/trace/trace_builder.rs:156-164) -------------------- */
nb200_status nb200_cols_alloc(nb200_ctx*, size_t n_cols, uint32_t log_size, nb200_cols** out);
/* non-owning view over caller-owned device memory (n_cols x 2^log_size words, column-major), e.g. a torch tensor */
nb200_status nb200_cols_from_device(nb200_ctx*, void* device_ptr, size_t n_cols, uint32_t log_size, nb200_cols** out);
void nb200_cols_free(nb200_ctx*, nb200_cols*);
size_t nb200_cols_count(const nb200_cols*);
uint32_t nb200_cols_log_size(const nb200_cols*);
void* nb200_cols_device_ptr(const nb200_cols*); /* column c starts at ptr + c * 2^log_size words */
/* host (n x 2^log_size, row = one column) -> device columns [first, first+n).
 * coset_order != 0: the host data is in trace (coset) order and the device applies
 * coset_order_to_circle_domain_order + bit_reverse_column (prover/src/trace/utils.rs:94-106,
 * utils_external.rs:24-39) — SURVEY §8(f1). */
nb200_status nb200_cols_upload(nb200_ctx*, nb200_cols*, size_t first, size_t n, const uint32_t* host, int coset_order);
nb200_status nb200_cols_download(nb200_ctx*, const nb200_cols*, size_t first, size_t n, uint32_t* host);
/* device-to-device: reorder columns already on the device from coset order (in place) */
nb200_status nb200_cols_finalize_order(nb200_ctx*, nb200_cols*);

/* ---- PolyOps (stwo prover/poly/circle/ops.rs) ------------------------------------------------------- */
/* PolyOps::precompute_twiddles(CanonicCoset(max_domain_log).circle_domain().half_coset)
 * — prover/src/machine.rs:186-194.  Idempotent; larger requests replace the cache. */
nb200_status nb200_twiddles_prepare(nb200_ctx*, uint32_t max_domain_log);
/* domain log the cached bank was built for (0 = none) */
uint32_t nb200_twiddles_domain_log(nb200_ctx*);
/* download the twiddle / inverse-twiddle buffers (each 2^(nb200_twiddles_domain_log-1) words) — test hook */
nb200_status nb200_twiddles_download(nb200_ctx*, uint32_t* tw, uint32_t* itw);
/* PolyOps::interpolate_columns: Circle iFFT in place, evaluations on CanonicCoset(log).circle_domain()
 * (bit-reversed) -> coefficients.   Called by TreeBuilder::extend_evals, prover/src/machine.rs:209-215. */
nb200_status nb200_interpolate(nb200_ctx*, nb200_cols* cols);
/* PolyOps::evaluate_polynomials: Circle FFT of the zero-extended coefficients onto
 * CanonicCoset(log+log_blowup).circle_domain() — the LDE inside TreeBuilder::commit, machine.rs:228.
 * `out` must be a batch of the same column count and log_size + log_blowup. */
nb200_status nb200_evaluate(nb200_ctx*, const nb200_cols* coeffs, uint32_t log_blowup, nb200_cols* out);
/* interpolate_columns + evaluate_polynomials in one call — TreeBuilder::extend_evals followed by the LDE of TreeBuilder::commit
 * (machine.rs:209-228) without the Merkle step: evals (read only) -> coeffs (same shape) and lde (log_size + log_blowup).  For
 * 2^16..2^22 rows this runs the fused three-kernel pipeline (csrc/fft_fused.cu); results equal nb200_interpolate + nb200_evaluate. */
nb200_status nb200_interpolate_evaluate(nb200_ctx*, const nb200_cols* evals, uint32_t log_blowup, nb200_cols* coeffs, nb200_cols* lde);
/* PolyOps::eval_at_point for every column of a batch at n_points QM31 circle points:
 * points = n_points x {x[4], y[4]}; out = n_cols x n_points x QM31 (column-major by column). */
nb200_status nb200_eval_at_points(nb200_ctx*, const nb200_cols* coeffs, const uint32_t* points_xy, size_t n_points, uint32_t* out_qm31);

/* ---- MerkleOps<Blake2sMerkleHasher> (stwo prover/vcs/prover.rs, core/vcs/blake2_merkle.rs) ----------- */
/* MerkleProver::commit over any mix of batches (sorted by column length, stable, as upstream):
 * node = H(left || right || values of the columns of this layer's size at this row). */
nb200_status nb200_merkle_commit(nb200_ctx*, const nb200_cols* const* batches, size_t n_batches, nb200_tree** out, uint8_t root[32]);
void nb200_tree_free(nb200_ctx*, nb200_tree*);
uint32_t nb200_tree_log_size(const nb200_tree*);
/* download one layer (log_size 0 = root layer): 32 * 2^layer_log bytes — test hook */
nb200_status nb200_tree_layer_download(nb200_ctx*, const nb200_tree*, uint32_t layer_log, uint8_t* out);
/* MerkleProver::decommit.  queries: for k < n_sizes, q_log_sizes[k] with q_counts[k] sorted positions taken
 * consecutively from q_positions.  Outputs are malloc'ed by the library; free with nb200_free. */
nb200_status nb200_merkle_decommit(nb200_ctx*, const nb200_tree*, const nb200_cols* const* batches, size_t n_batches,
                                   const uint32_t* q_log_sizes, const uint64_t* q_counts, const uint64_t* q_positions, size_t n_sizes,
                                   uint32_t** queried_values, size_t* n_queried,
                                   uint8_t** hash_witness, size_t* n_hashes,
                                   uint32_t** column_witness, size_t* n_column_witness);
/* The walk of nb200_merkle_decommit alone, on the host (no device needed): for a tree of 2^max_log leaves over columns of the given
 * log sizes (the caller's order) and the same queries, the column values it names as n_values (column index, row, queried ? 1 : 0)
 * triples and the hash witness as n_hashes (layer log, node) pairs, in proof order.  Outputs are malloc'ed; free with nb200_free. */
nb200_status nb200_merkle_decommit_plan(uint32_t max_log, const uint32_t* col_log_sizes, size_t n_cols,
                                        const uint32_t* q_log_sizes, const uint64_t* q_counts, const uint64_t* q_positions, size_t n_sizes,
                                        uint64_t** values, size_t* n_values, uint64_t** hashes, size_t* n_hashes);
void nb200_free(void*);
/* Blake2sMerkleHasher::hash_node on the host: H(left || right || values) with the selected construction (0 or 1, see
 * nb200_set_flavor); left/right both NULL for leaves.  Used to combine the Merkle caps of row-sharded sub-trees that
 * the ranks all-gather over NCCL (SURVEY §8e) and by a verifier-side shim. */
nb200_status nb200_hash_node(int merkle_hash, const uint8_t* left, const uint8_t* right, const uint32_t* values, size_t n_values, uint8_t out[32]);

/* ---- fused commitment: TreeBuilder::extend_evals + commit (machine.rs:208-263) ---------------------- */
/* In: evaluation batches (read only).  Out, per batch: the coefficient batch (interpolate) and the LDE batch
 * (log_size + log_blowup); coeffs_io[b] / lde_io[b] may be NULL (allocated by the library, owned by the
 * caller afterwards) or caller-provided batches of the right shape (reused across proofs).  Also the Merkle
 * tree over all LDE columns and its root.  This is the unit bench.py times. */
nb200_status nb200_commit_evals(nb200_ctx*, const nb200_cols* const* eval_batches, size_t n_batches, uint32_t log_blowup,
                                nb200_cols** coeffs_io /* n_batches */, nb200_cols** lde_io /* n_batches */,
                                nb200_tree** tree_out, uint8_t root[32]);

/* ---- host-column entry points: the reference hands over host `Vec<BaseColumn>`s (trace_builder.rs:156-164) ---- */
/* pinned host memory for trace columns (H2D at link speed, and real copy/compute overlap below) */
nb200_status nb200_host_alloc(size_t bytes, void** out);
void nb200_host_free(void*);
/* nb200_commit_evals from HOST columns: batch b is n_cols[b] x 2^log_sizes[b] words at host_batches[b].  Column chunks
 * are copied on a side stream while the previous chunk is transformed; with coset_order != 0 the device also applies
 * finalize_columns.  evals_io / coeffs_io / lde_io as in nb200_commit_evals (NULL entries are allocated). */
nb200_status nb200_commit_host(nb200_ctx*, const uint32_t* const* host_batches, const size_t* n_cols, const uint32_t* log_sizes,
                               size_t n_batches, int coset_order, uint32_t log_blowup, nb200_cols** evals_io, nb200_cols** coeffs_io,
                               nb200_cols** lde_io, nb200_tree** tree_out, uint8_t root[32]);

/* The same with a PACKED host format: batch b holds words of elem_bytes[b] = 1, 2 or 4 bytes (elem_bytes == NULL: all 4).
 * The reference's main trace is byte limbs, flags and 16-bit halves (prover/src/column.rs:22-604) stored as u32 BaseField
 * words; shipping them at their natural width cuts the PCIe payload of a 2^20-row proof from 1.4 GB to 0.36 GB.  The device
 * widens them (and applies finalize_columns when coset_order != 0); values must be canonical (< 2^31 - 1), which every
 * 1- or 2-byte word is. */
nb200_status nb200_commit_host_packed(nb200_ctx*, const void* const* host_batches, const uint32_t* elem_bytes, const size_t* n_cols,
                                      const uint32_t* log_sizes, size_t n_batches, int coset_order, uint32_t log_blowup,
                                      nb200_cols** evals_io, nb200_cols** coeffs_io, nb200_cols** lde_io, nb200_tree** tree_out, uint8_t root[32]);

/* ---- the keccak precompile extension's main trace, filled on the device from its side note ------------------------------------
 * The reference fills tree 1 of keccak_extensions() (prover/src/extensions/keccak/mod.rs:12-33) on the host from KeccakSideNote
 * (prover/src/trace/sidenote/keccak.rs:16-25) and hands over its BaseColumns; here only the side note crosses PCIe:
 *   inputs     = n_perms x 25 input lanes (lane x + 5 y),
 *   addresses  = n_perms base addresses (state byte k is at address + k),
 *   timestamps = n_perms x 200 previous timestamps, one per state byte.
 * Out: five new device batches (owned by the caller, nb200_cols_free) in commitment order and finalized order, ready for
 * nb200_scheme_commit:
 *   out[0] PermutationMemoryCheck, 2001 columns  (memory_check/trace.rs:32-123)
 *   out[1] KeccakRound 0 (rounds 0..15), 1705    (round/trace.rs:297-366)
 *   out[2] KeccakRound 1 (rounds 16..23), 1705
 *   out[3] the XorTable then BitNotAndTable multiplicities, 32 columns of 2^12 rows (bitwise_table/constraints.rs:46-68)
 *   out[4] the BitRotateTable multiplicity, 1 column of 2^11 rows (bit_rotate/mod.rs:69-91)
 * Log sizes: memory check max(log2ceil(n_perms), 4), KeccakRound 0 / 1 max(log2ceil(16 / 8 n_perms), 4) (compute_log_size).  Padding
 * rows of a round component hold the zero state and their lookups are counted; multiplicities are stored mod P.
 * NB200_ERR_ARG: n_perms == 0 or above 2^18 (the multiplicity counters are 32-bit), an address above 2^32 - 200, a timestamp of
 * 2^32 - 1.  Scratch memory (the side note on the device, the histograms) is released in stream order before the call returns. */
nb200_status nb200_keccak_main_trace(nb200_ctx*, size_t n_perms, const uint64_t* inputs, const uint32_t* addresses, const uint32_t* timestamps,
                                     nb200_cols** out);

/* ---- RamInitFinal's main trace, filled on the device from the keccak side note and the public initial memory -------------------
 * The reference builds RamInitFinal's columns (prover/src/extensions/ram_init_final.rs:458-511) on the host from the side note's
 * `last_access` map: one row per RAM byte address in ascending order, with the address bytes, the flag 1, the final value and the
 * final access counter bytes.  Here the map is rebuilt on the device from the same inputs nb200_keccak_main_trace takes plus the
 * public initial memory (n_init entries, init_addresses strictly ascending, init_values one byte each): permutation p reads the 200
 * bytes at addresses[p] with previous counters timestamps[p][k] and leaves the bytes of Keccak-f[1600](inputs[p]) with counter
 * timestamps[p][k] + 1; an initial-memory entry no permutation touches keeps its value with counter 0.  Rows are ordered by address,
 * and for each address the last access in permutation order gives the final state.
 * out: a caller-owned batch of 10 columns and 2^log_size rows, overwritten in finalized order; rows past the last address are zero.
 * *n_rows_out = the number of distinct addresses.
 * NB200_ERR_ARG: n_perms == 0 or above 2^18, an address above 2^32 - 200, a timestamp of 2^32 - 1, init addresses not strictly
 * ascending, more than 2^30 init entries, log_size outside [4, 30], `out` of another shape, or more distinct addresses than 2^log_size
 * (then *n_rows_out still holds the count: learning it costs one device-to-host read).  Scratch memory is released in stream order. */
nb200_status nb200_ram_init_final_trace(nb200_ctx*, size_t n_perms, const uint64_t* inputs, const uint32_t* addresses, const uint32_t* timestamps,
                                        size_t n_init, const uint32_t* init_addresses, const uint8_t* init_values, uint32_t log_size,
                                        nb200_cols* out, size_t* n_rows_out);

/* ---- the v1 main component's main trace, filled on the device from an ADD / ADDI program's step record --------------------------
 * The reference fills the main component's 347 columns (prover/src/column.rs) on the host, one row per executed step
 * (Machine::prove's MainTrace stage, machine.rs:147-173).  Here only the step record crosses PCIe: steps = NB200_V1_STEP_FIELDS arrays of
 * n_steps words each, field-major, in the order
 *   pc, instruction word, opcode (0 ADD, 1 ADDI), rd, rs1, op_c (rs2 for ADD, the sign-extended immediate for ADDI), value of rs1,
 *   value of rs2 or the immediate, previous value of rd, previous timestamps of the rs1 read, the rs2 read and the rd write (0 when not
 *   accessed), previous execution count of the instruction at pc
 * (add_chain.STEP_FIELDS), and final_ctr = the final execution count of each of the program's n_prog rows (FinalPrgMemoryCtr).  Step t is
 * trace row t (clk = t + 1, register timestamps 3 clk + {1, 2, 3}); rows from n_steps on are the reference's padding rows.  The rows are
 * the per-row fills of CpuChip, DecodingCheck types R / I, AddChip, ProgramMemCheck, RegisterMemCheck and Timestamp.
 * out: a caller-owned batch of 347 columns and 2^log_size rows, overwritten in finalized order.
 * NB200_ERR_ARG: log_size outside [4, 28], `out` of another shape, n_steps or n_prog above 2^log_size, an opcode other than ADD / ADDI, a
 * register index above 31, a previous timestamp not below the current one, a previous execution count of 2^32 - 1.  Scratch memory is
 * released in stream order. */
#define NB200_V1_STEP_FIELDS 13
nb200_status nb200_v1_main_trace(nb200_ctx*, size_t n_steps, const uint32_t* steps, size_t n_prog, const uint32_t* final_ctr, uint32_t log_size,
                                 nb200_cols* out);

/* ---- the same fill for a straight-line program of RV32I's ALU instructions -------------------------------------------------------
 * nb200_v1_main_trace's arguments, step record and kernel, for every RV32I register-register and register-immediate instruction but
 * LUI / AUIPC (add_chain.OPCODES).  The opcode field takes
 *    0 ADD     1 ADDI    2 SUB     3 SLL     4 SLT     5 SLTU    6 XOR     7 SRL     8 SRA     9 OR     10 AND
 *   11 SLTI   12 SLTIU  13 XORI   14 ORI    15 ANDI   16 SLLI   17 SRLI   18 SRAI
 * ADD, SUB ... AND are type R: op_c is rs2 and value_c its value.  ADDI and SLTI ... ANDI are type I: op_c = value_c = the sign-extended
 * 12-bit immediate.  SLLI, SRLI and SRAI are type I with a shift amount: op_c = value_c = the 5-bit amount.  The rows add the per-row fills
 * of SubChip, SltuChip, BitOpChip, SltChip, SllChip, SrlChip and SraChip and DecodingCheck's type I with a shift amount.
 * NB200_ERR_ARG: what nb200_v1_main_trace refuses but its opcode rule, and an opcode above 18, a shift amount above 31 on SLLI / SRLI /
 * SRAI, a type-I immediate that is not a sign-extended 12-bit value. */
nb200_status nb200_v1_alu_trace(nb200_ctx*, size_t n_steps, const uint32_t* steps, size_t n_prog, const uint32_t* final_ctr, uint32_t log_size,
                                nb200_cols* out);

/* ---- the same fill for a looping program: RV32I's branches, jumps, LUI and AUIPC ------------------------------------------------
 * nb200_v1_alu_trace's arguments, step record and kernel, for its 19 opcodes and the control-flow opcodes (add_chain.CONTROL_OPCODES)
 *   19 BEQ    20 BNE    21 BLT    22 BGE    23 BLTU   24 BGEU   25 JAL    26 JALR   27 LUI    28 AUIPC
 * Steps need not follow one another in pc: the row of step t holds its own pc, and the next pc (PcNext) follows from pc, the opcode and
 * the values.  pc_ctr_prev counts the earlier executions of the instruction at pc, final_ctr each program row's executions (0 for a row
 * that never ran).  Per type:
 *   B (BEQ ... BGEU): rd = op_a, the instruction's rs1 field, read through Reg3 (its value in rd_prev, which is ValueA); rs1 = op_b, the
 *     instruction's rs2 field, read through Reg1 (its value in value_b); op_c = value_c = the sign-extended, even 13-bit offset;
 *     ts1_prev and ts3_prev are the previous timestamps of op_b and op_a, ts2_prev = 0.  PcNext = pc + value_c when taken, else pc + 4.
 *   JAL (type J): rs1 = value_b = 0, op_c = value_c = the sign-extended, even 21-bit offset; ValueA = pc + 4, PcNext = pc + value_c.
 *   JALR (type I): rd, rs1, op_c and value_c as ADDI's; ValueA = pc + 4, PcNext = (value_b + value_c) with bit 0 cleared.
 *   LUI, AUIPC (type U): rs1 = value_b = 0, op_c = the 20-bit immediate, value_c = op_c << 12; ValueA = value_c, or pc + value_c.
 * The rows add the per-row fills of BneChip, BeqChip, BltuChip, BltChip, BgeuChip, BgeChip, JalChip, LuiChip, AuipcChip, JalrChip and
 * DecodingCheck's types B, U and J.  The fill does not check that the steps' pcs chain; the main component's next-row Pc constraint does.
 * NB200_ERR_ARG: what nb200_v1_alu_trace refuses but its opcode rule, and an opcode above 28, a JALR immediate that is not a sign-extended
 * 12-bit value, a branch offset that is not an even sign-extended 13-bit value, a JAL offset that is not an even sign-extended 21-bit
 * value, a U-type immediate of more than 20 bits. */
nb200_status nb200_v1_control_trace(nb200_ctx*, size_t n_steps, const uint32_t* steps, size_t n_prog, const uint32_t* final_ctr,
                                    uint32_t log_size, nb200_cols* out);

/* ---- one commitment over N GPUs (SURVEY §8e; one process per GPU, NCCL over NVLink inside the library) ------------------------
 * The reference has no multi-device path (SURVEY App. C); these entry points are what a multi-GPU `CudaBackend` would drive from
 * TreeBuilder::commit (machine.rs:208-263).  Rank 0 creates the id and hands it to the other ranks out of band (MPI, a file,
 * torch.distributed broadcast ...); world must be a power of two; NCCL is bound with dlopen (a libnccl already loaded into the
 * process is shared). */
size_t nb200_comm_unique_id_bytes(void);
nb200_status nb200_comm_get_unique_id(uint8_t* id_out);
nb200_status nb200_comm_init(nb200_ctx*, int rank, int world, const uint8_t* unique_id);
void nb200_comm_destroy(nb200_ctx*);
int nb200_comm_rank(const nb200_ctx*);
int nb200_comm_world(const nb200_ctx*);
/* the column range [first, first + count) of rank `rank`: contiguous, multiples of 16 columns (one Blake2s block) */
nb200_status nb200_shard_range(size_t total_cols, int world, int rank, size_t* first, size_t* count);
/* all-gather of a small host blob (Merkle caps, claimed sums, sampled values): out = world x bytes, rank order */
nb200_status nb200_comm_all_gather(nb200_ctx*, const uint8_t* mine, size_t bytes, uint8_t* out);
/* nb200_commit_evals of ONE tree by all ranks together: column-sharded fused iFFT+LDE -> NVLink exchange (grouped ncclSend/Recv of
 * packed row slices) -> row-sharded sub-tree hashing -> ncclAllGather of the world caps -> top levels on the host.
 * shard_evals = this rank's nb200_shard_range columns (2^log_size rows each; may be NULL when the range is empty);
 * replicated = smaller batches that follow in commitment order, identical on every rank.
 * Out: coefficients of this rank's columns, `rows` = ALL total_cols columns restricted to this rank's 2^(log_size+log_blowup)/world
 * LDE rows (what row-sharded constraint / DEEP kernels consume), the rank's sub-tree, the caps (world x 32 bytes, may be NULL) and
 * the root, bit-identical to the single-GPU root on every rank. */
nb200_status nb200_commit_sharded(nb200_ctx*, const nb200_cols* shard_evals, size_t total_cols, uint32_t log_size, uint32_t log_blowup,
                                  const nb200_cols* const* replicated, size_t n_replicated,
                                  nb200_cols** coeffs_out, nb200_cols** rows_out, nb200_tree** subtree_out, uint8_t* caps_out, uint8_t root[32]);

/* ---- Blake2sChannel (stwo core/channel/blake2s.rs; used at machine.rs:197-206,240,262) --------------- */
/* The Fiat-Shamir transcript is sequential host work; it is part of the library so that the Rust shim and the
 * coarse nb200_prove share one implementation.  ctx may be NULL (defaults for the flavour switches). */
typedef struct nb200_channel nb200_channel;
nb200_status nb200_channel_new(nb200_ctx*, nb200_channel** out);
nb200_status nb200_channel_clone(const nb200_channel*, nb200_channel** out);
void nb200_channel_free(nb200_channel*);
void nb200_channel_digest(const nb200_channel*, uint8_t out[32]);
void nb200_channel_mix_u64(nb200_channel*, uint64_t v);
void nb200_channel_mix_u32s(nb200_channel*, const uint32_t* words, size_t n);
void nb200_channel_mix_felts(nb200_channel*, const uint32_t* qm31s, size_t n);
void nb200_channel_mix_root(nb200_channel*, const uint8_t root[32]); /* Blake2sMerkleChannel::mix_root */
void nb200_channel_draw_felt(nb200_channel*, uint32_t out[4]);
void nb200_channel_draw_felts(nb200_channel*, size_t n, uint32_t* out);
void nb200_channel_draw_random_bytes(nb200_channel*, uint8_t out[32]);
/* The channel run by one device thread (what nb200_prove uses between FRI's inner layers), from the state (digest, n_sent): for each of
 * n steps, mix the 32-byte roots[i] (skipped when roots is NULL) and draw one felt into felts_out[4 i .. 4 i + 3]; the final state is
 * returned.  The draws honour nb200_set_flavor's draw_domain_sep. */
nb200_status nb200_device_channel_draw(nb200_ctx*, const uint8_t digest[32], uint64_t n_sent, const uint8_t* roots, size_t n,
                                       uint32_t* felts_out, uint8_t digest_out[32], uint64_t* n_sent_out);

/* ---- AIR: FrameworkComponent<E> as data (SSA bytecode recorded from `add_constraints`, traits.rs:45-50) ---- */
typedef struct nb200_air nb200_air;
nb200_status nb200_air_load(nb200_ctx*, const uint32_t* words, size_t n_words, nb200_air** out);
void nb200_air_free(nb200_air*);
uint32_t nb200_air_n_params(const nb200_air*);
uint32_t nb200_air_n_components(const nb200_air*);
/* the component's constraint count, LogUp constraints included (0 for an unknown component) */
uint32_t nb200_air_n_constraints(const nb200_air*, uint32_t component);
/* the CUDA C source a component's programs are specialised to at first use (NVRTC, sm_90a): which = 0 the constraint
 * program, 1 the logup (interaction trace) program, 2 the constraints of degree above 2 alone (evaluated on the extra half
 * coset of a component with log_expand = log_blowup + 1).  malloc'ed, NUL-terminated, free with nb200_free.  Works without a
 * device (ctx may have been NULL at nb200_air_load).  NB200_ERR_STATE (and *out = NULL): the program is too short to be
 * specialised and runs on the bytecode interpreter, or (which = 2) the component has no constraint of degree above 2.
 * which = 3: the constraint check of nb200_check_constraints (any program length; NB200_ERR_STATE only when the component has
 * no constraint). */
nb200_status nb200_air_kernel_source(const nb200_air*, uint32_t component, int which, char** out);
/* degree of each of the component's n constraints in the trace columns (masks 1, constants and parameters 0, products add,
 * sums take the maximum), and which of its n masks the constraints of degree above 2 read (flags[m] = 1) */
nb200_status nb200_air_constraint_degrees(const nb200_air*, uint32_t component, uint32_t* degrees, size_t n);
nb200_status nb200_air_d2_masks(const nb200_air*, uint32_t component, uint8_t* flags, size_t n);
/* file name (16 hex digits + ".cubin") under which that kernel is looked up in the cubin cache: <library dir>/jit_cache or
 * $NB200_JIT_CACHE.  `python -m nexus_zkvm_b200.build` pre-compiles the shipped machines' kernels there with nvcc. */
uint64_t nb200_kernel_source_key(const char* source);

/* ---- CommitmentSchemeProver<B, Blake2sMerkleChannel> (machine.rs:202-203) ------------------------------ */
typedef struct nb200_scheme nb200_scheme;
/* PcsConfig { pow_bits, FriConfig { log_blowup_factor, log_last_layer_degree_bound, n_queries } } (machine.rs:184) */
nb200_status nb200_scheme_new(nb200_ctx*, uint32_t pow_bits, uint32_t log_blowup, uint32_t log_last_layer_degree_bound,
                              uint32_t n_queries, nb200_scheme** out);
void nb200_scheme_free(nb200_scheme*);
/* Optional hint: log2 of the AIR's constraint degree bound relative to the trace (the reference's LOG_CONSTRAINT_DEGREE,
 * prover/src/components/mod.rs:12; = max log_expand of the loaded AIR, nb200_air_max_log_expand).  When it equals
 * log_blowup + 1, the sharded commit (nb200_scheme_commit_sharded) also evaluates the polynomials on the extra half-size coset
 * the quotient step needs.  Single-GPU commits ignore it: there the quotient step extends only the few columns its
 * constraints of degree above 2 read.  Results never depend on the hint. */
nb200_status nb200_scheme_set_constraint_log_degree(nb200_scheme*, uint32_t log_expand);
uint32_t nb200_air_max_log_expand(const nb200_air*);
/* tree_builder.extend_evals(batches...); tree_builder.commit(channel)  (machine.rs:208-263): interpolate, LDE,
 * Merkle, mix_root.  The evaluation batches are only read. */
nb200_status nb200_scheme_commit(nb200_scheme*, const nb200_cols* const* eval_batches, size_t n_batches, nb200_channel*, uint8_t root[32]);
/* the same from HOST columns (pipelined H2D, optional finalize_columns on the device); evals_out[b] receives the device
 * evaluation batches (owned by the caller; nb200_gen_interaction_trace reads them) */
nb200_status nb200_scheme_commit_host(nb200_scheme*, const uint32_t* const* host_batches, const size_t* n_cols, const uint32_t* log_sizes,
                                      size_t n_batches, int coset_order, nb200_channel*, uint8_t root[32], nb200_cols** evals_out);
/* packed host format (see nb200_commit_host_packed) */
nb200_status nb200_scheme_commit_host_packed(nb200_scheme*, const void* const* host_batches, const uint32_t* elem_bytes, const size_t* n_cols,
                                             const uint32_t* log_sizes, size_t n_batches, int coset_order, nb200_channel*, uint8_t root[32],
                                             nb200_cols** evals_out);
/* generate_interaction_trace for one component (machine.rs:242-260; LogupTraceGenerator semantics) from the committed
 * preprocessed (tree0) and main (tree1) evaluation batches; params = n_params QM31 (lookup elements).
 * Out: a new batch of 4 * n_logup_columns columns and the component's claimed sum.  SURVEY §8 row f2. */
nb200_status nb200_gen_interaction_trace(nb200_ctx*, const nb200_air*, uint32_t component,
                                         const nb200_cols* const* tree0, size_t n0, const nb200_cols* const* tree1, size_t n1,
                                         const uint32_t* params, size_t n_params, nb200_cols** out, uint32_t claimed_sum[4]);
/* stwo::prover::prove::<B, Blake2sMerkleChannel>(components, channel, commitment_scheme)  (machine.rs:286-290).
 * Requires the three trace trees to be committed.  Output: postcard(StarkProof) bytes, malloc'ed (nb200_free).
 * Returns NB200_ERR_CONSTRAINTS for ProvingError::ConstraintsNotSatisfied. */
nb200_status nb200_prove(nb200_scheme*, const nb200_air*, const uint32_t* params, size_t n_params, nb200_channel*,
                         uint8_t** proof_out, size_t* proof_len);
/* assert_constraints_on_polys (stwo-constraint-framework) for one component, on the GPU: every constraint is evaluated on every row of
 * the trace domain CanonicCoset(log_size) and tested for zero.  tree0 / tree1 / tree2 = the evaluation batches of the three committed
 * trees (commitment order, as committed); params = the table nb200_prove takes (lookup elements, cumsum shifts).  For constraint k
 * (declaration order as in nb200_air_constraint_degrees, the LogUp constraints last; n = the component's constraint count):
 * n_failing[k] = the rows where it does not hold, first_row[k] = the first of them in trace (coset) order — the index into the host
 * column before finalize_columns — or UINT64_MAX when it holds everywhere.  Returns NB200_OK whether or not a constraint fails
 * (also for a component without constraints, n = 0);
 * NB200_ERR_ARG for a missing or wrongly sized column, NB200_ERR_STATE when the generated check kernel is unavailable (NB200_JIT=0). */
nb200_status nb200_check_constraints(nb200_ctx*, const nb200_air*, uint32_t component,
                                     const nb200_cols* const* tree0, size_t n0, const nb200_cols* const* tree1, size_t n1,
                                     const nb200_cols* const* tree2, size_t n2, const uint32_t* params, size_t n_params,
                                     uint64_t* n_failing, uint64_t* first_row, size_t n);

/* ---- lookup-table multiplicities, counted on the GPU from the AIR's own lookups --------------------------------------------------
 * Every fraction's denominator is Relation::combine, sum_i alpha_i v_i - z; its relation is named by the z parameter and its tuple is
 * (v_0 .. v_n-1).  A table fraction has the numerator -m for one tree-1 column m (its multiplicity column) and a tuple of tree-0 columns
 * and constants; a lookup is any other fraction into a relation that has a table fraction.  Relations without one are ignored.
 * nb200_air_lookup_tables: per fraction of the component (declaration order; n = its fraction count): kind (0 ignored, 1 table, 2 lookup,
 * 3 does not parse where it would be needed), relation (the z parameter index; UINT32_MAX when the denominator does not parse) and arg (a
 * table: the index of its multiplicity column in tree 1; otherwise the tuple length).  No device needed.
 * nb200_air_count_kernel_source: the CUDA C of the component's count kernel (NVRTC, sm_90a; its own cubin-cache key), malloc'ed, free with
 * nb200_free; NB200_ERR_STATE when the component has neither a table nor a lookup, NB200_ERR_ARG when a fraction it needs does not parse.
 * It is an entry of its own rather than a fifth `which` of nb200_air_kernel_source, which keeps answering NB200_ERR_ARG outside 0-3. */
nb200_status nb200_air_lookup_tables(const nb200_air*, uint32_t component, uint32_t* kind, uint32_t* relation, uint32_t* arg, size_t n);
nb200_status nb200_air_count_kernel_source(const nb200_air*, uint32_t component, char** out);
/* The multiplicity column of every table fraction, written in place into the tree-1 batch that holds it (finalized order, mod P; whatever the
 * column held is overwritten): the sum of the numerators of the lookups whose tuple equals that row's, over every row of every component.
 * tree0 / tree1 = the evaluation batches of trees 0 and 1 in commitment and finalized order, before tree 1 is committed.  A lookup with a
 * nonzero numerator whose tuple is in no table row is unmatched: n_unmatched counts them, first_unmatched = (component, fraction, row in
 * trace order) of the smallest, or UINT32_MAX x 3.  Returns NB200_OK whether or not lookups were unmatched; NB200_ERR_ARG for a missing or
 * wrongly sized column, a needed fraction that does not parse, a tuple listed twice in one relation, or more than 2^33 lookups (rows x
 * lookup fractions); NB200_ERR_STATE with NB200_JIT=0 (the count has no interpreter).  Scratch is released in stream order. */
nb200_status nb200_table_multiplicities(nb200_ctx*, const nb200_air*, const nb200_cols* const* tree0, size_t n0, nb200_cols* const* tree1, size_t n1,
                                        uint64_t* n_unmatched, uint32_t first_unmatched[3]);
/* The same count, except for a tuple that several table rows of one relation list: the first of those rows (smallest component, table
 * fraction and row in trace order) gets its count and every other one is written as 0, as the reference's trace fill credits value k of a
 * padded range table to row k (Multiplicity8's table lists 0 nine times).  n_repeated = the rows written as 0 (table rows minus distinct
 * (relation, tuple) keys).  Arguments, outputs and every other refusal as nb200_table_multiplicities; its scratch adds 8 bytes per hash
 * slot (about 16 per table row), released in stream order. */
nb200_status nb200_table_multiplicities_first_row(nb200_ctx*, const nb200_air*, const nb200_cols* const* tree0, size_t n0,
                                                  nb200_cols* const* tree1, size_t n1, uint64_t* n_unmatched, uint32_t first_unmatched[3],
                                                  uint64_t* n_repeated);

/* ---- one PROOF over N GPUs ---------------------------------------------------------------------------------------------------
 * Every rank calls the same sequence (the Machine::prove order, machine.rs:197-290) with its own shard; transcript, roots and proof
 * bytes come out identical on all ranks and identical to the single-GPU proof.
 * nb200_scheme_commit_sharded = tree_builder.extend_evals + commit for a tree whose FIRST `total_big` columns (the main component's,
 * 2^log_size rows) are sharded: `big_shard` = this rank's nb200_shard_range of them (finalized order); `small` = the smaller batches that
 * follow in commitment order, identical on every rank; `replicate_cols` = indices (inside the big batch) of the columns some constraint
 * reads at a row offset (column.rs:17-19: Pc, IsPadding; the last LogUp secure column) — their LDE is kept in full on every rank;
 * keep_eval_rows != 0 keeps this rank's trace rows of all big columns for nb200_gen_interaction_trace_sharded (trees 0 and 1).
 * nb200_gen_interaction_trace_sharded = generate_interaction_trace of the sharded component: returns this rank's COLUMN shard of the
 * 4 * n_logup interaction columns (input of the next nb200_scheme_commit_sharded) and the claimed sum.  Components whose columns are
 * replicated use nb200_gen_interaction_trace.  nb200_prove then runs constraint rows, OODS, DEEP quotients and decommitment sharded,
 * composition / FRI / PoW replicated. */
nb200_status nb200_scheme_commit_sharded(nb200_scheme*, const nb200_cols* big_shard, size_t total_big, uint32_t log_size,
                                         const nb200_cols* const* small, size_t n_small, const uint32_t* replicate_cols, size_t n_replicate,
                                         int keep_eval_rows, nb200_channel*, uint8_t root[32]);
nb200_status nb200_gen_interaction_trace_sharded(nb200_scheme*, const nb200_air*, uint32_t component, const uint32_t* params, size_t n_params,
                                                 nb200_cols** shard_out, uint32_t claimed_sum[4]);

/* ---- backend-trait level operations ---------------------------------------------------------------------
 * The per-trait surface a Rust `struct CudaBackend;` shim binds when it implements Stwo's backend traits one by one
 * instead of calling the coarse nb200_prove (SURVEY §8b).  nb200_prove runs exactly this code.  A "secure column"
 * (SecureColumnByCoords) is a batch of 4 coordinate columns. */
/* ComponentProver::<B>::evaluate_constraint_quotients_on_domain for one component (built at machine.rs:265-285): extend
 * the committed polynomials the component reads to CanonicCoset(log_size + log_expand).circle_domain(), evaluate
 * sum_k coeffs[k] * constraint_k / vanishing on every row and ADD into accum (4 columns of that domain size).
 * coeffs = n_coeffs QM31 (= the component's n_constraints random-coefficient powers, first constraint first).
 * NB200_ERR_ARG for a component that reads columns of a sharded tree (nb200_scheme_commit_sharded): nb200_prove evaluates such a
 * component on the half domains only (nb200_constraint_quotients_half). */
nb200_status nb200_constraint_quotients(nb200_scheme*, const nb200_air*, uint32_t component, const uint32_t* params, size_t n_params,
                                        const uint32_t* coeffs, size_t n_coeffs, nb200_cols* accum);
/* The half-domain route nb200_prove takes (Q_HALF) for a component with log_expand = log_blowup + 1 whose LDE has more than 2^8 rows: ADDs
 * into three accumulators of 4 columns x 2^lde_log each (lde_log = log_size + log_blowup):
 *   q_d1      = every constraint's quotient on the committed LDE domain D1 = CanonicCoset(lde_log).circle_domain();
 *   q_high_d2 = the quotient of the constraints of degree > 2 alone on D2 = rows [0, 2^lde_log) of CanonicCoset(lde_log + 1).circle_domain()
 *               (bit-reversed);
 *   q_high_d1 = the same on D1.
 * Where the bytecode interpreter evaluates the component instead of the generated kernels (NB200_JIT=0, or an LDE of fewer than 2^10 rows)
 * every constraint counts as a high one: q_high_d2 and q_high_d1 then hold q itself.
 * NB200_ERR_ARG for a component that nb200_prove evaluates with Q_FULL (nb200_constraint_quotients).
 * A component that reads columns of a sharded tree takes the sharded route, as in nb200_prove: each rank evaluates its own rows, from its
 * LDE and D2 row slices and the full copies of the columns read at a row offset, and the accumulators are all-gathered, so every rank
 * holds all rows.  It needs the generated kernels (NB200_ERR_ARG without them), and NB200_ERR_ARG names a column read at a row offset
 * that was not listed in replicate_cols when its tree was committed. */
nb200_status nb200_constraint_quotients_half(nb200_scheme*, const nb200_air*, uint32_t component, const uint32_t* params, size_t n_params,
                                             const uint32_t* coeffs, size_t n_coeffs, nb200_cols* q_d1, nb200_cols* q_high_d2, nb200_cols* q_high_d1);
/* AccumulationOps::accumulate: a += b (element-wise, M31), same shapes */
nb200_status nb200_accumulate(nb200_ctx*, nb200_cols* a, const nb200_cols* b);
/* QuotientOps::accumulate_quotients (DEEP quotients) on CanonicCoset(log_size).circle_domain(): columns are numbered
 * through the batches in order; sample batch b = OODS point {x[4], y[4]} + entries [first_entry, first_entry+n_entries)
 * of (column, sampled value).  Out: a new secure column (4 x 2^log_size). */
typedef struct { uint32_t point[8]; size_t first_entry, n_entries; } nb200_sample_batch;
typedef struct { uint32_t column; uint32_t value[4]; } nb200_sample_entry;
nb200_status nb200_fri_quotients(nb200_ctx*, const nb200_cols* const* batches, size_t n_batches, uint32_t log_size,
                                 const nb200_sample_batch* sample_batches, size_t n_sample_batches,
                                 const nb200_sample_entry* entries, size_t n_entries, const uint32_t random_coeff[4], nb200_cols** out);
/* The same quotient over the LDEs (2^log_size rows) of the columns whose coefficients (2^(log_size - log_blowup) words each) the batches
 * hold, by the route nb200_prove takes: each sample batch's columns are combined on their coefficients and only the combinations are
 * extended.  Needs at least one sample batch and log_size >= log_blowup + 2. */
nb200_status nb200_fri_quotients_from_coeffs(nb200_ctx*, const nb200_cols* const* coeffs, size_t n_batches, uint32_t log_size, uint32_t log_blowup,
                                             const nb200_sample_batch* sample_batches, size_t n_sample_batches,
                                             const nb200_sample_entry* entries, size_t n_entries, const uint32_t random_coeff[4], nb200_cols** out);
/* Host only: the tables of that route.  Sample batches must list their entries in order (first_entry = the entries before them).
 * lines_out: per sample batch 24 words: point x (CM31 parts 0, 1 of x then of y, then 2, 3 of x then of y), A[4], B[4] (the sums of the
 * alpha-weighted line coefficients), random_coeff ^ n_entries [4], c[4] = conj(y) - y; alphas_out: per entry its alpha (4 words),
 * random_coeff ^ (1 + its index in the batch). */
nb200_status nb200_deep_plan(const nb200_sample_batch* sample_batches, size_t n_sample_batches, const nb200_sample_entry* entries, size_t n_entries,
                             const uint32_t random_coeff[4], uint32_t* lines_out, uint32_t* alphas_out);
/* FriOps::fold_circle_into_line: dst = dst * alpha^2 + fold(src); src = secure column on CanonicCoset(k).circle_domain(),
 * dst = secure column of 2^(k-1) values on LineDomain(Coset::half_odds(k-1)) */
nb200_status nb200_fold_circle_into_line(nb200_ctx*, nb200_cols* dst, const nb200_cols* src, const uint32_t alpha[4]);
/* FriOps::fold_line: src on LineDomain(Coset::half_odds(k)) (bit-reversed) -> new secure column of 2^(k-1) values */
nb200_status nb200_fold_line(nb200_ctx*, const nb200_cols* src, const uint32_t alpha[4], nb200_cols** dst_out);
/* GrindOps::grind: smallest nonce with >= pow_bits trailing zero bits in H(digest, nonce) (channel digest in, nonce out) */
nb200_status nb200_grind(nb200_ctx*, const uint8_t digest[32], uint32_t pow_bits, uint64_t* nonce_out);

#ifdef __cplusplus
}
#endif
#endif /* NB200_H */
