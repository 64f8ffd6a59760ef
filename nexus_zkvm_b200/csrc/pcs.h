// Internal interfaces between the proving orchestrator (prove.cu) and the kernel translation units.
#pragma once
#include "common.cuh"
#include "air.h"
#include "jit.h"
#include "device_channel.cuh"
#include <utility>

namespace nb {

// DEEP quotient descriptors (uploaded as-is)
struct QBatchDev {
  u32 prx[2], pry[2], pix[2], piy[2];  // CM31 parts of the sample point
  u32 A[4], B[4];                      // sum over the batch of the line coefficients alpha^k a_k, alpha^k b_k
  u32 coeff[4];                        // random_coeff ^ (columns in batch)
  u32 first, count;                    // entries [first, first+count)
};
struct QEntryDev { u32 c[4]; const u32* col; u32 pad[2]; };  // 32 bytes; c first so that it loads as one 128-bit word

// a sample batch of the combined route: numerator c G(x) - (A y + B), G = the batch's combination sum_k alpha^k f_k (deep_combine)
struct QLineDev {
  u32 prx[2], pry[2], pix[2], piy[2];  // CM31 parts of the sample point
  u32 A[4], B[4];                      // as in QBatchDev
  u32 coeff[4];                        // random_coeff ^ (columns in batch)
  u32 c[4];                            // conj(p.y) - p.y
};

nb200_status domain_points(nb200_ctx* ctx, u32 log_size, u32* d_x, u32* d_y);
nb200_status quotients_launch(nb200_ctx* ctx, const QBatchDev* h_batches, size_t n_batches, const QEntryDev* h_entries, size_t n_entries,
                              const u32* dom_x, const u32* dom_y, u32 log_size, u32* out /* 4 columns */, u32 row0 = 0, size_t n_rows = 0);
// g = per batch (4 columns of 2^log_n each, batch after batch) the sum over entries [first, first + count) of entry.c (QM31) x entry.col
nb200_status deep_combine(nb200_ctx* ctx, const uint2* h_ranges /* (first, count) */, size_t n_batches, const QEntryDev* h_entries, size_t n_entries,
                          u32 log_n, u32* g);
// out (4 columns of 2^log_size) = the DEEP quotient of the batches from their extended combinations g (4 columns of 2^log_size per batch)
nb200_status quotients_combined(nb200_ctx* ctx, const QLineDev* h_batches, size_t n_batches, const u32* g, const u32* dom_x, const u32* dom_y,
                                u32 log_size, u32* out);
nb200_status fold_circle_into_line(nb200_ctx* ctx, u32* dst, const u32* src, u32 src_log, qm31 alpha);
nb200_status fold_line(nb200_ctx* ctx, u32* dst, const u32* src, u32 src_log, qm31 alpha);
nb200_status fold_line(nb200_ctx* ctx, u32* dst, const u32* src, u32 src_log, const u32* d_alpha);   // alpha: 4 words in device memory
// the device channel (device_channel.cuh): mix the 32-byte root at d_root (skipped when null), draw a felt; d_rec = root words, then alpha
nb200_status channel_mix_draw(nb200_ctx* ctx, DevChannel* d_ch, const uint8_t* d_root, u32* d_rec, int domain_sep);
nb200_status add_inplace(nb200_ctx* ctx, u32* a, const u32* b, size_t n);
nb200_status table_mult_store(nb200_ctx* ctx, u32* dst, const unsigned long long* cnt, size_t n);   // dst[i] = cnt[i] mod P
// table_first_row.cu: every occupied slot of the built count hash names its key's first bin; *distinct += the occupied slots.  tables =
// (first bin, log size) per table fraction in bin order; owner = cap words of ~0.
nb200_status table_first_row_resolve(nb200_ctx* ctx, u32* slots, const u32* keys, u32 kw, u64 cap, u32 n_bins, const u32* tables, u32 n_tables,
                                     unsigned long long* owner, u32* distinct);
nb200_status grind(nb200_ctx* ctx, const uint8_t digest[32], u32 pow_bits, uint64_t* nonce_out);

// rows [0, 2^rows_log) of CanonicCoset(dom_log).circle_domain() (bit-reversed); rows_log == dom_log - 1 selects the first half of
// the domain; 0, 0 = the component's whole evaluation domain.  mask_cols are the columns evaluated on exactly those rows.
nb200_status constraint_eval(nb200_ctx* ctx, const AirComponent& c, const std::vector<const u32*>& mask_cols, const u32* d_params,
                             const std::vector<qm31>& coeffs, u32* const acc[4], const JitKernel* jk = nullptr, u32 rows_log = 0, u32 dom_log = 0,
                             u32 row0 = 0, size_t n_rows = 0,    // row0 / n_rows: only the rows [row0, row0 + n_rows) (pointers stay indexed by the global row)
                             u32* const acc_high[4] = nullptr);  // also: the constraints of degree above AIR_LOW_DEGREE alone (needs jit_usable)
nb200_status sub_scale_top_twiddle(nb200_ctx* ctx, u32* a, const u32* b, size_t n, u32 tw_log);  // a = (a - b) / (top-layer twiddle of canonic(tw_log))
nb200_status add_cols_strided(nb200_ctx* ctx, u32* dst, size_t dst_stride, const u32* src, size_t src_stride, size_t len, size_t n_cols);
nb200_status logup_generate(nb200_ctx* ctx, const AirComponent& c, const std::vector<const u32*>& mask_cols, const u32* d_params,
                            u32* d_out, qm31* claimed, const JitKernel* jk = nullptr);

nb200_status logup_rows(nb200_ctx* ctx, const AirComponent& c, const std::vector<const u32*>& mask_cols, const u32* d_params, u32* d_out, u32 rows_log, const JitKernel* jk);
nb200_status logup_finalize_last(nb200_ctx* ctx, u32 log_size, u32* last4, qm31* claimed);
nb200_status eval_at_points(nb200_ctx* ctx, const u32* coeffs, size_t n_cols, u32 log_size, const u32* points_xy, size_t n_points, u32* out_qm31);
// f(points[point]) of the 2^log_size coefficients at `coeffs`
struct EvalJob { const u32* coeffs; u32 log_size; u32 point; };
// every job in one launch and one round trip: out_qm31[i] = job i's value; points_xy = n_points x {x[4], y[4]}
nb200_status eval_at_points_multi(nb200_ctx* ctx, const std::vector<EvalJob>& jobs, const u32* points_xy, size_t n_points, u32* out_qm31);
nb200_status merkle_decommit(nb200_ctx* ctx, const nb200_tree* tree, const std::vector<ColRef>& cols_in,
                             const std::vector<std::pair<u32, std::vector<u64>>>& queries,
                             std::vector<u32>& queried_values, std::vector<uint8_t>& hash_witness, std::vector<u32>& column_witness);
nb200_status gather_u32(nb200_ctx* ctx, const std::vector<const u32*>& addrs, u32* host_out);
// the hashes (32 bytes each) and words at the given device addresses, fetched with one launch and one sync
nb200_status gather_batch(nb200_ctx* ctx, const std::vector<const uint8_t*>& hash_addrs, const std::vector<const u32*>& val_addrs, uint8_t* hashes_out, u32* vals_out);
// MerkleProver::decommit split in two: the host-only walk (plan), and the sorting of the gathered results into the decommitment (fill),
// so that many decommitments can share one gather
struct DecommitPlan {
  std::vector<std::pair<u32, u64>> vals;     // (column index in the caller's order, row), walk order
  std::vector<uint8_t> val_is_query;         // 1 -> queried_values, 0 -> column_witness
  std::vector<std::pair<u32, u64>> hashes;   // (layer, node): the hash witness, in order
};
void merkle_decommit_plan(u32 max_log, const std::vector<u32>& col_logs, const std::vector<std::pair<u32, std::vector<u64>>>& queries, DecommitPlan& plan);
void merkle_decommit_addrs(const DecommitPlan& plan, const nb200_tree* tree, const std::vector<ColRef>& cols,
                           std::vector<const uint8_t*>& hash_addrs, std::vector<const u32*>& val_addrs);
void merkle_decommit_fill(const DecommitPlan& plan, const uint8_t* hashes, const u32* vals,
                          std::vector<u32>& queried_values, std::vector<uint8_t>& hash_witness, std::vector<u32>& column_witness);

}  // namespace nb
