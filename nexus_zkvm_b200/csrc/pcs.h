// Internal interfaces between the proving orchestrator (prove.cu) and the kernel translation units.
#pragma once
#include "common.cuh"
#include "air.h"
#include "jit.h"
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

nb200_status domain_points(nb200_ctx* ctx, u32 log_size, u32* d_x, u32* d_y);
nb200_status quotients_launch(nb200_ctx* ctx, const QBatchDev* h_batches, size_t n_batches, const QEntryDev* h_entries, size_t n_entries,
                              const u32* dom_x, const u32* dom_y, u32 log_size, u32* out /* 4 columns */, u32 row0 = 0, size_t n_rows = 0);
nb200_status fold_circle_into_line(nb200_ctx* ctx, u32* dst, const u32* src, u32 src_log, qm31 alpha);
nb200_status fold_line(nb200_ctx* ctx, u32* dst, const u32* src, u32 src_log, qm31 alpha);
nb200_status add_inplace(nb200_ctx* ctx, u32* a, const u32* b, size_t n);
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
nb200_status merkle_decommit(nb200_ctx* ctx, const nb200_tree* tree, const std::vector<ColRef>& cols_in,
                             const std::vector<std::pair<u32, std::vector<u64>>>& queries,
                             std::vector<u32>& queried_values, std::vector<uint8_t>& hash_witness, std::vector<u32>& column_witness);
nb200_status gather_u32(nb200_ctx* ctx, const std::vector<const u32*>& addrs, u32* host_out);

}  // namespace nb
