// The resolve of nb200_table_multiplicities_first_row (table_first_row.cuh): every bin claims its key's slot with its (table, trace row)
// order, then every occupied slot is pointed at its smallest claim's bin and the occupied slots are counted.
#include "common.cuh"
#include "table_first_row.cuh"

namespace nb {
namespace {

constexpr u32 FR_BLOCK = 256;

__global__ void __launch_bounds__(FR_BLOCK) table_first_row_claim_kernel(const u32* __restrict__ slots, const u32* __restrict__ keys, u32 kw,
                                                                         u32 mask, const u32* __restrict__ tables, u32 n_tables, u32 n_bins,
                                                                         unsigned long long* owner) {
  const u32 b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n_bins) return;
  atomicMin(owner + first_row::key_slot(slots, keys, kw, mask, b), (unsigned long long)first_row::first_row_claim(tables, n_tables, b));
}

// every thread of a warp reaches the ballot: the occupied slots are counted once per warp
__global__ void __launch_bounds__(FR_BLOCK) table_first_row_slot_kernel(u32* __restrict__ slots, const unsigned long long* __restrict__ owner,
                                                                        u64 cap, u32* distinct) {
  const u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  const bool used = s < cap && first_row::own_slot(slots, reinterpret_cast<const u64*>(owner), s);
  const unsigned m = __ballot_sync(0xffffffffu, used);
  if ((threadIdx.x & 31u) == 0 && m) atomicAdd(distinct, (u32)__popc(m));
}

}  // namespace

nb200_status table_first_row_resolve(nb200_ctx* ctx, u32* slots, const u32* keys, u32 kw, u64 cap, u32 n_bins, const u32* tables, u32 n_tables,
                                     unsigned long long* owner, u32* distinct) {
  table_first_row_claim_kernel<<<(n_bins + FR_BLOCK - 1) / FR_BLOCK, FR_BLOCK, 0, ctx->stream>>>(slots, keys, kw, (u32)(cap - 1), tables, n_tables,
                                                                                                n_bins, owner);
  NB_LAUNCH_CHECK(ctx);
  table_first_row_slot_kernel<<<(u32)((cap + FR_BLOCK - 1) / FR_BLOCK), FR_BLOCK, 0, ctx->stream>>>(slots, owner, cap, distinct);
  NB_LAUNCH_CHECK(ctx);
  return NB200_OK;
}

}  // namespace nb
