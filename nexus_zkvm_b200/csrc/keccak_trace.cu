// The keccak precompile extension's main trace (tree 1 of keccak.KeccakMachine) filled on the device from its side note, in finalized
// order: what KeccakMachine.fill_main_trace() builds on the host followed by finalize_columns, without the host columns or their upload.
// One thread per finalized row position recomputes its row (up to 23 rounds from the permutation's input, keccak_trace.cuh), so
// consecutive threads write consecutive words of every column.  The table multiplicities are counted by a second pass over the round
// rows into u32 histograms (global atomics) and written out mod P by a third kernel.
#include "common.cuh"
#include "keccak_trace.cuh"
#include <algorithm>

namespace nb {
namespace {

constexpr u32 KT_BLOCK = 128;

struct AtomicInc {
  __device__ __forceinline__ void operator()(u32* p) const { atomicAdd(p, 1u); }
};

__global__ void __launch_bounds__(KT_BLOCK) keccak_mem_fill_kernel(const u64* __restrict__ inputs, const u32* __restrict__ addresses,
                                                                   const u32* __restrict__ timestamps, u32 n_perms, u32 log_size, u32* out) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (1u << log_size)) return;
  keccak::mem_row(inputs, addresses, timestamps, n_perms, log_size, i, out + i, (size_t)1 << log_size);
}

__global__ void __launch_bounds__(KT_BLOCK) keccak_round_fill_kernel(const u64* __restrict__ inputs, u32 n_perms, u32 rounds, u32 offset,
                                                                     u32 log_size, u32* out) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (1u << log_size)) return;
  const size_t n = (size_t)1 << log_size;
  keccak::ColumnSink s{out + i, n};
  const bool padding = keccak::round_component_row(inputs, n_perms, rounds, offset, log_size, i, s);
  out[(size_t)(keccak::ROUND_COLS - 1) * n + i] = padding ? 1u : 0u;
}

__global__ void __launch_bounds__(KT_BLOCK) keccak_round_count_kernel(const u64* __restrict__ inputs, u32 n_perms, u32 rounds, u32 offset,
                                                                      u32 log_size, u32* xor_hist, u32* nand_hist, u32* rot_hist) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (1u << log_size)) return;
  keccak::CountSink<AtomicInc> s{xor_hist, nand_hist, rot_hist};
  keccak::round_component_row(inputs, n_perms, rounds, offset, log_size, i, s);
}

// bitwise: 32 columns (XorTable's 16, then BitNotAndTable's) of 2^12 rows; rotate: 1 column of 2^11 rows; finalized order, mod P
__global__ void keccak_mult_kernel(const u32* __restrict__ xor_hist, const u32* __restrict__ nand_hist, const u32* __restrict__ rot_hist,
                                   u32* bitwise, u32* rotate) {
  const u32 e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= keccak::MULT_WORDS) return;
  const u32 v = keccak::mult_word(xor_hist, nand_hist, rot_hist, e);
  if (e < keccak::BITWISE_MULT_WORDS) bitwise[e] = v;
  else rotate[e - keccak::BITWISE_MULT_WORDS] = v;
}

u32 log2_ceil(size_t n) {
  u32 l = 0;
  while (((size_t)1 << l) < n) ++l;
  return l;
}

}  // namespace

// (index, rounds, offset) of the two KeccakRound components (extensions/keccak/mod.rs:15-24)
static const u32 kRoundSplit[2][2] = {{16, 0}, {8, 16}};

nb200_status keccak_main_trace(nb200_ctx* ctx, size_t n_perms, const uint64_t* inputs, const uint32_t* addresses, const uint32_t* timestamps,
                               nb200_cols** out) {
  NB_ARG(ctx, inputs && addresses && timestamps && out, "keccak_main_trace: null argument");
  NB_ARG(ctx, n_perms >= 1 && n_perms <= keccak::MAX_PERMS, "keccak_main_trace: n_perms must be in [1, 2^18]");
  for (size_t p = 0; p < n_perms; ++p)
    NB_ARG(ctx, addresses[p] <= 0xFFFFFFFFu - (keccak::STATE - 1), "keccak_main_trace: an address range of 200 bytes wraps 2^32");
  bool ts_max = false;
  for (size_t k = 0; k < n_perms * keccak::STATE; ++k) ts_max |= timestamps[k] == 0xFFFFFFFFu;
  NB_ARG(ctx, !ts_max, "keccak_main_trace: a timestamp of 2^32 - 1 has no successor");
  // log sizes as KeccakMachine.__init__ derives them (compute_log_size: at least 2^4 rows)
  const u32 mem_log = std::max(log2_ceil(n_perms), keccak::LOG_N_LANES);
  const u32 round_log[2] = {std::max(log2_ceil(n_perms * kRoundSplit[0][0]), keccak::LOG_N_LANES),
                            std::max(log2_ceil(n_perms * kRoundSplit[1][0]), keccak::LOG_N_LANES)};
  ColsPtr mem, rnd[2], bitwise, rotate;
  NB_TRY(alloc(ctx, mem, keccak::MEM_COLS, mem_log));
  NB_TRY(alloc(ctx, rnd[0], keccak::ROUND_COLS, round_log[0]));
  NB_TRY(alloc(ctx, rnd[1], keccak::ROUND_COLS, round_log[1]));
  NB_TRY(alloc(ctx, bitwise, 2 * keccak::BITWISE_MULT_COLS, keccak::BITWISE_LOG));
  NB_TRY(alloc(ctx, rotate, 1, keccak::ROTATE_LOG));
  // the side note on the device (inputs as u32 pairs) and the three histograms: scratch, freed in stream order below
  DevBuf d_in, d_addr, d_ts, hist;
  const size_t hist_words = 2 * ((size_t)1 << 16) + ((size_t)1 << keccak::ROTATE_LOG);
  NB_TRY(alloc(ctx, d_in, n_perms * 25 * 2));
  NB_TRY(alloc(ctx, d_addr, n_perms));
  NB_TRY(alloc(ctx, d_ts, n_perms * keccak::STATE));
  NB_TRY(alloc(ctx, hist, hist_words));
  NB_CUDA(ctx, cudaMemcpyAsync(d_in.p, inputs, n_perms * 25 * 8, cudaMemcpyHostToDevice, ctx->stream));
  NB_CUDA(ctx, cudaMemcpyAsync(d_addr.p, addresses, n_perms * 4, cudaMemcpyHostToDevice, ctx->stream));
  NB_CUDA(ctx, cudaMemcpyAsync(d_ts.p, timestamps, n_perms * keccak::STATE * 4, cudaMemcpyHostToDevice, ctx->stream));
  NB_CUDA(ctx, cudaMemsetAsync(hist.p, 0, hist_words * 4, ctx->stream));
  const u64* in = reinterpret_cast<const u64*>(d_in.p);
  const u32 np = (u32)n_perms;
  auto grid = [](u32 log) { return (u32)((((size_t)1 << log) + KT_BLOCK - 1) / KT_BLOCK); };
  keccak_mem_fill_kernel<<<grid(mem_log), KT_BLOCK, 0, ctx->stream>>>(in, d_addr.p, d_ts.p, np, mem_log, mem->d);
  NB_LAUNCH_CHECK(ctx);
  u32* xor_hist = hist.p;
  u32* nand_hist = xor_hist + ((size_t)1 << 16);
  u32* rot_hist = nand_hist + ((size_t)1 << 16);
  for (int k = 0; k < 2; ++k) {
    keccak_round_fill_kernel<<<grid(round_log[k]), KT_BLOCK, 0, ctx->stream>>>(in, np, kRoundSplit[k][0], kRoundSplit[k][1], round_log[k], rnd[k]->d);
    NB_LAUNCH_CHECK(ctx);
  }
  // padding rows count too: every row of both round components is a full round
  for (int k = 0; k < 2; ++k) {
    keccak_round_count_kernel<<<grid(round_log[k]), KT_BLOCK, 0, ctx->stream>>>(in, np, kRoundSplit[k][0], kRoundSplit[k][1], round_log[k],
                                                                                  xor_hist, nand_hist, rot_hist);
    NB_LAUNCH_CHECK(ctx);
  }
  keccak_mult_kernel<<<(keccak::MULT_WORDS + 255) / 256, 256, 0, ctx->stream>>>(xor_hist, nand_hist, rot_hist, bitwise->d, rotate->d);
  NB_LAUNCH_CHECK(ctx);
  out[0] = mem.release();
  out[1] = rnd[0].release();
  out[2] = rnd[1].release();
  out[3] = bitwise.release();
  out[4] = rotate.release();
  return NB200_OK;
}

}  // namespace nb
