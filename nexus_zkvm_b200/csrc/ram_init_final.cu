// RamInitFinal's main trace filled on the device (nb200_ram_init_final_trace): the keys (address, sequence) of every permutation access
// and initial-memory entry are radix-sorted with CUB, the first element of each address's run is marked and an inclusive scan over the
// marks numbers the addresses (their rows, ascending), the last element of each run is recorded as its row's source, and one thread per
// finalized position writes its row (ram_init_final.cuh) or a zero padding row.  The count of addresses is read back once to check it
// against the batch's 2^log_size rows.
#include "common.cuh"
#include "ram_init_final.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <algorithm>
#include <string>

namespace nb {
namespace {

constexpr u32 RF_BLOCK = 256;

__global__ void ram_keys_kernel(const u32* __restrict__ addresses, const u32* __restrict__ init_addresses, u32 n_acc, u32 n_elems, u64* keys,
                                u32* ids) {
  const u32 e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_elems) return;
  keys[e] = ram::access_key(addresses, init_addresses, n_acc, e);
  ids[e] = e;
}

// 1 where an address's run starts
__global__ void ram_heads_kernel(const u64* __restrict__ keys, u32 n_elems, u32* heads) {
  const u32 e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_elems) return;
  heads[e] = (e == 0 || ram::key_address(keys[e]) != ram::key_address(keys[e - 1])) ? 1u : 0u;
}

// the last element of each run is its row's source: row = (number of runs started up to e) - 1
__global__ void ram_tails_kernel(const u64* __restrict__ keys, const u32* __restrict__ ids, const u32* __restrict__ rank, u32 n_elems,
                                 u32* row_src) {
  const u32 e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_elems) return;
  if (e + 1 == n_elems || ram::key_address(keys[e]) != ram::key_address(keys[e + 1])) row_src[rank[e] - 1] = ids[e];
}

__global__ void ram_outputs_kernel(const u64* __restrict__ inputs, u32 n_perms, u64* outputs) {
  const u32 p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_perms) return;
  u64 a[25];
#pragma unroll
  for (int k = 0; k < 25; ++k) a[k] = inputs[(size_t)p * 25 + k];
  ram::keccak_f(a);
#pragma unroll
  for (int k = 0; k < 25; ++k) outputs[(size_t)p * 25 + k] = a[k];
}

// one thread per finalized position i: trace row finalized_src_row(i)
__global__ void ram_rows_kernel(const u32* __restrict__ row_src, u32 n_rows, u32 n_acc, const u64* __restrict__ outputs,
                                const u32* __restrict__ addresses, const u32* __restrict__ timestamps, const u32* __restrict__ init_addresses,
                                const uint8_t* __restrict__ init_values, u32 log_size, u32* out) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (1u << log_size)) return;
  const u32 r = (u32)finalized_src_row(i, log_size);
  u32 v[ram::COLS];
  if (r < n_rows) {
    ram::final_row(row_src[r], n_acc, outputs, addresses, timestamps, init_addresses, init_values, v);
  } else {
#pragma unroll
    for (u32 c = 0; c < ram::COLS; ++c) v[c] = 0;
  }
  const size_t n = (size_t)1 << log_size;
#pragma unroll
  for (u32 c = 0; c < ram::COLS; ++c) out[c * n + i] = v[c];
}

}  // namespace

nb200_status ram_init_final_trace(nb200_ctx* ctx, size_t n_perms, const uint64_t* inputs, const uint32_t* addresses, const uint32_t* timestamps,
                                  size_t n_init, const uint32_t* init_addresses, const uint8_t* init_values, uint32_t log_size, nb200_cols* out,
                                  size_t* n_rows_out) {
  NB_ARG(ctx, inputs && addresses && timestamps && out && n_rows_out && (n_init == 0 || (init_addresses && init_values)),
         "ram_init_final_trace: null argument");
  NB_ARG(ctx, n_perms >= 1 && n_perms <= keccak::MAX_PERMS, "ram_init_final_trace: n_perms must be in [1, 2^18]");
  NB_ARG(ctx, n_init <= ((size_t)1 << 30), "ram_init_final_trace: more than 2^30 initial-memory entries");
  NB_ARG(ctx, log_size >= keccak::LOG_N_LANES && log_size <= 30, "ram_init_final_trace: log_size must be in [4, 30]");
  NB_ARG(ctx, out->n_cols == ram::COLS && out->log_size == log_size, "ram_init_final_trace: out must be a batch of 10 columns of 2^log_size rows");
  *n_rows_out = 0;
  for (size_t p = 0; p < n_perms; ++p)
    NB_ARG(ctx, addresses[p] <= 0xFFFFFFFFu - (keccak::STATE - 1), "ram_init_final_trace: an address range of 200 bytes wraps 2^32");
  bool ts_max = false;
  for (size_t k = 0; k < n_perms * keccak::STATE; ++k) ts_max |= timestamps[k] == 0xFFFFFFFFu;
  NB_ARG(ctx, !ts_max, "ram_init_final_trace: a timestamp of 2^32 - 1 has no successor");
  for (size_t i = 1; i < n_init; ++i)
    NB_ARG(ctx, init_addresses[i - 1] < init_addresses[i], "ram_init_final_trace: initial-memory addresses must be strictly ascending");
  const u32 n_acc = (u32)(n_perms * keccak::STATE), n_elems = n_acc + (u32)n_init, np = (u32)n_perms;
  // scratch, freed in stream order when the call returns: the side note, the keys and element ids (twice: sort input and output), the run
  // marks and their scan, each row's source element, the permutation outputs and CUB's temporary storage
  DevBuf d_in, d_addr, d_ts, d_iaddr, d_ival, keys[2], ids[2], heads, rank, row_src, outputs, temp;
  NB_TRY(alloc(ctx, d_in, (size_t)np * 25 * 2));
  NB_TRY(alloc(ctx, d_addr, np));
  NB_TRY(alloc(ctx, d_ts, n_acc));
  NB_TRY(alloc(ctx, d_iaddr, n_init));
  NB_TRY(alloc(ctx, d_ival, (n_init + 3) / 4));
  for (int k = 0; k < 2; ++k) {
    NB_TRY(alloc(ctx, keys[k], (size_t)n_elems * 2));
    NB_TRY(alloc(ctx, ids[k], n_elems));
  }
  NB_TRY(alloc(ctx, heads, n_elems));
  NB_TRY(alloc(ctx, rank, n_elems));
  NB_TRY(alloc(ctx, row_src, (size_t)1 << log_size));
  NB_TRY(alloc(ctx, outputs, (size_t)np * 25 * 2));
  NB_CUDA(ctx, cudaMemcpyAsync(d_in.p, inputs, (size_t)np * 25 * 8, cudaMemcpyHostToDevice, ctx->stream));
  NB_CUDA(ctx, cudaMemcpyAsync(d_addr.p, addresses, (size_t)np * 4, cudaMemcpyHostToDevice, ctx->stream));
  NB_CUDA(ctx, cudaMemcpyAsync(d_ts.p, timestamps, (size_t)n_acc * 4, cudaMemcpyHostToDevice, ctx->stream));
  if (n_init) {
    NB_CUDA(ctx, cudaMemcpyAsync(d_iaddr.p, init_addresses, n_init * 4, cudaMemcpyHostToDevice, ctx->stream));
    NB_CUDA(ctx, cudaMemcpyAsync(d_ival.p, init_values, n_init, cudaMemcpyHostToDevice, ctx->stream));
  }
  u64* k_in = reinterpret_cast<u64*>(keys[0].p);
  u64* k_out = reinterpret_cast<u64*>(keys[1].p);
  auto grid = [](size_t n) { return (u32)((n + RF_BLOCK - 1) / RF_BLOCK); };
  ram_keys_kernel<<<grid(n_elems), RF_BLOCK, 0, ctx->stream>>>(d_addr.p, d_iaddr.p, n_acc, n_elems, k_in, ids[0].p);
  NB_LAUNCH_CHECK(ctx);
  size_t sort_bytes = 0, scan_bytes = 0;
  NB_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, k_in, k_out, ids[0].p, ids[1].p, (int)n_elems, 0, 64, ctx->stream));
  NB_CUDA(ctx, cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, heads.p, rank.p, (int)n_elems, ctx->stream));
  NB_TRY(alloc(ctx, temp, (std::max(sort_bytes, scan_bytes) + 3) / 4));
  size_t temp_bytes = sort_bytes;
  NB_CUDA(ctx, cub::DeviceRadixSort::SortPairs(temp.p, temp_bytes, k_in, k_out, ids[0].p, ids[1].p, (int)n_elems, 0, 64, ctx->stream));
  ram_heads_kernel<<<grid(n_elems), RF_BLOCK, 0, ctx->stream>>>(k_out, n_elems, heads.p);
  NB_LAUNCH_CHECK(ctx);
  temp_bytes = scan_bytes;
  NB_CUDA(ctx, cub::DeviceScan::InclusiveSum(temp.p, temp_bytes, heads.p, rank.p, (int)n_elems, ctx->stream));
  u32 n_rows = 0;
  NB_CUDA(ctx, cudaMemcpyAsync(&n_rows, rank.p + (n_elems - 1), 4, cudaMemcpyDeviceToHost, ctx->stream));
  NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  *n_rows_out = n_rows;
  NB_ARG(ctx, n_rows <= (1u << log_size), "ram_init_final_trace: more distinct addresses (" + std::to_string(n_rows) + ") than 2^log_size rows (" +
                                               std::to_string(1u << log_size) + ")");
  ram_tails_kernel<<<grid(n_elems), RF_BLOCK, 0, ctx->stream>>>(k_out, ids[1].p, rank.p, n_elems, row_src.p);
  NB_LAUNCH_CHECK(ctx);
  u64* outs = reinterpret_cast<u64*>(outputs.p);
  ram_outputs_kernel<<<grid(np), RF_BLOCK, 0, ctx->stream>>>(reinterpret_cast<const u64*>(d_in.p), np, outs);
  NB_LAUNCH_CHECK(ctx);
  ram_rows_kernel<<<grid((size_t)1 << log_size), RF_BLOCK, 0, ctx->stream>>>(row_src.p, n_rows, n_acc, outs, d_addr.p, d_ts.p, d_iaddr.p,
                                                                             reinterpret_cast<const uint8_t*>(d_ival.p), log_size, out->d);
  NB_LAUNCH_CHECK(ctx);
  return NB200_OK;
}

}  // namespace nb
