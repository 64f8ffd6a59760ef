// The row permutation of finalize_columns (nexus-zkvm prover/src/trace/utils.rs:94-106 + utils_external.rs:24-39): position i of a
// finalized (bit-reversed circle-domain order) column of 2^log_size rows holds row finalized_src_row(i) of the trace (coset) order column.
// Host and device: the keccak trace filler's host test (tests/test_keccak_fill_cpu.py) compiles it with g++.
#pragma once
#include <stddef.h>
#include "m31.cuh"

namespace nb {

NB_HD u32 brev32(u32 x) {
#if defined(__CUDA_ARCH__)
  return __brev(x);
#else
  x = ((x >> 1) & 0x55555555u) | ((x & 0x55555555u) << 1);
  x = ((x >> 2) & 0x33333333u) | ((x & 0x33333333u) << 2);
  x = ((x >> 4) & 0x0F0F0F0Fu) | ((x & 0x0F0F0F0Fu) << 4);
  x = ((x >> 8) & 0x00FF00FFu) | ((x & 0x00FF00FFu) << 8);
  return (x >> 16) | (x << 16);
#endif
}

// coset order -> circle-domain order -> bit-reversed: the trace row that finalized position i reads
NB_HD size_t finalized_src_row(u32 i, u32 log_size) {
  const u32 j = log_size ? (brev32(i) >> (32 - log_size)) : 0;
  const size_t n = (size_t)1 << log_size, half = n >> 1;
  return j < half ? ((size_t)j << 1) : (n - 1 - (((size_t)j - half) << 1));
}

}  // namespace nb
