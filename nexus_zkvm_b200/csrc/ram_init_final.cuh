// RamInitFinal's main trace (nexus-zkvm prover/src/extensions/ram_init_final.rs:458-511) from the keccak extension's side note and the
// public initial memory: one row per RAM byte address, in ascending address order (the side note's `last_access` BTreeMap), holding the
// address bytes, the flag 1, the byte's final value and its final access counter bytes; rows past the last address are zero.
// Every access is an element: element e < n_acc = 200 n_perms is byte e % 200 of permutation e / 200, element n_acc + i is initial-memory
// entry i.  Sorting the elements by key (address, sequence) puts each address's accesses in order, so the last element of an address's run
// gives its final state.  The same code runs in the kernels of ram_init_final.cu and, compiled as host C++, in
// tests/test_whole_machine_cpu.py, which compares it with the numpy columns of whole_machine.ram_init_final_columns.
#pragma once
#include "keccak_trace.cuh"

namespace nb {
namespace ram {

constexpr u32 COLS = 10;   // address bytes x 4, flag, final value, final counter bytes x 4 (ram_init_final.rs:83-89)

// sort key of element e: address << 32 | sequence, the sequence 0 for an initial-memory entry and 1 + p for permutation p's access
NB_HD u64 access_key(const u32* addresses, const u32* init_addresses, u32 n_acc, u32 e) {
  if (e < n_acc) {
    const u32 p = e / keccak::STATE;
    return (u64)(addresses[p] + e % keccak::STATE) << 32 | (u64)(p + 1);
  }
  return (u64)init_addresses[e - n_acc] << 32;
}

NB_HD u32 key_address(u64 key) { return (u32)(key >> 32); }

// the row of the address whose last element (in key order) is `e`: a permutation's access leaves the permutation's output byte with
// counter previous timestamp + 1 (chips/custom.rs: update_state_timestamps); an initial-memory entry no permutation touches keeps its
// value with counter 0.  outputs = n_perms x 25 lanes after Keccak-f[1600].
NB_HD void final_row(u32 e, u32 n_acc, const u64* outputs, const u32* addresses, const u32* timestamps, const u32* init_addresses,
                     const uint8_t* init_values, u32 v[COLS]) {
  u32 addr, value, counter;
  if (e < n_acc) {
    const u32 p = e / keccak::STATE, k = e % keccak::STATE;
    addr = addresses[p] + k;
    value = (u32)((outputs[(size_t)p * 25 + k / keccak::LANE] >> (8 * (k % keccak::LANE))) & 255);
    counter = timestamps[e] + 1;
  } else {
    addr = init_addresses[e - n_acc];
    value = init_values[e - n_acc];
    counter = 0;
  }
#pragma unroll
  for (u32 j = 0; j < 4; ++j) v[j] = (addr >> (8 * j)) & 255;
  v[4] = 1;
  v[5] = value;
#pragma unroll
  for (u32 j = 0; j < 4; ++j) v[6 + j] = (counter >> (8 * j)) & 255;
}

// Keccak-f[1600] of the 25 lanes in place
NB_HD void keccak_f(u64 a[25]) {
  for (u32 r = 0; r < 24; ++r) keccak::keccak_round(a, keccak::round_constant(r));
}

}  // namespace ram
}  // namespace nb
