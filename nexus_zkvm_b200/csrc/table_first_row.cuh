// The first-row rule of nb200_table_multiplicities_first_row: a tuple that several table rows of one relation list is credited to the first
// of them in (component, table fraction, trace row) order, as the reference's trace fill credits value k to row k
// (prover/src/chips/range_check/range8.rs:298 with extensions/multiplicity8.rs:194-204).  It runs between the generated count's build and
// probe (jit.cu gen_count_source).  After the build, `keys` holds every bin's key (relation, length, values) and every distinct key owns
// exactly one hash slot, whose bin won an arbitrary race; the resolve points each such slot at the key's first bin instead, so the unchanged
// probe adds every lookup there and the other bins of the key keep a zero counter.
//   per bin b:   owner[slot of b's key] = min(owner, first_row_claim(b)) — the claim's high word is unique and monotone in that order
//   per slot s:  slots[s] = the bin of owner[s]; the occupied slots are the distinct keys
// The hash and the key comparison are the generated source's khash / ksame, word for word; tests/test_table_first_row_cpu.py pins them equal
// and compiles this file as host C++.
#pragma once
#include "finalize_order.cuh"

namespace nb {
namespace first_row {

constexpr u32 EMPTY = 0xffffffffu;   // an empty hash slot (the generated source's NB_EMPTY)

NB_HD u32 key_hash(u32 rel, u32 len, const u32* v) {
  u64 h = ((u64)rel << 32 | len) * 0x9E3779B97F4A7C15ull;
  for (u32 i = 0; i < len; ++i) { h = (h ^ v[i]) * 0x9E3779B97F4A7C15ull; h ^= h >> 31; }
  return (u32)(h >> 32);
}

// k: a stored key (kw words: rel, len, values)
NB_HD bool key_same(const u32* k, u32 rel, u32 len, const u32* v) {
  if (k[0] != rel || k[1] != len) return false;
  for (u32 i = 0; i < len; ++i) if (k[2 + i] != v[i]) return false;
  return true;
}

// the slot that holds bin b's key: the key is in the hash, so the probe ends there
NB_HD u32 key_slot(const u32* slots, const u32* keys, u32 kw, u32 mask, u32 b) {
  const u32* k = keys + (u64)b * kw;
  const u32 rel = k[0], len = k[1];
  u32 s = key_hash(rel, len, k + 2) & mask;
  while (!key_same(keys + (u64)slots[s] * kw, rel, len, k + 2)) s = (s + 1) & mask;
  return s;
}

// bin b's claim: (tbase[t] + its trace row) << 32 | b, t = the table fraction holding b (tables[2 t] = its first bin, tables[2 t + 1] = its
// log size, ascending first bins; b - tbase[t] is the row's finalized position).  Fewer than 2^30 bins: the high word is unique.
NB_HD u64 first_row_claim(const u32* tables, u32 n_tables, u32 b) {
  u32 lo = 0, hi = n_tables - 1;   // the last table whose first bin is <= b
  while (lo < hi) {
    const u32 mid = (lo + hi + 1) >> 1;
    if (tables[2 * mid] <= b) lo = mid; else hi = mid - 1;
  }
  const u32 base = tables[2 * lo];
  const u32 order = base + (u32)finalized_src_row(b - base, tables[2 * lo + 1]);
  return (u64)order << 32 | b;
}

// slot s after every claim: an occupied slot names its key's first bin (the low word of its smallest claim); returns whether it is occupied
NB_HD bool own_slot(u32* slots, const u64* owner, u64 s) {
  if (slots[s] == EMPTY) return false;
  slots[s] = (u32)owner[s];
  return true;
}

}  // namespace first_row
}  // namespace nb
