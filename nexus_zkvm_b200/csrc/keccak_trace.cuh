// One row of the keccak precompile extension's main trace (tree 1), filled from its side note (nexus-zkvm
// prover/src/trace/sidenote/keccak.rs:16-25: per permutation 25 input lanes, one base address, 200 previous timestamps).
// The same code runs in the kernels of keccak_trace.cu and, compiled as host C++, in tests/test_keccak_fill_cpu.py, which compares
// every row with KeccakMachine.fill_main_trace().  Rows are addressed by their finalized position (finalize_order.cuh).
#pragma once
#include "m31.cuh"
#include "finalize_order.cuh"

namespace nb {
namespace keccak {

constexpr u32 LANE = 8;                      // bytes per 64-bit lane (round/constants.rs:45)
constexpr u32 STATE = 25 * LANE;             // 200 state bytes
constexpr u32 MEM_COLS = 2 * STATE + 3 * 2 * STATE + 2 * STATE + 1;   // memory_check/trace.rs:32-123: 2001
constexpr u32 ROUND_LANES = 25 + 20 + 5 * 4 + 25 + 24 * 3 + 50 + 1;   // round/trace.rs:297-366: 213
constexpr u32 ROUND_COLS = ROUND_LANES * LANE + 1;                     // 1705 (the last one is_padding)
constexpr u32 BITWISE_LOG = 12, BITWISE_MULT_COLS = 16;               // bitwise_table/mod.rs:61-62, preprocessed_columns.rs:38-40
constexpr u32 ROTATE_LOG = 11;                                        // bit_rotate/mod.rs:57
constexpr u32 LOG_N_LANES = 4;                                        // smallest component (round/component.rs:128)
// Largest permutation count: a multiplicity counter is a u32, and one bin receives at most 608 (XOR lookups per round row) x
// (2^22 + 2^21) rows at 2^18 permutations, < 2^32.
constexpr size_t MAX_PERMS = (size_t)1 << 18;

#define NB_KECCAK_RC                                                                                                   \
  0x0000000000000001ull, 0x0000000000008082ull, 0x800000000000808Aull, 0x8000000080008000ull, 0x000000000000808Bull,   \
  0x0000000080000001ull, 0x8000000080008081ull, 0x8000000000008009ull, 0x000000000000008Aull, 0x0000000000000088ull,   \
  0x0000000080008009ull, 0x000000008000000Aull, 0x000000008000808Bull, 0x800000000000008Bull, 0x8000000000008089ull,   \
  0x8000000000008003ull, 0x8000000000008002ull, 0x8000000000000080ull, 0x000000000000800Aull, 0x800000008000000Aull,   \
  0x8000000080008081ull, 0x8000000000008080ull, 0x0000000080000001ull, 0x8000000080008008ull
#if defined(__CUDACC__)
__constant__ u64 kRoundConstants[24] = {NB_KECCAK_RC};
#endif

// RC[i] of round i (FIPS 202 Algorithm 6)
NB_HD u64 round_constant(u32 i) {
#if defined(__CUDA_ARCH__)
  return kRoundConstants[i];
#else
  static const u64 t[24] = {NB_KECCAK_RC};
  return t[i];
#endif
}

// rho offset of lane x + 5 y (FIPS 202 Algorithm 2); called with constants only, so it folds away
NB_HD u32 rho(u32 k) {
  const u32 r[25] = {0, 1, 62, 28, 27, 36, 44, 6, 55, 20, 3, 10, 43, 25, 39, 41, 45, 15, 21, 8, 18, 2, 61, 56, 14};
  return r[k];
}

NB_HD u64 rotl64(u64 v, u32 r) { return r ? (v << r) | (v >> (64 - r)) : v; }

// one round on lanes a[x + 5 y] (round/mod.rs:11-51)
NB_HD void keccak_round(u64 a[25], u64 rc) {
  u64 c[5], b[25];
#pragma unroll
  for (int x = 0; x < 5; ++x) c[x] = a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20];
#pragma unroll
  for (int x = 0; x < 5; ++x) {
    const u64 d = c[(x + 4) % 5] ^ rotl64(c[(x + 1) % 5], 1);
#pragma unroll
    for (int y = 0; y < 5; ++y) a[x + 5 * y] ^= d;
  }
#pragma unroll
  for (int x = 0; x < 5; ++x)
#pragma unroll
    for (int y = 0; y < 5; ++y) b[y + ((2 * x + 3 * y) % 5) * 5] = rotl64(a[x + 5 * y], rho(x + 5 * y));
#pragma unroll
  for (int i = 0; i < 25; ++i) a[i] = b[i] ^ (~b[(i % 5 + 1) % 5 + 5 * (i / 5)] & b[(i % 5 + 2) % 5 + 5 * (i / 5)]);
  a[0] ^= rc;
}

// ---- lookups: the keys the three tables are counted under ------------------------------------------------------------------
// byte j of a bitwise lookup (a, b): histogram bin (a_j << 8) | b_j
NB_HD u32 bitwise_key(u64 a, u64 b, u32 j) { return (u32)(((a >> (8 * j)) & 255) << 8 | ((b >> (8 * j)) & 255)); }
// byte j of a rotation of a by r (bits = r % 8): BitRotateTable row 8 a_j + bits
NB_HD u32 rotate_key(u64 a, u32 bits, u32 j) { return (u32)(8 * ((a >> (8 * j)) & 255) + bits); }
// BitwiseAccumulator (bitwise_table/constraints.rs:46-68): trace row `row` of multiplicity column `col` (0..15) counts the lookups
// (a, b) with a = (col / 4) << 6 | row >> 6, b = (col % 4) << 6 | row & 63
NB_HD u32 bitwise_mult_key(u32 col, u32 row) {
  const u32 a = (col >> 2) << 6 | (row >> 6), b = (col & 3) << 6 | (row & 63);
  return a << 8 | b;
}
NB_HD u32 mod_p(u32 v) { return v >= P31 ? v - P31 : v; }   // counts are below 2^32 < 2 P
constexpr u32 BITWISE_MULT_WORDS = 2 * BITWISE_MULT_COLS << BITWISE_LOG;
constexpr u32 MULT_WORDS = BITWISE_MULT_WORDS + (1u << ROTATE_LOG);
// word e < MULT_WORDS of the multiplicity columns in finalized order, mod P: XorTable's 16 columns of 2^12 rows, BitNotAndTable's 16,
// then BitRotateTable's one column of 2^11 rows (row 8 byte + bits)
NB_HD u32 mult_word(const u32* xor_hist, const u32* nand_hist, const u32* rot_hist, u32 e) {
  if (e < BITWISE_MULT_WORDS) {
    const u32 col = e >> BITWISE_LOG, i = e & ((1u << BITWISE_LOG) - 1);
    const u32 key = bitwise_mult_key(col % BITWISE_MULT_COLS, (u32)finalized_src_row(i, BITWISE_LOG));
    return mod_p((col < BITWISE_MULT_COLS ? xor_hist : nand_hist)[key]);
  }
  return mod_p(rot_hist[finalized_src_row(e - BITWISE_MULT_WORDS, ROTATE_LOG)]);
}

// ---- round component: generate_round_component_trace (round/trace.rs:297-366) ----------------------------------------------
// Sink: lane(v) stores the next allocated lane (8 byte columns), xor_lookup / nand_lookup (a, b) and rot_lookup (a, bits) count the
// table lookups of one lane.  On return a[] holds the round's output state.
template <class Sink>
NB_HD void round_row(u64 a[25], u64 rc, Sink& s) {
  auto xr = [&](u64 x, u64 y) { s.xor_lookup(x, y); const u64 r = x ^ y; s.lane(r); return r; };
  auto nand = [&](u64 x, u64 y) { s.nand_lookup(x, y); const u64 r = ~x & y; s.lane(r); return r; };
  // rotate_left (round/constraints.rs:158-193): lanes bits_low, bits_high, out
  auto rot = [&](u64 x, u32 r) {
    if (r == 0) return x;
    const u32 bits = r % 8;
    s.rot_lookup(x, bits);
    const u64 ones = 0x0101010101010101ull;
    s.lane((x << bits) & (ones * ((0xFFu << bits) & 0xFFu)));
    s.lane((x >> (8 - bits)) & (ones * (0xFFu >> (8 - bits))));
    const u64 out = rotl64(x, r);
    s.lane(out);
    return out;
  };
#pragma unroll
  for (int i = 0; i < 25; ++i) s.lane(a[i]);
  u64 c[5];
#pragma unroll
  for (int x = 0; x < 5; ++x) {                                   // theta
    u64 acc = a[x];
#pragma unroll
    for (int i = 1; i < 5; ++i) acc = xr(acc, a[x + 5 * i]);
    c[x] = acc;
  }
  u64 d[5];
#pragma unroll
  for (int x = 0; x < 5; ++x) {
    const u64 r = rot(c[(x + 1) % 5], 1);
    d[x] = xr(c[(x + 4) % 5], r);
  }
#pragma unroll
  for (int x = 0; x < 5; ++x)
#pragma unroll
    for (int y = 0; y < 5; ++y) a[x + 5 * y] = xr(a[x + 5 * y], d[x]);
  u64 b[25];
#pragma unroll
  for (int x = 0; x < 5; ++x)                                     // rho and pi
#pragma unroll
    for (int y = 0; y < 5; ++y) b[y + ((2 * x + 3 * y) % 5) * 5] = rot(a[x + 5 * y], rho(x + 5 * y));
#pragma unroll
  for (int x = 0; x < 5; ++x)                                     // chi
#pragma unroll
    for (int y = 0; y < 5; ++y) {
      const u64 n = nand(b[(x + 1) % 5 + 5 * y], b[(x + 2) % 5 + 5 * y]);
      a[x + 5 * y] = xr(b[x + 5 * y], n);
    }
  a[0] = xr(a[0], rc);                                            // iota
}

// Row `i` (finalized position) of KeccakRound { rounds, offset } of 2^log_size rows: trace row perm * rounds + t holds the state of
// permutation perm before round offset + t; rows from n_perms * rounds on are padding: the zero state with RC[offset + row % rounds].
// inputs = n_perms x 25 lanes.  Returns is_padding.
template <class Sink>
NB_HD bool round_component_row(const u64* inputs, u32 n_perms, u32 rounds, u32 offset, u32 log_size, u32 i, Sink& s) {
  const u32 row = (u32)finalized_src_row(i, log_size);
  const u32 perm = row / rounds, t = row % rounds;
  u64 a[25];
  const bool padding = perm >= n_perms;
#pragma unroll
  for (int k = 0; k < 25; ++k) a[k] = padding ? 0 : inputs[(size_t)perm * 25 + k];
  if (!padding)
    for (u32 r = 0; r < offset + t; ++r) keccak_round(a, round_constant(r));
  round_row(a, round_constant(offset + t), s);
  return padding;
}

// column writer: lane k of the row goes to byte columns 8 k .. 8 k + 7 at out[col * stride]
struct ColumnSink {
  u32* out;
  size_t stride;
  u32 col = 0;
  NB_HD void lane(u64 v) {
#pragma unroll
    for (u32 j = 0; j < LANE; ++j) out[(size_t)(col + j) * stride] = (u32)((v >> (8 * j)) & 255);
    col += LANE;
  }
  NB_HD void xor_lookup(u64, u64) {}
  NB_HD void nand_lookup(u64, u64) {}
  NB_HD void rot_lookup(u64, u32) {}
};

// lookup counter: Inc()(u32*) adds one to a bin (an atomic add on the device)
template <class Inc>
struct CountSink {
  u32 *xor_hist, *nand_hist, *rot_hist;   // 2^16, 2^16 and 2^11 bins
  NB_HD void lane(u64) {}
  NB_HD void xor_lookup(u64 a, u64 b) {
#pragma unroll
    for (u32 j = 0; j < LANE; ++j) Inc()(xor_hist + bitwise_key(a, b, j));
  }
  NB_HD void nand_lookup(u64 a, u64 b) {
#pragma unroll
    for (u32 j = 0; j < LANE; ++j) Inc()(nand_hist + bitwise_key(a, b, j));
  }
  NB_HD void rot_lookup(u64 a, u32 bits) {
#pragma unroll
    for (u32 j = 0; j < LANE; ++j) Inc()(rot_hist + rotate_key(a, bits, j));
  }
};

// ---- PermutationMemoryCheck: generate_keccak_mem_check_trace (memory_check/trace.rs:32-123) -------------------------------
// Row `i` (finalized position) of 2^log_size rows into out[col * stride], col < MEM_COLS: input state bytes, output state bytes, then
// (lo, hi) 16-bit limbs of address + k, previous timestamp and previous timestamp + 1 for the 200 state bytes k, the address carries
// (low limb == 0xFFFF), the timestamp carries, is_padding.  Padding rows (from n_perms on) are zero but for is_padding.
// The caller guarantees address + 199 and timestamp + 1 below 2^32.
NB_HD void mem_row(const u64* inputs, const u32* addresses, const u32* timestamps, u32 n_perms, u32 log_size, u32 i, u32* out, size_t stride) {
  const u32 perm = (u32)finalized_src_row(i, log_size);
  auto put = [&](u32 col, u32 v) { out[(size_t)col * stride] = v; };
  if (perm >= n_perms) {
    for (u32 c = 0; c + 1 < MEM_COLS; ++c) put(c, 0);
    put(MEM_COLS - 1, 1);
    return;
  }
  u64 a[25];
#pragma unroll
  for (int k = 0; k < 25; ++k) a[k] = inputs[(size_t)perm * 25 + k];
#pragma unroll
  for (u32 k = 0; k < STATE; ++k) put(k, (u32)((a[k / LANE] >> (8 * (k % LANE))) & 255));
  for (u32 r = 0; r < 24; ++r) keccak_round(a, round_constant(r));
#pragma unroll
  for (u32 k = 0; k < STATE; ++k) put(STATE + k, (u32)((a[k / LANE] >> (8 * (k % LANE))) & 255));
  const u32 base = addresses[perm];
  const u32* ts = timestamps + (size_t)perm * STATE;
  for (u32 k = 0; k < STATE; ++k) {
    const u32 addr = base + k, prev = ts[k], next = prev + 1;
    put(2 * STATE + 2 * k, addr & 0xFFFF);
    put(2 * STATE + 2 * k + 1, addr >> 16);
    put(4 * STATE + 2 * k, prev & 0xFFFF);
    put(4 * STATE + 2 * k + 1, prev >> 16);
    put(6 * STATE + 2 * k, next & 0xFFFF);
    put(6 * STATE + 2 * k + 1, next >> 16);
    put(8 * STATE + k, (addr & 0xFFFF) == 0xFFFF);
    put(9 * STATE + k, (prev & 0xFFFF) == 0xFFFF);
  }
  put(MEM_COLS - 1, 0);
}

}  // namespace keccak
}  // namespace nb
