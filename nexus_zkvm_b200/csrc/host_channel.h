// Host-side Fiat-Shamir transcript: Blake2sChannel + Blake2sMerkleChannel::mix_root
// (stwo core/channel/blake2s.rs, core/vcs/blake2_merkle.rs), as used by the reference at
// nexus-zkvm prover/src/machine.rs:197-206,240,262 and inside stwo::prover::prove (machine.rs:286-290).
// The channel serialises the protocol, it is not data-parallel work: it stays on the host (SURVEY.md §8 a6), except between FRI's
// inner layers, where device_channel.cuh runs the same steps and this channel replays them.
#pragma once
#include "blake2s.cuh"
#include <vector>
#include <array>

namespace nb {

typedef std::array<uint8_t, 32> Hash32;

struct HostChannel {
  Hash32 digest;
  uint64_t n_challenges = 0, n_sent = 0;
  int draw_domain_sep = 0;  // [risk] newer upstream revisions append a 0x00 byte in draw_random_bytes
  HostChannel() { digest.fill(0); }
  void update_digest(const uint8_t d[32]) { memcpy(digest.data(), d, 32); n_challenges += 1; n_sent = 0; }
  void mix_u32s(const u32* w, size_t n) {
    Blake2sHost b; b.update(digest.data(), 32);
    for (size_t i = 0; i < n; ++i) { uint8_t le[4] = {(uint8_t)w[i], (uint8_t)(w[i] >> 8), (uint8_t)(w[i] >> 16), (uint8_t)(w[i] >> 24)}; b.update(le, 4); }
    uint8_t out[32]; b.finalize(out); update_digest(out);
  }
  void mix_u64(uint64_t v) { u32 w[2] = {(u32)v, (u32)(v >> 32)}; mix_u32s(w, 2); }
  void mix_felts(const qm31* f, size_t n) { mix_u32s(n ? f[0].c : nullptr, 4 * n); }
  void mix_root(const uint8_t root[32]) {
    Blake2sHost b; b.update(digest.data(), 32); b.update(root, 32);
    uint8_t out[32]; b.finalize(out); update_digest(out);
  }
  void draw_random_bytes(uint8_t out[32]) {
    uint8_t in[65]; memcpy(in, digest.data(), 32); memset(in + 32, 0, 33);
    for (int i = 0; i < 8; ++i) in[32 + i] = (uint8_t)(n_sent >> (8 * i));
    n_sent += 1;
    Blake2sHost b; b.update(in, draw_domain_sep ? 65 : 64); b.finalize(out);
  }
  void draw_base_felts(u32 out[8]) {
    while (true) {
      uint8_t r[32]; draw_random_bytes(r);
      bool ok = true;
      for (int i = 0; i < 8; ++i) {
        u32 w = (u32)r[4 * i] | ((u32)r[4 * i + 1] << 8) | ((u32)r[4 * i + 2] << 16) | ((u32)r[4 * i + 3] << 24);
        if (w >= 2 * P31) ok = false;
        out[i] = w >= P31 ? w - P31 : w;
      }
      if (ok) return;
    }
  }
  qm31 draw_felt() { u32 f[8]; draw_base_felts(f); return qm31_make(f[0], f[1], f[2], f[3]); }
  void draw_felts(size_t n, qm31* out) {
    u32 f[8]; int have = 0;
    for (size_t i = 0; i < n; ++i) {
      if (have == 0) { draw_base_felts(f); have = 8; }
      int o = 8 - have;
      out[i] = qm31_make(f[o], f[o + 1], f[o + 2], f[o + 3]);
      have -= 4;
    }
  }
  u32 trailing_zeros() const {
    u32 tz = 0;
    for (int i = 0; i < 16; ++i) {
      uint8_t b = digest[i];
      if (b == 0) { tz += 8; continue; }
      while ((b & 1) == 0) { ++tz; b >>= 1; }
      return tz;
    }
    return 128;
  }
};

}  // namespace nb
