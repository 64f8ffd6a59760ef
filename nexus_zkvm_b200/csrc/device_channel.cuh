// The Blake2s Fiat-Shamir channel (host_channel.h) run by one device thread, for the stretch of the protocol in which the host has
// nothing to add: FRI's inner layers, where every round is "commit a folded layer, mix its root, draw the next folding alpha".  The
// state lives in device memory, so the layers are queued back to back without a host round trip; the host channel replays the same
// steps afterwards from the roots and checks every alpha (prove.cu: fri_commit).
#pragma once
#include "blake2s.cuh"

namespace nb {

// HostChannel's digest and n_sent (n_challenges is not read by any draw)
struct DevChannel { u32 digest[8]; u32 n_sent[2]; u32 pad[6]; };

#if defined(__CUDACC__)
// RFC 7693 Blake2s-256 of the 64 bytes m, followed by one zero byte when `extra_zero` (HostChannel::draw_random_bytes with draw_domain_sep)
__device__ __forceinline__ void dev_b2s_64(const u32 (&m)[16], bool extra_zero, u32 (&h)[8]) {
  b2s_init(h);
  if (!extra_zero) { b2s_compress(h, m, 64u, 0u, 0xFFFFFFFFu, 0u); return; }
  b2s_compress(h, m, 64u, 0u, 0u, 0u);
  u32 z[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) z[i] = 0;
  b2s_compress(h, z, 65u, 0u, 0xFFFFFFFFu, 0u);
}

// HostChannel::mix_root
__device__ __forceinline__ void dev_mix_root(DevChannel& c, const u32 (&root)[8]) {
  u32 m[16], h[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { m[i] = c.digest[i]; m[8 + i] = root[i]; }
  dev_b2s_64(m, false, h);
#pragma unroll
  for (int i = 0; i < 8; ++i) c.digest[i] = h[i];
  c.n_sent[0] = c.n_sent[1] = 0;
}

// HostChannel::draw_felt: draw_random_bytes until no word is >= 2P, then the first four words reduced mod P
__device__ __forceinline__ void dev_draw_felt(DevChannel& c, bool domain_sep, u32 (&out)[4]) {
  while (true) {
    u32 m[16], h[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) m[i] = c.digest[i];
    m[8] = c.n_sent[0]; m[9] = c.n_sent[1];
#pragma unroll
    for (int i = 10; i < 16; ++i) m[i] = 0;
    if (++c.n_sent[0] == 0) ++c.n_sent[1];
    dev_b2s_64(m, domain_sep, h);
    bool ok = true;
#pragma unroll
    for (int i = 0; i < 8; ++i) ok = ok && h[i] < 2 * P31;
    if (ok) {
#pragma unroll
      for (int i = 0; i < 4; ++i) out[i] = h[i] >= P31 ? h[i] - P31 : h[i];
      return;
    }
  }
}
#endif

}  // namespace nb
