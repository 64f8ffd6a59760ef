// Circle FFT / iFFT over M31 for batches of columns (PolyOps::interpolate / PolyOps::evaluate).
// Replaces the SimdBackend `ifft` / `rfft` reached from TreeBuilder::extend_evals and TreeBuilder::commit at
// nexus-zkvm prover/src/machine.rs:208-263 (and prover2/machine/src/prove.rs:70-105).
//
// Algorithm (identical butterfly network to stwo's CPU backend so results are bit-exact):
//   values are in bit-reversed circle-domain order; layer i pairs indices that differ in bit i with
//   twiddle index h = idx >> (i+1); layer 0 uses the circle (y) twiddles derived from the first line layer
//   ([x, y] -> [y, -y, -x, x]), layers >= 1 use line (x) twiddles; interpolate runs layers 0..n-1 with
//   ibutterfly and scales by 2^-n, evaluate runs n-1..0 with butterfly on zero-extended coefficients.
//
// Kernel structure (integer work bounded by HBM traffic and INT32 issue, no tensor cores):
//   A transform of 2^n is split into passes of <= 13 layers.  A pass owns a contiguous range of layers
//   [lo, lo+L); each CTA stages a tile of 2^T words (2^L "rows" x 2^W contiguous words, W = T-L) of CB columns
//   into shared memory with coalesced 128-bit accesses, runs the L layers there in rounds of <= 4 layers (every
//   thread holds 16 words in registers: a radix-16 butterfly network per round), and writes the tile back.
//   Twiddles of a round are fetched with vector loads into registers and reused for the CB columns of the CTA.
//   Shared memory is XOR-swizzled; tests/test_layout.py proves every access pattern conflict-free.
//   `fft_tile_kernel<INV,T,W>` is the compile-time specialised fast path; `fft_pass_kernel` is the generic
//   fallback for shapes outside the specialised set.
#include "fft_common.cuh"
#include "circle_host.h"
#include <map>
#include <mutex>

namespace nb {

// NZ: (forward, top pass of a zero-extended input) the top NZ layers of the pass have all-zero odd inputs -> copies
template <bool INV, int T, int W, int CB, int NZ>
__global__ void __launch_bounds__(1 << (T - 4), (T >= 13 ? 2 : 3)) fft_tile_kernel(const FftPass p) {
  extern __shared__ __align__(16) u32 sm[];
  constexpr int L = T - W;
  constexpr int NT = 1 << (T - 4);
  constexpr int NFULL = L / 4, REM = L % 4, NROUNDS = NFULL + (REM ? 1 : 0);
  const u32 lo = p.lo, n = p.n;
  const u32 tid = threadIdx.x;
  const u32 tile = blockIdx.x;
  const u32 mid_bits = W ? lo - W : 0;
  const u32 tile_mid = tile & ((1u << mid_bits) - 1u);
  const u32 tile_hi = tile >> mid_bits;
  const size_t gbase = ((size_t)tile_hi << (lo + L)) | ((size_t)tile_mid << W);
  const u32 col0 = blockIdx.y * CB;
  const u32 ncb = min((u32)CB, p.n_cols - col0);

  // ---- staging geometry: thread `tid` moves the 4 x uint4 at s_it = (tid + it*NT)*4.  For NT*4 >= 512 the swizzle
  // bits (5, 6, 8) are not touched by `it`, so physical and global offsets are affine in `it` (no per-access math).
  constexpr bool AFFINE = (NT * 4 >= 512) && (W <= T - 2);
  const u32 s0 = tid * 4;
  const u32 phys0 = swz2(s0);
  const size_t g0 = W ? (gbase | ((size_t)(s0 >> W) << lo) | (s0 & ((1u << W) - 1u))) : (gbase | s0);
  const size_t gstep = W ? ((size_t)((NT * 4) >> W) << lo) : (size_t)(NT * 4);

  // ---- stage in: 128-bit coalesced global loads -> swizzled shared.
  // FUSE_TOP (forward passes whose layer count is 4k+1): the pass's top layer pairs s with s + 2^(T-1), i.e. the uint4 a thread moves at
  // `it` with the one at `it + 2`, and its twiddle is one value per tile — so it is applied here, on the way into shared memory, instead
  // of costing a whole shared-memory round (16 LDS + 16 STS + a barrier per thread and column) for 8 butterflies.
  constexpr bool FUSE_TOP = !INV && REM == 1 && L > 1;
  constexpr int NROUNDS_RUN = FUSE_TOP ? NFULL : NROUNDS;
  if (FUSE_TOP) {
    const u32 t2 = (NZ > 0) ? 0u : __ldg(p.tw2 + (p.tw_len - (1u << (p.tn - (lo + L - 1)))) + tile_hi);
    // all loads first (see the plain path below), then the top-layer butterflies and the shared stores
    constexpr int SBF = (CB >= 2) ? 2 : 1;   // two columns (up to 8 x 128 bits) in flight per thread
#pragma unroll
    for (int cb0 = 0; cb0 < CB; cb0 += SBF) {
    uint4 va[SBF][2], vb[SBF][2];
#pragma unroll
    for (int cc = 0; cc < SBF; ++cc) {
      const int c = cb0 + cc;
      const u32* __restrict__ scol = p.src + (size_t)(col0 + (c < (int)ncb ? c : 0)) * p.src_stride;
#pragma unroll
      for (int it = 0; it < 2; ++it) {
        size_t g, g2;
        if (AFFINE) { g = g0 + it * gstep; g2 = g0 + (it + 2) * gstep; }
        else {
          const u32 s = (tid + it * NT) * 4, s2 = (tid + (it + 2) * NT) * 4;
          g = W ? (gbase | ((size_t)(s >> W) << lo) | (s & ((1u << W) - 1u))) : (gbase | s);
          g2 = W ? (gbase | ((size_t)(s2 >> W) << lo) | (s2 & ((1u << W) - 1u))) : (gbase | s2);
        }
        va[cc][it] = make_uint4(0, 0, 0, 0); vb[cc][it] = make_uint4(0, 0, 0, 0);
        if (c < (int)ncb && g < p.src_len) va[cc][it] = __ldg(reinterpret_cast<const uint4*>(scol + g));
        if (NZ == 0 && c < (int)ncb && g2 < p.src_len) vb[cc][it] = __ldg(reinterpret_cast<const uint4*>(scol + g2));
      }
    }
#pragma unroll
    for (int cc = 0; cc < SBF; ++cc) {
      const int c = cb0 + cc;
      if (c < (int)ncb) {
#pragma unroll
        for (int it = 0; it < 2; ++it) {
          const u32 ph = AFFINE ? (phys0 + it * NT * 4) : swz2((tid + it * NT) * 4);
          const u32 ph2 = AFFINE ? (phys0 + (it + 2) * NT * 4) : swz2((tid + (it + 2) * NT) * 4);
          uint4 a = va[cc][it], b4 = vb[cc][it];
          if (NZ > 0) b4 = a;   // the partner is a zero-extension word: v0 + t*0 = v0 - t*0
          else { butterfly_dbl(a.x, b4.x, t2); butterfly_dbl(a.y, b4.y, t2); butterfly_dbl(a.z, b4.z, t2); butterfly_dbl(a.w, b4.w, t2); }
          *reinterpret_cast<uint4*>(sm + (c << T) + ph) = a;
          *reinterpret_cast<uint4*>(sm + (c << T) + ph2) = b4;
        }
      }
    }
    }
  } else {
    // Loads of SB columns (SB * 4 x 128 bits per thread) are all issued before the first shared store: the compiler otherwise emits
    // load-4 / store-4 per column, i.e. CB serialised global-memory latencies per CTA.
    constexpr int SB = (CB >= 2) ? 2 : 1;
#pragma unroll
    for (int cb0 = 0; cb0 < CB; cb0 += SB) {
      uint4 buf[SB][4];
#pragma unroll
      for (int cc = 0; cc < SB; ++cc) {
        const int c = cb0 + cc;
        const u32* __restrict__ scol = p.src + (size_t)(col0 + (c < (int)ncb ? c : 0)) * p.src_stride;
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          size_t g;
          if (AFFINE) g = g0 + it * gstep;
          else {
            const u32 s = (tid + it * NT) * 4;
            g = W ? (gbase | ((size_t)(s >> W) << lo) | (s & ((1u << W) - 1u))) : (gbase | s);
          }
          buf[cc][it] = make_uint4(0, 0, 0, 0);
          if (c < (int)ncb && g < p.src_len) buf[cc][it] = __ldg(reinterpret_cast<const uint4*>(scol + g));
        }
      }
#pragma unroll
      for (int cc = 0; cc < SB; ++cc) {
        const int c = cb0 + cc;
        if (c < (int)ncb) {
#pragma unroll
          for (int it = 0; it < 4; ++it) {
            const u32 ph = AFFINE ? (phys0 + it * NT * 4) : swz2((tid + it * NT) * 4);
            *reinterpret_cast<uint4*>(sm + (c << T) + ph) = buf[cc][it];
          }
        }
      }
    }
  }
  __syncthreads();

#pragma unroll
  for (int rr = 0; rr < NROUNDS_RUN; ++rr) {
    const int ri = INV ? rr : NROUNDS_RUN - 1 - rr;
    const int b = ri < NFULL ? W + 4 * ri : T - 4;
    const int jlo = ri < NFULL ? 0 : 4 - REM;
    const u32 tau_hi = tid >> b, tau_lo = tid & ((1u << b) - 1u);
    u32 triv = 0u;
    if (!INV && NZ > 0) {
#pragma unroll
      for (int j = 0; j < 4; ++j) if (b + j - W >= L - NZ) triv |= 1u << j;
    }
    // twiddles: layer j of the round is global layer i = lo + b + j - W; the (8 >> j) twiddles of a thread are contiguous
    u32 tw[15] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (j >= jlo) {
        const u32 i = lo + b + j - W;
        const u32 hbase = (tile_hi << (L - (b + j - W) - 1)) | (tau_hi << (3 - j));
        const u32* __restrict__ src = (W == 0 && b + j == 0) ? (p.ctw2 + hbase) : (p.tw2 + (p.tw_len - (1u << (p.tn - i))) + hbase);
        if (j == 0) {
          uint4 a = __ldg(reinterpret_cast<const uint4*>(src)), c4 = __ldg(reinterpret_cast<const uint4*>(src) + 1);
          tw[0] = a.x; tw[1] = a.y; tw[2] = a.z; tw[3] = a.w; tw[4] = c4.x; tw[5] = c4.y; tw[6] = c4.z; tw[7] = c4.w;
        } else if (j == 1) {
          uint4 a = __ldg(reinterpret_cast<const uint4*>(src));
          tw[8] = a.x; tw[9] = a.y; tw[10] = a.z; tw[11] = a.w;
        } else if (j == 2) {
          uint2 a = __ldg(reinterpret_cast<const uint2*>(src));
          tw[12] = a.x; tw[13] = a.y;
        } else {
          tw[14] = __ldg(src);
        }
      }
    }
    const u32 sbase = (tau_hi << (b + 4)) | tau_lo;
    if (b == 0) {
      // the 16 words of a thread are contiguous: 4 x 128-bit shared accesses
      const u32 a0 = swz2(sbase), a1 = swz2(sbase | 4u), a2 = swz2(sbase | 8u), a3 = swz2(sbase | 12u);
#pragma unroll
      for (int c = 0; c < CB; ++c) {
        if (c < (int)ncb) {
          u32* smc = sm + (c << T);
          u32 v[16];
          uint4 q0 = *reinterpret_cast<uint4*>(smc + a0), q1 = *reinterpret_cast<uint4*>(smc + a1);
          uint4 q2 = *reinterpret_cast<uint4*>(smc + a2), q3 = *reinterpret_cast<uint4*>(smc + a3);
          v[0] = q0.x; v[1] = q0.y; v[2] = q0.z; v[3] = q0.w; v[4] = q1.x; v[5] = q1.y; v[6] = q1.z; v[7] = q1.w;
          v[8] = q2.x; v[9] = q2.y; v[10] = q2.z; v[11] = q2.w; v[12] = q3.x; v[13] = q3.y; v[14] = q3.z; v[15] = q3.w;
          radix16<INV>(v, tw, jlo, triv);
          *reinterpret_cast<uint4*>(smc + a0) = make_uint4(v[0], v[1], v[2], v[3]);
          *reinterpret_cast<uint4*>(smc + a1) = make_uint4(v[4], v[5], v[6], v[7]);
          *reinterpret_cast<uint4*>(smc + a2) = make_uint4(v[8], v[9], v[10], v[11]);
          *reinterpret_cast<uint4*>(smc + a3) = make_uint4(v[12], v[13], v[14], v[15]);
        }
      }
    } else {
      u32 addr[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) addr[k] = swz2(sbase | ((u32)k << b));
#pragma unroll
      for (int c = 0; c < CB; ++c) {
        if (c < (int)ncb) {
          u32* smc = sm + (c << T);
          u32 v[16];
#pragma unroll
          for (int k = 0; k < 16; ++k) v[k] = smc[addr[k]];
          radix16<INV>(v, tw, jlo, triv);
#pragma unroll
          for (int k = 0; k < 16; ++k) smc[addr[k]] = v[k];
        }
      }
    }
    __syncthreads();
  }

  // ---- stage out
#pragma unroll
  for (int c = 0; c < CB; ++c) {
    if (c < (int)ncb) {
      u32* __restrict__ dcol = p.dst + (size_t)(col0 + c) * p.dst_stride;
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        u32 ph; size_t g;
        if (AFFINE) { ph = phys0 + it * NT * 4; g = g0 + it * gstep; }
        else {
          const u32 s = (tid + it * NT) * 4;
          ph = swz2(s);
          g = W ? (gbase | ((size_t)(s >> W) << lo) | (s & ((1u << W) - 1u))) : (gbase | s);
        }
        uint4 v = *reinterpret_cast<const uint4*>(sm + (c << T) + ph);
        if (p.apply_scale) { const u32 sc2 = p.scale << 1; v.x = m31_mul_dbl(v.x, sc2); v.y = m31_mul_dbl(v.y, sc2); v.z = m31_mul_dbl(v.z, sc2); v.w = m31_mul_dbl(v.w, sc2); }
        *reinterpret_cast<uint4*>(dcol + g) = v;
      }
    }
  }
}

// =====================================================================================================
// generic fallback (runtime tile shape)
// =====================================================================================================
__device__ __forceinline__ u32 swz(u32 s) { return s ^ ((s >> 4) & 31u); }

template <bool INV>
__global__ void __launch_bounds__(512) fft_pass_kernel(const FftPass p) {
  extern __shared__ u32 sm[];
  const u32 T = p.T, W = p.W, L = T - W, lo = p.lo, n = p.n;
  const u32 nthreads = blockDim.x;  // 2^(T-4)
  const u32 tid = threadIdx.x;
  const u32 tile = blockIdx.x;
  const u32 mid_bits = lo > W ? lo - W : 0;  // lo == 0 implies W == 0
  const u32 tile_mid = tile & ((1u << mid_bits) - 1u);
  const u32 tile_hi = tile >> mid_bits;
  const size_t gbase = ((size_t)tile_hi << (lo + L)) | ((size_t)tile_mid << W);
  const u32 wmask = (1u << W) - 1u;
  const u32 col0 = blockIdx.y * p.cb;
  const u32 ncb = min(p.cb, p.n_cols - col0);
  const u32 tile_words = 1u << T;

  for (u32 c = 0; c < ncb; ++c) {
    const u32* __restrict__ scol = p.src + (size_t)(col0 + c) * p.src_stride;
    u32* smc = sm + ((size_t)c << T);
    for (u32 s = tid; s < tile_words; s += nthreads) {
      size_t g = gbase | ((size_t)(s >> W) << lo) | (s & wmask);
      u32 v = g < p.src_len ? __ldg(scol + g) : 0u;
      smc[swz(s)] = v;
    }
  }
  __syncthreads();

  const u32 nfull = L >> 2, rem = L & 3u;
  const u32 nrounds = nfull + (rem ? 1u : 0u);
  for (u32 rr = 0; rr < nrounds; ++rr) {
    const u32 ri = INV ? rr : nrounds - 1 - rr;
    u32 b, jlo;
    if (ri < nfull) { b = W + 4 * ri; jlo = 0; } else { b = T - 4; jlo = 4 - rem; }
    const u32 tau_hi = tid >> b, tau_lo = tid & ((1u << b) - 1u);
    u32 tw[15];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if ((u32)j >= jlo) {
        const u32 i = lo + b + j - W;
        const u32 hbase = ((tile_hi << (L - (b + j - W) - 1)) | (tau_hi << (3 - j)));
#pragma unroll
        for (int kk = 0; kk < (8 >> j); ++kk) {
          const int off = (j == 0 ? 0 : j == 1 ? 8 : j == 2 ? 12 : 14) + kk;
          tw[off] = (i == 0) ? circle_tw(p.tw, p.tw_len, p.tn, hbase + kk) : line_tw(p.tw, p.tw_len, p.tn, i, hbase + kk);
        }
      }
    }
    const u32 sbase = (tau_hi << (b + 4)) | tau_lo;
    for (u32 c = 0; c < ncb; ++c) {
      u32* smc = sm + ((size_t)c << T);
      u32 v[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) v[k] = smc[swz(sbase | ((u32)k << b))];
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int j = INV ? jj : 3 - jj;
        if ((u32)j >= jlo) {
#pragma unroll
          for (int m = 0; m < 8; ++m) {
            const int k0 = ((m >> j) << (j + 1)) | (m & ((1 << j) - 1));
            const int k1 = k0 | (1 << j);
            const int off = (j == 0 ? 0 : j == 1 ? 8 : j == 2 ? 12 : 14) + (m >> j);
            if (INV) ibutterfly(v[k0], v[k1], tw[off]);
            else butterfly(v[k0], v[k1], tw[off]);
          }
        }
      }
#pragma unroll
      for (int k = 0; k < 16; ++k) smc[swz(sbase | ((u32)k << b))] = v[k];
    }
    __syncthreads();
  }

  for (u32 c = 0; c < ncb; ++c) {
    u32* __restrict__ dcol = p.dst + (size_t)(col0 + c) * p.dst_stride;
    const u32* smc = sm + ((size_t)c << T);
    for (u32 s = tid; s < tile_words; s += nthreads) {
      size_t g = gbase | ((size_t)(s >> W) << lo) | (s & wmask);
      u32 v = smc[swz(s)];
      if (p.apply_scale) v = m31_mul(v, p.scale);
      dcol[g] = v;
    }
  }
}

// Generic small transform (n <= 8): one CTA per column, whole column in shared memory, layer by layer.
struct FftSmall {
  const u32* src; u32* dst; size_t src_stride, dst_stride, src_len;
  const u32* tw; u32 tw_len; u32 n_cols, n;
  u32 y0;      // n <= 2: (inverse of) y of half_coset.initial
  u32 scale, apply_scale;
};
template <bool INV>
__global__ void fft_small_kernel(const FftSmall p) {
  extern __shared__ u32 sm[];
  const u32 n = p.n, len = 1u << n, half = len >> 1;
  const u32 c = blockIdx.x;
  const u32* __restrict__ scol = p.src + (size_t)c * p.src_stride;
  u32* __restrict__ dcol = p.dst + (size_t)c * p.dst_stride;
  for (u32 s = threadIdx.x; s < len; s += blockDim.x) sm[s] = s < p.src_len ? scol[s] : 0u;
  __syncthreads();
  for (u32 ll = 0; ll < n; ++ll) {
    const u32 i = INV ? ll : n - 1 - ll;
    for (u32 idx = threadIdx.x; idx < half; idx += blockDim.x) {
      u32 h = idx >> i, l = idx & ((1u << i) - 1u);
      u32 i0 = (h << (i + 1)) + l, i1 = i0 + (1u << i);
      u32 t;
      if (i == 0) {
        if (n <= 2) t = (h & 1u) ? (P31 - p.y0) : p.y0;   // n == 1: [y]; n == 2: [y, -y]
        else t = circle_tw(p.tw, p.tw_len, n, h);
      } else {
        t = line_tw(p.tw, p.tw_len, n, i, h);
      }
      u32 a = sm[i0], b = sm[i1];
      if (INV) ibutterfly(a, b, t); else butterfly(a, b, t);
      sm[i0] = a; sm[i1] = b;
    }
    __syncthreads();
  }
  for (u32 s = threadIdx.x; s < len; s += blockDim.x) {
    u32 v = sm[s];
    if (p.apply_scale) v = m31_mul(v, p.scale);
    dcol[s] = v;
  }
}

// out[i] = in[src(i)]: coset order -> circle-domain order -> bit-reversed  (finalize_columns,
// nexus-zkvm prover/src/trace/utils.rs:94-106 + utils_external.rs:24-39); src words are EB bytes wide (packed host format)
template <int EB>
__global__ void reorder_kernel(const void* __restrict__ src, u32* __restrict__ dst, u32 log_size, size_t total, int coset_order) {
  size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  size_t n = (size_t)1 << log_size;
  size_t c = e >> log_size;
  u32 i = (u32)(e & (n - 1));
  size_t s = i;
  if (coset_order) {
    u32 j = log_size ? (__brev(i) >> (32 - log_size)) : 0;
    size_t half = n >> 1;
    s = j < half ? ((size_t)j << 1) : (n - 1 - (((size_t)j - half) << 1));
  }
  u32 v;
  if (EB == 1) v = reinterpret_cast<const uint8_t*>(src)[c * n + s];
  else if (EB == 2) v = reinterpret_cast<const uint16_t*>(src)[c * n + s];
  else v = reinterpret_cast<const u32*>(src)[c * n + s];
  dst[e] = v;
}

nb200_status reorder_coset_to_bitrev(nb200_ctx* ctx, const u32* src, u32* dst, size_t n_cols, u32 log_size) {
  return expand_reorder(ctx, src, 4, dst, n_cols, log_size, 1);
}

// packed host words (elem_bytes = 1, 2 or 4) -> u32 columns, optionally applying finalize_columns' permutation
nb200_status expand_reorder(nb200_ctx* ctx, const void* src, u32 elem_bytes, u32* dst, size_t n_cols, u32 log_size, int coset_order) {
  NB_ARG(ctx, (const void*)src != (const void*)dst, "reorder must be out of place");
  NB_ARG(ctx, elem_bytes == 1 || elem_bytes == 2 || elem_bytes == 4, "packed columns: 1, 2 or 4 bytes per word");
  size_t total = n_cols << log_size;
  if (total == 0) return NB200_OK;
  u32 threads = 256;
  size_t blocks = (total + threads - 1) / threads;
  if (elem_bytes == 1) reorder_kernel<1><<<(u32)blocks, threads, 0, ctx->stream>>>(src, dst, log_size, total, coset_order);
  else if (elem_bytes == 2) reorder_kernel<2><<<(u32)blocks, threads, 0, ctx->stream>>>(src, dst, log_size, total, coset_order);
  else reorder_kernel<4><<<(u32)blocks, threads, 0, ctx->stream>>>(src, dst, log_size, total, coset_order);
  NB_LAUNCH_CHECK(ctx);
  return NB200_OK;
}

// ---- circle-twiddle tables (layer 0 of each transform size), owned by the ctx (freed in nb200_ctx_destroy) ----
struct CircleTables { std::map<u32, std::pair<u32*, u32*>> by_log; };
void fft_drop_tables(nb200_ctx* ctx) {
  CircleTables* ct = (CircleTables*)ctx->fft_tables;
  if (!ct) return;
  for (auto& kv : ct->by_log) { cudaFree(kv.second.first); cudaFree(kv.second.second); }
  delete ct;
  ctx->fft_tables = nullptr;
}
nb200_status fft_circle_tables(nb200_ctx* ctx, u32 n, const u32** fwd, const u32** inv) {
  if (!ctx->fft_tables) ctx->fft_tables = new CircleTables();
  CircleTables& ct = *(CircleTables*)ctx->fft_tables;   // tables hold values derived from the generator, not pointers into the bank
  auto it = ct.by_log.find(n);
  if (it == ct.by_log.end()) {
    u32 *f = nullptr, *g = nullptr;
    size_t len = (size_t)1 << (n - 1);
    NB_CUDA(ctx, cudaMalloc(&f, len * 4));
    if (cudaMalloc(&g, len * 4) != cudaSuccess) { cudaFree(f); cudaGetLastError(); return set_err(ctx, NB200_ERR_OOM, "circle tables"); }
    u32 thr = 256, blk = (u32)((len + thr - 1) / thr);
    circle_table_kernel<<<blk, thr, 0, ctx->stream>>>(ctx->tw.d_tw, 1u << ctx->tw.half_log, n, f);
    NB_LAUNCH_CHECK(ctx);
    circle_table_kernel<<<blk, thr, 0, ctx->stream>>>(ctx->tw.d_itw, 1u << ctx->tw.half_log, n, g);
    NB_LAUNCH_CHECK(ctx);
    it = ct.by_log.emplace(n, std::make_pair(f, g)).first;
  }
  *fwd = it->second.first; *inv = it->second.second;
  return NB200_OK;
}

// ---- pass planning ----
struct PassPlan { u32 lo, T, W; };
static void plan_passes(u32 n, std::vector<PassPlan>& out) {
  // contiguous pass over the low layers, then strided passes (tile rows x 2^W contiguous words, W >= 4)
  out.clear();
  if (n <= 13) { out.push_back(PassPlan{0, n, 0}); return; }
  u32 rest_min = n - 13;                      // layers left if the contiguous pass takes 13
  u32 npass = (rest_min + 8) / 9;             // strided passes of <= 9 layers
  u32 LA = n - npass * 8;                     // give the strided passes 8 layers each when possible
  if (LA < 9) LA = 9;
  if (LA > 13) LA = 13;
  // the 12-layer contiguous kernel (4 columns per CTA, 3 CTAs/SM) is the most efficient one: prefer it when the strided passes can
  // absorb the extra layer (a 9-layer strided pass applies its top layer while staging, see FUSE_TOP): 2^21 = 12 + 9
  if (LA == 13 && n - 12 <= 9 * npass) LA = 12;
  out.push_back(PassPlan{0, LA, 0});
  u32 rest = n - LA, lo = LA;
  for (u32 k = 0; k < npass; ++k) {
    u32 L = rest / npass + (k < rest % npass ? 1 : 0);
    if (L == 9) out.push_back(PassPlan{lo, 13, 4});
    else out.push_back(PassPlan{lo, 12, 12 - L});
    lo += L;
  }
}

template <bool INV, int T, int W, int CB, int NZ>
static nb200_status launch_tile(nb200_ctx* ctx, const FftPass& p) {
  constexpr int threads = 1 << (T - 4);
  constexpr size_t smem = (size_t)CB << (T + 2);
  static bool attr_set[NB_MAX_DEVICES] = {false};   // cudaFuncSetAttribute is per device
  if (!attr_set[ctx->device % NB_MAX_DEVICES]) {
    NB_CUDA(ctx, cudaFuncSetAttribute(fft_tile_kernel<INV, T, W, CB, NZ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set[ctx->device % NB_MAX_DEVICES] = true;
  }
  dim3 grid(1u << (p.n - T), (u32)((p.n_cols + CB - 1) / CB));
  fft_tile_kernel<INV, T, W, CB, NZ><<<grid, threads, smem, ctx->stream>>>(p);
  NB_LAUNCH_CHECK(ctx);
  return NB200_OK;
}

// returns true if a specialised kernel exists for (T, W)
template <bool INV>
static bool launch_fast(nb200_ctx* ctx, const FftPass& p, nb200_status* st) {
  // zero-extension specialisations exist for the strided (top) passes of forward transforms only
  const u32 nz = (!INV && p.W > 0 && p.lo + p.T - p.W == p.n && p.ztop < p.n) ? (p.n - p.ztop >= 2 ? 2u : 1u) : 0u;
#define NB_CASE(TT, WW, CBB) if (p.T == TT && p.W == WW) { *st = launch_tile<INV, TT, WW, CBB, 0>(ctx, p); return true; }
#define NB_CASEZ(TT, WW, CBB)                                                                          \
  if (p.T == TT && p.W == WW) {                                                                        \
    if (INV || nz == 0) *st = launch_tile<INV, TT, WW, CBB, 0>(ctx, p);                                \
    else if (nz == 1) *st = launch_tile<false, TT, WW, CBB, 1>(ctx, p);                                \
    else *st = launch_tile<false, TT, WW, CBB, 2>(ctx, p);                                             \
    return true;                                                                                       \
  }
  NB_CASE(9, 0, 4) NB_CASE(10, 0, 4) NB_CASE(11, 0, 4) NB_CASE(12, 0, 4) NB_CASE(13, 0, 2)
  NB_CASEZ(12, 4, 4) NB_CASEZ(12, 5, 4) NB_CASEZ(12, 6, 4) NB_CASEZ(12, 7, 4) NB_CASEZ(12, 8, 4) NB_CASEZ(13, 4, 2)
#undef NB_CASE
#undef NB_CASEZ
  return false;
}

template <bool INV>
static nb200_status launch_pass(nb200_ctx* ctx, const PassPlan& pl, const u32* src, size_t src_stride, size_t src_len,
                                u32* dst, size_t dst_stride, size_t n_cols, u32 n, bool scale, u32 ztop = 0xffffffffu, u32 tw_log = 0) {
  FftPass p;
  p.tn = tw_log ? tw_log : n;
  p.src = src; p.dst = dst; p.src_stride = src_stride; p.dst_stride = dst_stride; p.src_len = src_len;
  p.tw = INV ? ctx->tw.d_itw : ctx->tw.d_tw;
  p.tw_len = 1u << ctx->tw.half_log;
  const u32 *cf = nullptr, *ci = nullptr;
  NB_TRY(fft_circle_tables(ctx, p.tn, &cf, &ci));
  p.ctw2 = INV ? ci : cf;
  p.tw2 = INV ? ctx->tw.d_itw2 : ctx->tw.d_tw2;
  p.n_cols = (u32)n_cols; p.n = n; p.lo = pl.lo; p.T = pl.T; p.W = pl.W;
  p.cb = pl.T >= 13 ? 2 : 4;
  if (p.cb > n_cols) p.cb = (u32)n_cols;
  p.scale = 0; p.apply_scale = 0; p.ztop = ztop < n ? ztop : n;
  if (scale) { p.apply_scale = 1; p.scale = m31_inv((u32)(1u << n) % P31); }
  // 128-bit staging needs 16-byte aligned columns
  bool aligned = ((((uintptr_t)src) | ((uintptr_t)dst)) & 15u) == 0 && (src_stride % 4 == 0) && (dst_stride % 4 == 0) && (src_len % 4 == 0);
  nb200_status st = NB200_OK;
  if (aligned && launch_fast<INV>(ctx, p, &st)) return st;
  u32 threads = 1u << (pl.T - 4);
  size_t smem = (size_t)p.cb << (pl.T + 2);
  dim3 grid(1u << (n - pl.T), (u32)((n_cols + p.cb - 1) / p.cb));
  static bool attr_set[NB_MAX_DEVICES] = {false};   // one flag per (template instance, device)
  if (!attr_set[ctx->device % NB_MAX_DEVICES]) {
    NB_CUDA(ctx, cudaFuncSetAttribute(fft_pass_kernel<INV>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    attr_set[ctx->device % NB_MAX_DEVICES] = true;
  }
  fft_pass_kernel<INV><<<grid, threads, smem, ctx->stream>>>(p);
  NB_LAUNCH_CHECK(ctx);
  return NB200_OK;
}

template <bool INV>
static nb200_status launch_small(nb200_ctx* ctx, const u32* src, size_t src_stride, size_t src_len, u32* dst, size_t dst_stride,
                                 size_t n_cols, u32 n, bool scale) {
  FftSmall p;
  p.src = src; p.dst = dst; p.src_stride = src_stride; p.dst_stride = dst_stride; p.src_len = src_len;
  p.tw = INV ? ctx->tw.d_itw : ctx->tw.d_tw;
  p.tw_len = 1u << ctx->tw.half_log;
  p.n_cols = (u32)n_cols; p.n = n;
  p.y0 = 0;
  if (n >= 1 && n <= 2) {
    u32 y = HCoset::half_odds(n - 1).at(0).y;
    p.y0 = INV ? m31_inv(y) : y;
  }
  p.scale = 0; p.apply_scale = 0;
  if (scale) { p.apply_scale = 1; p.scale = m31_inv((u32)(1u << n) % P31); }
  u32 half = n ? (1u << (n - 1)) : 1;
  u32 threads = half < 32 ? 32 : (half > 256 ? 256 : half);
  size_t smem = (size_t)4 << n;
  fft_small_kernel<INV><<<(u32)n_cols, threads, smem, ctx->stream>>>(p);
  NB_LAUNCH_CHECK(ctx);
  return NB200_OK;
}

static const u32 SMALL_MAX_LOG = 8;

nb200_status fft_interpolate(nb200_ctx* ctx, const u32* src, u32* data, size_t n_cols, u32 n, u32 tw_log) {
  if (n_cols == 0) return NB200_OK;
  NB_ARG(ctx, n <= 30, "interpolate: log size too large");
  if (n == 0) {  // constant polynomial: coeff == value
    if (src != data) NB_CUDA(ctx, cudaMemcpyAsync(data, src, n_cols * 4, cudaMemcpyDeviceToDevice, ctx->stream));
    return NB200_OK;
  }
  const u32 tn = tw_log ? tw_log : n;
  NB_ARG(ctx, tn == n || (tn == n + 1 && n > SMALL_MAX_LOG), "interpolate: half-domain transforms need tw_log == n + 1 and n > 8");
  NB_ARG(ctx, ctx->tw.d_tw && ctx->tw.half_log + 1 >= tn, "interpolate: twiddles not prepared for this size");
  size_t len = (size_t)1 << n;
  if (n <= SMALL_MAX_LOG) return launch_small<true>(ctx, src, len, len, data, len, n_cols, n, true);
  std::vector<PassPlan> plan;
  plan_passes(n, plan);
  for (size_t k = 0; k < plan.size(); ++k)
    NB_TRY(launch_pass<true>(ctx, plan[k], k == 0 ? src : data, len, len, data, len, n_cols, n, k + 1 == plan.size(), 0xffffffffu, tn));
  return NB200_OK;
}

nb200_status fft_evaluate(nb200_ctx* ctx, const u32* src, u32 src_log, u32* dst, u32 n, size_t n_cols, u32 tw_log) {
  if (n_cols == 0) return NB200_OK;
  NB_ARG(ctx, src_log <= n && n <= 30, "evaluate: bad sizes");
  size_t slen = (size_t)1 << src_log, len = (size_t)1 << n;
  if (n == 0) {
    if (src != dst) NB_CUDA(ctx, cudaMemcpyAsync(dst, src, n_cols * 4, cudaMemcpyDeviceToDevice, ctx->stream));
    return NB200_OK;
  }
  const u32 tn = tw_log ? tw_log : n;
  NB_ARG(ctx, tn == n || (tn == n + 1 && n > SMALL_MAX_LOG), "evaluate: half-domain transforms need tw_log == n + 1 and n > 8");
  NB_ARG(ctx, ctx->tw.d_tw && ctx->tw.half_log + 1 >= tn, "evaluate: twiddles not prepared for this size");
  NB_ARG(ctx, src != dst || src_log == n, "evaluate: in-place requires equal sizes");
  if (n <= SMALL_MAX_LOG) return launch_small<false>(ctx, src, slen, slen, dst, len, n_cols, n, false);
  std::vector<PassPlan> plan;
  plan_passes(n, plan);
  for (size_t k = plan.size(); k-- > 0;) {
    bool first = (k + 1 == plan.size());
    if (first) NB_TRY(launch_pass<false>(ctx, plan[k], src, slen, slen, dst, len, n_cols, n, false, src_log, tn));
    else NB_TRY(launch_pass<false>(ctx, plan[k], dst, len, len, dst, len, n_cols, n, false, 0xffffffffu, tn));
  }
  return NB200_OK;
}

}  // namespace nb
