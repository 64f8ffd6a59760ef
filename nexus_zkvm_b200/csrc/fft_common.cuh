// Shared device helpers of the Circle FFT kernels (fft.cu: per-pass tile kernels; fft_fused.cu: the commit pipeline
// with the fused iFFT-tail / LDE-head kernel).  See fft.cu for the algorithm and the reference call sites.
#pragma once
#include "common.cuh"

namespace nb {

#ifndef NB_MAX_SHARD_RANKS
#define NB_MAX_SHARD_RANKS 16
#endif
struct FftPass {
  const u32* src;     // source columns (column c at src + c*src_stride); zero-extended beyond src_len
  u32* dst;           // destination columns
  size_t src_stride, dst_stride;
  size_t src_len;     // valid words per source column
  const u32* tw;      // twiddle (or inverse twiddle) bank
  const u32* tw2;     // the same bank doubled (2t), for m31_mul_dbl
  const u32* ctw2;    // DOUBLED circle (layer 0) twiddles of this transform size, 2^(n-1) words
  u32 tw_len;         // bank length (2^k)
  u32 n_cols;
  u32 n;              // log size of the transform
  u32 lo;             // first layer of this pass
  u32 T, W;           // tile log, width log (L = T - W layers)
  u32 cb;             // columns per CTA
  u32 scale;          // multiply outputs by this (interpolate last pass) if apply_scale
  u32 apply_scale;
  u32 tn;             // log size of the canonic domain whose twiddle arrays are used (= n, or n + 1 for the half-domain transforms)
  u32 ztop;           // forward transforms of zero-extended input: layers >= ztop are copies (= log2 of the source length)
  // row-sharded destination (one proof over N GPUs): rows [q << shard_log, (q + 1) << shard_log) of every column belong to rank q, whose row-slice
  // buffer (column stride 2^shard_log) is mapped at shard_dst[q] — peer memory over NVLink for q != this rank.  0 = off (dst / dst_stride are used).
  u32 shard_log = 0;
  size_t shard_col0 = 0;  // index of this batch's column 0 inside the row-slice buffers
  u32* shard_dst[NB_MAX_SHARD_RANKS] = {nullptr};
};

__device__ __forceinline__ void butterfly(u32& v0, u32& v1, u32 t) {
  u32 tmp = m31_mul(v1, t);
  v1 = m31_sub(v0, tmp);
  v0 = m31_add(v0, tmp);
}
__device__ __forceinline__ void ibutterfly(u32& v0, u32& v1, u32 it) {
  u32 tmp = v0;
  v0 = m31_add(tmp, v1);
  v1 = m31_mul(m31_sub(tmp, v1), it);
}

// twiddle of layer i (>= 1) at index h for a transform of log size n
__device__ __forceinline__ u32 line_tw(const u32* __restrict__ tw, u32 tw_len, u32 n, u32 i, u32 h) {
  return __ldg(tw + (tw_len - (1u << (n - i)) + h));
}
// circle twiddle (layer 0) at index h: from the first line layer, [x, y] -> [y, -y, -x, x]
__device__ __forceinline__ u32 circle_tw(const u32* __restrict__ tw, u32 tw_len, u32 n, u32 h) {
  const u32* l1 = tw + (tw_len - (1u << (n - 1)));
  u32 q = h >> 2, r = h & 3u;
  u32 x = __ldg(l1 + 2 * q), y = __ldg(l1 + 2 * q + 1);
  u32 v = (r < 2) ? y : x;
  return (r == 1 || r == 2) ? (P31 - v) : v;
}
static __global__ void circle_table_kernel(const u32* __restrict__ tw, u32 tw_len, u32 n, u32* __restrict__ out) {
  u32 h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h < (1u << (n - 1))) out[h] = circle_tw(tw, tw_len, n, h) << 1;  // doubled, see m31_mul_dbl
}

// =====================================================================================================
// fast path: compile-time tile shape
// =====================================================================================================
// swizzle keeps aligned groups of 4 words intact (128-bit accesses) and is conflict-free for: 128-bit staging,
// the 128-bit round at bit 0, and the 32-bit rounds at every bit position used by the schedules below.
__device__ __forceinline__ u32 swz2(u32 s) { return s ^ (((s >> 5) & 3u) << 2) ^ (((s >> 8) & 1u) << 4); }

// a * t mod P with the twiddle pre-doubled (t2 = 2t < 2^32): the 64-bit product a * t2 has (a*t) >> 31 in its high
// word and 2 * ((a*t) mod 2^31) in its low word, so the Mersenne fold is one shifted add (LEA.HI) and one min — the
// mask and the funnel shift of the plain form disappear, which matters because the ALU pipe is the binding one.
__device__ __forceinline__ u32 m31_mul_dbl(u32 a, u32 t2) {
  u64 p = (u64)a * t2;
  u32 s = ((u32)p >> 1) + (u32)(p >> 32);
  return umin32(s, s - P31);
}
__device__ __forceinline__ void butterfly_dbl(u32& v0, u32& v1, u32 t2) {
  u32 tmp = m31_mul_dbl(v1, t2);
  v1 = m31_sub(v0, tmp);
  v0 = m31_add(v0, tmp);
}
__device__ __forceinline__ void ibutterfly_dbl(u32& v0, u32& v1, u32 it2) {
  u32 tmp = v0;
  v0 = m31_add(tmp, v1);
  v1 = m31_mul_dbl(m31_sub(tmp, v1), it2);
}

template <bool INV>
__device__ __forceinline__ void radix16(u32 (&v)[16], const u32 (&tw)[15], const int jlo, const u32 triv = 0u) {
  // tw holds DOUBLED twiddles.  triv bit j (forward only): layer j of this round sits at or above the zero-extension
  // boundary, its odd inputs are known zeros, so the butterfly degenerates to a copy (no arithmetic).
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    const int j = INV ? jj : 3 - jj;
    if (j >= jlo) {
      if (!INV && ((triv >> j) & 1u)) {
#pragma unroll
        for (int m = 0; m < 8; ++m) {
          const int k0 = ((m >> j) << (j + 1)) | (m & ((1 << j) - 1));
          v[k0 | (1 << j)] = v[k0];
        }
      } else {
#pragma unroll
        for (int m = 0; m < 8; ++m) {
          const int k0 = ((m >> j) << (j + 1)) | (m & ((1 << j) - 1));
          const int k1 = k0 | (1 << j);
          const int off = (j == 0 ? 0 : j == 1 ? 8 : j == 2 ? 12 : 14) + (m >> j);
          if (INV) ibutterfly_dbl(v[k0], v[k1], tw[off]);
          else butterfly_dbl(v[k0], v[k1], tw[off]);
        }
      }
    }
  }
}


// a*ta + b*tb mod P with both constants pre-doubled: the two 64-bit products (each < 2^63) are summed BEFORE the Mersenne fold, so a
// radix-4 step needs one fold for t*(v1 +- s*v3) = t*v1 +- (t*s)*v3 instead of two butterflies' worth (fft_fused.cu, radix16p).
__device__ __forceinline__ u32 m31_mul2_dbl(u32 a, u32 ta2, u32 b, u32 tb2) {
  const u64 p = (u64)a * ta2 + (u64)b * tb2;   // = 2 X, X = a*ta + b*tb < 2 P^2
  u32 hi = (u32)(p >> 32);                      // X >> 31 < 2 P
  hi = umin32(hi, hi - P31);
  const u32 s = ((u32)p >> 1) + hi;             // (X mod 2^31) + (X >> 31 mod P) <= 2 P
  return umin32(s, s - P31);
}

// One radix-16 round (4 layers) as two radix-4 steps with PRODUCT twiddles: for the layer pair (j+1, j) with twiddles s (layer j+1), t_a / t_b
// (layer j, even / odd index) the table holds pt_a = t_a*s and pt_b = P - t_b*s (doubled).  Forward:  t_a*(v1 + s*v3) = t_a*v1 + pt_a*v3 and
// t_b*(v1 - s*v3) = t_b*v1 + pt_b*v3; inverse:  ia*(v0-v1) + ib*(v2-v3)  and  is*(ia*(v0-v1) - ib*(v2-v3)) = pia*(v0-v1) + pib*(v2-v3).
// 25 instructions (14 on the ALU pipe) per four butterflies instead of 28 (16): field arithmetic is exact, so the results are identical.
// tw: as radix16 (15 doubled twiddles); pt[0..7]: products of layer 0 with layer 1, pt[8..9]: of layer 2 with layer 3.
template <bool INV>
__device__ __forceinline__ void radix4p(u32& v0, u32& v1, u32& v2, u32& v3, const u32 ta, const u32 tb, const u32 s, const u32 pa, const u32 pb) {
  if (!INV) {
    const u32 tmp = m31_mul_dbl(v2, s);
    const u32 a0 = m31_add(v0, tmp), a2 = m31_sub(v0, tmp);
    const u32 b1 = m31_mul2_dbl(v1, ta, v3, pa), b3 = m31_mul2_dbl(v1, tb, v3, pb);
    v0 = m31_add(a0, b1); v1 = m31_sub(a0, b1); v2 = m31_add(a2, b3); v3 = m31_sub(a2, b3);
  } else {
    const u32 d01 = m31_sub(v0, v1), d23 = m31_sub(v2, v3), b0 = m31_add(v0, v1), b2 = m31_add(v2, v3);
    v0 = m31_add(b0, b2);
    v2 = m31_mul_dbl(m31_sub(b0, b2), s);
    v1 = m31_mul2_dbl(d01, ta, d23, tb);
    v3 = m31_mul2_dbl(d01, pa, d23, pb);
  }
}
template <bool INV>
__device__ __forceinline__ void radix16p(u32 (&v)[16], const u32 (&tw)[15], const u32 (&pt)[10]) {
  if (INV) {
#pragma unroll
    for (int g = 0; g < 4; ++g) radix4p<true>(v[4 * g], v[4 * g + 1], v[4 * g + 2], v[4 * g + 3], tw[2 * g], tw[2 * g + 1], tw[8 + g], pt[2 * g], pt[2 * g + 1]);
#pragma unroll
    for (int r = 0; r < 4; ++r) radix4p<true>(v[r], v[r + 4], v[r + 8], v[r + 12], tw[12], tw[13], tw[14], pt[8], pt[9]);
  } else {
#pragma unroll
    for (int r = 0; r < 4; ++r) radix4p<false>(v[r], v[r + 4], v[r + 8], v[r + 12], tw[12], tw[13], tw[14], pt[8], pt[9]);
#pragma unroll
    for (int g = 0; g < 4; ++g) radix4p<false>(v[4 * g], v[4 * g + 1], v[4 * g + 2], v[4 * g + 3], tw[2 * g], tw[2 * g + 1], tw[8 + g], pt[2 * g], pt[2 * g + 1]);
  }
}

// ---- asynchronous global -> shared copies (LDGSTS): no registers, no issue slots between request and use ----
__device__ __forceinline__ void cp_async16(u32 smem_addr, const void* g, bool valid) {
  const int sz = valid ? 16 : 0;   // src-size 0: nothing is read, the 16 bytes are zero-filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(smem_addr), "l"(g), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

// circle (layer 0) twiddle tables of a transform size, cached per ctx (fft.cu)
nb200_status fft_circle_tables(nb200_ctx* ctx, u32 n, const u32** fwd, const u32** inv);

}  // namespace nb
