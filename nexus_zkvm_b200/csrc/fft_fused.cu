// The commit transforms as ONE pipeline: evaluations -> coefficients (Circle iFFT) -> LDE (Circle FFT on the blown-up
// domain), i.e. TreeBuilder::extend_evals + the evaluate_polynomials inside TreeBuilder::commit at
// nexus-zkvm prover/src/machine.rs:208-263, for a batch of columns of 2^n rows (16 <= n <= 22).
//
//   A  fft_tile_async_kernel<INV>   layers 0..LA-1 of the iFFT, contiguous 2^LA-word tiles          read 4 B   write 4 B
//   B  fft_mid_kernel               the iFFT's strided tail (layers LA..n-1, 2^-n scaling) -> the coefficients are written
//                                   ONCE, stay in shared memory, and the same CTA runs the strided HEAD of every forward
//                                   transform that consumes them: both halves of the LDE (its top layer pairs a coefficient
//                                   with a zero-extension word, i.e. it is a copy), and on request the two halves of the
//                                   half-coset extension D2 the quotient step needs (prove.cu component_quotients)
//                                                                                                   read 4 B   write 4 + 8 (+ 8) B
//   C  fft_tile_async_kernel<FWD>   layers LA-1..0 of each forward transform, contiguous tiles       read 8 B   write 8 B
//
// per trace element — 40 B against the 44 B of four independent passes, one launch and one global->shared staging less,
// and none of B's forward inputs is ever read from memory.
//
// Staging uses cp.async (LDGSTS.128) with one commit group per column: the first radix-16 round of column c starts as soon
// as ITS tile has landed while the tiles of the later columns are still in flight, instead of every column waiting for the
// whole synchronous stage-in.
// Butterfly network, twiddle addressing and the shared-memory swizzle are those of fft.cu, so results are bit-identical
// to the per-pass kernels: tests/test_gpu_bench_size_parity.py, tests/test_gpu_commit_parity.py.
#include "fft_common.cuh"
#include <type_traits>

namespace nb {

template <int I, int N, class F>
__device__ __forceinline__ void static_for(F&& f) {
  if constexpr (I < N) {
    f(std::integral_constant<int, I>{});
    static_for<I + 1, N>(f);
  }
}

template <int CB>
__device__ __forceinline__ void wait_column(const int c) {   // c is a literal after unrolling: groups c+1.. may still be in flight
  const int pending = CB - 1 - c;
  if (pending <= 0) cp_async_wait<0>();
  else if (pending == 1) cp_async_wait<1>();
  else if (pending == 2) cp_async_wait<2>();
  else cp_async_wait<3>();
}

// ---- tile geometry shared by stage-in / stage-out: thread `tid` moves the 4 x uint4 at s_it = (tid + it*NT)*4 ----
template <int T, int W>
struct TileGeo {
  static constexpr int NT = 1 << (T - 4);
  static_assert((NT * 4 >= 512) && (W <= T - 2), "affine staging geometry (see fft.cu)");
  u32 phys0; size_t g0, gstep;
  __device__ __forceinline__ TileGeo(u32 lo, size_t gbase) {
    const u32 s0 = threadIdx.x * 4;
    phys0 = swz2(s0);
    g0 = W ? (gbase | ((size_t)(s0 >> W) << lo) | (s0 & ((1u << W) - 1u))) : (gbase | s0);
    gstep = W ? ((size_t)((NT * 4) >> W) << lo) : (size_t)(NT * 4);
  }
};

template <int T, int W, int CB>
__device__ __forceinline__ void stage_in_async(const TileGeo<T, W>& geo, const u32* __restrict__ src, size_t src_stride, size_t src_len,
                                               u32 col0, u32 ncb, u32* sm) {
  constexpr int NT = 1 << (T - 4);
  const u32 sm_base = (u32)__cvta_generic_to_shared(sm);
#pragma unroll
  for (int c = 0; c < CB; ++c) {
    const u32* __restrict__ scol = src + (size_t)(col0 + (c < (int)ncb ? c : 0)) * src_stride;
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const size_t g = geo.g0 + it * geo.gstep;
      const bool ok = c < (int)ncb && g < src_len;
      cp_async16(sm_base + (((u32)c << T) + geo.phys0 + it * NT * 4) * 4u, ok ? (const void*)(scol + g) : (const void*)scol, ok);
    }
    cp_async_commit();
  }
}

template <int T, int W, int CB>
__device__ __forceinline__ void stage_out(const TileGeo<T, W>& geo, const u32* sm, u32* __restrict__ dst, size_t dst_stride, u32 col0, u32 ncb, size_t gsub = 0) {
  constexpr int NT = 1 << (T - 4);
#pragma unroll
  for (int c = 0; c < CB; ++c) {
    if (c < (int)ncb) {
      u32* __restrict__ dcol = dst + (size_t)(col0 + c) * dst_stride - gsub;
#pragma unroll
      for (int it = 0; it < 4; ++it)
        *reinterpret_cast<uint4*>(dcol + geo.g0 + it * geo.gstep) = *reinterpret_cast<const uint4*>(sm + (c << T) + geo.phys0 + it * NT * 4);
    }
  }
}

// One radix-16 round (<= 4 butterfly layers) over the CB column tiles of a CTA: column c is read at sm_src + c*2^T and written at
// sm_dst + c*2^T (equal pointers = in place).  RI = position of the round inside the pass (0 = lowest layers), as in fft.cu.
// SCALE: multiply the outputs by sc2/2 (the 2^-n of interpolate).  WAITC: this is the first round after an asynchronous stage-in.
// PROD: full 4-layer rounds run as two radix-4 steps with product twiddles (fft_common.cuh radix16p; ptw2 = product bank).
template <bool INV, int T, int W, int CB, int RI, bool SCALE, bool WAITC, int NZ, bool PROD = false>
__device__ __forceinline__ void tile_round(const u32* __restrict__ tw2, const u32* __restrict__ ctw2, const u32 tw_len, const u32 tn, const u32 lo,
                                           const u32 tile_hi, const u32* sm_src, u32* sm_dst, const u32 ncb, const u32 sc2,
                                           const u32* __restrict__ ptw2 = nullptr) {
  static_assert(!PROD || W > 0, "product twiddles of the circle layer (W == 0) have no table");
  constexpr int L = T - W, NFULL = L / 4, REM = L % 4;
  constexpr int b = RI < NFULL ? W + 4 * RI : T - 4;
  constexpr int jlo = RI < NFULL ? 0 : 4 - REM;
  const u32 tid = threadIdx.x;
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
      const u32* __restrict__ src = (W == 0 && b + j == 0) ? (ctw2 + hbase) : (tw2 + (tw_len - (1u << (tn - i))) + hbase);
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
  constexpr bool USEP = PROD && jlo == 0 && NZ == 0;
  u32 pt[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  if (USEP) {
    {
      const u32 hbase = (tile_hi << (L - (b - W) - 1)) | (tau_hi << 3);
      const u32* __restrict__ src = ptw2 + (tw_len - (1u << (tn - (lo + b - W)))) + hbase;
      uint4 a = __ldg(reinterpret_cast<const uint4*>(src)), c4 = __ldg(reinterpret_cast<const uint4*>(src) + 1);
      pt[0] = a.x; pt[1] = a.y; pt[2] = a.z; pt[3] = a.w; pt[4] = c4.x; pt[5] = c4.y; pt[6] = c4.z; pt[7] = c4.w;
    }
    {
      const u32 hbase = (tile_hi << (L - (b + 2 - W) - 1)) | (tau_hi << 1);
      const uint2 a = __ldg(reinterpret_cast<const uint2*>(ptw2 + (tw_len - (1u << (tn - (lo + b + 2 - W)))) + hbase));
      pt[8] = a.x; pt[9] = a.y;
    }
  }
  const u32 sbase = (tau_hi << (b + 4)) | tau_lo;
  if (b == 0) {
    // the 16 words of a thread are contiguous: 4 x 128-bit shared accesses
    const u32 a0 = swz2(sbase), a1 = swz2(sbase | 4u), a2 = swz2(sbase | 8u), a3 = swz2(sbase | 12u);
#pragma unroll
    for (int c = 0; c < CB; ++c) {
      if (WAITC) { wait_column<CB>(c); __syncthreads(); }
      if (c < (int)ncb) {
        const u32* sc = sm_src + (c << T);
        u32* dc = sm_dst + (c << T);
        u32 v[16];
        uint4 q0 = *reinterpret_cast<const uint4*>(sc + a0), q1 = *reinterpret_cast<const uint4*>(sc + a1);
        uint4 q2 = *reinterpret_cast<const uint4*>(sc + a2), q3 = *reinterpret_cast<const uint4*>(sc + a3);
        v[0] = q0.x; v[1] = q0.y; v[2] = q0.z; v[3] = q0.w; v[4] = q1.x; v[5] = q1.y; v[6] = q1.z; v[7] = q1.w;
        v[8] = q2.x; v[9] = q2.y; v[10] = q2.z; v[11] = q2.w; v[12] = q3.x; v[13] = q3.y; v[14] = q3.z; v[15] = q3.w;
        if (USEP) radix16p<INV>(v, tw, pt); else radix16<INV>(v, tw, jlo, triv);
        if (SCALE) {
#pragma unroll
          for (int k = 0; k < 16; ++k) v[k] = m31_mul_dbl(v[k], sc2);
        }
        *reinterpret_cast<uint4*>(dc + a0) = make_uint4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<uint4*>(dc + a1) = make_uint4(v[4], v[5], v[6], v[7]);
        *reinterpret_cast<uint4*>(dc + a2) = make_uint4(v[8], v[9], v[10], v[11]);
        *reinterpret_cast<uint4*>(dc + a3) = make_uint4(v[12], v[13], v[14], v[15]);
      }
    }
  } else {
    u32 addr[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      addr[k] = swz2(sbase | ((u32)k << b));
      if (PROD) asm volatile("" : "+r"(addr[k]));   // keep the 16 addresses live across the columns (ptxas otherwise rematerialises them per column: +300 ALU-pipe instructions)
    }
#pragma unroll
    for (int c = 0; c < CB; ++c) {
      if (WAITC) { wait_column<CB>(c); __syncthreads(); }
      if (c < (int)ncb) {
        const u32* sc = sm_src + (c << T);
        u32* dc = sm_dst + (c << T);
        u32 v[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) v[k] = sc[addr[k]];
        if (USEP) radix16p<INV>(v, tw, pt); else radix16<INV>(v, tw, jlo, triv);
        if (SCALE) {
#pragma unroll
          for (int k = 0; k < 16; ++k) v[k] = m31_mul_dbl(v[k], sc2);
        }
#pragma unroll
        for (int k = 0; k < 16; ++k) dc[addr[k]] = v[k];
      }
    }
  }
}

// ================================================================================================================
// A / C: one pass over a contiguous-or-strided tile with asynchronous staging (same work as fft.cu's fft_tile_kernel)
// ================================================================================================================
template <bool INV, int T, int W, int CB, int MINB>
__global__ void __launch_bounds__(1 << (T - 4), MINB) fft_tile_async_kernel(const FftPass p) {
  extern __shared__ __align__(16) u32 sm[];
  constexpr int L = T - W;
  constexpr int NROUNDS = L / 4 + ((L % 4) ? 1 : 0);
  const u32 lo = p.lo;
  const u32 tile = blockIdx.x;
  const u32 mid_bits = W ? lo - W : 0;
  const u32 tile_mid = tile & ((1u << mid_bits) - 1u);
  const u32 tile_hi = tile >> mid_bits;
  const size_t gbase = ((size_t)tile_hi << (lo + L)) | ((size_t)tile_mid << W);
  const u32 col0 = blockIdx.y * CB;
  const u32 ncb = min((u32)CB, p.n_cols - col0);
  const TileGeo<T, W> geo(lo, gbase);
  stage_in_async<T, W, CB>(geo, p.src, p.src_stride, p.src_len, col0, ncb, sm);
  static_for<0, NROUNDS>([&](auto rr) {   // (the 2^-n scaling of interpolate is applied by fft_mid_kernel)
    constexpr int RR = decltype(rr)::value;
    constexpr int RI = INV ? RR : NROUNDS - 1 - RR;
    tile_round<INV, T, W, CB, RI, false, RR == 0, 0>(p.tw2, p.ctw2, p.tw_len, p.tn, lo, tile_hi, sm, sm, ncb, 0u);
    __syncthreads();
  });
  if (W == 0 && p.shard_log) {
    // the tile's rows all belong to one rank: the finished tile goes straight into that rank's row-slice buffer (a peer store over NVLink unless it
    // is ours) — the re-shard of the commitment happens here, tile by tile, while the other CTAs are still computing
    const u32 q = (u32)(gbase >> p.shard_log);
    stage_out<T, W, CB>(geo, sm, p.shard_dst[q] + (p.shard_col0 << p.shard_log), (size_t)1 << p.shard_log, col0, ncb, (size_t)q << p.shard_log);
  } else {
    stage_out<T, W, CB>(geo, sm, p.dst, p.dst_stride, col0, ncb);
  }
}

// ================================================================================================================
// B: iFFT tail -> coefficients -> heads of the forward transforms, one CTA per (tile, CB columns)
// ================================================================================================================
struct FftMid {
  const u32* src; size_t src_stride;        // A's output: 2^n words per column
  u32* coeffs; size_t coeff_stride;         // coefficients out (may alias src: a CTA reads its tile completely before it writes)
  const u32* itw2; const u32* tw2; u32 tw_len;
  const u32* iptw2; const u32* ptw2;        // product banks (radix16p)
  u32 n_cols, n, lo;                        // this pass owns inverse layers [lo, n)
  u32 sc2;                                  // 2 * 2^-n (doubled for m31_mul_dbl)
  u32 nfwd;                                 // forward heads to run (<= 4)
  u32* fdst[4]; size_t fstride[4];          // destination (already offset to the 2^n-word block this head fills) and its column stride
  u32 ftn[4];                               // log size of the canonic domain whose twiddles the head uses
  u32 fhi[4];                               // index of that block among the 2^n-word blocks of the forward transform (the bits above n)
};

template <int T, int W, int CB, int MINB, bool PROD>
__global__ void __launch_bounds__(1 << (T - 4), MINB) fft_mid_kernel(const FftMid p) {
  extern __shared__ __align__(16) u32 sm[];
  constexpr int L = T - W;
  constexpr int NROUNDS = L / 4 + ((L % 4) ? 1 : 0);
  u32* S0 = sm;                  // coefficient tiles
  u32* S1 = sm + (CB << T);      // working tiles of the forward heads
  const u32 lo = p.lo;
  const u32 tile = blockIdx.x;
  const u32 mid_bits = lo - W;
  const u32 tile_mid = tile & ((1u << mid_bits) - 1u);
  const u32 tile_hi = tile >> mid_bits;          // 0: lo + L == n (checked by the host)
  const size_t gbase = ((size_t)tile_hi << (lo + L)) | ((size_t)tile_mid << W);
  const u32 col0 = blockIdx.y * CB;
  const u32 ncb = min((u32)CB, p.n_cols - col0);
  const TileGeo<T, W> geo(lo, gbase);
  stage_in_async<T, W, CB>(geo, p.src, p.src_stride, (size_t)1 << p.n, col0, ncb, S0);
  // ---- inverse layers lo..n-1, scaled: S0 = coefficients
  static_for<0, NROUNDS>([&](auto rr) {
    constexpr int RR = decltype(rr)::value;
    tile_round<true, T, W, CB, RR, RR == NROUNDS - 1, RR == 0, 0, PROD>(p.itw2, nullptr, p.tw_len, p.n, lo, tile_hi, S0, S0, ncb, p.sc2, p.iptw2);
    __syncthreads();
  });
  stage_out<T, W, CB>(geo, S0, p.coeffs, p.coeff_stride, col0, ncb);
  // ---- forward heads: layers n-1..lo of a transform whose layers >= n are copies (zero-extended input); S0 is only read
#pragma unroll 1
  for (u32 f = 0; f < p.nfwd; ++f) {
    const u32 fhi = (p.fhi[f] << (p.n - lo - L)) | tile_hi;
    const u32 ftn = p.ftn[f];
    static_for<0, NROUNDS>([&](auto rr) {
      constexpr int RR = decltype(rr)::value;
      constexpr int RI = NROUNDS - 1 - RR;
      tile_round<false, T, W, CB, RI, false, false, 0, PROD>(p.tw2, nullptr, p.tw_len, ftn, lo, fhi, RR == 0 ? S0 : S1, S1, ncb, 0u, p.ptw2);
      __syncthreads();
    });
    stage_out<T, W, CB>(geo, S1, p.fdst[f], p.fstride[f], col0, ncb);
    __syncthreads();   // S1 is rewritten by the next head
  }
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
template <class K>
static nb200_status set_smem(nb200_ctx* ctx, K kernel, size_t smem, bool* flags) {
  if (!flags[ctx->device % NB_MAX_DEVICES]) {
    NB_CUDA(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    flags[ctx->device % NB_MAX_DEVICES] = true;
  }
  return NB200_OK;
}

template <bool INV, int T, int CB, int MINB>
static nb200_status launch_contig(nb200_ctx* ctx, const u32* src, size_t src_stride, u32* dst, size_t dst_stride, size_t n_cols, u32 n, u32 tn,
                                  const RowScatter* sc = nullptr, int which = 0) {
  FftPass p;
  p.shard_log = 0; p.shard_col0 = 0;
  for (int q = 0; q < NB_MAX_SHARD_RANKS; ++q) p.shard_dst[q] = nullptr;
  if (sc) {
    NB_ARG(ctx, !INV && sc->world <= NB_MAX_SHARD_RANKS && sc->log_slice >= (u32)T && sc->log_slice <= n, "row scatter: slice smaller than a tile");
    p.shard_log = sc->log_slice; p.shard_col0 = sc->col0;
    for (int q = 0; q < sc->world; ++q) p.shard_dst[q] = which ? sc->hx_rows[q] : sc->lde_rows[q];
  }
  p.src = src; p.dst = dst; p.src_stride = src_stride; p.dst_stride = dst_stride; p.src_len = (size_t)1 << n;
  p.tw = INV ? ctx->tw.d_itw : ctx->tw.d_tw;
  p.tw2 = INV ? ctx->tw.d_itw2 : ctx->tw.d_tw2;
  p.tw_len = 1u << ctx->tw.half_log;
  const u32 *cf = nullptr, *ci = nullptr;
  NB_TRY(fft_circle_tables(ctx, tn, &cf, &ci));
  p.ctw2 = INV ? ci : cf;
  p.n_cols = (u32)n_cols; p.n = n; p.lo = 0; p.T = T; p.W = 0; p.cb = CB; p.scale = 0; p.apply_scale = 0; p.tn = tn; p.ztop = n;
  constexpr size_t smem = (size_t)CB << (T + 2);
  static bool flags[NB_MAX_DEVICES] = {false};
  NB_TRY(set_smem(ctx, fft_tile_async_kernel<INV, T, 0, CB, MINB>, smem, flags));
  dim3 grid(1u << (n - T), (u32)((n_cols + CB - 1) / CB));
  fft_tile_async_kernel<INV, T, 0, CB, MINB><<<grid, 1 << (T - 4), smem, ctx->stream>>>(p);
  NB_LAUNCH_CHECK(ctx);
  return NB200_OK;
}

template <int T, int W, int CB, int MINB, bool PROD = false>
static nb200_status launch_mid(nb200_ctx* ctx, const FftMid& p) {
  constexpr size_t smem = (size_t)2 * CB << (T + 2);
  static bool flags[NB_MAX_DEVICES] = {false};
  NB_TRY(set_smem(ctx, fft_mid_kernel<T, W, CB, MINB, PROD>, smem, flags));
  dim3 grid(1u << (p.n - T), (u32)((p.n_cols + CB - 1) / CB));
  fft_mid_kernel<T, W, CB, MINB, PROD><<<grid, 1 << (T - 4), smem, ctx->stream>>>(p);
  NB_LAUNCH_CHECK(ctx);
  return NB200_OK;
}

struct FusedPlan { u32 LA, Lm; };
static bool fused_plan(u32 n, FusedPlan* pl) {
  if (n < 16 || n > 22) return false;
  pl->LA = n <= 21 ? 12 : 13;
  pl->Lm = n - pl->LA;
  return true;
}

bool fft_fused_supported(u32 n, u32 log_blowup, const void* a, const void* b, const void* c) {
  FusedPlan pl;
  if (log_blowup < 1 || log_blowup > 2 || !fused_plan(n, &pl)) return false;
  return (((uintptr_t)a | (uintptr_t)b | (uintptr_t)c) & 15u) == 0;
}

// evals (n_cols x 2^n, read only) -> coeffs (n_cols x 2^n) and lde (n_cols x 2^(n+bl)); optionally half_ext (n_cols x 2^(n+bl)):
// the same polynomials on the first half of CanonicCoset(n+bl+1).circle_domain() (fft.cu's half-domain transform).
nb200_status fft_commit_transforms(nb200_ctx* ctx, const u32* evals, u32* coeffs, u32* lde, u32* half_ext, size_t n_cols, u32 n, u32 bl, const RowScatter* scatter) {
  if (n_cols == 0) return NB200_OK;
  FusedPlan pl;
  NB_ARG(ctx, fused_plan(n, &pl) && bl >= 1 && bl <= 2, "commit transforms: unsupported shape for the fused pipeline");
  const u32 m = n + bl;                       // LDE log size
  NB_ARG(ctx, ctx->tw.d_tw && ctx->tw.half_log + 1 >= (half_ext ? m + 1 : m), "commit transforms: twiddles not prepared for this size");
  NB_ARG(ctx, !half_ext || bl == 1, "commit transforms: the half-coset extension is produced for blow-up 2 only");
  const size_t len = (size_t)1 << n, mlen = (size_t)1 << m;
  // A
  if (pl.LA == 12) NB_TRY((launch_contig<true, 12, 4, 3>(ctx, evals, len, coeffs, len, n_cols, n, n)));
  else NB_TRY((launch_contig<true, 13, 2, 2>(ctx, evals, len, coeffs, len, n_cols, n, n)));
  // B
  FftMid p;
  p.src = coeffs; p.src_stride = len; p.coeffs = coeffs; p.coeff_stride = len;
  p.itw2 = ctx->tw.d_itw2; p.tw2 = ctx->tw.d_tw2; p.tw_len = 1u << ctx->tw.half_log;
  p.iptw2 = ctx->tw.d_iptw2; p.ptw2 = ctx->tw.d_ptw2;
  p.n_cols = (u32)n_cols; p.n = n; p.lo = pl.LA; p.sc2 = m31_inv((u32)(1u << n) % P31) << 1;
  p.nfwd = 0;
  for (u32 r = 0; r < (1u << bl); ++r) {
    p.fdst[p.nfwd] = lde + ((size_t)r << n); p.fstride[p.nfwd] = mlen; p.ftn[p.nfwd] = m; p.fhi[p.nfwd] = r; ++p.nfwd;
  }
  if (half_ext) {
    for (u32 r = 0; r < 2; ++r) {
      p.fdst[p.nfwd] = half_ext + ((size_t)r << n); p.fstride[p.nfwd] = mlen; p.ftn[p.nfwd] = m + 1; p.fhi[p.nfwd] = r; ++p.nfwd;
    }
  }
  switch (pl.Lm) {
    case 4: NB_TRY((launch_mid<12, 8, 2, 3>(ctx, p))); break;
    case 5: NB_TRY((launch_mid<12, 7, 2, 3>(ctx, p))); break;
    case 6: NB_TRY((launch_mid<12, 6, 2, 3>(ctx, p))); break;
    case 7: NB_TRY((launch_mid<12, 5, 2, 3>(ctx, p))); break;
    case 8: NB_TRY((launch_mid<12, 4, 2, 3, true>(ctx, p))); break;
    case 9: NB_TRY((launch_mid<13, 4, 1, 2>(ctx, p))); break;
    default: return set_err(ctx, NB200_ERR_STATE, "commit transforms: plan");
  }
  // C: the contiguous low layers of every forward transform (each 2^n-word block is independent below layer n: run them as
  // one launch over the 2^m-word columns)
  auto fwd_low = [&](u32* buf, u32 tn, int which) -> nb200_status {
    if (pl.LA == 12) return launch_contig<false, 12, 4, 3>(ctx, buf, mlen, buf, mlen, n_cols, m, tn, scatter, which);
    return launch_contig<false, 13, 2, 2>(ctx, buf, mlen, buf, mlen, n_cols, m, tn, scatter, which);
  };
  NB_TRY(fwd_low(lde, m, 0));
  if (half_ext) NB_TRY(fwd_low(half_ext, m + 1, 1));
  return NB200_OK;
}

// TreeBuilder::extend_evals + the LDE of TreeBuilder::commit for one batch: the fused pipeline when the shape allows, else per-transform passes
// `scatter` (one proof over N GPUs): the last pass of the LDE (and of the D2 evaluation) stores every finished tile into the row-slice buffer of the
// rank that owns its rows instead of `lde` / `half_ext` (which then hold intermediates only); *scattered tells the caller whether that happened — the
// per-transform fallback cannot, and leaves complete columns in `lde` / `half_ext` for a copy-based re-shard.
nb200_status commit_transforms(nb200_ctx* ctx, const u32* evals, u32* coeffs, u32* lde, u32* half_ext, size_t n_cols, u32 n, u32 bl, const RowScatter* scatter, bool* scattered) {
  if (scattered) *scattered = false;
  if (n_cols == 0) return NB200_OK;
  if (fft_fused_supported(n, bl, evals, coeffs, lde) && (!half_ext || (bl == 1 && ((uintptr_t)half_ext & 15u) == 0))) {
    FusedPlan pl;
    const bool can = scatter && scattered && fused_plan(n, &pl) && scatter->world <= NB_MAX_SHARD_RANKS && scatter->log_slice >= pl.LA;
    if (scattered) *scattered = can;
    return fft_commit_transforms(ctx, evals, coeffs, lde, half_ext, n_cols, n, bl, can ? scatter : nullptr);
  }
  NB_TRY(fft_interpolate(ctx, evals, coeffs, n_cols, n));
  NB_TRY(fft_evaluate(ctx, coeffs, n, lde, n + bl, n_cols));
  if (half_ext) NB_TRY(fft_evaluate(ctx, coeffs, n, half_ext, n + bl, n_cols, n + bl + 1));
  return NB200_OK;
}

// can the last LDE pass store straight into row-slice buffers of 2^log_slice rows?  (the same answer on every rank: it depends on sizes only)
bool commit_transforms_can_scatter(u32 n, u32 bl, u32 log_slice, int world) {
  FusedPlan pl;
  return bl == 1 && fused_plan(n, &pl) && world <= NB_MAX_SHARD_RANKS && log_slice >= pl.LA;
}

}  // namespace nb
