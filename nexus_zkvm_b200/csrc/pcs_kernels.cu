// Kernels of the polynomial commitment scheme's opening phase:
//   - DEEP / FRI quotients   (QuotientOps::accumulate_quotients,  stwo prover/backend/*/quotients.rs, core/pcs/quotients.rs)
//   - FRI folding            (FriOps::fold_circle_into_line / fold_line, stwo prover/backend/*/fri.rs)
//   - proof of work          (GrindOps::grind)
//   - secure-column helpers  (AccumulationOps::accumulate, domain point tables, gathers)
// all reached from stwo::prover::prove at nexus-zkvm prover/src/machine.rs:286-290.
// Every kernel is one thread per row/pair with coalesced 32-bit column accesses (columns are SoA: a QM31 column is 4
// coordinate columns, exactly the layout the Merkle kernels hash).  Field arithmetic is exact, so the re-association
// of sums used here (per-batch sum of line terms hoisted to the host) is bit-exact with the reference formula.
#include "pcs.h"
#include "blake2s.cuh"
#include "device_channel.cuh"
#include "circle_host.h"

namespace nb {

__constant__ cpoint c_gen_pow2_pcs[31];

static nb200_status ensure_gen_table(nb200_ctx* ctx) {
  static bool up[64] = {false};
  if (!up[ctx->device & 63]) {
    NB_CUDA(ctx, cudaMemcpyToSymbol(c_gen_pow2_pcs, gen_table().pow2, sizeof(cpoint) * 31));
    up[ctx->device & 63] = true;
  }
  return NB200_OK;
}

// x/y of CanonicCoset(log).circle_domain() in bit-reversed order.  Position i holds the point of index init + step jj of the half coset
// half_odds(log-1) (initial = subgroup_gen(log+1), step = subgroup_gen(log-1); jj = bit-reversed i modulo the half), conjugated in the
// second half.  With jj = lo + 2^k hi that point is P_lo[lo] + P_hi[hi]: two small tables (domain_tables_kernel) and one group addition
// per point instead of a 31-step scalar multiplication.  The group law is exact, so the words do not depend on how the sum is split.
__device__ __forceinline__ cpoint point_of_index(u32 idx) {
  cpoint r{1, 0};
#pragma unroll 1
  for (int b = 0; b < 31; ++b) if ((idx >> b) & 1u) r = cp_add(r, c_gen_pow2_pcs[b]);
  return r;
}
// lo[t] = (init + step t) G for t < 2^k; hi[t] = (step 2^k t) G for t < 2^(log_size - 1 - k)
__global__ void domain_tables_kernel(u32 log_size, u32 k, cpoint* __restrict__ lo, cpoint* __restrict__ hi) {
  const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
  const u32 init = 1u << (31 - (log_size + 1));
  const u32 step = (log_size - 1 == 0) ? 0u : (1u << (31 - (log_size - 1)));
  const u32 n_lo = 1u << k, n_hi = 1u << (log_size - 1 - k);
  if (t < n_lo) lo[t] = point_of_index((init + (u32)(((u64)step * t) & 0x7fffffffu)) & 0x7fffffffu);
  else if (t - n_lo < n_hi) hi[t - n_lo] = point_of_index((u32)(((u64)step * ((u64)(t - n_lo) << k)) & 0x7fffffffu));
}
__global__ void domain_points_kernel(u32 log_size, u32 k, const cpoint* __restrict__ lo, const cpoint* __restrict__ hi,
                                     u32* __restrict__ xs, u32* __restrict__ ys) {
  u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  u32 n = 1u << log_size;
  if (i >= n) return;
  u32 j = __brev(i) >> (32 - log_size);
  u32 half = n >> 1;
  u32 jj = j < half ? j : j - half;
  const cpoint r = cp_add(lo[jj & ((1u << k) - 1)], hi[jj >> k]);
  xs[i] = r.x;
  ys[i] = j < half ? r.y : m31_neg(r.y);
}
nb200_status domain_points(nb200_ctx* ctx, u32 log_size, u32* d_x, u32* d_y) {
  NB_TRY(ensure_gen_table(ctx));
  NB_ARG(ctx, log_size >= 1 && log_size <= 30, "domain_points: log size");
  const u32 k = (log_size - 1) / 2, n_tab = (1u << k) + (1u << (log_size - 1 - k));
  cpoint* d_tab = nullptr;
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d_tab, (size_t)n_tab * sizeof(cpoint)));
  u32 n = 1u << log_size, thr = 256;
  domain_tables_kernel<<<(n_tab + thr - 1) / thr, thr, 0, ctx->stream>>>(log_size, k, d_tab, d_tab + (1u << k));
  NB_LAUNCH_CHECK(ctx);
  domain_points_kernel<<<(n + thr - 1) / thr, thr, 0, ctx->stream>>>(log_size, k, d_tab, d_tab + (1u << k), d_x, d_y);
  NB_LAUNCH_CHECK(ctx);
  dfree(ctx, d_tab);   // ordered after the kernels on the stream
  return NB200_OK;
}

// ---- DEEP quotients ----
__global__ void __launch_bounds__(256) quotients_kernel(const QBatchDev* __restrict__ batches, u32 n_batches, const QEntryDev* __restrict__ entries,
                                                        const u32* __restrict__ dom_x, const u32* __restrict__ dom_y, u32 log_size,
                                                        u32* __restrict__ o0, u32* __restrict__ o1, u32* __restrict__ o2, u32* __restrict__ o3, u32 row0, u32 row_end) {
  const u32 row = row0 + blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= row_end) return;
  const u32 x = __ldg(dom_x + row), y = __ldg(dom_y + row);
  qm31 acc = qm31_zero();
  for (u32 b = 0; b < n_batches; ++b) {
    const QBatchDev* qb = batches + b;
    // numerator = sum_k c_k f_k(row) - (A y + B)
    // sums of 64-bit products: four products (< 2^62 each) plus a reduced carry-in fit in 64 bits, so reduce after every fourth
    // entry.  The four column loads of a group are issued before any arithmetic (the loop is otherwise latency bound: one dependent
    // pointer + data load per entry).
    u64 s0 = 0, s1 = 0, s2 = 0, s3 = 0;
    const u32 first = qb->first, count = qb->count;
    const QEntryDev* en = entries + first;
    u32 e = 0;
    for (; e + 4 <= count; e += 4) {
      const u32* c0p = en[e].col; const u32* c1p = en[e + 1].col; const u32* c2p = en[e + 2].col; const u32* c3p = en[e + 3].col;
      const u32 f0 = __ldg(c0p + row), f1 = __ldg(c1p + row), f2 = __ldg(c2p + row), f3 = __ldg(c3p + row);
      const uint4 k0 = __ldg(reinterpret_cast<const uint4*>(en[e].c)), k1 = __ldg(reinterpret_cast<const uint4*>(en[e + 1].c));
      const uint4 k2 = __ldg(reinterpret_cast<const uint4*>(en[e + 2].c)), k3 = __ldg(reinterpret_cast<const uint4*>(en[e + 3].c));
      s0 += (u64)f0 * k0.x + (u64)f1 * k1.x + (u64)f2 * k2.x + (u64)f3 * k3.x;
      s1 += (u64)f0 * k0.y + (u64)f1 * k1.y + (u64)f2 * k2.y + (u64)f3 * k3.y;
      s2 += (u64)f0 * k0.z + (u64)f1 * k1.z + (u64)f2 * k2.z + (u64)f3 * k3.z;
      s3 += (u64)f0 * k0.w + (u64)f1 * k1.w + (u64)f2 * k2.w + (u64)f3 * k3.w;
      s0 = m31_red64(s0); s1 = m31_red64(s1); s2 = m31_red64(s2); s3 = m31_red64(s3);
    }
    for (; e < count; ++e) {   // at most three left: still within 64 bits
      const uint4 c = __ldg(reinterpret_cast<const uint4*>(en[e].c));
      const u32 f = __ldg(en[e].col + row);
      s0 += (u64)f * c.x; s1 += (u64)f * c.y; s2 += (u64)f * c.z; s3 += (u64)f * c.w;
    }
    qm31 numer = qm31_make(m31_red64(s0), m31_red64(s1), m31_red64(s2), m31_red64(s3));
    qm31 A = qm31_make(qb->A[0], qb->A[1], qb->A[2], qb->A[3]);
    qm31 B = qm31_make(qb->B[0], qb->B[1], qb->B[2], qb->B[3]);
    numer = qm31_sub(numer, qm31_add(qm31_mul_m31(A, y), B));
    // denominator = (prx - x) * piy - (pry - y) * pix   (CM31)
    cm31 prx{qb->prx[0], qb->prx[1]}, pry{qb->pry[0], qb->pry[1]}, pix{qb->pix[0], qb->pix[1]}, piy{qb->piy[0], qb->piy[1]};
    cm31 dx{m31_sub(prx.a, x), prx.b}, dy{m31_sub(pry.a, y), pry.b};
    cm31 den = cm31_sub(cm31_mul(dx, piy), cm31_mul(dy, pix));
    qm31 cf = qm31_make(qb->coeff[0], qb->coeff[1], qb->coeff[2], qb->coeff[3]);
    acc = qm31_add(qm31_mul(acc, cf), qm31_mul_cm31(numer, cm31_inv(den)));
  }
  o0[row] = acc.c[0]; o1[row] = acc.c[1]; o2[row] = acc.c[2]; o3[row] = acc.c[3];
}

// cm31_inv of four values with one field inversion: Montgomery's trick on their norms a^2 + b^2 (the norm of a nonzero value is nonzero,
// -1 being no square mod P).  When a norm is zero the product is zero, and each value is inverted on its own as cm31_inv does (0 -> 0).
__device__ __forceinline__ void cm31_inv4(const cm31 (&d)[4], cm31 (&out)[4]) {
  u32 n[4], ni[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) n[r] = m31_add(m31_mul(d[r].a, d[r].a), m31_mul(d[r].b, d[r].b));
  const u32 p01 = m31_mul(n[0], n[1]), p012 = m31_mul(p01, n[2]), p = m31_mul(p012, n[3]);
  if (p != 0) {
    u32 t = m31_inv(p);                              // 1 / (n0 n1 n2 n3)
    ni[3] = m31_mul(t, p012); t = m31_mul(t, n[3]);  // t = 1 / (n0 n1 n2)
    ni[2] = m31_mul(t, p01);  t = m31_mul(t, n[2]);  // t = 1 / (n0 n1)
    ni[1] = m31_mul(t, n[0]); ni[0] = m31_mul(t, n[1]);
  } else {
#pragma unroll
    for (int r = 0; r < 4; ++r) ni[r] = m31_inv(n[r]);
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) out[r] = cm31{m31_mul(d[r].a, ni[r]), m31_neg(m31_mul(d[r].b, ni[r]))};
}

// s[r][j] += sum over the entries of coordinate j of en[e].c times word (row + r) of column en[e].col, for r < 4: the column reads of
// quotients_kernel_x4 and deep_combine_kernel.  Every column is read with 128-bit loads (512 contiguous bytes per warp and column instead
// of 128: the sweep jumps 2^log_size words from column to column, so longer bursts matter for DRAM efficiency) and the per-entry
// constants are fetched once for four rows.  Lazy reduction: four products (< 2^62 each) plus a reduced carry-in fit in 64 bits, so the
// sums are reduced after every group of four entries; on return each s[r][j] holds a reduced value plus at most three products.
__device__ __forceinline__ void sum_entries_x4(const QEntryDev* __restrict__ en, u32 count, u32 row, u64 (&s)[4][4]) {
  u32 e = 0;
  for (; e + 8 <= count; e += 8) {   // eight columns (128 bytes) in flight per thread: two groups of four, one reduction per group
    uint4 f[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) f[u] = __ldg(reinterpret_cast<const uint4*>(en[e + u].col + row));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      uint4 k[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) k[u] = __ldg(reinterpret_cast<const uint4*>(en[e + 4 * h + u].c));
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const u32 fr[4] = {f[4 * h + u].x, f[4 * h + u].y, f[4 * h + u].z, f[4 * h + u].w};
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          s[r][0] += (u64)fr[r] * k[u].x; s[r][1] += (u64)fr[r] * k[u].y; s[r][2] += (u64)fr[r] * k[u].z; s[r][3] += (u64)fr[r] * k[u].w;
        }
      }
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int j = 0; j < 4; ++j) s[r][j] = m31_red64(s[r][j]);
    }
  }
  for (; e + 4 <= count; e += 4) {   // four columns in flight per thread (the loop is latency bound otherwise), then one reduction
    uint4 f[4], k[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) f[u] = __ldg(reinterpret_cast<const uint4*>(en[e + u].col + row));
#pragma unroll
    for (int u = 0; u < 4; ++u) k[u] = __ldg(reinterpret_cast<const uint4*>(en[e + u].c));
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const u32 fr[4] = {f[u].x, f[u].y, f[u].z, f[u].w};
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        s[r][0] += (u64)fr[r] * k[u].x; s[r][1] += (u64)fr[r] * k[u].y; s[r][2] += (u64)fr[r] * k[u].z; s[r][3] += (u64)fr[r] * k[u].w;
      }
    }
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[r][j] = m31_red64(s[r][j]);
  }
  for (; e < count; ++e) {           // at most three left: still within 64 bits
    const uint4 f = __ldg(reinterpret_cast<const uint4*>(en[e].col + row));
    const uint4 k = __ldg(reinterpret_cast<const uint4*>(en[e].c));
    const u32 fr[4] = {f.x, f.y, f.z, f.w};
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      s[r][0] += (u64)fr[r] * k.x; s[r][1] += (u64)fr[r] * k.y; s[r][2] += (u64)fr[r] * k.z; s[r][3] += (u64)fr[r] * k.w;
    }
  }
}

// Four consecutive rows per thread (sum_entries_x4), their four denominators inverted together (cm31_inv4).  Same field values as
// quotients_kernel.
__global__ void __launch_bounds__(128) quotients_kernel_x4(const QBatchDev* __restrict__ batches, u32 n_batches, const QEntryDev* __restrict__ entries,
                                                           const u32* __restrict__ dom_x, const u32* __restrict__ dom_y, u32 log_size,
                                                           u32* __restrict__ o0, u32* __restrict__ o1, u32* __restrict__ o2, u32* __restrict__ o3, u32 row0, u32 row_end) {
  const u32 row = row0 + (blockIdx.x * blockDim.x + threadIdx.x) * 4u;
  if (row >= row_end) return;
  const uint4 xv = __ldg(reinterpret_cast<const uint4*>(dom_x + row)), yv = __ldg(reinterpret_cast<const uint4*>(dom_y + row));
  const u32 xs[4] = {xv.x, xv.y, xv.z, xv.w}, ys[4] = {yv.x, yv.y, yv.z, yv.w};
  qm31 acc[4] = {qm31_zero(), qm31_zero(), qm31_zero(), qm31_zero()};
  for (u32 b = 0; b < n_batches; ++b) {
    const QBatchDev* qb = batches + b;
    u64 s[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[r][j] = 0;
    sum_entries_x4(entries + qb->first, qb->count, row, s);
    const qm31 A = qm31_make(qb->A[0], qb->A[1], qb->A[2], qb->A[3]);
    const qm31 B = qm31_make(qb->B[0], qb->B[1], qb->B[2], qb->B[3]);
    const cm31 prx{qb->prx[0], qb->prx[1]}, pry{qb->pry[0], qb->pry[1]}, pix{qb->pix[0], qb->pix[1]}, piy{qb->piy[0], qb->piy[1]};
    const qm31 cf = qm31_make(qb->coeff[0], qb->coeff[1], qb->coeff[2], qb->coeff[3]);
    cm31 den[4], inv[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const cm31 dx{m31_sub(prx.a, xs[r]), prx.b}, dy{m31_sub(pry.a, ys[r]), pry.b};
      den[r] = cm31_sub(cm31_mul(dx, piy), cm31_mul(dy, pix));
    }
    cm31_inv4(den, inv);
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      qm31 numer = qm31_make(m31_red64(s[r][0]), m31_red64(s[r][1]), m31_red64(s[r][2]), m31_red64(s[r][3]));
      numer = qm31_sub(numer, qm31_add(qm31_mul_m31(A, ys[r]), B));
      acc[r] = qm31_add(qm31_mul(acc[r], cf), qm31_mul_cm31(numer, inv[r]));
    }
  }
  *reinterpret_cast<uint4*>(o0 + row) = make_uint4(acc[0].c[0], acc[1].c[0], acc[2].c[0], acc[3].c[0]);
  *reinterpret_cast<uint4*>(o1 + row) = make_uint4(acc[0].c[1], acc[1].c[1], acc[2].c[1], acc[3].c[1]);
  *reinterpret_cast<uint4*>(o2 + row) = make_uint4(acc[0].c[2], acc[1].c[2], acc[2].c[2], acc[3].c[2]);
  *reinterpret_cast<uint4*>(o3 + row) = make_uint4(acc[0].c[3], acc[1].c[3], acc[2].c[3], acc[3].c[3]);
}

nb200_status quotients_launch(nb200_ctx* ctx, const QBatchDev* h_batches, size_t n_batches, const QEntryDev* h_entries, size_t n_entries,
                              const u32* dom_x, const u32* dom_y, u32 log_size, u32* out /* 4 columns */, u32 row0, size_t n_rows) {
  QBatchDev* d_b = nullptr; QEntryDev* d_e = nullptr;
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d_b, n_batches * sizeof(QBatchDev)));
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d_e, n_entries * sizeof(QEntryDev)));
  NB_CUDA(ctx, cudaMemcpyAsync(d_b, h_batches, n_batches * sizeof(QBatchDev), cudaMemcpyHostToDevice, ctx->stream));
  NB_CUDA(ctx, cudaMemcpyAsync(d_e, h_entries, n_entries * sizeof(QEntryDev), cudaMemcpyHostToDevice, ctx->stream));
  size_t n = (size_t)1 << log_size;
  const size_t nr = n_rows ? n_rows : n;      // rows [row0, row0 + nr) of the domain (a rank's slice in a multi-GPU proof); pointers are indexed by the global row
  const u32 row_end = (u32)(row0 + nr);
  bool aligned = log_size >= 2 && (row0 % 4 == 0) && (nr % 4 == 0) && ((((uintptr_t)out) | ((uintptr_t)dom_x) | ((uintptr_t)dom_y)) & 15u) == 0;
  for (size_t e = 0; e < n_entries && aligned; ++e) aligned = (((uintptr_t)h_entries[e].col) & 15u) == 0;
  if (aligned) {
    u32 thr = 128; size_t nt = nr / 4;
    quotients_kernel_x4<<<(u32)((nt + thr - 1) / thr), thr, 0, ctx->stream>>>(d_b, (u32)n_batches, d_e, dom_x, dom_y, log_size,
                                                                             out, out + n, out + 2 * n, out + 3 * n, row0, row_end);
  } else {
    u32 thr = 256;
    quotients_kernel<<<(u32)((nr + thr - 1) / thr), thr, 0, ctx->stream>>>(d_b, (u32)n_batches, d_e, dom_x, dom_y, log_size,
                                                                          out, out + n, out + 2 * n, out + 3 * n, row0, row_end);
  }
  NB_LAUNCH_CHECK(ctx);
  // no sync: the host tables may go once the copies above have returned (a copy from pageable host memory is staged by then), and the
  // frees are ordered after the kernel on the stream
  dfree(ctx, d_b); dfree(ctx, d_e);
  return NB200_OK;
}

// ---- DEEP quotients from combined coefficients (deep_quotients in prove.cu) ----
// The numerator of sample batch b is sum_k (alpha_k c_b) f_k(x) - (A_b y + B_b) = c_b G_b(x) - (A_b y + B_b) with G_b = sum_k alpha_k f_k.
// G_b is formed on the columns' coefficients (half the words of their LDE) and extended once; the row kernel then reads G_b's four
// coordinate columns per batch instead of every column.  Field arithmetic is exact, so the quotient is the same word for word.

// g (4 coordinate columns of 2^log_n per batch, batch after batch) = per batch b, sum over its entries of alpha_k (entry.c) times the
// coefficient column entry.col.  One thread per four coefficients of one batch: grid (coefficient blocks, batches).
__global__ void __launch_bounds__(128, 8) deep_combine_kernel(const uint2* __restrict__ ranges /* (first entry, count) per batch */,
                                                           const QEntryDev* __restrict__ entries, u32 log_n, u32* __restrict__ g) {
  const u32 i = (blockIdx.x * blockDim.x + threadIdx.x) * 4u;
  const size_t n = (size_t)1 << log_n;
  if (i >= n) return;
  const uint2 rg = __ldg(ranges + blockIdx.y);
  u64 s[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int j = 0; j < 4; ++j) s[r][j] = 0;
  sum_entries_x4(entries + rg.x, rg.y, i, s);
  u32* gb = g + ((size_t)blockIdx.y * 4) * n;
#pragma unroll
  for (int j = 0; j < 4; ++j)
    *reinterpret_cast<uint4*>(gb + j * n + i) = make_uint4(m31_red64(s[0][j]), m31_red64(s[1][j]), m31_red64(s[2][j]), m31_red64(s[3][j]));
}
nb200_status deep_combine(nb200_ctx* ctx, const uint2* h_ranges, size_t n_batches, const QEntryDev* h_entries, size_t n_entries, u32 log_n, u32* g) {
  NB_ARG(ctx, log_n >= 2 && (((uintptr_t)g) & 15u) == 0, "deep_combine: 4-word aligned columns of at least 4 coefficients");
  for (size_t e = 0; e < n_entries; ++e) NB_ARG(ctx, (((uintptr_t)h_entries[e].col) & 15u) == 0, "deep_combine: 4-word aligned columns");
  uint2* d_r = nullptr; QEntryDev* d_e = nullptr;
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d_r, n_batches * sizeof(uint2)));
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d_e, n_entries * sizeof(QEntryDev)));
  NB_CUDA(ctx, cudaMemcpyAsync(d_r, h_ranges, n_batches * sizeof(uint2), cudaMemcpyHostToDevice, ctx->stream));
  NB_CUDA(ctx, cudaMemcpyAsync(d_e, h_entries, n_entries * sizeof(QEntryDev), cudaMemcpyHostToDevice, ctx->stream));
  const u32 thr = 128;
  const size_t nt = ((size_t)1 << log_n) / 4;
  deep_combine_kernel<<<dim3((u32)((nt + thr - 1) / thr), (u32)n_batches), thr, 0, ctx->stream>>>(d_r, d_e, log_n, g);
  NB_LAUNCH_CHECK(ctx);
  dfree(ctx, d_r); dfree(ctx, d_e);   // ordered after the kernel on the stream (see quotients_launch)
  return NB200_OK;
}

// out (4 columns of 2^log_size) = the DEEP quotient from g, the extended combinations (4 columns of 2^log_size per batch).  Four rows per
// thread; the denominators and the chaining by random_coeff ^ (columns in batch) are those of quotients_kernel_x4.
__global__ void __launch_bounds__(128) quotients_combined_kernel(const QLineDev* __restrict__ batches, u32 n_batches, const u32* __restrict__ g,
                                                                 const u32* __restrict__ dom_x, const u32* __restrict__ dom_y, u32 log_size,
                                                                 u32* __restrict__ o0, u32* __restrict__ o1, u32* __restrict__ o2, u32* __restrict__ o3) {
  const size_t n = (size_t)1 << log_size;
  const u32 row = (blockIdx.x * blockDim.x + threadIdx.x) * 4u;
  if (row >= n) return;
  const uint4 xv = __ldg(reinterpret_cast<const uint4*>(dom_x + row)), yv = __ldg(reinterpret_cast<const uint4*>(dom_y + row));
  const u32 xs[4] = {xv.x, xv.y, xv.z, xv.w}, ys[4] = {yv.x, yv.y, yv.z, yv.w};
  qm31 acc[4] = {qm31_zero(), qm31_zero(), qm31_zero(), qm31_zero()};
  for (u32 b = 0; b < n_batches; ++b) {
    const QLineDev* qb = batches + b;
    const u32* gb = g + ((size_t)b * 4) * n + row;
    uint4 v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = __ldg(reinterpret_cast<const uint4*>(gb + j * n));
    const qm31 A = qm31_make(qb->A[0], qb->A[1], qb->A[2], qb->A[3]);
    const qm31 B = qm31_make(qb->B[0], qb->B[1], qb->B[2], qb->B[3]);
    const qm31 c = qm31_make(qb->c[0], qb->c[1], qb->c[2], qb->c[3]);
    const cm31 prx{qb->prx[0], qb->prx[1]}, pry{qb->pry[0], qb->pry[1]}, pix{qb->pix[0], qb->pix[1]}, piy{qb->piy[0], qb->piy[1]};
    const qm31 cf = qm31_make(qb->coeff[0], qb->coeff[1], qb->coeff[2], qb->coeff[3]);
    const u32 gx[4] = {v[0].x, v[0].y, v[0].z, v[0].w}, gy[4] = {v[1].x, v[1].y, v[1].z, v[1].w};
    const u32 gz[4] = {v[2].x, v[2].y, v[2].z, v[2].w}, gw[4] = {v[3].x, v[3].y, v[3].z, v[3].w};
    cm31 den[4], inv[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const cm31 dx{m31_sub(prx.a, xs[r]), prx.b}, dy{m31_sub(pry.a, ys[r]), pry.b};
      den[r] = cm31_sub(cm31_mul(dx, piy), cm31_mul(dy, pix));
    }
    cm31_inv4(den, inv);
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      qm31 numer = qm31_mul(c, qm31_make(gx[r], gy[r], gz[r], gw[r]));
      numer = qm31_sub(numer, qm31_add(qm31_mul_m31(A, ys[r]), B));
      acc[r] = qm31_add(qm31_mul(acc[r], cf), qm31_mul_cm31(numer, inv[r]));
    }
  }
  *reinterpret_cast<uint4*>(o0 + row) = make_uint4(acc[0].c[0], acc[1].c[0], acc[2].c[0], acc[3].c[0]);
  *reinterpret_cast<uint4*>(o1 + row) = make_uint4(acc[0].c[1], acc[1].c[1], acc[2].c[1], acc[3].c[1]);
  *reinterpret_cast<uint4*>(o2 + row) = make_uint4(acc[0].c[2], acc[1].c[2], acc[2].c[2], acc[3].c[2]);
  *reinterpret_cast<uint4*>(o3 + row) = make_uint4(acc[0].c[3], acc[1].c[3], acc[2].c[3], acc[3].c[3]);
}
nb200_status quotients_combined(nb200_ctx* ctx, const QLineDev* h_batches, size_t n_batches, const u32* g, const u32* dom_x, const u32* dom_y,
                                u32 log_size, u32* out /* 4 columns */) {
  NB_ARG(ctx, log_size >= 2 && ((((uintptr_t)out) | ((uintptr_t)g) | ((uintptr_t)dom_x) | ((uintptr_t)dom_y)) & 15u) == 0,
         "quotients_combined: 4-word aligned columns of at least 4 rows");
  QLineDev* d_b = nullptr;
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d_b, n_batches * sizeof(QLineDev)));
  NB_CUDA(ctx, cudaMemcpyAsync(d_b, h_batches, n_batches * sizeof(QLineDev), cudaMemcpyHostToDevice, ctx->stream));
  const size_t n = (size_t)1 << log_size;
  const u32 thr = 128;
  quotients_combined_kernel<<<(u32)((n / 4 + thr - 1) / thr), thr, 0, ctx->stream>>>(d_b, (u32)n_batches, g, dom_x, dom_y, log_size,
                                                                                   out, out + n, out + 2 * n, out + 3 * n);
  NB_LAUNCH_CHECK(ctx);
  dfree(ctx, d_b);
  return NB200_OK;
}

// ---- FRI folds ----
__device__ __forceinline__ qm31 ld_q(const u32* c, size_t n, size_t i) { return qm31_make(c[i], c[n + i], c[2 * n + i], c[3 * n + i]); }
__device__ __forceinline__ void st_q(u32* c, size_t n, size_t i, qm31 v) { c[i] = v.c[0]; c[n + i] = v.c[1]; c[2 * n + i] = v.c[2]; c[3 * n + i] = v.c[3]; }

// dst[i] = dst[i] * alpha^2 + (f0' + alpha f1'),  (f0', f1') = ibutterfly(src[2i], src[2i+1], 1/y_i)
__global__ void fold_circle_kernel(u32* __restrict__ dst, const u32* __restrict__ src, u32 src_log, const u32* __restrict__ itw, u32 tw_len,
                                   qm31 alpha, qm31 alpha_sq) {
  const size_t n = (size_t)1 << src_log, m = n >> 1;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  // circle inverse twiddle of layer 0 at h = i (same derivation as the FFT: [x, y] -> [y, -y, -x, x])
  u32 t;
  if (src_log <= 2) {
    t = 0;  // handled by the caller through explicit twiddles (tiny domains never reach FRI in practice)
  } else {
    const u32* l1 = itw + (tw_len - (1u << (src_log - 1)));
    u32 q = (u32)i >> 2, r = (u32)i & 3u;
    u32 x = __ldg(l1 + 2 * q), y = __ldg(l1 + 2 * q + 1);
    u32 v = (r < 2) ? y : x;
    t = (r == 1 || r == 2) ? (P31 - v) : v;
  }
  qm31 f0 = ld_q(src, n, 2 * i), f1 = ld_q(src, n, 2 * i + 1);
  qm31 s = qm31_add(f0, f1), d = qm31_mul_m31(qm31_sub(f0, f1), t);
  qm31 fp = qm31_add(qm31_mul(alpha, d), s);
  qm31 cur = ld_q(dst, m, i);
  st_q(dst, m, i, qm31_add(qm31_mul(cur, alpha_sq), fp));
}
// dst[i] = f0' + alpha f1',  (f0', f1') = ibutterfly(src[2i], src[2i+1], 1/x_i); alpha is read from d_alpha (device memory) when it is set
__global__ void fold_line_kernel(u32* __restrict__ dst, const u32* __restrict__ src, u32 src_log, const u32* __restrict__ itw, u32 tw_len, qm31 alpha,
                                 const u32* __restrict__ d_alpha) {
  const size_t n = (size_t)1 << src_log, m = n >> 1;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  if (d_alpha) alpha = qm31_make(__ldg(d_alpha), __ldg(d_alpha + 1), __ldg(d_alpha + 2), __ldg(d_alpha + 3));
  u32 t = __ldg(itw + (tw_len - (1u << src_log)) + i);
  qm31 f0 = ld_q(src, n, 2 * i), f1 = ld_q(src, n, 2 * i + 1);
  qm31 s = qm31_add(f0, f1), d = qm31_mul_m31(qm31_sub(f0, f1), t);
  st_q(dst, m, i, qm31_add(s, qm31_mul(alpha, d)));
}
nb200_status fold_circle_into_line(nb200_ctx* ctx, u32* dst, const u32* src, u32 src_log, qm31 alpha) {
  NB_ARG(ctx, src_log >= 3, "fold_circle_into_line: domain too small");
  NB_ARG(ctx, ctx->tw.d_itw && ctx->tw.half_log + 1 >= src_log, "fold_circle_into_line: twiddles");
  size_t m = (size_t)1 << (src_log - 1);
  u32 thr = 256;
  fold_circle_kernel<<<(u32)((m + thr - 1) / thr), thr, 0, ctx->stream>>>(dst, src, src_log, ctx->tw.d_itw, 1u << ctx->tw.half_log, alpha, qm31_mul(alpha, alpha));
  NB_LAUNCH_CHECK(ctx);
  return NB200_OK;
}
static nb200_status fold_line_launch(nb200_ctx* ctx, u32* dst, const u32* src, u32 src_log, qm31 alpha, const u32* d_alpha) {
  NB_ARG(ctx, src_log >= 1, "fold_line: domain too small");
  NB_ARG(ctx, ctx->tw.d_itw && ctx->tw.half_log >= src_log, "fold_line: twiddles");
  size_t m = (size_t)1 << (src_log - 1);
  u32 thr = 256;
  fold_line_kernel<<<(u32)((m + thr - 1) / thr), thr, 0, ctx->stream>>>(dst, src, src_log, ctx->tw.d_itw, 1u << ctx->tw.half_log, alpha, d_alpha);
  NB_LAUNCH_CHECK(ctx);
  return NB200_OK;
}
nb200_status fold_line(nb200_ctx* ctx, u32* dst, const u32* src, u32 src_log, qm31 alpha) { return fold_line_launch(ctx, dst, src, src_log, alpha, nullptr); }
nb200_status fold_line(nb200_ctx* ctx, u32* dst, const u32* src, u32 src_log, const u32* d_alpha) {
  return fold_line_launch(ctx, dst, src, src_log, qm31_zero(), d_alpha);
}

// ---- the channel between FRI's inner layers (device_channel.cuh): one thread mixes the root a Merkle commit just wrote (unless root is
// null) and draws the next alpha; rec receives the root's 8 words (zeros without a root) and the alpha's 4
__global__ void channel_mix_draw_kernel(DevChannel* __restrict__ ch, const u32* __restrict__ root, u32* __restrict__ rec, int domain_sep) {
  DevChannel c = *ch;
  u32 r[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { r[i] = root ? root[i] : 0u; rec[i] = r[i]; }
  if (root) dev_mix_root(c, r);
  u32 a[4];
  dev_draw_felt(c, domain_sep != 0, a);
#pragma unroll
  for (int i = 0; i < 4; ++i) rec[8 + i] = a[i];
  *ch = c;
}
nb200_status channel_mix_draw(nb200_ctx* ctx, DevChannel* d_ch, const uint8_t* d_root, u32* d_rec, int domain_sep) {
  channel_mix_draw_kernel<<<1, 1, 0, ctx->stream>>>(d_ch, (const u32*)d_root, d_rec, domain_sep);
  NB_LAUNCH_CHECK(ctx);
  return NB200_OK;
}

// ---- accumulate (AccumulationOps::accumulate): a[i] += b[i] over 4-coordinate columns ----
__global__ void add_inplace_kernel(u32* __restrict__ a, const u32* __restrict__ b, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = m31_add(a[i], b[i]);
}
nb200_status add_inplace(nb200_ctx* ctx, u32* a, const u32* b, size_t n) {
  u32 thr = 256;
  add_inplace_kernel<<<(u32)((n + thr - 1) / thr), thr, 0, ctx->stream>>>(a, b, n);
  NB_LAUNCH_CHECK(ctx);
  return NB200_OK;
}

// ---- table multiplicities (nb200_table_multiplicities): a table fraction's column (finalized order) = its bins' u64 counters mod P ----
__global__ void table_mult_store_kernel(u32* __restrict__ dst, const unsigned long long* __restrict__ cnt, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = (u32)(cnt[i] % P31);
}
nb200_status table_mult_store(nb200_ctx* ctx, u32* dst, const unsigned long long* cnt, size_t n) {
  u32 thr = 256;
  table_mult_store_kernel<<<(u32)((n + thr - 1) / thr), thr, 0, ctx->stream>>>(dst, cnt, n);
  NB_LAUNCH_CHECK(ctx);
  return NB200_OK;
}

// a[i] = (a[i] - b[i]) / t, t = the top-layer (line layer tw_log - 1) twiddle of CanonicCoset(tw_log)'s FFT on the first half of the domain.
// Used to split a polynomial of 2^tw_log coefficients into its low and high halves from evaluations on two half-size domains (prove.cu).
__global__ void sub_scale_kernel(u32* __restrict__ a, const u32* __restrict__ b, size_t n, const u32* __restrict__ itw_top) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const u32 it = __ldg(itw_top);
  if (i < n) a[i] = m31_mul(m31_sub(a[i], b[i]), it);
}
nb200_status sub_scale_top_twiddle(nb200_ctx* ctx, u32* a, const u32* b, size_t n, u32 tw_log) {
  NB_ARG(ctx, ctx->tw.d_itw && tw_log >= 2 && ctx->tw.half_log + 1 >= tw_log, "sub_scale_top_twiddle: twiddles");
  // TwiddleTree layout: the array of layer i of canonic(n) starts at tw_len - 2^(n - i); layer n - 1 has one entry
  const u32* it = ctx->tw.d_itw + (((size_t)1 << ctx->tw.half_log) - 2);
  u32 thr = 256;
  sub_scale_kernel<<<(u32)((n + thr - 1) / thr), thr, 0, ctx->stream>>>(a, b, n, it);
  NB_LAUNCH_CHECK(ctx);
  return NB200_OK;
}
// dst[c * dst_stride + i] += src[c * src_stride + i], i < len
__global__ void add_cols_kernel(u32* __restrict__ dst, size_t dst_stride, const u32* __restrict__ src, size_t src_stride, size_t len) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < len) { u32* d = dst + blockIdx.y * dst_stride + i; *d = m31_add(*d, src[blockIdx.y * src_stride + i]); }
}
nb200_status add_cols_strided(nb200_ctx* ctx, u32* dst, size_t dst_stride, const u32* src, size_t src_stride, size_t len, size_t n_cols) {
  u32 thr = 256;
  add_cols_kernel<<<dim3((u32)((len + thr - 1) / thr), (u32)n_cols), thr, 0, ctx->stream>>>(dst, dst_stride, src, src_stride, len);
  NB_LAUNCH_CHECK(ctx);
  return NB200_OK;
}

// ---- proof of work: smallest nonce with trailing_zeros(Blake2s(digest || nonce_le)) >= pow_bits ----
__global__ void grind_kernel(const u32 d0, const u32 d1, const u32 d2, const u32 d3, const u32 d4, const u32 d5, const u32 d6, const u32 d7,
                             u64 base, u32 pow_bits, unsigned long long* __restrict__ result) {
  u64 nonce = base + (u64)blockIdx.x * blockDim.x + threadIdx.x;
  u32 h[8]; b2s_init(h);
  u32 m[16] = {d0, d1, d2, d3, d4, d5, d6, d7, (u32)nonce, (u32)(nonce >> 32), 0, 0, 0, 0, 0, 0};
  b2s_compress(h, m, 40, 0, 0xFFFFFFFFu, 0);
  // trailing zeros of the first 16 bytes as a little-endian u128
  u32 tz;
  if (h[0]) tz = __ffs(h[0]) - 1;
  else if (h[1]) tz = 32 + __ffs(h[1]) - 1;
  else if (h[2]) tz = 64 + __ffs(h[2]) - 1;
  else if (h[3]) tz = 96 + __ffs(h[3]) - 1;
  else tz = 128;
  if (tz >= pow_bits) atomicMin(result, (unsigned long long)nonce);
}
nb200_status grind(nb200_ctx* ctx, const uint8_t digest[32], u32 pow_bits, uint64_t* nonce_out) {
  NB_ARG(ctx, ctx->pow_variant == 0, "grind: only pow_variant 0 is implemented");
  NB_ARG(ctx, pow_bits <= 64, "grind: pow_bits too large");
  u32 d[8];
  for (int i = 0; i < 8; ++i) d[i] = (u32)digest[4 * i] | ((u32)digest[4 * i + 1] << 8) | ((u32)digest[4 * i + 2] << 16) | ((u32)digest[4 * i + 3] << 24);
  unsigned long long* d_res = nullptr;
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d_res, 8));
  const unsigned long long none = ~0ull;
  u64 base = 0;
  // chunk size grows with the expected work so tiny pow_bits stay cheap
  u32 blocks = pow_bits <= 12 ? 64 : (u32)ctx->sm_count * 32;
  const u32 thr = 256;
  while (true) {
    NB_CUDA(ctx, cudaMemcpyAsync(d_res, &none, 8, cudaMemcpyHostToDevice, ctx->stream));
    grind_kernel<<<blocks, thr, 0, ctx->stream>>>(d[0], d[1], d[2], d[3], d[4], d[5], d[6], d[7], base, pow_bits, d_res);
    NB_LAUNCH_CHECK(ctx);
    unsigned long long r;
    NB_CUDA(ctx, cudaMemcpyAsync(&r, d_res, 8, cudaMemcpyDeviceToHost, ctx->stream));
    NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (r != none) { *nonce_out = r; break; }
    base += (u64)blocks * thr;
  }
  dfree(ctx, d_res);
  return NB200_OK;
}

}  // namespace nb
