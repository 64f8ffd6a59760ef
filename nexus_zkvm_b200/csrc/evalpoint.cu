// PolyOps::eval_at_point for batches of coefficient columns at QM31 circle points (OODS sampling inside
// CommitmentSchemeProver::prove_values, reached from stwo::prover::prove at nexus-zkvm
// prover/src/machine.rs:286-290).
//
// f(p) = sum_i c_i * prod_b m_b^{bit b of i},  m = [p.y, p.x, pi(p.x), pi^2(p.x), ...]  (stwo backend/cpu/circle.rs
// eval_at_point + core/poly/utils.rs fold).  Field arithmetic is exact, so any summation order is bit-exact.
// One sweep over the coefficients (HBM-bound): a CTA owns 2^Q consecutive coefficients, thread t accumulates
// c[j*2^LB + t] * w_mid[j] with lazily reduced 64-bit accumulators, multiplies by its own low-bit weight,
// the CTA reduces and applies the weight of its block index; a second kernel adds the per-CTA partials.  Any number of (column, point)
// pairs of any sizes go into one launch of each kernel (OODS sampling evaluates every committed column in one round trip).
#include "pcs.h"
#include <algorithm>

namespace nb {

static constexpr u32 EP_THREADS = 256;
static constexpr u32 EP_LB = 8;    // low bits handled across threads
static constexpr u32 EP_QMAX = 15; // coefficients per CTA (log)

__device__ __forceinline__ qm31 load_q(const u32* p) { return qm31_make(p[0], p[1], p[2], p[3]); }

// One (column, point) evaluation of a batched launch: its CTAs are [cta0, cta0 + 2^(log_size - Q)), Q = min(log_size, EP_QMAX), and the
// point's factors [y, x, pi(x), ...] start at factors + fac_off.
struct EvalJobDev { const u32* coeffs; u32 log_size, fac_off, cta0, pad; };

// grid: one CTA per block of 2^Q coefficients of every job; partials[cta] = the block's weighted sum
__global__ void __launch_bounds__(EP_THREADS) eval_points_partial_kernel(const EvalJobDev* __restrict__ jobs, u32 n_jobs, const u32* __restrict__ factors,
                                                                        u32* __restrict__ partials /* [cta][4] */) {
  __shared__ __align__(16) u32 wmid[128 * 4];
  __shared__ u32 red[EP_THREADS / 32][4];
  __shared__ u32 s_job;
  const u32 t = threadIdx.x;
  if (t == 0) {   // the last job whose first CTA is at or before this one
    u32 lo = 0, hi = n_jobs - 1;
    while (lo < hi) { const u32 mid = (lo + hi + 1) >> 1; if (jobs[mid].cta0 <= blockIdx.x) lo = mid; else hi = mid - 1; }
    s_job = lo;
  }
  __syncthreads();
  const EvalJobDev job = jobs[s_job];
  const u32 log_size = job.log_size;
  const u32 Q = log_size < EP_QMAX ? log_size : EP_QMAX;
  const u32 blk = blockIdx.x - job.cta0;
  const u32 LB = Q < EP_LB ? Q : EP_LB;
  const u32 nj = 1u << (Q - LB);
  const u32* f = factors + job.fac_off;
  // mid weights
  if (t < nj) {
    qm31 w = qm31_one();
    for (u32 b = 0; b < Q - LB; ++b) if ((t >> b) & 1u) w = qm31_mul(w, load_q(f + 4 * (LB + b)));
    wmid[4 * t] = w.c[0]; wmid[4 * t + 1] = w.c[1]; wmid[4 * t + 2] = w.c[2]; wmid[4 * t + 3] = w.c[3];
  }
  __syncthreads();
  qm31 acc = qm31_zero();
  if (t < (1u << LB)) {
    const u32* c = job.coeffs + ((size_t)blk << Q);
    u64 a0 = 0, a1 = 0, a2 = 0, a3 = 0;
    // raw 64-bit products: four of them (< 2^62 each) plus a reduced carry-in fit, so reduce after every fourth term; the four
    // coefficient loads of a group are issued together
    u32 j = 0;
    // eight coefficient loads (two reduction groups) are in flight per thread before any arithmetic: the sweep is latency bound otherwise
    for (; j + 8 <= nj; j += 8) {
      u32 v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = __ldg(c + ((size_t)(j + u) << LB) + t);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint4 w0 = *reinterpret_cast<const uint4*>(wmid + 4 * (j + 4 * h)), w1 = *reinterpret_cast<const uint4*>(wmid + 4 * (j + 4 * h) + 4);
        const uint4 w2 = *reinterpret_cast<const uint4*>(wmid + 4 * (j + 4 * h) + 8), w3 = *reinterpret_cast<const uint4*>(wmid + 4 * (j + 4 * h) + 12);
        const u32 v0 = v[4 * h], v1 = v[4 * h + 1], v2 = v[4 * h + 2], v3 = v[4 * h + 3];
        a0 += (u64)v0 * w0.x + (u64)v1 * w1.x + (u64)v2 * w2.x + (u64)v3 * w3.x;
        a1 += (u64)v0 * w0.y + (u64)v1 * w1.y + (u64)v2 * w2.y + (u64)v3 * w3.y;
        a2 += (u64)v0 * w0.z + (u64)v1 * w1.z + (u64)v2 * w2.z + (u64)v3 * w3.z;
        a3 += (u64)v0 * w0.w + (u64)v1 * w1.w + (u64)v2 * w2.w + (u64)v3 * w3.w;
        a0 = m31_red64(a0); a1 = m31_red64(a1); a2 = m31_red64(a2); a3 = m31_red64(a3);
      }
    }
    for (; j + 4 <= nj; j += 4) {
      const u32 v0 = __ldg(c + ((size_t)j << LB) + t), v1 = __ldg(c + ((size_t)(j + 1) << LB) + t);
      const u32 v2 = __ldg(c + ((size_t)(j + 2) << LB) + t), v3 = __ldg(c + ((size_t)(j + 3) << LB) + t);
      const uint4 w0 = *reinterpret_cast<const uint4*>(wmid + 4 * j), w1 = *reinterpret_cast<const uint4*>(wmid + 4 * j + 4);
      const uint4 w2 = *reinterpret_cast<const uint4*>(wmid + 4 * j + 8), w3 = *reinterpret_cast<const uint4*>(wmid + 4 * j + 12);
      a0 += (u64)v0 * w0.x + (u64)v1 * w1.x + (u64)v2 * w2.x + (u64)v3 * w3.x;
      a1 += (u64)v0 * w0.y + (u64)v1 * w1.y + (u64)v2 * w2.y + (u64)v3 * w3.y;
      a2 += (u64)v0 * w0.z + (u64)v1 * w1.z + (u64)v2 * w2.z + (u64)v3 * w3.z;
      a3 += (u64)v0 * w0.w + (u64)v1 * w1.w + (u64)v2 * w2.w + (u64)v3 * w3.w;
      a0 = m31_red64(a0); a1 = m31_red64(a1); a2 = m31_red64(a2); a3 = m31_red64(a3);
    }
    for (; j < nj; ++j) {
      const u32 v = __ldg(c + ((size_t)j << LB) + t);
      const uint4 w = *reinterpret_cast<const uint4*>(wmid + 4 * j);
      a0 += (u64)v * w.x; a1 += (u64)v * w.y; a2 += (u64)v * w.z; a3 += (u64)v * w.w;
    }
    acc = qm31_make(m31_red64(a0), m31_red64(a1), m31_red64(a2), m31_red64(a3));
    // low-bit weight of this thread
    qm31 w = qm31_one();
    for (u32 b = 0; b < LB; ++b) if ((t >> b) & 1u) w = qm31_mul(w, load_q(f + 4 * b));
    acc = qm31_mul(acc, w);
  }
  // block reduction (field additions)
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    u32 x = acc.c[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x = m31_add(x, __shfl_xor_sync(0xffffffffu, x, o));
    if ((t & 31u) == 0) red[t >> 5][k] = x;
  }
  __syncthreads();
  if (t == 0) {
    qm31 s = qm31_zero();
    for (u32 w = 0; w < EP_THREADS / 32; ++w) s = qm31_add(s, qm31_make(red[w][0], red[w][1], red[w][2], red[w][3]));
    qm31 wb = qm31_one();
    for (u32 b = Q; b < log_size; ++b) if ((blk >> (b - Q)) & 1u) wb = qm31_mul(wb, load_q(f + 4 * b));
    s = qm31_mul(s, wb);
    u32* o = partials + (size_t)blockIdx.x * 4;
    o[0] = s.c[0]; o[1] = s.c[1]; o[2] = s.c[2]; o[3] = s.c[3];
  }
}

// out[job] = the sum of its CTAs' partials
__global__ void eval_points_sum_kernel(const EvalJobDev* __restrict__ jobs, u32 n_jobs, const u32* __restrict__ partials, u32* __restrict__ out) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_jobs) return;
  const EvalJobDev job = jobs[i];
  const u32 Q = job.log_size < EP_QMAX ? job.log_size : EP_QMAX;
  const u32 nblk = 1u << (job.log_size - Q);
  const u32* p = partials + (size_t)job.cta0 * 4;
  qm31 s = qm31_zero();
  for (u32 b = 0; b < nblk; ++b) s = qm31_add(s, qm31_make(p[4 * b], p[4 * b + 1], p[4 * b + 2], p[4 * b + 3]));
  out[4 * i] = s.c[0]; out[4 * i + 1] = s.c[1]; out[4 * i + 2] = s.c[2]; out[4 * i + 3] = s.c[3];
}

// Every job in one partial launch and one sum launch: one upload (jobs + every point's factors), one copy back, one sync.
nb200_status eval_at_points_multi(nb200_ctx* ctx, const std::vector<EvalJob>& jobs, const u32* points_xy, size_t n_points, u32* out_qm31) {
  if (jobs.empty()) return NB200_OK;
  // factors per point, up to the largest log size it is evaluated at: [y, x, pi(x), ...] (a smaller column uses a prefix)
  std::vector<u32> max_log(n_points, 1);
  for (const EvalJob& j : jobs) {
    NB_ARG(ctx, j.point < n_points && j.log_size <= 30, "eval_at_points: point index or log size");
    max_log[j.point] = std::max(max_log[j.point], j.log_size);
  }
  std::vector<u32> fac_off(n_points);
  size_t fac_words = 0;
  for (size_t p = 0; p < n_points; ++p) { fac_off[p] = (u32)fac_words; fac_words += (size_t)max_log[p] * 4; }
  std::vector<EvalJobDev> jd(jobs.size());
  size_t ctas = 0;
  for (size_t i = 0; i < jobs.size(); ++i) {
    const u32 Q = jobs[i].log_size < EP_QMAX ? jobs[i].log_size : EP_QMAX;
    jd[i] = EvalJobDev{jobs[i].coeffs, jobs[i].log_size, fac_off[jobs[i].point], (u32)ctas, 0};
    ctas += (size_t)1 << (jobs[i].log_size - Q);
  }
  NB_ARG(ctx, ctas < 0x7fffffffu && jobs.size() < 0x7fffffffu, "eval_at_points: too many evaluations in one launch");
  const size_t job_bytes = jobs.size() * sizeof(EvalJobDev);
  std::vector<uint8_t> up(job_bytes + fac_words * 4);
  memcpy(up.data(), jd.data(), job_bytes);
  u32* fac = (u32*)(up.data() + job_bytes);
  for (size_t p = 0; p < n_points; ++p) {
    const u32* xy = points_xy + 8 * p;
    qm31 x = qm31_make(xy[0], xy[1], xy[2], xy[3]), y = qm31_make(xy[4], xy[5], xy[6], xy[7]);
    for (u32 b = 0; b < max_log[p]; ++b) {
      qm31 v;
      if (b == 0) v = y; else { v = x; x = qm31_double_x(x); }
      memcpy(fac + fac_off[p] + 4 * b, v.c, 16);
    }
  }
  uint8_t* d = nullptr;
  const size_t n_out = jobs.size();
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d, up.size() + (ctas + n_out) * 16));
  const EvalJobDev* d_jobs = (const EvalJobDev*)d;
  const u32* d_fac = (const u32*)(d + job_bytes);
  u32* d_part = (u32*)(d + up.size());
  u32* d_out = d_part + ctas * 4;
  cudaError_t e = cudaMemcpyAsync(d, up.data(), up.size(), cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) {
    eval_points_partial_kernel<<<(u32)ctas, EP_THREADS, 0, ctx->stream>>>(d_jobs, (u32)n_out, d_fac, d_part);
    eval_points_sum_kernel<<<(u32)((n_out + 127) / 128), 128, 0, ctx->stream>>>(d_jobs, (u32)n_out, d_part, d_out);
    ctx->launches += 2;
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(out_qm31, d_out, n_out * 16, cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);   // also: `up` has been consumed
  dfree(ctx, d);
  if (e != cudaSuccess) return set_err(ctx, NB200_ERR_CUDA, std::string("eval_at_points: ") + cudaGetErrorString(e));
  return NB200_OK;
}

// every column of a batch at every point: out = n_cols x n_points QM31s
nb200_status eval_at_points(nb200_ctx* ctx, const u32* coeffs, size_t n_cols, u32 log_size, const u32* points_xy, size_t n_points, u32* out_qm31) {
  if (n_cols == 0 || n_points == 0) return NB200_OK;
  std::vector<EvalJob> jobs;
  for (size_t c = 0; c < n_cols; ++c)
    for (size_t p = 0; p < n_points; ++p) jobs.push_back(EvalJob{coeffs + (c << log_size), log_size, (u32)p});
  return eval_at_points_multi(ctx, jobs, points_xy, n_points, out_qm31);
}

}  // namespace nb
