// AIR bytecode interpreter kernels:
//  (1) constraint / quotient evaluation over the blow-up domain — replaces
//      ComponentProver::<SimdBackend>::evaluate_constraint_quotients_on_domain (FrameworkComponent + SimdDomainEvaluator),
//      reached from stwo::prover::prove at nexus-zkvm prover/src/machine.rs:286-290; the constraints themselves are
//      the reference's `add_constraints` bodies (prover/src/components/mod.rs:48-57) recorded as bytecode;
//  (2) LogUp interaction-trace generation (LogupTraceGenerator::{write_frac, finalize_col, finalize_last}) — replaces the
//      CPU-SIMD generate_interaction_trace at machine.rs:242-247 / traits.rs:124-145 (SURVEY.md §8 row f2).
// One thread per row; the program is uniform across the grid (no divergence); virtual registers live in shared
// memory laid out [register][thread] so every access is conflict-free; column reads are coalesced.
#include "common.cuh"
#include "air.h"
#include "jit.h"
#include "circle_host.h"

namespace nb {

struct MaskDev { const u32* ptr; int32_t off; u32 pad; };

struct InterpArgs {
  const uint4* prog; u32 n_instr;
  const MaskDev* masks;
  const u32* params;       // n_params x 4
  u32 nb, ne;              // register counts
  u32 log_size, eval_log;  // trace / evaluation domain logs
  // constraint mode
  const u32* coeff;        // n_constraints x 4 (random-coefficient powers in declaration order)
  const u32* dinv;         // 2^(eval_log - log_size) vanishing inverses (bit-reversed coset order)
  u32* acc[4];             // accumulator columns (+=)
  // logup mode
  const u32* batching;     // fraction -> batch
  u32* out;                // 4 * n_batches columns of 2^log_size
  u32 n_batches;
};

// constraint-framework utils: offset_bit_reversed_circle_domain_index
__device__ __forceinline__ u32 offset_row(u32 i, u32 domain_log, u32 eval_log, int32_t off) {
  u32 prev = __brev(i) >> (32 - eval_log);
  u32 half = 1u << (eval_log - 1);
  int64_t step = (int64_t)off * (int64_t)(1u << (eval_log - domain_log - 1));
  int64_t v;
  if (prev < half) { v = ((int64_t)prev + step) % (int64_t)half; if (v < 0) v += half; }
  else { v = ((int64_t)prev - step) % (int64_t)half; if (v < 0) v += half; v += half; }
  return __brev((u32)v) >> (32 - eval_log);
}

#define BR(r) sm[(r) * BD + tid]
#define ER(r, k) sm[(nb + 4 * (r) + (k)) * BD + tid]

template <int BD, bool LOGUP>
__global__ void __launch_bounds__(BD) interp_kernel(const InterpArgs a) {
  extern __shared__ u32 sm[];
  const u32 tid = threadIdx.x;
  const u32 row = blockIdx.x * BD + tid;  // grids are exact multiples of BD (domains are >= BD or BD is clamped)
  const u32 nb = a.nb;
  qm31 row_res = qm31_zero();
  u32 k = 0;
  // logup state
  qm31 fn = qm31_zero(), fd = qm31_one(), running = qm31_zero();
  u32 cur_batch = 0; bool have = false;
  const size_t n_rows = (size_t)1 << a.log_size;

  for (u32 pc = 0; pc < a.n_instr; ++pc) {
    const uint4 in = __ldg(a.prog + pc);
    switch (in.x) {
      case OP_LOADM: {
        const MaskDev m = a.masks[in.z];
        u32 r = (LOGUP || m.off == 0) ? row : offset_row(row, a.log_size, a.eval_log, m.off);
        BR(in.y) = m.ptr ? __ldg(m.ptr + r) : 0u;
      } break;
      case OP_CONSTB: BR(in.y) = in.z; break;
      case OP_ADDB: BR(in.y) = m31_add(BR(in.z), BR(in.w)); break;
      case OP_SUBB: BR(in.y) = m31_sub(BR(in.z), BR(in.w)); break;
      case OP_MULB: BR(in.y) = m31_mul(BR(in.z), BR(in.w)); break;
      case OP_NEGB: BR(in.y) = m31_neg(BR(in.z)); break;
      case OP_PARAME: {
        const u32* p = a.params + 4 * in.z;
        ER(in.y, 0) = __ldg(p); ER(in.y, 1) = __ldg(p + 1); ER(in.y, 2) = __ldg(p + 2); ER(in.y, 3) = __ldg(p + 3);
      } break;
      case OP_ADDE: {
#pragma unroll
        for (int c = 0; c < 4; ++c) ER(in.y, c) = m31_add(ER(in.z, c), ER(in.w, c));
      } break;
      case OP_SUBE: {
#pragma unroll
        for (int c = 0; c < 4; ++c) ER(in.y, c) = m31_sub(ER(in.z, c), ER(in.w, c));
      } break;
      case OP_MULE: {
        qm31 x = qm31_make(ER(in.z, 0), ER(in.z, 1), ER(in.z, 2), ER(in.z, 3));
        qm31 y = qm31_make(ER(in.w, 0), ER(in.w, 1), ER(in.w, 2), ER(in.w, 3));
        qm31 r = qm31_mul(x, y);
        ER(in.y, 0) = r.c[0]; ER(in.y, 1) = r.c[1]; ER(in.y, 2) = r.c[2]; ER(in.y, 3) = r.c[3];
      } break;
      case OP_NEGE: {
#pragma unroll
        for (int c = 0; c < 4; ++c) ER(in.y, c) = m31_neg(ER(in.z, c));
      } break;
      case OP_ADDEB: {
        u32 b = BR(in.w);
        u32 e0 = ER(in.z, 0), e1 = ER(in.z, 1), e2 = ER(in.z, 2), e3 = ER(in.z, 3);
        ER(in.y, 0) = m31_add(e0, b); ER(in.y, 1) = e1; ER(in.y, 2) = e2; ER(in.y, 3) = e3;
      } break;
      case OP_SUBEB: {
        u32 b = BR(in.w);
        u32 e0 = ER(in.z, 0), e1 = ER(in.z, 1), e2 = ER(in.z, 2), e3 = ER(in.z, 3);
        ER(in.y, 0) = m31_sub(e0, b); ER(in.y, 1) = e1; ER(in.y, 2) = e2; ER(in.y, 3) = e3;
      } break;
      case OP_MULEB: {
        u32 b = BR(in.w);
#pragma unroll
        for (int c = 0; c < 4; ++c) ER(in.y, c) = m31_mul(ER(in.z, c), b);
      } break;
      case OP_BTOE: {
        u32 b = BR(in.z);
        ER(in.y, 0) = b; ER(in.y, 1) = 0; ER(in.y, 2) = 0; ER(in.y, 3) = 0;
      } break;
      case OP_LOADME: {
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const MaskDev m = a.masks[in.z + c];
          u32 r = (LOGUP || m.off == 0) ? row : offset_row(row, a.log_size, a.eval_log, m.off);
          ER(in.y, c) = m.ptr ? __ldg(m.ptr + r) : 0u;
        }
      } break;
      case OP_CONSTRB: {
        if (!LOGUP) {
          u32 v = BR(in.z);
          const u32* cf = a.coeff + 4 * k;
#pragma unroll
          for (int c = 0; c < 4; ++c) row_res.c[c] = m31_add(row_res.c[c], m31_mul(__ldg(cf + c), v));
          ++k;
        }
      } break;
      case OP_CONSTRE: {
        if (!LOGUP) {
          qm31 v = qm31_make(ER(in.z, 0), ER(in.z, 1), ER(in.z, 2), ER(in.z, 3));
          const u32* cf = a.coeff + 4 * k;
          qm31 cq = qm31_make(__ldg(cf), __ldg(cf + 1), __ldg(cf + 2), __ldg(cf + 3));
          row_res = qm31_add(row_res, qm31_mul(cq, v));
          ++k;
        }
      } break;
      case OP_FRAC: {
        if (LOGUP) {
          u32 b = __ldg(a.batching + k);
          if (have && b != cur_batch) {
            running = qm31_add(running, qm31_mul(fn, qm31_inv(fd)));
#pragma unroll
            for (int c = 0; c < 4; ++c) a.out[((size_t)(4 * cur_batch + c) << a.log_size) + row] = running.c[c];
            fn = qm31_zero(); fd = qm31_one();
          }
          cur_batch = b; have = true;
          qm31 nu = qm31_make(ER(in.z, 0), ER(in.z, 1), ER(in.z, 2), ER(in.z, 3));
          qm31 de = qm31_make(ER(in.w, 0), ER(in.w, 1), ER(in.w, 2), ER(in.w, 3));
          fn = qm31_add(qm31_mul(fn, de), qm31_mul(nu, fd));
          fd = qm31_mul(fd, de);
          ++k;
        }
      } break;
      default: break;
    }
  }
  if (LOGUP) {
    if (have) {
      running = qm31_add(running, qm31_mul(fn, qm31_inv(fd)));
#pragma unroll
      for (int c = 0; c < 4; ++c) a.out[((size_t)(4 * cur_batch + c) << a.log_size) + row] = running.c[c];
    }
    (void)n_rows;
  } else {
    u32 di = __ldg(a.dinv + (row >> a.log_size));
#pragma unroll
    for (int c = 0; c < 4; ++c) a.acc[c][row] = m31_add(a.acc[c][row], m31_mul(row_res.c[c], di));
  }
}
#undef BR
#undef ER

// ---- small utilities: column sum, coset-order prefix sum ----
__global__ void sum_columns_kernel(const u32* __restrict__ cols, u32 log_size, u32* __restrict__ partial /* [col][block] */) {
  __shared__ u32 red[32];
  const u32 col = blockIdx.y;
  const u32* c = cols + ((size_t)col << log_size);
  size_t n = (size_t)1 << log_size;
  u64 acc = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) acc += c[i];
  u32 v = m31_reduce64(acc);
  for (int o = 16; o > 0; o >>= 1) v = m31_add(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    u32 s = 0;
    for (u32 w = 0; w < blockDim.x / 32; ++w) s = m31_add(s, red[w]);
    partial[col * gridDim.x + blockIdx.x] = s;
  }
}

__device__ __forceinline__ u32 coset_pos(u32 i, u32 log_size) {
  // bit_reverse_index(coset_index_to_circle_domain_index(i, n), n)
  u32 d = (i & 1u) ? (((2u << log_size) - i) >> 1) : (i >> 1);
  return log_size ? (__brev(d) >> (32 - log_size)) : 0;
}
// tmp[i] = col[pos(i)] - shift   (coset order)
__global__ void coset_gather_shift_kernel(const u32* __restrict__ col, u32 log_size, u32 shift, u32* __restrict__ tmp) {
  u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < (1u << log_size)) tmp[i] = m31_sub(col[coset_pos(i, log_size)], shift);
}
__global__ void coset_scatter_kernel(const u32* __restrict__ tmp, u32 log_size, u32* __restrict__ col) {
  u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < (1u << log_size)) col[coset_pos(i, log_size)] = tmp[i];
}
// inclusive scan (mod P) of chunks of 1024; block totals to `totals`
__global__ void scan_block_kernel(u32* __restrict__ data, size_t n, u32* __restrict__ totals) {
  __shared__ u32 wsum[32];
  size_t i = (size_t)blockIdx.x * 1024 + threadIdx.x;
  u32 v = i < n ? data[i] : 0u;
  const u32 lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int o = 1; o < 32; o <<= 1) { u32 t = __shfl_up_sync(0xffffffffu, v, o); if (lane >= (u32)o) v = m31_add(v, t); }
  if (lane == 31) wsum[w] = v;
  __syncthreads();
  if (w == 0) {
    u32 s = wsum[lane];
    for (int o = 1; o < 32; o <<= 1) { u32 t = __shfl_up_sync(0xffffffffu, s, o); if (lane >= (u32)o) s = m31_add(s, t); }
    wsum[lane] = s;
  }
  __syncthreads();
  if (w > 0) v = m31_add(v, wsum[w - 1]);
  if (i < n) data[i] = v;
  if (threadIdx.x == 1023 && totals) totals[blockIdx.x] = v;
}
__global__ void scan_add_kernel(u32* __restrict__ data, size_t n, const u32* __restrict__ totals_scanned) {
  size_t i = (size_t)blockIdx.x * 1024 + threadIdx.x;
  if (blockIdx.x > 0 && i < n) data[i] = m31_add(data[i], totals_scanned[blockIdx.x - 1]);
}
static nb200_status inclusive_scan(nb200_ctx* ctx, u32* d, size_t n) {
  size_t nblk = (n + 1023) / 1024;
  u32* totals = nullptr;
  if (nblk > 1) NB_CUDA(ctx, dmalloc(ctx, (void**)&totals, nblk * 4));
  scan_block_kernel<<<(u32)nblk, 1024, 0, ctx->stream>>>(d, n, totals);
  NB_LAUNCH_CHECK(ctx);
  if (nblk > 1) {
    NB_TRY(inclusive_scan(ctx, totals, nblk));
    scan_add_kernel<<<(u32)nblk, 1024, 0, ctx->stream>>>(d, n, totals);
    NB_LAUNCH_CHECK(ctx);
    dfree(ctx, totals);
  }
  return NB200_OK;
}

// ---- host drivers ----
static nb200_status upload_prog(nb200_ctx* ctx, const std::vector<AirInstr>& prog, uint4** d_prog) {
  static_assert(sizeof(AirInstr) == sizeof(uint4), "instr layout");
  NB_CUDA(ctx, dmalloc(ctx, (void**)d_prog, prog.size() * sizeof(uint4)));
  NB_CUDA(ctx, cudaMemcpyAsync(*d_prog, prog.data(), prog.size() * sizeof(uint4), cudaMemcpyHostToDevice, ctx->stream));
  return NB200_OK;
}

template <bool LOGUP>
static nb200_status launch_interp(nb200_ctx* ctx, InterpArgs& a, u32 domain_log) {
  size_t rows = (size_t)1 << domain_log;
  size_t per_thread = ((size_t)a.nb + 4 * (size_t)a.ne) * 4;
  // pick the block size that fits the register file in shared memory (<= 200 KB)
  u32 bd = 128;
  while (bd > 32 && per_thread * bd > 200 * 1024) bd >>= 1;
  while ((size_t)bd > rows) bd >>= 1;
  NB_ARG(ctx, bd >= 16 || rows < 16, "air: too many virtual registers for the interpreter");
  NB_ARG(ctx, per_thread * bd <= 200 * 1024, "air: too many virtual registers for the interpreter");
  size_t smem = per_thread * bd;
  if (smem == 0) smem = 4;
  u32 blocks = (u32)(rows / bd);
#define NB_LAUNCH_INTERP(BDV)                                                                                                   \
  {                                                                                                                             \
    NB_CUDA(ctx, cudaFuncSetAttribute(interp_kernel<BDV, LOGUP>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));     \
    interp_kernel<BDV, LOGUP><<<blocks, BDV, smem, ctx->stream>>>(a);                                                           \
  }
  switch (bd) {
    case 128: NB_LAUNCH_INTERP(128) break;
    case 64: NB_LAUNCH_INTERP(64) break;
    case 32: NB_LAUNCH_INTERP(32) break;
    case 16: NB_LAUNCH_INTERP(16) break;
    case 8: NB_LAUNCH_INTERP(8) break;
    case 4: NB_LAUNCH_INTERP(4) break;
    case 2: NB_LAUNCH_INTERP(2) break;
    default: NB_LAUNCH_INTERP(1) break;
  }
#undef NB_LAUNCH_INTERP
  NB_LAUNCH_CHECK(ctx);
  return NB200_OK;
}

// Evaluate the component's constraints on its evaluation domain and accumulate  sum_k coeff_k * c_k / vanishing  into acc.
// mask_cols[m]: device pointer of mask m's column evaluated on CanonicCoset(eval_log).circle_domain().
nb200_status constraint_eval(nb200_ctx* ctx, const AirComponent& c, const std::vector<const u32*>& mask_cols, const u32* d_params,
                             const std::vector<qm31>& coeffs, u32* const acc[4], const JitKernel* jk, u32 rows_log, u32 dom_log, u32 row0, size_t n_rows,
                             u32* const acc_high[4]) {
  NB_ARG(ctx, mask_cols.size() == c.masks.size() && coeffs.size() == c.n_constraints, "constraint_eval: shape");
  // rows [0, 2^rows_log) of CanonicCoset(dom_log).circle_domain() in bit-reversed order: the whole domain or its first half
  if (rows_log == 0 && dom_log == 0) rows_log = dom_log = c.eval_log();
  NB_ARG(ctx, dom_log > c.log_size && (rows_log == dom_log || rows_log + 1 == dom_log) && rows_log >= c.log_size, "constraint_eval: row range");
  const u32 elog = dom_log;
  // vanishing inverses: coset_vanishing(CanonicCoset(log_size).coset, eval_domain.at(i)) for i < 2^(dom_log - log_size), bit-reversed
  // (the vanishing polynomial is constant on each block of 2^log_size rows; a first-half row range uses the first half of the table)
  std::vector<u32> dinv((size_t)1 << (dom_log - c.log_size));
  {
    HCircleDomain ed = HCircleDomain::canonic(elog);
    HCoset tc = HCoset::odds(c.log_size);
    // rotate to the canonic coset: p - initial + step/2 ; then double x (log_size - 1) times
    u32 shift = idx_add(idx_neg(tc.initial_index), tc.step_index >> 1);
    for (size_t i = 0; i < dinv.size(); ++i) {
      u32 x = index_to_point(idx_add(ed.index_at(i), shift)).x;
      for (u32 k = 1; k < c.log_size; ++k) x = m31_double_x(x);
      dinv[bit_reverse_u32((u32)i, dom_log - c.log_size)] = m31_inv(x);
    }
  }
  std::vector<MaskDev> hm(c.masks.size());
  for (size_t m = 0; m < hm.size(); ++m) { hm[m].ptr = mask_cols[m]; hm[m].off = c.masks[m].off; hm[m].pad = 0; }
  uint4* d_prog = nullptr; MaskDev* d_masks = nullptr; u32 *d_coeff = nullptr, *d_dinv = nullptr;
  NB_TRY(upload_prog(ctx, c.prog, &d_prog));
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d_masks, hm.size() * sizeof(MaskDev)));
  NB_CUDA(ctx, cudaMemcpyAsync(d_masks, hm.data(), hm.size() * sizeof(MaskDev), cudaMemcpyHostToDevice, ctx->stream));
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d_coeff, coeffs.size() * 16));
  NB_CUDA(ctx, cudaMemcpyAsync(d_coeff, coeffs.data(), coeffs.size() * 16, cudaMemcpyHostToDevice, ctx->stream));
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d_dinv, dinv.size() * 4));
  NB_CUDA(ctx, cudaMemcpyAsync(d_dinv, dinv.data(), dinv.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
  nb200_status st;
  const bool use_jit = jit_usable(jk, c, rows_log);
  if (row0 != 0 || n_rows != 0) NB_ARG(ctx, use_jit, "constraint_eval: a row range needs the specialised kernel");
  NB_ARG(ctx, !acc_high || use_jit, "constraint_eval: the high-degree accumulators need the specialised kernel");
  if (use_jit) {
    // NVRTC-specialised kernel (jit.cu): same arithmetic, registers instead of the shared-memory register file
    const u32** d_cols = nullptr;
    NB_CUDA(ctx, dmalloc(ctx, (void**)&d_cols, mask_cols.size() * sizeof(u32*)));
    NB_CUDA(ctx, cudaMemcpyAsync(d_cols, mask_cols.data(), mask_cols.size() * sizeof(u32*), cudaMemcpyHostToDevice, ctx->stream));
    std::vector<u32> tab;
    jit_coeff_table(coeffs, tab);
    u32* d_tab = nullptr;
    NB_CUDA(ctx, dmalloc(ctx, (void**)&d_tab, tab.size() * 4 + 16));
    NB_CUDA(ctx, cudaMemcpyAsync(d_tab, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    st = jit_launch_constraints(ctx, *jk, d_cols, d_params, d_tab, d_dinv, acc, rows_log, dom_log, row0, n_rows, acc_high);
    cudaStreamSynchronize(ctx->stream);
    dfree(ctx, (void*)d_cols); dfree(ctx, d_tab);
  } else {
    InterpArgs a{};
    a.prog = d_prog; a.n_instr = (u32)c.prog.size(); a.masks = d_masks; a.params = d_params;
    a.nb = c.n_base_regs; a.ne = c.n_ext_regs; a.log_size = c.log_size; a.eval_log = elog;
    a.coeff = d_coeff; a.dinv = d_dinv;
    for (int k = 0; k < 4; ++k) a.acc[k] = acc[k];
    st = launch_interp<false>(ctx, a, rows_log);
  }
  // host vectors were consumed by async copies: make sure they are done before the vectors die
  cudaStreamSynchronize(ctx->stream);
  dfree(ctx, d_prog); dfree(ctx, d_masks); dfree(ctx, d_coeff); dfree(ctx, d_dinv);
  return st;
}

nb200_status logup_finalize_last(nb200_ctx* ctx, u32 log_size, u32* last4, qm31* claimed);

// LogupTraceGenerator: fills 4 * n_logup_cols columns (bit-reversed circle-domain order) and returns the claimed sum.
// mask_cols[m]: device pointer of mask m's trace column on the trace domain (nullptr for masks the program never reads).
nb200_status logup_generate(nb200_ctx* ctx, const AirComponent& c, const std::vector<const u32*>& mask_cols, const u32* d_params,
                            u32* d_out, qm31* claimed, const JitKernel* jk) {
  const u32 ncols = c.n_logup_cols();
  *claimed = qm31_zero();
  if (ncols == 0) return NB200_OK;
  NB_ARG(ctx, mask_cols.size() == c.masks.size(), "logup_generate: shape");
  std::vector<MaskDev> hm(c.masks.size());
  for (size_t m = 0; m < hm.size(); ++m) { hm[m].ptr = (c.masks[m].off == 0 && c.masks[m].tree != 2) ? mask_cols[m] : nullptr; hm[m].off = 0; hm[m].pad = 0; }
  uint4* d_prog = nullptr; MaskDev* d_masks = nullptr; u32* d_batch = nullptr;
  NB_TRY(upload_prog(ctx, c.logup_prog, &d_prog));
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d_masks, hm.size() * sizeof(MaskDev)));
  NB_CUDA(ctx, cudaMemcpyAsync(d_masks, hm.data(), hm.size() * sizeof(MaskDev), cudaMemcpyHostToDevice, ctx->stream));
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d_batch, c.batching.size() * 4));
  NB_CUDA(ctx, cudaMemcpyAsync(d_batch, c.batching.data(), c.batching.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
  InterpArgs a{};
  a.prog = d_prog; a.n_instr = (u32)c.logup_prog.size(); a.masks = d_masks; a.params = d_params;
  a.nb = c.lg_base_regs; a.ne = c.lg_ext_regs; a.log_size = c.log_size; a.eval_log = c.log_size;
  a.batching = d_batch; a.out = d_out; a.n_batches = ncols;
  if (jk && jk->kernel && jk->log_size == c.log_size && ((size_t)1 << c.log_size) >= JIT_BLOCK) {
    // NVRTC-specialised kernel (jit.cu gen_logup_source): same arithmetic as the bytecode loop below
    std::vector<const u32*> ptrs(hm.size());
    for (size_t m = 0; m < hm.size(); ++m) ptrs[m] = hm[m].ptr;
    const u32** d_cols = nullptr;
    NB_CUDA(ctx, dmalloc(ctx, (void**)&d_cols, std::max<size_t>(ptrs.size(), 1) * sizeof(u32*)));
    NB_CUDA(ctx, cudaMemcpyAsync(d_cols, ptrs.data(), ptrs.size() * sizeof(u32*), cudaMemcpyHostToDevice, ctx->stream));
    nb200_status js = jit_launch_logup(ctx, *jk, d_cols, d_params, d_out, c.log_size);
    cudaStreamSynchronize(ctx->stream);
    dfree(ctx, (void*)d_cols);
    NB_TRY(js);
  } else {
    NB_TRY(launch_interp<true>(ctx, a, c.log_size));
  }
  dfree(ctx, d_prog); dfree(ctx, d_masks); dfree(ctx, d_batch);
  return logup_finalize_last(ctx, c.log_size, d_out + ((size_t)(4 * (ncols - 1)) << c.log_size), claimed);
}

// the row kernel alone on 2^rows_log rows (a rank's slice of the trace domain): out = 4 * n_logup_cols columns of 2^rows_log rows
nb200_status logup_rows(nb200_ctx* ctx, const AirComponent& c, const std::vector<const u32*>& mask_cols, const u32* d_params, u32* d_out, u32 rows_log, const JitKernel* jk) {
  NB_ARG(ctx, mask_cols.size() == c.masks.size() && jk && jk->kernel && jk->log_size == c.log_size, "logup_rows: needs the specialised kernel");
  std::vector<const u32*> ptrs(c.masks.size());
  for (size_t m = 0; m < ptrs.size(); ++m) ptrs[m] = (c.masks[m].off == 0 && c.masks[m].tree != 2) ? mask_cols[m] : nullptr;
  const u32** d_cols = nullptr;
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d_cols, std::max<size_t>(ptrs.size(), 1) * sizeof(u32*)));
  NB_CUDA(ctx, cudaMemcpyAsync(d_cols, ptrs.data(), ptrs.size() * sizeof(u32*), cudaMemcpyHostToDevice, ctx->stream));
  nb200_status js = jit_launch_logup(ctx, *jk, d_cols, d_params, d_out, rows_log);
  cudaStreamSynchronize(ctx->stream);
  dfree(ctx, (void*)d_cols);
  return js;
}

// finalize_last on the FULL last secure column (4 coordinate columns of 2^log_size rows): claimed sum, shift by claimed / 2^n, prefix sum in coset order
nb200_status logup_finalize_last(nb200_ctx* ctx, u32 log_size, u32* last, qm31* claimed) {
  const size_t n = (size_t)1 << log_size;
  const u32 sb = 64;
  u32* d_part = nullptr;
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d_part, 4 * sb * 4));
  sum_columns_kernel<<<dim3(sb, 4), 256, 0, ctx->stream>>>(last, log_size, d_part);
  NB_LAUNCH_CHECK(ctx);
  std::vector<u32> part(4 * sb);
  NB_CUDA(ctx, cudaMemcpyAsync(part.data(), d_part, part.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
  NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  qm31 cs = qm31_zero();
  for (int k = 0; k < 4; ++k) for (u32 b = 0; b < sb; ++b) cs.c[k] = m31_add(cs.c[k], part[k * sb + b]);
  *claimed = cs;
  qm31 shift = qm31_mul_m31(cs, m31_inv((u32)(n % P31)));
  u32* tmp = nullptr;
  NB_CUDA(ctx, dmalloc(ctx, (void**)&tmp, n * 4));
  u32 thr = 256, blk = (u32)((n + thr - 1) / thr);
  for (int k = 0; k < 4; ++k) {
    u32* col = last + ((size_t)k << log_size);
    coset_gather_shift_kernel<<<blk, thr, 0, ctx->stream>>>(col, log_size, shift.c[k], tmp);
    NB_LAUNCH_CHECK(ctx);
    NB_TRY(inclusive_scan(ctx, tmp, n));
    coset_scatter_kernel<<<blk, thr, 0, ctx->stream>>>(tmp, log_size, col);
    NB_LAUNCH_CHECK(ctx);
  }
  cudaStreamSynchronize(ctx->stream);
  dfree(ctx, tmp); dfree(ctx, d_part);
  return NB200_OK;
}

}  // namespace nb
