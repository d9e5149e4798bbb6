// em.cu -- Stage B: EM / VBEM over equivalence classes on H100 (sm_90a).
//
// Replaces CollapsedEMOptimizer::optimize (src/inference/CollapsedEMOptimizer.cpp:732-1035)
// and its update kernels EMUpdate_ (:178-234) / VBEMUpdate_ (:241-328).
//
// Design (DESIGN.md "Stage B"): the class<->transcript map is held twice in HBM,
// class-major and transcript-major, so that one iteration is two segmented
// reductions with NO atomics and a fixed summation order:
//   P1 (class-major):  denom_c = sum_i theta[t_i] * w_ci ;  scale_c = count_c / denom_c
//   P2 (txp-major):    alpha'_t = base_t + theta_t * sum_c w_ct * scale_c
//                      + convergence test + theta'_t (VBEM: exp(digamma(alpha'+prior) - logNorm))
// Both passes stream each warp's range of the SELL-32 entry arrays into shared
// memory with 1-D bulk (TMA) copies on an mbarrier ring and gather theta / scale
// from L2.  A persistent cooperative kernel runs the whole iteration loop with two
// grid barriers per iteration.  The per-phase kernels launch P1 and P2 (or P2's
// partial alpha') separately: variant 0 on one GPU, and the NCCL multi-GPU path,
// where an all-reduce sits between P2's partials and the update.
#include <cooperative_groups.h>
#include <cub/cub.cuh>
#include <float.h>
#include <math.h>
#include <stdarg.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "common.cuh"
#include "em_internal.h"

#include "em_kernels.cuh"

namespace sb {

// ---------------------------------------------------------------------------
// the iteration kernels: [0] = plain EM, [1] = VBEM (compile-time variants: the NaN guard exists in EM only, the
// digamma/exp epilogue in VBEM only).  Every one takes EM_SMEM bytes of dynamic shared memory.
// ---------------------------------------------------------------------------
static const void* const K_PERSISTENT[2] = {(const void*)k_em_persistent<false>, (const void*)k_em_persistent<true>};
static const void* const K_PERSISTENT_MGPU[2] = {(const void*)k_em_persistent_mgpu<false>,
                                                 (const void*)k_em_persistent_mgpu<true>};
static void (*const K_P1[2])(EmArgs) = {k_em_p1<false>, k_em_p1<true>};
static void (*const K_P2[2])(EmArgs, uint32_t) = {k_em_p2<false>, k_em_p2<true>};
static void (*const K_P2_PARTIAL[2])(EmArgs) = {k_em_p2_partial<false>, k_em_p2_partial<true>};

// ---------------------------------------------------------------------------
// prepare kernels
// ---------------------------------------------------------------------------

// CollapsedEMOptimizer.cpp:778-823 : per-transcript initialisation.
__global__ void k_txp_init(uint32_t M, const double* __restrict__ projected,
                           const double* __restrict__ eff_in,
                           const uint64_t* __restrict__ unique, sb_em_params p,
                           double totalWeight, double* __restrict__ effLens,
                           double* __restrict__ prior, double* __restrict__ alpha0) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  double el = p.no_length_correction ? 100.0 : eff_in[i];
  effLens[i] = el;
  prior[i] = p.per_txp_prior ? p.vb_prior : p.vb_prior * el;
  double uniqueCount = (double)unique[i] + 0.5;
  double wi = p.init_uniform ? 100.0 : (uniqueCount * 1e-3 * el);
  double a;
  if (p.init_uniform) {
    a = wi;
  } else {
    double uniformPrior = totalWeight / (double)M;
    double fracObserved = fmin(0.999, totalWeight / p.num_required_frags);
    double uniAbund = p.alt_init ? wi : uniformPrior;
    a = __dadd_rn(__dmul_rn(projected[i], fracObserved), __dmul_rn(uniAbund, (1.0 - fracObserved)));
  }
  alpha0[i] = a;
}

// :830-873 (and MappingPipelineStages.cpp:116-125): the combined weight of every entry of one class before the
// normalisation, written to cw[b, e); returns their sum
__device__ __forceinline__ double class_weights(uint64_t b, uint64_t e, double count, const uint32_t* __restrict__ tids,
                                                const double* __restrict__ aux, const double* __restrict__ effLens,
                                                int no_rich_eq, int eq_class_mode, double* __restrict__ cw) {
  double wsum = 0.0;
  for (uint64_t j = b; j < e; ++j) {
    double el = effLens[tids[j]];
    if (el <= 1.0) el = 1.0;
    double w = no_rich_eq ? 1.0 : aux[j];
    double probStartPos = 1.0 / el;
    double wt = eq_class_mode ? w : __dmul_rn(__dmul_rn(count, w), probStartPos);
    cw[j] = wt;
    wsum = __dadd_rn(wsum, wt);
  }
  return wsum;
}

// :830-873 combined weights, :330-394 degenerate marking, singleton folding.
// One thread per class (one-time work).  sortkey = first transcript of a kept class.
__global__ void k_class_combine(uint64_t C, uint32_t M, const uint64_t* __restrict__ off,
                                const uint32_t* __restrict__ tids,
                                const double* __restrict__ aux,
                                const uint64_t* __restrict__ counts,
                                const double* __restrict__ effLens,
                                const double* __restrict__ alpha0, sb_em_params p,
                                double* __restrict__ cw, uint64_t* __restrict__ packed,
                                uint32_t* __restrict__ sortkey, uint32_t* __restrict__ cls_map,
                                double* __restrict__ single, uint8_t* __restrict__ valid,
                                unsigned long long* __restrict__ n_degenerate) {
  uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const uint64_t b = off[c], e = off[c + 1];
  const double count = (double)counts[c];
  const double wsum = class_weights(b, e, count, tids, aux, effLens, p.no_rich_eq, p.eq_class_mode, cw);
  const double wnorm = 1.0 / wsum;
  double denom = 0.0;
  for (uint64_t j = b; j < e; ++j) {
    double v = __dmul_rn(cw[j], wnorm);
    cw[j] = v;
    double d = __dmul_rn(alpha0[tids[j]], v);
    if (!isnan(d)) denom = __dadd_rn(denom, d);
  }
  const bool ok = !(denom <= MIN_EQ_W);
  valid[c] = ok ? 1 : 0;
  uint64_t len = e - b;
  uint64_t pk = 0;
  uint32_t key = M;  // dropped classes sort last
  uint32_t cmap = 0xffffffffu;  // class -> accumulator (samplers): 0x80000000|tid for singletons
  if (!ok) {
    atomicAdd(n_degenerate, 1ull);
  } else if (len == 1) {
    atomicAdd(&single[tids[b]], count);  // integer-valued: order independent
    cmap = 0x80000000u | tids[b];
  } else if (len > 1) {
    pk = (1ull << 32) | len;             // (class count, entry count)
    key = tids[b];
  }
  packed[c] = pk;
  sortkey[c] = key;
  cls_map[c] = cmap;
}

// --skipQuant --dumpEqWeights (MappingPipelineStages.cpp:112-162): the combined weights alone, normalised per class
__global__ void k_eq_combined(uint64_t C, const uint64_t* __restrict__ off, const uint32_t* __restrict__ tids,
                              const double* __restrict__ aux, const uint64_t* __restrict__ counts,
                              const double* __restrict__ effLens, int no_rich_eq, double* __restrict__ cw) {
  uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const uint64_t b = off[c], e = off[c + 1];
  const double wnorm = 1.0 / class_weights(b, e, (double)counts[c], tids, aux, effLens, no_rich_eq, 0, cw);
  for (uint64_t j = b; j < e; ++j) cw[j] = __dmul_rn(cw[j], wnorm);
}

// second-level key: (locality group, length bucket); dropped rows last
__global__ void k_bucket_key(uint64_t n, const uint32_t* __restrict__ order,
                             const uint64_t* __restrict__ packed, uint32_t group,
                             uint32_t* __restrict__ key, uint32_t* __restrict__ val) {
  uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const uint64_t pk = packed[order ? order[p] : p];
  const uint32_t len = (uint32_t)(pk & 0xffffffffu);
  key[p] = pk ? ((uint32_t)(p / group) << 9) | min(len, 511u) : 0xffffffffu;
  val[p] = order ? order[p] : (uint32_t)p;
}

__global__ void k_gather_u64(uint64_t n, const uint32_t* __restrict__ order,
                             const uint64_t* __restrict__ src, uint64_t* __restrict__ dst) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[order[i]];
}

// Compact the kept classes in their final order; histogram of transcript occurrences.
__global__ void k_compact(uint64_t C, const uint32_t* __restrict__ order,
                          const uint64_t* __restrict__ off,
                          const uint32_t* __restrict__ tids, const double* __restrict__ cw,
                          const uint64_t* __restrict__ counts,
                          const uint64_t* __restrict__ packed_sorted,
                          const uint64_t* __restrict__ packed_scan,
                          uint32_t* __restrict__ m_off, uint32_t* __restrict__ m_idx,
                          double* __restrict__ m_w, double* __restrict__ m_cnt,
                          uint32_t* __restrict__ ent_cls, uint32_t* __restrict__ tcnt,
                          uint32_t* __restrict__ cls_map) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C) return;
  if (packed_sorted[i] == 0) return;
  const uint64_t c = order[i];
  const uint64_t s = packed_scan[i];
  const uint32_t cid = (uint32_t)(s >> 32);
  uint32_t o = (uint32_t)(s & 0xffffffffu);
  m_off[cid] = o;
  m_cnt[cid] = (double)counts[c];
  cls_map[c] = cid;
  for (uint64_t j = off[c]; j < off[c + 1]; ++j, ++o) {
    uint32_t t = tids[j];
    m_idx[o] = t;
    m_w[o] = cw[j];
    ent_cls[o] = cid;
    atomicAdd(&tcnt[t], 1u);
  }
}

__global__ void k_iota(uint32_t n, uint32_t* __restrict__ v) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) v[i] = i;
}

// per transcript: packed (active flag, occurrence count) for the rank scan
__global__ void k_row_pack(uint32_t M, const uint32_t* __restrict__ tcnt,
                           uint64_t* __restrict__ packed) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < M) packed[i] = tcnt[i] ? ((1ull << 32) | tcnt[i]) : 0ull;
}
// rank space (active transcripts in ascending id): CSR offsets + id of each rank
__global__ void k_rank_fill(uint32_t M, const uint32_t* __restrict__ tcnt,
                            const uint64_t* __restrict__ scan, uint32_t* __restrict__ t_off,
                            uint32_t* __restrict__ rank_tid, uint64_t* __restrict__ rank_packed) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  if (tcnt[i]) {
    uint32_t rk = (uint32_t)(scan[i] >> 32);
    t_off[rk] = (uint32_t)(scan[i] & 0xffffffffu);
    rank_tid[rk] = i;
    rank_packed[rk] = (1ull << 32) | tcnt[i];
  }
}
// final rows: row r holds rank rowperm[r]; state vectors gathered into row space
__global__ void k_row_fill(uint32_t R, const uint32_t* __restrict__ rowperm,
                           const uint32_t* __restrict__ rank_tid, const double* __restrict__ prior,
                           const double* __restrict__ base, const double* __restrict__ alpha0,
                           uint32_t* __restrict__ row_tid, uint32_t* __restrict__ tid_row,
                           double* __restrict__ r_prior, double* __restrict__ r_base,
                           double* __restrict__ r_alpha0) {
  uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const uint32_t t = rank_tid[rowperm[r]];
  row_tid[r] = t;
  tid_row[t] = r;
  r_prior[r] = prior[t];
  r_base[r] = base[t];
  r_alpha0[r] = alpha0[t];
}
// transcript-major CSR (rank order) from the stable sort permutation
__global__ void k_gather_csc(uint32_t nnz, const uint32_t* __restrict__ perm,
                             const uint32_t* __restrict__ ent_cls,
                             const double* __restrict__ m_w, uint32_t* __restrict__ t_idx,
                             double* __restrict__ t_w) {
  uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nnz) return;
  uint32_t j = perm[k];
  t_idx[k] = ent_cls[j];
  t_w[k] = m_w[j];
}
__global__ void k_remap(uint32_t n, const uint32_t* __restrict__ src,
                        const uint32_t* __restrict__ map, uint32_t* __restrict__ dst) {
  uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) dst[k] = map[src[k]];
}

// ---- CSR -> SELL-32 -------------------------------------------------------------
// one warp per slice: row lengths, slice width (= max non-long length, exact), base index (= smallest gather index of
// its SELL rows).  A slice whose indices do not fit 16 bits relative to the base (IDX_PAD is reserved) sends its rows
// to the long-row path (counts: [0] long rows, [2] of which fallback rows).
__global__ void k_sell_widths(uint32_t n_rows, uint32_t n_slices, const uint32_t* __restrict__ rowperm,
                              const uint32_t* __restrict__ csr_off, const uint32_t* __restrict__ csr_idx,
                              uint16_t* __restrict__ len16, uint32_t* __restrict__ width,
                              uint32_t* __restrict__ sbase, uint32_t* __restrict__ counts) {
  const uint32_t s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (s >= n_slices) return;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t row = s * 32 + lane;
  uint32_t len = 0, lo = 0xffffffffu, hi = 0;   // len: of a SELL row (0: long or absent)
  bool sell = false;
  if (row < n_rows) {
    const uint32_t cr = rowperm ? rowperm[row] : row;
    const uint32_t b = csr_off[cr];
    len = csr_off[cr + 1] - b;
    sell = len <= LMAX;
    if (!sell) {
      len16[row] = LEN_LONG;
      atomicAdd(&counts[0], 1u);
      len = 0;
    }
    for (uint32_t j = 0; j < len; ++j) {
      lo = min(lo, csr_idx[b + j]);
      hi = max(hi, csr_idx[b + j]);
    }
  }
  uint32_t width_s = len;
  for (int o = 16; o > 0; o >>= 1) {
    width_s = max(width_s, __shfl_xor_sync(0xffffffffu, width_s, o));
    lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  const bool fallback = hi >= lo && hi - lo >= (uint32_t)IDX_PAD;
  if (sell) {
    len16[row] = fallback ? LEN_LONG : (uint16_t)len;
    if (fallback) {
      atomicAdd(&counts[0], 1u);
      atomicAdd(&counts[2], 1u);
    }
  }
  if (lane == 0) {
    width[s] = fallback ? 0u : width_s;
    sbase[s] = hi >= lo ? lo : 0u;
  }
}
__global__ void k_sell_fill(uint32_t n_rows, uint32_t n_slices, const uint32_t* __restrict__ rowperm,
                            const uint32_t* __restrict__ csr_off, const uint32_t* __restrict__ csr_idx,
                            const double* __restrict__ csr_w, const uint32_t* __restrict__ slice_ptr,
                            const uint32_t* __restrict__ sbase, const uint16_t* __restrict__ len16,
                            uint16_t* __restrict__ s_idx, double* __restrict__ s_w,
                            uint32_t* __restrict__ long_rows, uint32_t* __restrict__ long_cursor) {
  const uint32_t s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (s >= n_slices) return;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t row = s * 32 + lane;
  // entry j of lane l: in the groups of 4 (j < width & ~3) at (first column * 32) + (j / 4) * 128 + l * 4 + (j % 4),
  // in the remainder columns at (first column + j) * 32 + l (em_kernels.cuh: run_phase)
  const size_t first = (size_t)slice_ptr[s] * 32;
  const uint32_t width = slice_ptr[s + 1] - slice_ptr[s];
  const uint32_t grouped = width & ~3u;
  auto pos = [&](uint32_t j) {
    return j < grouped ? first + (size_t)(j >> 2) * 128 + lane * 4 + (j & 3u) : first + (size_t)j * 32 + lane;
  };
  const uint32_t base = sbase[s];
  uint32_t n = 0;
  if (row < n_rows) {
    const uint32_t cr = rowperm ? rowperm[row] : row;
    const uint32_t b = csr_off[cr], e = csr_off[cr + 1];
    if (len16[row] == LEN_LONG) {
      const uint32_t pos = atomicAdd(long_cursor, 1u);
      long_rows[3 * pos] = row;
      long_rows[3 * pos + 1] = b;
      long_rows[3 * pos + 2] = e;
    } else {
      n = e - b;
      for (uint32_t j = 0; j < n; ++j) {
        s_idx[pos(j)] = (uint16_t)(csr_idx[b + j] - base);
        s_w[pos(j)] = csr_w[b + j];
      }
    }
  }
  // padding: weight 0 and the index that gathers the zero slot
  for (uint32_t j = n; j < width; ++j) {
    s_idx[pos(j)] = IDX_PAD;
    s_w[pos(j)] = 0.0;
  }
}
// contiguous, work-balanced slice ranges per warp: work(slice) = width + overhead
__global__ void k_warp_ranges(uint32_t n_slices, const uint32_t* __restrict__ slice_ptr,
                              uint32_t overhead, uint32_t n_warps, uint32_t* __restrict__ warp_begin) {
  const uint32_t wid = blockIdx.x * blockDim.x + threadIdx.x;
  if (wid > n_warps) return;
  if (wid == n_warps || n_slices == 0) { warp_begin[wid] = n_slices; return; }
  const uint64_t total = (uint64_t)slice_ptr[n_slices] + (uint64_t)overhead * n_slices;
  const uint64_t target = total * wid / n_warps;
  uint32_t lo = 0, hi = n_slices;  // first slice whose cumulative work (before it) >= target
  while (lo < hi) {
    uint32_t mid = (lo + hi) >> 1;
    uint64_t wk = (uint64_t)slice_ptr[mid] + (uint64_t)overhead * mid;
    if (wk >= target) hi = mid; else lo = mid + 1;
  }
  warp_begin[wid] = lo;
}

// deterministic single-block reduction: out[0] = sum_i f(i)
// mode 0: a[i]+b[i] over all i ; mode 1: a[i]+b[i] over inactive i
__global__ void k_sum1(uint32_t M, const double* __restrict__ a, const double* __restrict__ b,
                       const uint32_t* __restrict__ tid_row, int mode, double* __restrict__ out) {
  __shared__ double scratch[32];
  double acc = 0.0;
  for (uint32_t i = threadIdx.x; i < M; i += blockDim.x) {
    if (mode == 1 && tid_row[i] != 0xffffffffu) continue;
    acc += a[i] + b[i];
  }
  acc = block_reduce<false>(acc, scratch);
  if (threadIdx.x == 0) out[0] = acc;
}

// iteration-0 state (exact logNorm), in whatever index space the caller iterates in
__global__ void k_theta0(uint32_t n, int vbem, const double* __restrict__ alpha0,
                         const double* __restrict__ prior, const double* __restrict__ sum0,
                         double* __restrict__ alpha, double* __restrict__ theta) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double a = alpha0[i];
  alpha[i] = a;
  if (vbem) {
    double logNorm = digamma_pos(sum0[0]);
    double ap = a + prior[i];
    theta[i] = theta_of<true>(a, ap, logNorm);
  } else {
    theta[i] = a;
  }
}

// row space -> transcript space.  Inactive transcripts (in no kept multi-transcript
// class) hold base (+1.0 after exactly one EM iteration: alphasPrime starts at 1.0).
__global__ void k_finalize(uint32_t M, const uint32_t* __restrict__ tid_row,
                           const double* __restrict__ base, double bias,
                           const double* __restrict__ r_alpha, double* __restrict__ alpha) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  uint32_t r = tid_row[i];
  alpha[i] = (r == 0xffffffffu) ? base[i] + bias : r_alpha[r];
}

__global__ void k_reset_maxrel(unsigned long long* maxrel, uint32_t par) { maxrel[par] = 0ull; }

// multi-GPU: per-transcript update over ALL transcripts from the all-reduced alpha'.
// Every rank computes the same values, so every rank takes the same decisions.
template <bool VBEM>
__global__ void __launch_bounds__(256)
k_em_update(const __grid_constant__ EmArgs A, const double* __restrict__ red, uint32_t M,
            uint32_t it) {
  __shared__ double scratch[32];
  const uint32_t par = it & 1u;
  double logNorm = 0.0;
  if (VBEM) {
    if (it == 0) logNorm = digamma_pos(A.sum0);
    else logNorm = digamma_pos(sum_partials(A.sum_partial + (size_t)(par ^ 1u) * gridDim.x,
                                                 gridDim.x, 0.0, scratch));
  }
  const double bias = (it == 0) ? A.first_bias : 0.0;
  double sum = 0.0, mx = 0.0;
  for (uint32_t t = blockIdx.x * 256 + threadIdx.x; t < M; t += gridDim.x * 256) {
    const double na = red[t] + bias;
    const double old = A.alpha[t];
    if (na > ALPHA_CHECK_CUTOFF) mx = fmax(mx, fabs(old - na) / na);
    A.alpha[t] = na;
    const double ap = na + A.prior[t];
    sum += ap;
    A.theta[t] = theta_of<VBEM>(na, ap, logNorm);
  }
  double bs = block_reduce<false>(sum, scratch);
  double bm = block_reduce<true>(mx, scratch);
  if (threadIdx.x == 0) {
    A.sum_partial[(size_t)par * gridDim.x + blockIdx.x] = bs;
    if (bm > 0.0) atomicMax(&A.maxrel[par], (unsigned long long)__double_as_longlong(bm));
  }
}

}  // namespace sb

// ===========================================================================
// host side
// ===========================================================================
using namespace sb;

namespace sb {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace sb

extern "C" const char* sb_last_error(void) { return sb::g_err; }
extern "C" int sb_version(void) { return 100; }
extern "C" int sb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

extern "C" void sb_em_default_params(sb_em_params* p) {
  memset(p, 0, sizeof(*p));
  p->use_vbem = 1;        // SalmonDefaults.hpp useVBOpt
  p->per_txp_prior = 1;   // perTranscriptPrior
  p->vb_prior = 1e-2;
  p->tol = 0.01;
  p->num_required_frags = 5e7;
  p->min_iter = 100;
  p->max_iter = 10000;
}

extern "C" sb_em_ctx* sb_em_create(int device) {
  int n = sb_device_count();
  if (n <= 0) {
    set_error("no CUDA device available (libsalmon_b200 has no CPU fallback)");
    return nullptr;
  }
  if (device < 0 || device >= n) {
    set_error("device %d out of range (0..%d)", device, n - 1);
    return nullptr;
  }
  if (cudaSetDevice(device) != cudaSuccess) {
    set_error("cannot initialise device %d: %s", device, cudaGetErrorString(cudaGetLastError()));
    return nullptr;
  }
  sb_em_ctx* c = new sb_em_ctx(device);
  int rc = c->res.stream(&c->stream, cudaStreamNonBlocking);
  for (int i = 0; i < 4 && rc == SB_OK; ++i) rc = c->res.event(&c->ev[i], cudaEventDefault);
  if (rc != SB_OK) { delete c; return nullptr; }
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, device);
  c->n_sm = prop.multiProcessorCount;
  c->l2_bytes = (size_t)prop.l2CacheSize;
  // development overrides of the tuning defaults (sweeps over the test-suite)
  if (const char* e = getenv("SB_EM_GROUP_CM")) { const int v = atoi(e); if (v >= 32 && !(v & (v - 1))) c->sell_group_cm = v; }
  if (const char* e = getenv("SB_EM_GROUP_TM")) { const int v = atoi(e); if (v >= 32 && !(v & (v - 1))) c->sell_group_tm = v; }
  return c;
}

extern "C" void sb_em_destroy(sb_em_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  for (void* p : c->x_opened) cudaIpcCloseMemHandle(p);
  sb_em_comm_destroy(c);
  delete c;
}

extern "C" int sb_em_set_option(sb_em_ctx* c, const char* key, int64_t value) {
  if (!c || !key) { set_error("null argument"); return SB_ERR_INVALID; }
  if (!strcmp(key, "variant")) c->variant = (int)value;
  else if (!strcmp(key, "blocks_per_sm")) { c->blocks_per_sm = (int)value; c->prepared = false; }
  else if (!strcmp(key, "sell_group_cm") || !strcmp(key, "sell_group_tm")) {
    if (value < 32 || value > (1 << 20) || (value & (value - 1))) { set_error("sell_group must be a power of two >= 32"); return SB_ERR_INVALID; }
    (key[11] == 'c' ? c->sell_group_cm : c->sell_group_tm) = (int)value; c->prepared = false;
  }
  else if (!strcmp(key, "push_pass")) { c->push_pass = (int)value; }
  else if (!strcmp(key, "sample_offset")) { c->sample_offset = (uint32_t)value; }
  else if (!strcmp(key, "rebalance")) { c->rebalance = (int)value; c->prepared = false; }
  else { set_error("unknown option '%s'", key); return SB_ERR_INVALID; }
  return SB_OK;
}

// Figures of the prepared layout (per matrix: suffix _cm = class-major, _tm = transcript-major).
extern "C" int sb_em_get_info(sb_em_ctx* c, const char* key, int64_t* value) {
  if (!c || !key || !value) { set_error("null argument"); return SB_ERR_INVALID; }
  if (!c->prepared) { set_error("sb_em_get_info before sb_em_prepare"); return SB_ERR_STATE; }
  // bytes one iteration streams: SELL entries (2-byte index + 8-byte weight) and the long rows' CSR (4 + 8 bytes)
  auto stream = [](const SellDev& m) { return (int64_t)m.n_cols * 32 * 10 + (int64_t)m.long_entries * 12; };
  if (!strcmp(key, "stream_bytes")) { *value = stream(c->cm) + stream(c->tm); return SB_OK; }
  // warps of the grid the slice ranges were cut for, and the columns one warp's ring holds
  if (!strcmp(key, "warps")) { *value = (int64_t)c->grid * (EM_THREADS / 32); return SB_OK; }
  if (!strcmp(key, "ring_cols")) { *value = (int64_t)EM_CH * EM_RING; return SB_OK; }
  // s of the fixed-point sum of (alpha' + prior): units of 2^-s, 20 unless the counts and priors are large
  if (!strcmp(key, "sum_scale_log2")) { *value = c->sum_scale_log2; return SB_OK; }
  const size_t n = strlen(key);
  const SellDev* m = nullptr;
  if (n > 3 && !strcmp(key + n - 3, "_cm")) m = &c->cm;
  else if (n > 3 && !strcmp(key + n - 3, "_tm")) m = &c->tm;
  const std::string k(key, m ? n - 3 : n);
  if (m && k == "stream_bytes") *value = stream(*m);
  else if (m && k == "sell_cols") *value = m->n_cols;
  else if (m && k == "long_rows") *value = m->n_long;
  else if (m && k == "long_entries") *value = (int64_t)m->long_entries;
  else if (m && k == "fallback_rows") *value = m->n_fallback;
  else { set_error("unknown info key '%s'", key); return SB_ERR_INVALID; }
  return SB_OK;
}

extern "C" int sb_em_upload(sb_em_ctx* c, const sb_eq_csr* eq, const double* projected,
                            const double* eff_len, const uint64_t* unique) {
  if (!c || !eq || !projected || !eff_len || !unique) { set_error("null argument"); return SB_ERR_INVALID; }
  if (eq->n_classes && (!eq->off || !eq->counts)) { set_error("null CSR arrays"); return SB_ERR_INVALID; }
  SB_CUDA(cudaSetDevice(c->device));
  const uint64_t C = eq->n_classes;
  const uint32_t M = eq->n_txps;
  const uint64_t nnz = C ? eq->off[C] : 0;
  if (M == 0) { set_error("no transcripts"); return SB_ERR_INVALID; }
  if (nnz >= 0xfffffff0ull || C >= 0xfffffff0ull) {
    set_error("eq-class table too large for 32-bit device offsets (nnz=%llu)", (unsigned long long)nnz);
    return SB_ERR_INVALID;
  }
  if (nnz && (!eq->tids || !eq->weights)) { set_error("null CSR arrays"); return SB_ERR_INVALID; }
  c->C = C; c->M = M; c->nnz = nnz;
  c->prepared = false;
  SB_TRY(c->res.grow(&c->d_off, C + 1));
  SB_TRY(c->res.grow(&c->d_tids, nnz));
  SB_TRY(c->res.grow(&c->d_aux, nnz));
  SB_TRY(c->res.grow(&c->d_counts, C));
  SB_TRY(c->res.grow(&c->d_projected, M));
  SB_TRY(c->res.grow(&c->d_eff_in, M));
  SB_TRY(c->res.grow(&c->d_unique, M));
  cudaStream_t st = c->stream;
  if (C) {
    SB_CUDA(cudaMemcpyAsync(c->d_off, eq->off, (C + 1) * 8, cudaMemcpyHostToDevice, st));
    SB_CUDA(cudaMemcpyAsync(c->d_counts, eq->counts, C * 8, cudaMemcpyHostToDevice, st));
  } else {
    uint64_t z = 0;
    SB_CUDA(cudaMemcpyAsync(c->d_off, &z, 8, cudaMemcpyHostToDevice, st));
  }
  if (nnz) {
    SB_CUDA(cudaMemcpyAsync(c->d_tids, eq->tids, nnz * 4, cudaMemcpyHostToDevice, st));
    SB_CUDA(cudaMemcpyAsync(c->d_aux, eq->weights, nnz * 8, cudaMemcpyHostToDevice, st));
  }
  SB_CUDA(cudaMemcpyAsync(c->d_projected, projected, (size_t)M * 8, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(c->d_eff_in, eff_len, (size_t)M * 8, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(c->d_unique, unique, (size_t)M * 8, cudaMemcpyHostToDevice, st));
  // serial host sum, same order as the reference (:778-781)
  double tw = 0.0;
  for (uint32_t i = 0; i < M; ++i) tw += projected[i];
  c->total_weight = tw;
  // inputs of the bound on sum(alpha' + prior) that sb_em_prepare scales the fixed-point sum by
  double cs = 0.0, es = 0.0;
  for (uint64_t k = 0; k < C; ++k) cs += (double)eq->counts[k];
  for (uint32_t i = 0; i < M; ++i) es += fabs(eff_len[i]);
  c->count_sum = cs;
  c->eff_abs_sum = es;
  c->h2d_bytes = (C + 1) * 8 + C * 8 + nnz * 12 + (size_t)M * 24;
  SB_CUDA(cudaStreamSynchronize(st));
  c->uploaded = true;
  return SB_OK;
}

static inline unsigned nblk(uint64_t n, unsigned t) { return (unsigned)((n + t - 1) / t); }

static int bits_for(uint64_t n) {  // bits needed to represent values 0..n
  int b = 1;
  while (b < 32 && (1ull << b) <= n) ++b;
  return b;
}

// stable sort of (key,val) u32 pairs through the context's scratch buffers;
// result in d_sort_keys2 / d_sort_vals2
static int sort_pairs(sb_em_ctx* c, uint32_t n, int end_bit) {
  size_t tb = c->tmp_bytes;
  SB_CUDA(cub::DeviceRadixSort::SortPairs(c->d_tmp, tb, c->d_sort_keys, c->d_sort_keys2,
                                          c->d_sort_vals, c->d_sort_vals2, (int)n, 0, end_bit,
                                          c->stream));
  c->launches += 1 + 2 * ((end_bit + 7) / 8);
  return SB_OK;
}
static int scan_u64(sb_em_ctx* c, const uint64_t* in, uint64_t* out, uint64_t n) {
  size_t tb = c->tmp_bytes;
  SB_CUDA(cub::DeviceScan::ExclusiveSum(c->d_tmp, tb, in, out, (int)n, c->stream));
  c->launches += 2;
  return SB_OK;
}

// epilogue overhead of a slice in columns, for cutting the warp ranges: P1 (and plain EM's P2), VBEM's P2
constexpr uint32_t OVERHEAD_P1 = 3, OVERHEAD_P2 = 12;
static uint32_t overhead_tm(const sb_em_ctx* c) { return c->params.use_vbem ? OVERHEAD_P2 : OVERHEAD_P1; }

// modelled cost of a slice in columns: its width plus the epilogue overhead (slices of long rows only cost nothing)
static double slice_cost(const std::vector<uint32_t>& sp, uint32_t s, uint32_t overhead) {
  return (double)(sp[s + 1] - sp[s]) + (sp[s + 1] > sp[s] ? (double)overhead : 0.0);
}

// CSR (rows optionally permuted by rowperm) -> SELL-32 + long-row list + warp ranges
static int build_sell(sb_em_ctx* c, SellDev& m, uint32_t n_rows, const uint32_t* rowperm,
                      const uint32_t* csr_off, const uint32_t* csr_idx, const double* csr_w,
                      uint32_t pad_idx, uint32_t overhead, uint32_t n_warps) {
  cudaStream_t st = c->stream;
  m.n_rows = n_rows;
  m.n_slices = (n_rows + 31) / 32;
  m.csr_idx = csr_idx;
  m.csr_w = csr_w;
  m.zero = pad_idx;
  SB_TRY(c->res.grow(&m.len, (size_t)n_rows));
  SB_TRY(c->res.grow(&m.width, (size_t)m.n_slices + 1));
  SB_TRY(c->res.grow(&m.slice_ptr, (size_t)m.n_slices + 1));
  SB_TRY(c->res.grow(&m.base, (size_t)m.n_slices + 1));
  SB_TRY(c->res.grow(&m.warp_begin, (size_t)n_warps + 1));
  uint32_t* d_nlong = (uint32_t*)(c->d_scalars + 8);   // [0] long rows, [1] fill cursor, [2] fallback rows
  SB_CUDA(cudaMemsetAsync(d_nlong, 0, 16, st));
  SB_CUDA(cudaMemsetAsync(m.width, 0, ((size_t)m.n_slices + 1) * 4, st));
  if (m.n_slices) {
    k_sell_widths<<<nblk(m.n_slices, 8), 256, 0, st>>>(n_rows, m.n_slices, rowperm, csr_off, csr_idx, m.len, m.width,
                                                       m.base, d_nlong);
    c->launches++;
  }
  {
    size_t tb = c->tmp_bytes;
    SB_CUDA(cub::DeviceScan::ExclusiveSum(c->d_tmp, tb, m.width, m.slice_ptr, (int)(m.n_slices + 1), st));
    c->launches += 2;
  }
  uint32_t ncols = 0;
  SB_CUDA(cudaMemcpyAsync(&ncols, m.slice_ptr + m.n_slices, 4, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(&m.n_long, d_nlong, 4, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(&m.n_fallback, d_nlong + 2, 4, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  m.n_cols = ncols;
  SB_TRY(c->res.grow(&m.idx, (size_t)ncols * 32 + 32));
  SB_TRY(c->res.grow(&m.w, (size_t)ncols * 32 + 32));
  SB_TRY(c->res.grow(&m.long_rows, (size_t)3 * m.n_long + 3));
  SB_CUDA(cudaMemsetAsync(m.idx, 0xff, ((size_t)ncols * 32 + 32) * 2, st));
  SB_CUDA(cudaMemsetAsync(m.w, 0, ((size_t)ncols * 32 + 32) * 8, st));
  if (m.n_slices) {
    k_sell_fill<<<nblk(m.n_slices, 8), 256, 0, st>>>(n_rows, m.n_slices, rowperm, csr_off, csr_idx,
                                                     csr_w, m.slice_ptr, m.base, m.len, m.idx,
                                                     m.w, m.long_rows, d_nlong + 1);
    c->launches++;
  }
  m.n_block = 0;
  m.long_entries = 0;
  if (m.n_long > 0) {
    // every long row is reduced independently with a fixed tree, so the list order does
    // not affect results.  Longest first: the first n_block rows (> LWARP entries) take
    // the block path, the rest are dealt round-robin to warps (longest-processing-time).
    std::vector<uint32_t> h((size_t)3 * m.n_long);
    SB_CUDA(cudaMemcpyAsync(h.data(), m.long_rows, h.size() * 4, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    std::vector<uint32_t> ord(m.n_long);
    for (uint32_t i = 0; i < m.n_long; ++i) ord[i] = i;
    std::sort(ord.begin(), ord.end(), [&](uint32_t x, uint32_t y) {
      const uint32_t lx = h[3 * x + 2] - h[3 * x + 1], ly = h[3 * y + 2] - h[3 * y + 1];
      return lx != ly ? lx > ly : h[3 * x] < h[3 * y];
    });
    for (uint32_t i = 0; i < m.n_long; ++i) {
      if (h[3 * ord[i] + 2] - h[3 * ord[i] + 1] > LWARP) m.n_block = i + 1;
      m.long_entries += h[3 * i + 2] - h[3 * i + 1];
    }
    std::vector<uint32_t> h2(h.size());
    for (uint32_t i = 0; i < m.n_long; ++i)
      for (int k = 0; k < 3; ++k) h2[3 * i + k] = h[3 * ord[i] + k];
    SB_CUDA(cudaMemcpyAsync(m.long_rows, h2.data(), h2.size() * 4, cudaMemcpyHostToDevice, st));
    SB_CUDA(cudaStreamSynchronize(st));
  }
  k_warp_ranges<<<nblk(n_warps + 1, 256), 256, 0, st>>>(m.n_slices, m.slice_ptr, overhead, n_warps, m.warp_begin);
  c->launches++;
  return SB_OK;
}

static int em_rebalance(sb_em_ctx* c);

extern "C" int sb_em_prepare(sb_em_ctx* c, const sb_em_params* p, sb_em_stats* stats) {
  if (!c || !p) { set_error("null argument"); return SB_ERR_INVALID; }
  if (!c->uploaded) { set_error("sb_em_prepare before sb_em_upload"); return SB_ERR_STATE; }
  if (!(p->vb_prior >= 0.0) || !std::isfinite(p->vb_prior)) {
    set_error("the VB prior (--vbPrior) must be a finite number >= 0, not %g", p->vb_prior);
    return SB_ERR_INVALID;
  }
  // Unit of P2's fixed-point sum of (alpha' + prior) over the active rows (em_kernels.cuh: P2Acc).  An iteration's
  // alpha' add up to the counts of the classes it keeps, plus 1.0 per transcript in the first plain-EM iteration; the
  // priors add vb_prior per transcript or per unit of effective length.  Twice that bound B leaves room for rounding,
  // and the largest s <= 20 with 2B * 2^s < 2^62 keeps every row's term and the grid's total inside 64 bits.
  {
    const double prior_sum = p->per_txp_prior ? p->vb_prior * (double)c->M
                                              : p->vb_prior * (p->no_length_correction ? 100.0 * (double)c->M : c->eff_abs_sum);
    const double bound = 2.0 * (c->count_sum + (double)c->M + prior_sum);
    if (!std::isfinite(bound)) {
      set_error("the class counts and priors sum to %g, which the EM cannot represent", bound);
      return SB_ERR_INVALID;
    }
    int e2 = 0;
    frexp(bound, &e2);   // bound < 2^e2
    c->sum_scale_log2 = std::min(20, 62 - e2);
  }
  SB_CUDA(cudaSetDevice(c->device));
  cudaStream_t st = c->stream;
  c->params = *p;
  c->launches = 0;
  const uint64_t C = c->C;
  const uint32_t M = c->M;
  const uint64_t nnz = c->nnz;
  const bool row_space = c->nranks <= 1 && !c->fused_loopback;
  SB_CUDA(cudaEventRecord(c->ev[0], st));

  // launch geometry first: the slice ranges are cut for this grid
  int occ = 0;
  for (int v = 0; v < 2; ++v) {
    SB_CUDA(cudaFuncSetAttribute(K_PERSISTENT[v], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)EM_SMEM));
    SB_CUDA(cudaFuncSetAttribute((const void*)K_P1[v], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)EM_SMEM));
    SB_CUDA(cudaFuncSetAttribute((const void*)K_P2[v], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)EM_SMEM));
    SB_CUDA(cudaFuncSetAttribute((const void*)K_P2_PARTIAL[v], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)EM_SMEM));
    SB_CUDA(cudaFuncSetAttribute(K_PERSISTENT_MGPU[v], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)EM_SMEM));
  }
  const int vb = p->use_vbem ? 1 : 0;
  SB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, (c->nranks > 1 || c->fused_loopback) ? K_PERSISTENT_MGPU[vb] : K_PERSISTENT[vb],
                                                        EM_THREADS, EM_SMEM));
  if (occ < 1) { set_error("persistent EM kernel does not fit on an SM"); return SB_ERR_CUDA; }
  if (c->blocks_per_sm > 0) occ = std::min(occ, c->blocks_per_sm);
  c->grid = (uint32_t)(occ * c->n_sm);
  c->occ = occ;
  const uint32_t n_warps = c->grid * (EM_THREADS / 32);

  const uint64_t NP = std::max<uint64_t>(C, M) + 1;
  const uint64_t NS = std::max<uint64_t>(std::max<uint64_t>(C, nnz), (uint64_t)M) + 1;
  SB_TRY(c->res.grow(&c->d_efflens, M));
  SB_TRY(c->res.grow(&c->d_prior, M));
  SB_TRY(c->res.grow(&c->d_alpha0, M));
  SB_TRY(c->res.grow(&c->d_alpha, M));
  SB_TRY(c->res.grow(&c->d_theta, (size_t)M + 4));
  SB_CUDA(cudaMemsetAsync(c->d_theta, 0, ((size_t)M + 4) * 8, st));
  SB_TRY(c->res.grow(&c->d_base, M));
  SB_TRY(c->res.grow(&c->d_cw, nnz));
  SB_TRY(c->res.grow(&c->d_packed, NP));
  SB_TRY(c->res.grow(&c->d_packed2, NP));
  SB_TRY(c->res.grow(&c->d_packed_scan, NP));
  SB_TRY(c->res.grow(&c->d_valid, C));
  SB_TRY(c->res.grow(&c->d_cls_map, C));
  SB_TRY(c->res.grow(&c->d_scalars, 64));
  SB_TRY(c->res.grow(&c->d_tcnt, M));
  SB_TRY(c->res.grow(&c->d_tid_row, M));
  SB_TRY(c->res.grow(&c->d_sort_keys, NS));
  SB_TRY(c->res.grow(&c->d_sort_vals, NS));
  SB_TRY(c->res.grow(&c->d_sort_keys2, NS));
  SB_TRY(c->res.grow(&c->d_sort_vals2, NS));
  SB_TRY(c->res.grow(&c->d_order, NS));
  SB_CUDA(cudaMemsetAsync(c->d_base, 0, (size_t)M * 8, st));
  SB_CUDA(cudaMemsetAsync(c->d_scalars, 0, 64 * 8, st));
  SB_CUDA(cudaMemsetAsync(c->d_tcnt, 0, (size_t)M * 4, st));
  SB_CUDA(cudaMemsetAsync(c->d_tid_row, 0xff, (size_t)M * 4, st));

  // scratch for cub
  size_t t1 = 0, t2 = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, t1, c->d_packed, c->d_packed_scan, (int)NP, st);
  {
    uint32_t* k = nullptr; uint32_t* v = nullptr;
    cub::DeviceRadixSort::SortPairs(nullptr, t2, k, k, v, v, (int)NS, 0, 32, st);
  }
  size_t need = std::max(t1, t2);
  if (need > c->tmp_bytes) {
    SB_TRY(c->res.grow((unsigned char**)&c->d_tmp, need));
    c->tmp_bytes = need;
  }

  k_txp_init<<<nblk(M, 256), 256, 0, st>>>(M, c->d_projected, c->d_eff_in, c->d_unique, *p,
                                            c->total_weight, c->d_efflens, c->d_prior, c->d_alpha0);
  c->launches++;
  unsigned long long* d_ndeg = (unsigned long long*)(c->d_scalars + 0);
  if (C) {
    k_class_combine<<<nblk(C, 128), 128, 0, st>>>(C, M, c->d_off, c->d_tids, c->d_aux, c->d_counts,
                                                   c->d_efflens, c->d_alpha0, *p, c->d_cw,
                                                   c->d_packed, c->d_sort_keys, c->d_cls_map,
                                                   c->d_base, c->d_valid, d_ndeg);
    // (1) locality order: classes by first transcript id
    k_iota<<<nblk(C, 256), 256, 0, st>>>((uint32_t)C, c->d_sort_vals);
    c->launches += 2;
    SB_TRY(sort_pairs(c, (uint32_t)C, bits_for(M)));
    SB_CUDA(cudaMemcpyAsync(c->d_order, c->d_sort_vals2, C * 4, cudaMemcpyDeviceToDevice, st));
    // (2) inside groups of SELL_GROUP classes, bucket by label length
    k_bucket_key<<<nblk(C, 256), 256, 0, st>>>(C, c->d_order, c->d_packed, (uint32_t)c->sell_group_cm, c->d_sort_keys, c->d_sort_vals);
    c->launches++;
    SB_TRY(sort_pairs(c, (uint32_t)C, 32));
    SB_CUDA(cudaMemcpyAsync(c->d_order, c->d_sort_vals2, C * 4, cudaMemcpyDeviceToDevice, st));
    k_gather_u64<<<nblk(C, 256), 256, 0, st>>>(C, c->d_order, c->d_packed, c->d_packed2);
    c->launches++;
  }
  SB_CUDA(cudaMemsetAsync(c->d_packed2 + C, 0, 8, st));
  SB_TRY(scan_u64(c, c->d_packed2, c->d_packed_scan, C + 1));
  uint64_t tot = 0;
  SB_CUDA(cudaMemcpyAsync(&tot, c->d_packed_scan + C, 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(&c->n_degenerate, d_ndeg, 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  const uint32_t Cm = (uint32_t)(tot >> 32);
  const uint32_t nnzm = (uint32_t)(tot & 0xffffffffu);
  c->n_cls = Cm; c->nnzm = nnzm;

  // compact class-major CSR in final class order
  SB_TRY(c->res.grow(&c->m_off, (size_t)Cm + 1));
  SB_TRY(c->res.grow(&c->m_idx, (size_t)nnzm + 1));
  SB_TRY(c->res.grow(&c->m_idx_state, (size_t)nnzm + 1));
  SB_TRY(c->res.grow(&c->m_w, (size_t)nnzm + 1));
  SB_TRY(c->res.grow(&c->d_cnt, (size_t)Cm));
  SB_TRY(c->res.grow(&c->d_scale, (size_t)Cm + 4));
  SB_TRY(c->res.grow(&c->d_ent_cls, (size_t)nnzm));
  SB_CUDA(cudaMemsetAsync(c->d_scale, 0, ((size_t)Cm + 4) * 8, st));
  SB_CUDA(cudaMemcpyAsync(c->m_off + Cm, &nnzm, 4, cudaMemcpyHostToDevice, st));
  if (C) {
    k_compact<<<nblk(C, 128), 128, 0, st>>>(C, c->d_order, c->d_off, c->d_tids, c->d_cw, c->d_counts,
                                             c->d_packed2, c->d_packed_scan, c->m_off, c->m_idx,
                                             c->m_w, c->d_cnt, c->d_ent_cls, c->d_tcnt, c->d_cls_map);
    c->launches++;
  }
  // transcript-major CSR in rank order: stable radix sort of (tid, entry) pairs
  if (nnzm) {
    SB_CUDA(cudaMemcpyAsync(c->d_sort_keys, c->m_idx, (size_t)nnzm * 4, cudaMemcpyDeviceToDevice, st));
    k_iota<<<nblk(nnzm, 256), 256, 0, st>>>(nnzm, c->d_sort_vals);
    c->launches++;
    SB_TRY(sort_pairs(c, nnzm, bits_for(M)));
  }
  k_row_pack<<<nblk(M, 256), 256, 0, st>>>(M, c->d_tcnt, c->d_packed);
  c->launches++;
  SB_CUDA(cudaMemsetAsync(c->d_packed + M, 0, 8, st));
  SB_TRY(scan_u64(c, c->d_packed, c->d_packed_scan, (uint64_t)M + 1));
  uint64_t tot2 = 0;
  SB_CUDA(cudaMemcpyAsync(&tot2, c->d_packed_scan + M, 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  const uint32_t R = (uint32_t)(tot2 >> 32);
  if ((uint32_t)(tot2 & 0xffffffffu) != nnzm) {
    set_error("internal: transcript-major entry count mismatch");
    return SB_ERR_STATE;
  }
  c->n_rows = R;
  SB_TRY(c->res.grow(&c->t_off, (size_t)R + 1));
  SB_TRY(c->res.grow(&c->t_idx, (size_t)nnzm + 1));
  SB_TRY(c->res.grow(&c->t_w, (size_t)nnzm + 1));
  SB_TRY(c->res.grow(&c->d_rank_tid, (size_t)R + 1));
  SB_TRY(c->res.grow(&c->d_rowperm, (size_t)R + 1));
  SB_TRY(c->res.grow(&c->d_row_tid, (size_t)R + 1));
  SB_TRY(c->res.grow(&c->r_alpha, (size_t)R + 1));
  SB_TRY(c->res.grow(&c->r_theta, (size_t)R + 4));
  SB_CUDA(cudaMemsetAsync(c->r_theta, 0, ((size_t)R + 4) * 8, st));
  SB_TRY(c->res.grow(&c->r_prior, (size_t)R + 1));
  SB_TRY(c->res.grow(&c->r_base, (size_t)R + 1));
  SB_TRY(c->res.grow(&c->r_alpha0, (size_t)R + 1));
  SB_CUDA(cudaMemcpyAsync(c->t_off + R, &nnzm, 4, cudaMemcpyHostToDevice, st));
  // rank_packed reuses d_packed2 (class packing no longer needed)
  k_rank_fill<<<nblk(M, 256), 256, 0, st>>>(M, c->d_tcnt, c->d_packed_scan, c->t_off, c->d_rank_tid,
                                             c->d_packed2);
  c->launches++;
  if (nnzm) {
    k_gather_csc<<<nblk(nnzm, 256), 256, 0, st>>>(nnzm, c->d_sort_vals2, c->d_ent_cls, c->m_w,
                                                   c->t_idx, c->t_w);
    c->launches++;
  }
  // rows: ranks bucketed by occurrence count inside groups of SELL_GROUP
  if (R) {
    k_bucket_key<<<nblk(R, 256), 256, 0, st>>>(R, nullptr, c->d_packed2, (uint32_t)c->sell_group_tm, c->d_sort_keys, c->d_sort_vals);
    c->launches++;
    SB_TRY(sort_pairs(c, R, 32));
    SB_CUDA(cudaMemcpyAsync(c->d_rowperm, c->d_sort_vals2, (size_t)R * 4, cudaMemcpyDeviceToDevice, st));
    k_row_fill<<<nblk(R, 256), 256, 0, st>>>(R, c->d_rowperm, c->d_rank_tid, c->d_prior, c->d_base,
                                              c->d_alpha0, c->d_row_tid, c->d_tid_row, c->r_prior,
                                              c->r_base, c->r_alpha0);
    c->launches++;
  }
  // class-major gather index: row ids (single GPU) or transcript ids (multi GPU)
  if (nnzm) {
    if (row_space) {
      k_remap<<<nblk(nnzm, 256), 256, 0, st>>>(nnzm, c->m_idx, c->d_tid_row, c->m_idx_state);
      c->launches++;
    } else {
      SB_CUDA(cudaMemcpyAsync(c->m_idx_state, c->m_idx, (size_t)nnzm * 4, cudaMemcpyDeviceToDevice, st));
    }
  }
  // SELL-32 copies.  overhead = per-slice epilogue cost in "columns" for the work split
  SB_TRY(build_sell(c, c->cm, Cm, nullptr, c->m_off, c->m_idx_state, c->m_w, row_space ? R : M, OVERHEAD_P1, n_warps));
  SB_TRY(build_sell(c, c->tm, R, c->d_rowperm, c->t_off, c->t_idx, c->t_w, Cm, overhead_tm(c), n_warps));

  // iteration-0 reductions
  double* d_sum0 = c->d_scalars + 16;
  double* d_inact = c->d_scalars + 17;
  k_sum1<<<1, 1024, 0, st>>>(M, c->d_alpha0, c->d_prior, c->d_tid_row, 0, d_sum0);
  k_sum1<<<1, 1024, 0, st>>>(M, c->d_base, c->d_prior, c->d_tid_row, 1, d_inact);
  c->launches += 2;
  SB_CUDA(cudaMemcpyAsync(&c->sum0, d_sum0, 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(&c->inactive_sum, d_inact, 8, cudaMemcpyDeviceToHost, st));
  SB_TRY(c->res.grow(&c->d_sum_partial, (size_t)2 * std::max<uint32_t>(c->grid, 4096)));
  SB_CUDA(cudaStreamSynchronize(st));
  c->prepared = true;
  // measured re-cut of the warp ranges (persistent kernels only: they carry the per-warp phase timers)
  c->rebalance_rounds_done = 0;
  if (c->variant == 1 && (c->nranks <= 1 || (c->peers_ready && c->M <= c->x_cap)) && p->max_iter > 0) {
    for (int r = 0; r < c->rebalance; ++r) {
      int rc = em_rebalance(c);
      if (rc != SB_OK) { c->prepared = false; return rc; }
          c->rebalance_rounds_done++;
    }
  }
  const uint32_t prep_launches = c->launches;
  SB_CUDA(cudaEventRecord(c->ev[1], st));
  SB_CUDA(cudaEventSynchronize(c->ev[1]));
  float ms = 0;
  cudaEventElapsedTime(&ms, c->ev[0], c->ev[1]);
  c->prepare_ms = ms;
  c->prepared = true;
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->n_degenerate = c->n_degenerate;
    stats->n_multi_classes = Cm;
    stats->nnz_multi = nnzm;
    stats->n_active_txps = R;
    stats->prepare_ms = ms;
    stats->gpu_launches = prep_launches;
  }
  return SB_OK;
}

static Sell sell_view(const SellDev& m) {
  Sell s;
  s.slice_ptr = m.slice_ptr; s.base = m.base; s.len = m.len; s.idx = m.idx; s.w = m.w; s.warp_begin = m.warp_begin;
  s.long_rows = m.long_rows; s.csr_idx = m.csr_idx; s.csr_w = m.csr_w;
  s.n_rows = m.n_rows; s.n_slices = m.n_slices; s.n_long = m.n_long;
  s.n_block = m.n_block;
  s.zero = m.zero;
  return s;
}

static void fill_args(sb_em_ctx* c, EmArgs& A, bool row_space) {
  memset(&A, 0, sizeof(A));
  A.cm = sell_view(c->cm);
  A.tm = sell_view(c->tm);
  // the bootstrap driver's overrides apply only while it is running (ov_active): the buffers outlive it, and a later
  // optimize on the same context must not see the last replicate's resampled counts (bootstrap overrides)
  const bool ov = c->ov_active;
  A.c_cnt = (ov && c->ov_cnt) ? c->ov_cnt : c->d_cnt; A.scale = c->d_scale;
  if (row_space) {
    A.alpha = c->r_alpha; A.theta = c->r_theta; A.prior = c->r_prior;
    A.base = (ov && c->ov_base_row) ? c->ov_base_row : c->r_base;
    A.row_tid = nullptr;
  } else {
    A.alpha = c->d_alpha; A.theta = c->d_theta; A.prior = c->d_prior; A.base = c->d_base;
    A.row_tid = c->d_row_tid;
    A.tid_row = c->d_tid_row;
  }
  A.sum_partial = c->d_sum_partial;
  A.maxrel = (unsigned long long*)(c->d_scalars + 24);
  A.inactive_sum = ov ? c->ov_inactive_sum : c->inactive_sum;
  A.sum0 = ov ? c->ov_sum0 : c->sum0;
  A.sum_scale = ldexp(1.0, c->sum_scale_log2);
  A.min_eq_w = ov ? c->ov_min_eq_w : DBL_MIN;
  A.first_bias = ov ? 0.0 : (c->params.use_vbem ? 0.0 : 1.0);
  A.tol = c->params.tol; A.min_iter = c->params.min_iter; A.max_iter = c->params.max_iter;
  A.out = (uint32_t*)(c->d_scalars + 32);
  A.lq = (unsigned int*)(c->d_scalars + 44);
  A.dbg = c->dbg_enabled ? c->d_dbg : nullptr;
  A.dbg_it = c->dbg_it;
}

// ---------------------------------------------------------------------------
// multi-GPU: NCCL is loaded at run time (dlopen) so the library has no link-time
// dependency on it; torch's bundled libnccl.so.2 is picked up when present.
// ---------------------------------------------------------------------------
#include <dlfcn.h>
namespace {
struct NcclUid { char b[128]; };  // ncclUniqueId (NCCL_UNIQUE_ID_BYTES = 128), passed by value
struct NcclFns {
  void* h = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, NcclUid, int) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
NcclFns g_nccl;
int nccl_load() {
  if (g_nccl.h) return SB_OK;
  const char* names[] = {"libnccl.so.2", "libnccl.so", nullptr};
  void* h = nullptr;
  for (int i = 0; names[i] && !h; ++i) h = dlopen(names[i], RTLD_NOW | RTLD_GLOBAL);
  if (!h) { set_error("cannot dlopen libnccl.so.2: %s", dlerror()); return SB_ERR_NCCL; }
  g_nccl.GetUniqueId = (decltype(g_nccl.GetUniqueId))dlsym(h, "ncclGetUniqueId");
  g_nccl.CommInitRank = (decltype(g_nccl.CommInitRank))dlsym(h, "ncclCommInitRank");
  g_nccl.AllReduce = (decltype(g_nccl.AllReduce))dlsym(h, "ncclAllReduce");
  g_nccl.AllGather = (decltype(g_nccl.AllGather))dlsym(h, "ncclAllGather");
  g_nccl.CommDestroy = (decltype(g_nccl.CommDestroy))dlsym(h, "ncclCommDestroy");
  g_nccl.GetErrorString = (decltype(g_nccl.GetErrorString))dlsym(h, "ncclGetErrorString");
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllReduce || !g_nccl.AllGather || !g_nccl.CommDestroy) {
    set_error("libnccl is missing required symbols");
    return SB_ERR_NCCL;
  }
  g_nccl.h = h;
  return SB_OK;
}
#define SB_NCCL(call)                                                            \
  do {                                                                           \
    int _r = (call);                                                             \
    if (_r != 0) {                                                               \
      set_error("%s:%d: %s -> nccl error %d (%s)", __FILE__, __LINE__, #call, _r, \
                g_nccl.GetErrorString ? g_nccl.GetErrorString(_r) : "?");        \
      return SB_ERR_NCCL;                                                        \
    }                                                                            \
  } while (0)
}  // namespace

extern "C" int sb_nccl_unique_id(void* out128) {
  if (!out128) { set_error("null argument"); return SB_ERR_INVALID; }
  SB_TRY(nccl_load());
  SB_NCCL(g_nccl.GetUniqueId(out128));
  return SB_OK;
}
// ---- host-level communicator of the C++ multi-GPU driver (one process per GPU; NCCL underneath) ---------------------
// The once-per-run reductions at the end of mapping (M-sized vectors), the exchange of the CUDA IPC handles of the
// fused EM kernel and the gathering of posterior samples go through it; the per-iteration exchange of the EM does not
// (k_em_persistent_mgpu moves it inside the kernel).
struct sb_comm {
  int rank = 0, nranks = 1, device = 0;
  void* nccl = nullptr;
  cudaStream_t stream = nullptr;
  unsigned char* d_buf = nullptr;
  sb::Resources res;
  sb_comm(int rank_, int nranks_, int device_) : rank(rank_), nranks(nranks_), device(device_), res(device_) {}
};
extern "C" sb_comm* sb_comm_create(int rank, int nranks, const void* nccl_uid128, int device) {
  if (nranks < 1 || rank < 0 || rank >= nranks || (nranks > 1 && !nccl_uid128)) { set_error("sb_comm_create: bad arguments"); return nullptr; }
  if (nranks == 1) return new sb_comm(rank, nranks, device);
  if (nccl_load() != SB_OK) return nullptr;
  if (cudaSetDevice(device) != cudaSuccess) { set_error("sb_comm_create: cannot use device %d", device); return nullptr; }
  sb_comm* cm = new sb_comm(rank, nranks, device);
  if (cm->res.stream(&cm->stream, cudaStreamDefault) != SB_OK) { delete cm; return nullptr; }
  NcclUid u;
  memcpy(u.b, nccl_uid128, 128);
  const int r = g_nccl.CommInitRank(&cm->nccl, nranks, u, rank);
  if (r != 0) {
    set_error("ncclCommInitRank -> %d (%s)", r, g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
    delete cm; return nullptr;
  }
  return cm;
}
extern "C" void sb_comm_destroy(sb_comm* cm) {
  if (!cm) return;
  if (cm->nccl && g_nccl.CommDestroy) g_nccl.CommDestroy(cm->nccl);
  delete cm;
}
extern "C" int sb_comm_rank(const sb_comm* cm) { return cm ? cm->rank : 0; }
extern "C" int sb_comm_size(const sb_comm* cm) { return cm ? cm->nranks : 1; }
// in place over host buffers; dtype: 0 = f64, 1 = u64; op: 0 sum, 2 max, 3 min (ncclRedOp_t)
extern "C" int sb_comm_allreduce(sb_comm* cm, void* buf, size_t n, int dtype, int op) {
  if (!cm || (n && !buf)) { set_error("null argument"); return SB_ERR_INVALID; }
  if (cm->nranks == 1 || n == 0) return SB_OK;
  SB_CUDA(cudaSetDevice(cm->device));
  SB_TRY(cm->res.grow(&cm->d_buf, n * 8));
  SB_CUDA(cudaMemcpyAsync(cm->d_buf, buf, n * 8, cudaMemcpyHostToDevice, cm->stream));
  SB_NCCL(g_nccl.AllReduce(cm->d_buf, cm->d_buf, n, dtype == 0 ? /*ncclFloat64*/ 8 : /*ncclUint64*/ 5, op, cm->nccl, cm->stream));
  SB_CUDA(cudaMemcpyAsync(buf, cm->d_buf, n * 8, cudaMemcpyDeviceToHost, cm->stream));
  SB_CUDA(cudaStreamSynchronize(cm->stream));
  return SB_OK;
}
// recv = nranks x bytes (rank order); host buffers
extern "C" int sb_comm_allgather(sb_comm* cm, const void* send, void* recv, size_t bytes) {
  if (!cm || !send || !recv) { set_error("null argument"); return SB_ERR_INVALID; }
  if (cm->nranks == 1) { memcpy(recv, send, bytes); return SB_OK; }
  const size_t padded = (bytes + 15) & ~(size_t)15;
  SB_CUDA(cudaSetDevice(cm->device));
  SB_TRY(cm->res.grow(&cm->d_buf, padded * (size_t)(cm->nranks + 1)));
  SB_CUDA(cudaMemcpyAsync(cm->d_buf, send, bytes, cudaMemcpyHostToDevice, cm->stream));
  SB_NCCL(g_nccl.AllGather(cm->d_buf, cm->d_buf + padded, padded, /*ncclInt8*/ 0, cm->nccl, cm->stream));
  std::vector<unsigned char> tmp(padded * (size_t)cm->nranks);
  SB_CUDA(cudaMemcpyAsync(tmp.data(), cm->d_buf + padded, tmp.size(), cudaMemcpyDeviceToHost, cm->stream));
  SB_CUDA(cudaStreamSynchronize(cm->stream));
  for (int r = 0; r < cm->nranks; ++r) memcpy((unsigned char*)recv + (size_t)r * bytes, tmp.data() + (size_t)r * padded, bytes);
  return SB_OK;
}
// the fused multi-GPU EM on this communicator: exchange the exchange blocks' CUDA IPC handles and map the peers
extern "C" int sb_em_peer_setup(sb_em_ctx* c, sb_comm* cm, uint32_t max_txps) {
  if (!c || !cm) { set_error("null argument"); return SB_ERR_INVALID; }
  if (cm->nranks == 1) return SB_OK;
  unsigned char mine[64];
  SB_TRY(sb_em_peer_handle(c, max_txps, mine));
  std::vector<unsigned char> all((size_t)64 * cm->nranks);
  SB_TRY(sb_comm_allgather(cm, mine, all.data(), 64));
  return sb_em_peer_open(c, cm->rank, cm->nranks, all.data());
}

extern "C" int sb_em_comm_init(sb_em_ctx* c, int rank, int nranks, const void* uid) {
  if (!c || !uid || nranks < 1 || rank < 0 || rank >= nranks) { set_error("bad argument"); return SB_ERR_INVALID; }
  SB_TRY(nccl_load());
  SB_CUDA(cudaSetDevice(c->device));
  NcclUid u;
  memcpy(u.b, uid, 128);
  void* comm = nullptr;
  SB_NCCL(g_nccl.CommInitRank(&comm, nranks, u, rank));
  c->nccl_comm = comm;
  c->rank = rank;
  c->nranks = nranks;
  c->prepared = false;  // gather windows depend on the index space
  return SB_OK;
}
extern "C" int sb_em_comm_destroy(sb_em_ctx* c) {
  if (!c) return SB_OK;
  if (c->nccl_comm && g_nccl.CommDestroy) {
    g_nccl.CommDestroy(c->nccl_comm);
    c->nccl_comm = nullptr;
  }
  c->nranks = 1;
  c->rank = 0;
  return SB_OK;
}

// ---- exchange blocks for the fused multi-GPU kernel (CUDA IPC over NVLink P2P); layout: XchgLayout ----------
extern "C" int sb_em_peer_handle(sb_em_ctx* c, uint32_t max_txps, void* out64) {
  if (!c || !out64 || !max_txps) { set_error("null argument"); return SB_ERR_INVALID; }
  SB_CUDA(cudaSetDevice(c->device));
  if (c->x_block && c->x_cap < max_txps) { set_error("exchange block already allocated for %u transcripts", c->x_cap); return SB_ERR_STATE; }
  if (!c->x_block) {   // both buffers are made before either is recorded: a failure leaves the context as it was
    const size_t bytes = XchgLayout(max_txps, 64).bytes() + 64 * 8;   // G * ceil(M / G) <= M + 63 for every G <= 64
    unsigned char* xb = nullptr;
    uint32_t* xf = nullptr;
    int rc = c->res.alloc(&xb, bytes);
    if (rc == SB_OK) rc = c->res.alloc(&xf, 1);
    if (rc == SB_OK) {
      const cudaError_t e = cudaMemset(xb, 0, bytes);
      if (e != cudaSuccess) { set_error("clearing the exchange block: %s", cudaGetErrorString(e)); rc = SB_ERR_CUDA; }
    }
    if (rc != SB_OK) { c->res.release(xb); c->res.release(xf); return rc; }
    c->x_block = xb; c->d_xfail = xf; c->x_cap = max_txps;
  }
  cudaIpcMemHandle_t h;
  SB_CUDA(cudaIpcGetMemHandle(&h, c->x_block));
  static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(out64, &h, 64);
  return SB_OK;
}

// handles: nranks x 64 bytes (every rank's sb_em_peer_handle, all-gathered by the host layer).  nranks == 1 is a
// loop-back (the rank is its own and only peer): the fused kernel's exchange logic on one GPU, for tests.
extern "C" int sb_em_peer_open(sb_em_ctx* c, int rank, int nranks, const void* handles) {
  if (!c || !handles || nranks < 1 || nranks > 64 || rank < 0 || rank >= nranks) { set_error("bad arguments"); return SB_ERR_INVALID; }
  if (!c->x_block) { set_error("sb_em_peer_open before sb_em_peer_handle"); return SB_ERR_STATE; }
  SB_CUDA(cudaSetDevice(c->device));
  std::vector<unsigned char*> ptrs(nranks, nullptr);
  for (int q = 0; q < nranks; ++q) {
    if (q == rank) { ptrs[q] = c->x_block; continue; }
    cudaIpcMemHandle_t h;
    memcpy(&h, (const char*)handles + (size_t)q * 64, 64);
    void* p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) { set_error("cudaIpcOpenMemHandle(rank %d): %s", q, cudaGetErrorString(e)); cudaGetLastError(); return SB_ERR_CUDA; }
    ptrs[q] = (unsigned char*)p;
    c->x_opened.push_back(p);
  }
  if (!c->d_peers) SB_TRY(c->res.alloc(&c->d_peers, 64));
  SB_CUDA(cudaMemcpy(c->d_peers, ptrs.data(), (size_t)nranks * sizeof(unsigned char*), cudaMemcpyHostToDevice));
  c->rank = rank; c->nranks = nranks;
  c->peers_ready = true;
  c->fused_loopback = (nranks == 1);
  c->prepared = false;   // the index space of the class-major matrix depends on it
  return SB_OK;
}

// Fused path: one cooperative launch per run on every rank; the partial alpha' are pushed to their owners, the owners
// push theta back, all inside the kernel over the peers' exchange blocks (see k_em_persistent_mgpu).
static int em_run_multi_gpu_fused(sb_em_ctx* c, EmArgs& A, uint32_t* out,
                                  uint32_t* launches, uint32_t* loop_launches, float* loop_ms) {
  cudaStream_t st = c->stream;
  const uint32_t M = c->M;
  const int vb = c->params.use_vbem ? 1 : 0;
  const XchgLayout X(M, (uint32_t)c->nranks);
  SB_CUDA(cudaMemsetAsync(c->d_xfail, 0, 4, st));
  SB_TRY(c->res.grow(&c->d_part, (size_t)M));
  // locally inactive transcripts contribute their (constant) folded singleton mass
  SB_CUDA(cudaMemcpyAsync(c->d_part, c->d_base, (size_t)M * 8, cudaMemcpyDeviceToDevice, st));
  A.part_out = c->d_part;
  A.push_pass = (c->push_pass >= 0) ? (uint32_t)c->push_pass : (c->nranks > 2 ? 1u : 0u);
  if (c->grid > XAUX) { set_error("multi-GPU EM: grid of %u blocks exceeds the exchange block's aux area", c->grid); return SB_ERR_STATE; }
  A.theta = reinterpret_cast<double*>(c->x_block + X.off_theta());
  A.inactive_sum = 0.0;
  A.peers = c->d_peers; A.rank = (uint32_t)c->rank; A.nranks = (uint32_t)c->nranks; A.M = M;
  A.epoch0 = c->x_epoch; A.xfail = c->d_xfail;
  void* args[] = {(void*)&A};
  SB_CUDA(cudaEventRecord(c->ev[2], st));
  SB_CUDA(cudaLaunchCooperativeKernel(K_PERSISTENT_MGPU[vb], dim3(c->grid), dim3(EM_THREADS), args, EM_SMEM, st));
  SB_CUDA(cudaEventRecord(c->ev[3], st));
  *launches += 1; *loop_launches += 1;
  uint32_t fail = 0;
  SB_CUDA(cudaMemcpyAsync(out, A.out, 16, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(&fail, c->d_xfail, 4, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(c->d_alpha, c->x_block + X.off_alpha(), (size_t)M * 8, cudaMemcpyDeviceToDevice, st));
  SB_CUDA(cudaStreamSynchronize(st));
  cudaEventElapsedTime(loop_ms, c->ev[2], c->ev[3]);
  c->x_epoch += out[3];
  if (fail) { set_error("multi-GPU EM: a peer GPU did not reach the in-kernel barrier (rank %d of %d)", c->rank, c->nranks); return SB_ERR_NCCL; }
  return SB_OK;
}

// One iteration = P1, P2-partial, all-reduce(alpha'), update.  Classes stay sharded.
static int em_run_multi_gpu(sb_em_ctx* c, EmArgs& A, uint32_t* out,
                            uint32_t* launches, uint32_t* loop_launches, float* loop_ms) {
  cudaStream_t st = c->stream;
  const uint32_t M = c->M;
  const int vb = c->params.use_vbem ? 1 : 0;
  if (!c->nccl_comm) { set_error("multi-GPU EM: neither peers (sb_em_peer_open) nor NCCL (sb_em_comm_init) are set up"); return SB_ERR_STATE; }
  SB_TRY(c->res.grow(&c->d_part, (size_t)M));
  SB_TRY(c->res.grow(&c->d_part_red, (size_t)M));
  // locally inactive transcripts contribute their (constant) folded singleton mass
  SB_CUDA(cudaMemcpyAsync(c->d_part, c->d_base, (size_t)M * 8, cudaMemcpyDeviceToDevice, st));
  A.part_out = c->d_part;
  A.inactive_sum = 0.0;  // the update covers every transcript
  const uint32_t ugrid = std::min<uint32_t>(4096u, (M + 255) / 256);
  uint32_t it = 0;
  bool converged = false;
  SB_CUDA(cudaEventRecord(c->ev[2], st));
  while (it < A.min_iter || (it < A.max_iter && !converged)) {
    k_reset_maxrel<<<1, 1, 0, st>>>(A.maxrel, it & 1u);
    K_P1[vb]<<<c->grid, EM_THREADS, EM_SMEM, st>>>(A);
    K_P2_PARTIAL[vb]<<<c->grid, EM_THREADS, EM_SMEM, st>>>(A);
    SB_NCCL(g_nccl.AllReduce(c->d_part, c->d_part_red, (size_t)M, /*ncclFloat64*/ 8, /*ncclSum*/ 0,
                             c->nccl_comm, st));
    if (vb) k_em_update<true><<<ugrid, 256, 0, st>>>(A, c->d_part_red, M, it);
    else k_em_update<false><<<ugrid, 256, 0, st>>>(A, c->d_part_red, M, it);
    *launches += 5; *loop_launches += 4;
    ++it;
    if (it >= A.min_iter) {
      unsigned long long mr = 0;
      SB_CUDA(cudaMemcpyAsync(&mr, A.maxrel + ((it - 1) & 1u), 8, cudaMemcpyDeviceToHost, st));
      SB_CUDA(cudaStreamSynchronize(st));
      double d;
      memcpy(&d, &mr, 8);
      converged = !(d > A.tol);
    }
  }
  SB_CUDA(cudaEventRecord(c->ev[3], st));
  SB_CUDA(cudaStreamSynchronize(st));
  cudaEventElapsedTime(loop_ms, c->ev[2], c->ev[3]);
  out[0] = it; out[1] = converged; out[2] = (it - 1) & 1u;
  return SB_OK;
}

extern "C" int sb_em_run(sb_em_ctx* c, sb_em_stats* stats) {
  if (!c) { set_error("null argument"); return SB_ERR_INVALID; }
  if (!c->prepared) { set_error("sb_em_run before sb_em_prepare"); return SB_ERR_STATE; }
  SB_CUDA(cudaSetDevice(c->device));
  cudaStream_t st = c->stream;
  const uint32_t M = c->M;
  const uint32_t R = c->n_rows;
  const bool multi_gpu = c->nranks > 1 || c->fused_loopback;
  const int vb = c->params.use_vbem ? 1 : 0;
  uint32_t launches = 0;
  SB_CUDA(cudaEventRecord(c->ev[0], st));
  // restart from the prepared state
  double* d_sum0 = c->d_scalars + 16;
  const bool fused = multi_gpu && c->peers_ready && c->M <= c->x_cap && c->variant == 1;
  const bool ov = c->ov_active;
  if (multi_gpu) {
    // fused path: the replicated theta lives in the rank's exchange block (the owners push into it)
    double* theta0 = fused ? reinterpret_cast<double*>(c->x_block + XchgLayout(M, (uint32_t)c->nranks).off_theta()) : c->d_theta;
    k_theta0<<<nblk(M, 256), 256, 0, st>>>(M, c->params.use_vbem, c->d_alpha0, c->d_prior, d_sum0,
                                            c->d_alpha, theta0);
    ++launches;
  } else if (R) {
    k_theta0<<<nblk(R, 256), 256, 0, st>>>(R, c->params.use_vbem,
                                            (ov && c->ov_alpha0_row) ? c->ov_alpha0_row : c->r_alpha0,
                                            c->r_prior, ov ? c->d_scalars + 18 : d_sum0,
                                            c->r_alpha, c->r_theta);
    ++launches;
  }
  SB_CUDA(cudaMemsetAsync(c->d_scalars + 24, 0, 16 * 8, st));
  SB_CUDA(cudaMemsetAsync(c->d_scalars + 44, 0, 16, st));   // long-row queues
  EmArgs A;
  fill_args(c, A, !multi_gpu);
  uint32_t out[4] = {0, 0, 0, 0};
  float loop_ms = 0;
  uint32_t loop_launches = 0;
  if (c->params.max_iter == 0 && c->params.min_iter == 0) {
    // nothing to iterate
  } else if (multi_gpu) {
    int r = fused ? em_run_multi_gpu_fused(c, A, out, &launches, &loop_launches, &loop_ms)
                  : em_run_multi_gpu(c, A, out, &launches, &loop_launches, &loop_ms);
    if (r != SB_OK) return r;
  } else if (c->variant == 1) {
    void* args[] = {(void*)&A};
    SB_CUDA(cudaEventRecord(c->ev[2], st));
    SB_CUDA(cudaLaunchCooperativeKernel(K_PERSISTENT[vb], dim3(c->grid), dim3(EM_THREADS), args, EM_SMEM, st));
    SB_CUDA(cudaEventRecord(c->ev[3], st));
    ++launches; ++loop_launches;
    SB_CUDA(cudaMemcpyAsync(out, A.out, 16, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    cudaEventElapsedTime(&loop_ms, c->ev[2], c->ev[3]);
  } else {
    // one launch per phase; the host reads the convergence flag only where the
    // reference's loop condition can change (it >= min_iter).
    uint32_t it = 0;
    bool converged = false;
    SB_CUDA(cudaEventRecord(c->ev[2], st));
    while (it < A.min_iter || (it < A.max_iter && !converged)) {
      k_reset_maxrel<<<1, 1, 0, st>>>(A.maxrel, it & 1u);
      K_P1[vb]<<<c->grid, EM_THREADS, EM_SMEM, st>>>(A);
      K_P2[vb]<<<c->grid, EM_THREADS, EM_SMEM, st>>>(A, it);
      launches += 3; loop_launches += 2;
      ++it;
      if (it >= A.min_iter) {
        unsigned long long mr = 0;
        SB_CUDA(cudaMemcpyAsync(&mr, A.maxrel + ((it - 1) & 1u), 8, cudaMemcpyDeviceToHost, st));
        SB_CUDA(cudaStreamSynchronize(st));
        double d;
        memcpy(&d, &mr, 8);
        converged = !(d > A.tol);
      }
    }
    SB_CUDA(cudaEventRecord(c->ev[3], st));
    SB_CUDA(cudaStreamSynchronize(st));
    cudaEventElapsedTime(&loop_ms, c->ev[2], c->ev[3]);
    out[0] = it; out[1] = converged; out[2] = (it - 1) & 1u;
  }
  c->iters = out[0];
  c->converged = out[1];
  if (out[0] > 0) {
    unsigned long long mr = 0;
    SB_CUDA(cudaMemcpy(&mr, A.maxrel + out[2], 8, cudaMemcpyDeviceToHost));
    memcpy(&c->max_rel_diff, &mr, 8);
  } else {
    c->max_rel_diff = -DBL_MAX;
  }
  if (!multi_gpu) {
    // row space -> transcript space (+ inactive transcripts)
    if (out[0] > 0) {
      double bias = (!ov && !c->params.use_vbem && out[0] == 1) ? 1.0 : 0.0;
      k_finalize<<<nblk(M, 256), 256, 0, st>>>(M, c->d_tid_row, (ov && c->ov_base_tid) ? c->ov_base_tid : c->d_base,
                                                bias, c->r_alpha, c->d_alpha);
    } else {
      SB_CUDA(cudaMemcpyAsync(c->d_alpha, (ov && c->ov_alpha0_tid) ? c->ov_alpha0_tid : c->d_alpha0, (size_t)M * 8,
                              cudaMemcpyDeviceToDevice, st));
    }
    ++launches;
  }
  SB_CUDA(cudaEventRecord(c->ev[1], st));
  SB_CUDA(cudaEventSynchronize(c->ev[1]));
  float ms = 0;
  cudaEventElapsedTime(&ms, c->ev[0], c->ev[1]);
  c->run_ms = ms;
  c->launches += launches;
  if (stats) {
    stats->iters = c->iters;
    stats->converged = c->converged;
    stats->max_rel_diff = c->max_rel_diff;
    stats->n_degenerate = c->n_degenerate;
    stats->n_multi_classes = c->n_cls;
    stats->nnz_multi = c->nnzm;
    stats->n_active_txps = c->n_rows;
    stats->prepare_ms = c->prepare_ms;
    stats->run_ms = ms;
    stats->loop_kernel_ms = loop_ms;
    stats->loop_kernel_launches = loop_launches;
    stats->gpu_launches = launches;
  }
  return SB_OK;
}

// Measured re-balancing (a static split by column count does not predict a warp's phase time, and every warp waits
// at the two grid barriers for the slowest).  One short instrumented run of the persistent kernel accumulates, per
// warp, the duration of P1 and P2 and of their home streams (em_kernels.cuh: SB_ACC_*).  Every slice is given the
// measured time density of the warp that streamed it (damped towards the mean) times its modelled cost, and the
// ranges are re-cut so that every warp gets total / n_warps of that measured time.  The long rows are not charged to
// any warp: they are taken from the phase's work queue by whichever warp is free.  Deterministic given the
// measurements; the results of the iteration do not depend on the split (each row's sum is computed by one lane in a
// fixed order wherever the row lands).
static int em_recut(sb::SellDev& m, uint32_t overhead, const std::vector<unsigned long long>& dbg, int slot_total,
                    int slot_sell, uint32_t n_warps) {
  if (m.n_slices == 0 || n_warps == 0) return SB_OK;
  std::vector<uint32_t> sp((size_t)m.n_slices + 1), wb((size_t)n_warps + 1);
  SB_CUDA(cudaMemcpy(sp.data(), m.slice_ptr, sp.size() * 4, cudaMemcpyDeviceToHost));
  SB_CUDA(cudaMemcpy(wb.data(), m.warp_begin, wb.size() * 4, cudaMemcpyDeviceToHost));
  auto cost = [&](uint32_t s) { return slice_cost(sp, s, overhead); };
  std::vector<double> dens(n_warps, 0.0);
  double sell_total = 0.0, dens_sum = 0.0, work_sum = 0.0;
  for (uint32_t w = 0; w < n_warps; ++w) {
    // the SELL tap fires at the end of the home stream: the density is home-stream time over the range's work
    const double T = (double)dbg[(size_t)w * DBG_SLOTS + slot_total];
    const double Ts = std::min(T, (double)dbg[(size_t)w * DBG_SLOTS + slot_sell]);
    double W = 0.0;
    for (uint32_t s = wb[w]; s < wb[w + 1]; ++s) W += cost(s);
    if (W > 0.0) { dens[w] = Ts / W; dens_sum += Ts; work_sum += W; }
    sell_total += Ts;
  }
  if (!(sell_total > 0.0) || !(work_sum > 0.0)) return SB_OK;
  const double dens_mean = dens_sum / work_sum;
  // cumulative measured time over slices
  std::vector<double> F((size_t)m.n_slices + 1, 0.0);
  {
    uint32_t w = 0;
    for (uint32_t s = 0; s < m.n_slices; ++s) {
      while (w + 1 < n_warps && s >= wb[w + 1]) ++w;
      const double d = dens[w] > 0.0 ? 0.75 * dens[w] + 0.25 * dens_mean : dens_mean;   // damped
      F[s + 1] = F[s] + d * cost(s);
    }
  }
  const double total = F[m.n_slices];
  std::vector<uint32_t> nb((size_t)n_warps + 1);
  nb[0] = 0;
  nb[n_warps] = m.n_slices;
  uint32_t s = 0;
  for (uint32_t w = 1; w < n_warps; ++w) {
    const double level = total * w / n_warps;
    while (s < m.n_slices && 0.5 * (F[s] + F[s + 1]) < level) ++s;   // a slice goes to the warp that holds its midpoint
    nb[w] = s;
  }
  SB_CUDA(cudaMemcpy(m.warp_begin, nb.data(), nb.size() * 4, cudaMemcpyHostToDevice));
  return SB_OK;
}

constexpr uint32_t REBALANCE_ITERS = 8;   // measured iterations of the instrumented run (the first is not timed)

static int em_rebalance(sb_em_ctx* c) {
  const uint32_t n_warps = c->grid * (EM_THREADS / 32);
  SB_TRY(c->res.grow(&c->d_dbg, (size_t)n_warps * DBG_SLOTS));
  SB_CUDA(cudaMemsetAsync(c->d_dbg, 0, (size_t)n_warps * DBG_SLOTS * 8, c->stream));
  const sb_em_params saved = c->params;
  const uint32_t saved_it = c->dbg_it;
  const bool saved_en = c->dbg_enabled;
  c->params.min_iter = c->params.max_iter = REBALANCE_ITERS + 1;
  c->dbg_it = DBG_ACCUMULATE;
  c->dbg_enabled = true;
  int rc = sb_em_run(c, nullptr);
  c->params = saved; c->dbg_it = saved_it; c->dbg_enabled = saved_en;
  if (rc != SB_OK) return rc;
  std::vector<unsigned long long> dbg((size_t)n_warps * DBG_SLOTS);
  SB_CUDA(cudaMemcpy(dbg.data(), c->d_dbg, dbg.size() * 8, cudaMemcpyDeviceToHost));
  SB_TRY(em_recut(c->cm, OVERHEAD_P1, dbg, 0, 3, n_warps));
  SB_TRY(em_recut(c->tm, overhead_tm(c), dbg, 1, 4, n_warps));
  return SB_OK;
}

extern "C" int sb_em_download(sb_em_ctx* c, double* alpha_out, sb_em_stats* stats) {
  if (!c || !alpha_out) { set_error("null argument"); return SB_ERR_INVALID; }
  if (!c->prepared) { set_error("sb_em_download before sb_em_prepare"); return SB_ERR_STATE; }
  SB_CUDA(cudaSetDevice(c->device));
  SB_CUDA(cudaMemcpyAsync(alpha_out, c->d_alpha, (size_t)c->M * 8, cudaMemcpyDeviceToHost, c->stream));
  SB_CUDA(cudaStreamSynchronize(c->stream));
  // truncation + alphaSum, serial in reference order (:1004-1014, EMUtils.cpp:55-67)
  double alphaSum = 0.0;
  for (uint32_t i = 0; i < c->M; ++i) {
    if (alpha_out[i] <= 1e-8) alpha_out[i] = 0.0;
    alphaSum += alpha_out[i];
  }
  if (stats) stats->alpha_sum = alphaSum;
  return (alphaSum < DBL_MIN) ? 1 : SB_OK;   // :1016-1020 -> false
}

extern "C" int sb_em_get_combined(sb_em_ctx* c, double* combined_out, uint8_t* valid_out) {
  if (!c) { set_error("null argument"); return SB_ERR_INVALID; }
  if (!c->prepared) { set_error("not prepared"); return SB_ERR_STATE; }
  SB_CUDA(cudaSetDevice(c->device));
  if (combined_out && c->nnz)
    SB_CUDA(cudaMemcpy(combined_out, c->d_cw, c->nnz * 8, cudaMemcpyDeviceToHost));
  if (valid_out && c->C) SB_CUDA(cudaMemcpy(valid_out, c->d_valid, c->C, cudaMemcpyDeviceToHost));
  return SB_OK;
}

extern "C" int sb_eq_combined_weights(sb_em_ctx* c, const sb_eq_csr* eq, const double* eff_len, int no_rich_eq,
                                      double* combined_out) {
  if (!c || !eq || !eff_len || !combined_out) { set_error("null argument"); return SB_ERR_INVALID; }
  const uint32_t M = eq->n_txps;
  std::vector<double> zeros(M, 0.0);   // the projected and unique counts play no part here
  std::vector<uint64_t> uzeros(M, 0);
  SB_TRY(sb_em_upload(c, eq, zeros.data(), eff_len, uzeros.data()));
  const uint64_t C = c->C, nnz = c->nnz;
  if (!nnz) return SB_OK;
  cudaStream_t st = c->stream;
  SB_TRY(c->res.grow(&c->d_cw, nnz));
  k_eq_combined<<<nblk(C, 128), 128, 0, st>>>(C, c->d_off, c->d_tids, c->d_aux, c->d_counts, c->d_eff_in,
                                               no_rich_eq ? 1 : 0, c->d_cw);
  SB_CUDA(cudaGetLastError());
  SB_CUDA(cudaMemcpyAsync(combined_out, c->d_cw, nnz * 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return SB_OK;
}

// --bootstrapReproject (CollapsedEMOptimizer.cpp:495-505): one more update of the single-GPU loop, from the alpha and
// theta the last sb_em_run left in row space, against the class counts `cnt` (compact classes) and the folded
// singleton counts base_row / base_tid, dropping classes whose denominator is at most min_eq_w.  The iteration index
// continues the run's, so P2's lagged logNorm reads the partial sums the run's last iteration wrote.  The result
// replaces d_alpha.
static int em_reproject(sb_em_ctx* c, const double* cnt, const double* base_row, const double* base_tid,
                        double min_eq_w) {
  cudaStream_t st = c->stream;
  const int vb = c->params.use_vbem ? 1 : 0;
  const uint32_t it = c->iters;
  EmArgs A;
  fill_args(c, A, true);
  A.c_cnt = cnt;
  A.base = base_row;
  A.min_eq_w = min_eq_w;
  k_reset_maxrel<<<1, 1, 0, st>>>(A.maxrel, it & 1u);
  K_P1[vb]<<<c->grid, EM_THREADS, EM_SMEM, st>>>(A);
  K_P2[vb]<<<c->grid, EM_THREADS, EM_SMEM, st>>>(A, it);
  k_finalize<<<nblk(c->M, 256), 256, 0, st>>>(c->M, c->d_tid_row, base_tid, 0.0, c->r_alpha, c->d_alpha);
  SB_CUDA(cudaGetLastError());
  c->launches += 4;
  return SB_OK;
}

extern "C" int sb_em_optimize(sb_em_ctx* c, const sb_eq_csr* eq, const sb_em_params* p,
                              const double* projected, const double* eff_len,
                              const uint64_t* unique, double* alpha_out, sb_em_stats* stats) {
  sb_em_stats local;
  sb_em_stats* s = stats ? stats : &local;
  SB_TRY(sb_em_upload(c, eq, projected, eff_len, unique));
  SB_TRY(sb_em_prepare(c, p, s));
  uint32_t prep_launches = s->gpu_launches;
  SB_TRY(sb_em_run(c, s));
  s->gpu_launches += prep_launches;
  return sb_em_download(c, alpha_out, s);
}

extern "C" int sb_flush_l2(sb_em_ctx* c) {
  if (!c) { set_error("null argument"); return SB_ERR_INVALID; }
  SB_CUDA(cudaSetDevice(c->device));
  size_t bytes = std::max<size_t>(c->l2_bytes * 2, (size_t)256 << 20);
  SB_TRY(c->res.grow((unsigned char**)&c->d_flush, bytes));
  SB_CUDA(cudaMemsetAsync(c->d_flush, (int)(c->flush_ctr++ & 0xff), bytes, c->stream));
  SB_CUDA(cudaStreamSynchronize(c->stream));
  return SB_OK;
}

extern "C" int sb_host_register(void* ptr, size_t bytes) {
  if (!ptr || !bytes) { set_error("null argument"); return SB_ERR_INVALID; }
  if (sb_device_count() <= 0) { set_error("no CUDA device available"); return SB_ERR_NO_DEVICE; }
  SB_CUDA(cudaHostRegister(ptr, bytes, cudaHostRegisterDefault));
  return SB_OK;
}
extern "C" int sb_host_unregister(void* ptr) {
  if (!ptr) { set_error("null argument"); return SB_ERR_INVALID; }
  SB_CUDA(cudaHostUnregister(ptr));
  return SB_OK;
}

extern "C" int sb_debug_device_memory(uint64_t* out3) {
  if (!out3) { set_error("null argument"); return SB_ERR_INVALID; }
  for (int i = 0; i < 3; ++i) out3[i] = g_resource_stats[i].load();
  return SB_OK;
}

extern "C" int sb_em_debug_timeline(sb_em_ctx* c, uint64_t* out, uint32_t iteration) {
  if (!c) { set_error("null argument"); return SB_ERR_INVALID; }
  if (!c->prepared) { set_error("not prepared"); return SB_ERR_STATE; }
  SB_CUDA(cudaSetDevice(c->device));
  const uint32_t n_warps = c->grid * (EM_THREADS / 32);
  if (!out) {
    // arm: the next sb_em_run records iteration `iteration`
    SB_TRY(c->res.grow(&c->d_dbg, (size_t)n_warps * DBG_SLOTS));
    SB_CUDA(cudaMemset(c->d_dbg, 0, (size_t)n_warps * DBG_SLOTS * 8));
    c->dbg_it = iteration;
    c->dbg_enabled = true;
    return (int)n_warps;
  }
  if (!c->d_dbg) { set_error("timeline not armed"); return SB_ERR_STATE; }
  SB_CUDA(cudaMemcpy(out, c->d_dbg, (size_t)n_warps * DBG_SLOTS * 8, cudaMemcpyDeviceToHost));
  return (int)n_warps;
}

#include "sampling.cuh"
