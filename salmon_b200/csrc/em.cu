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
// Both passes stream fixed-size windows ("tiles") of the entry arrays into shared
// memory with 1-D bulk (TMA) copies on an mbarrier ring and gather theta / scale
// from L2.  A persistent cooperative kernel runs the whole iteration loop with two
// grid barriers per iteration; the multi-kernel variant launches P1 / P2 separately
// (used for the multi-GPU path where an all-reduce sits between P2 and the update).
#include <cooperative_groups.h>
#include <cub/cub.cuh>
#include <float.h>
#include <math.h>
#include <stdarg.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "em_internal.h"

#include "em_kernels.cuh"

namespace sb {

// ---------------------------------------------------------------------------
// kernel configurations: ring chunk (columns) x resident blocks per SM
// ---------------------------------------------------------------------------
struct KernelSet {
  const char* name;
  int ch, ring;      // ring chunk (columns) x chunks in flight per warp
  size_t smem;
  // [0] = plain EM, [1] = VBEM (compile-time variants: the NaN guard exists in EM only, the digamma/exp epilogue in VBEM only)
  const void* persistent[2];
  const void* persistent_mgpu[2];
  void (*p1[2])(EmArgs);
  void (*p2[2])(EmArgs, uint32_t);
  void (*p2_partial[2])(EmArgs);
};
template <int CH, int RING, int MINB>
static KernelSet make_set(const char* name) {
  KernelSet k;
  k.name = name;
  k.ch = CH;
  k.ring = RING;
  k.smem = em_smem<CH, RING>();
  k.persistent[0] = (const void*)k_em_persistent<CH, RING, MINB, false>;
  k.persistent[1] = (const void*)k_em_persistent<CH, RING, MINB, true>;
  k.persistent_mgpu[0] = (const void*)k_em_persistent_mgpu<CH, RING, MINB, false>;
  k.persistent_mgpu[1] = (const void*)k_em_persistent_mgpu<CH, RING, MINB, true>;
  k.p1[0] = k_em_p1<CH, RING, MINB, false>;
  k.p1[1] = k_em_p1<CH, RING, MINB, true>;
  k.p2[0] = k_em_p2<CH, RING, MINB, false>;
  k.p2[1] = k_em_p2<CH, RING, MINB, true>;
  k.p2_partial[0] = k_em_p2_partial<CH, RING, MINB, false>;
  k.p2_partial[1] = k_em_p2_partial<CH, RING, MINB, true>;
  return k;
}
// chunk columns x ring depth x resident blocks per SM (shared memory per block = 8 warps x CH x RING x 384 B):
//   0: 16x2 b2 (96 KB, 16 warps/SM)   1: 8x4 b2   2: 8x3 b3 (72 KB, 24 warps/SM)   3: 8x2 b4 (48 KB, 32 warps/SM)
constexpr int N_KERNEL_SETS = 4;
static const KernelSet& kernel_set(int cfg) {
  static const KernelSet sets[N_KERNEL_SETS] = {
      make_set<16, 2, 2>("ch16r2b2"), make_set<8, 4, 2>("ch8r4b2"), make_set<8, 3, 3>("ch8r3b3"),
      make_set<8, 2, 4>("ch8r2b4"),
  };
  if (cfg < 0 || cfg >= N_KERNEL_SETS) cfg = 0;
  return sets[cfg];
}

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
  double wsum = 0.0;
  for (uint64_t j = b; j < e; ++j) {
    double el = effLens[tids[j]];
    if (el <= 1.0) el = 1.0;
    double w = p.no_rich_eq ? 1.0 : aux[j];
    double probStartPos = 1.0 / el;
    double wt = p.eq_class_mode ? w : __dmul_rn(__dmul_rn(count, w), probStartPos);
    cw[j] = wt;
    wsum = __dadd_rn(wsum, wt);
  }
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
// one warp per slice: row lengths, slice width (= max non-long length)
__global__ void k_sell_widths(uint32_t n_rows, uint32_t n_slices, uint32_t lmax,
                              const uint32_t* __restrict__ rowperm,
                              const uint32_t* __restrict__ csr_off, uint16_t* __restrict__ len16,
                              uint32_t* __restrict__ width, uint32_t* __restrict__ n_long) {
  const uint32_t s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (s >= n_slices) return;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t row = s * 32 + lane;
  uint32_t len = 0;
  if (row < n_rows) {
    const uint32_t cr = rowperm ? rowperm[row] : row;
    len = csr_off[cr + 1] - csr_off[cr];
    if (len > lmax) {
      len16[row] = LEN_LONG;
      atomicAdd(n_long, 1u);
      len = 0;
    } else {
      len16[row] = (uint16_t)len;
    }
  }
  for (int o = 16; o > 0; o >>= 1) len = max(len, __shfl_xor_sync(0xffffffffu, len, o));
  if (lane == 0) width[s] = (len + 3u) & ~3u;   // whole column groups of 4 (em_kernels.cuh: run_phase)
}
__global__ void k_sell_fill(uint32_t n_rows, uint32_t n_slices, const uint32_t* __restrict__ rowperm,
                            const uint32_t* __restrict__ csr_off, const uint32_t* __restrict__ csr_idx,
                            const double* __restrict__ csr_w, const uint32_t* __restrict__ slice_ptr,
                            const uint16_t* __restrict__ len16, uint32_t pad_idx,
                            uint32_t* __restrict__ s_idx, double* __restrict__ s_w,
                            uint32_t* __restrict__ long_rows, uint32_t* __restrict__ long_cursor) {
  const uint32_t s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (s >= n_slices) return;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t row = s * 32 + lane;
  // group-of-4 layout: entry j of lane l sits at (first column * 32) + (j / 4) * 128 + l * 4 + (j % 4)
  const size_t base = (size_t)slice_ptr[s] * 32 + (size_t)lane * 4;
  const uint32_t width = slice_ptr[s + 1] - slice_ptr[s];
  auto pos = [&](uint32_t j) { return base + (size_t)(j >> 2) * 128 + (j & 3u); };
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
        s_idx[pos(j)] = csr_idx[b + j];
        s_w[pos(j)] = csr_w[b + j];
      }
    }
  }
  // padding: weight 0 and a gather index that always reads 0.0 (slot one past the end)
  for (uint32_t j = n; j < width; ++j) {
    s_idx[pos(j)] = pad_idx;
    s_w[pos(j)] = 0.0;
  }
}
// contiguous, work-balanced slice ranges per warp: work(slice) = width + overhead
__global__ void k_warp_ranges(uint32_t n_slices, const uint32_t* __restrict__ slice_ptr,
                              uint32_t overhead, uint32_t n_warps, const uint64_t* __restrict__ targets,
                              uint32_t* __restrict__ warp_begin) {
  const uint32_t wid = blockIdx.x * blockDim.x + threadIdx.x;
  if (wid > n_warps) return;
  if (wid == n_warps || n_slices == 0) { warp_begin[wid] = n_slices; return; }
  const uint64_t total = (uint64_t)slice_ptr[n_slices] + (uint64_t)overhead * n_slices;
  const uint64_t target = targets ? targets[wid] : total * wid / n_warps;
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

// Grow-only device buffers: capacity is remembered per pointer slot so that repeated
// optimize() calls on same-sized problems never touch cudaMalloc/cudaFree again.
#include <unordered_map>
static std::unordered_map<void**, size_t>& cap_table() {
  static thread_local std::unordered_map<void**, size_t> t;
  return t;
}
template <typename T>
static int dev_alloc(T** p, size_t n) {
  if (n == 0) n = 1;
  const size_t bytes = n * sizeof(T);
  auto& caps = cap_table();
  auto it = caps.find((void**)p);
  if (*p && it != caps.end() && it->second >= bytes) return SB_OK;
  if (*p) { cudaFree(*p); *p = nullptr; }
  const size_t want = bytes + bytes / 16 + 256;  // a little slack against small size changes
  cudaError_t e = cudaMalloc((void**)p, want);
  if (e != cudaSuccess) {
    set_error("cudaMalloc(%zu bytes) failed: %s", want, cudaGetErrorString(e));
    caps.erase((void**)p);
    return SB_ERR_NOMEM;
  }
  caps[(void**)p] = want;
  return SB_OK;
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
  sb_em_ctx* c = new sb_em_ctx();
  c->device = device;
  if (cudaSetDevice(device) != cudaSuccess ||
      cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) {
    set_error("cannot initialise device %d: %s", device, cudaGetErrorString(cudaGetLastError()));
    delete c;
    return nullptr;
  }
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, device);
  c->n_sm = prop.multiProcessorCount;
  c->l2_bytes = (size_t)prop.l2CacheSize;
  for (int i = 0; i < 4; ++i) cudaEventCreate(&c->ev[i]);
  // development overrides of the tuning defaults (sweeps over the test-suite)
  if (const char* e = getenv("SB_EM_CONFIG")) { const int v = atoi(e); if (v >= 0 && v < N_KERNEL_SETS) c->config = v; }
  if (const char* e = getenv("SB_EM_LWARP")) { const int v = atoi(e); if (v >= 1) c->lwarp = v; }
  if (const char* e = getenv("SB_EM_BALANCE")) c->balance_long = atoi(e);
  if (const char* e = getenv("SB_EM_GROUP_CM")) { const int v = atoi(e); if (v >= 32 && !(v & (v - 1))) c->sell_group_cm = v; }
  if (const char* e = getenv("SB_EM_GROUP_TM")) { const int v = atoi(e); if (v >= 32 && !(v & (v - 1))) c->sell_group_tm = v; }
  return c;
}

static void free_sell(SellDev& m) {
  void** ptrs[] = {(void**)&m.slice_ptr, (void**)&m.width, (void**)&m.len, (void**)&m.idx,
                   (void**)&m.w, (void**)&m.warp_begin, (void**)&m.long_rows, (void**)&m.targets,
                   };
  for (void** p : ptrs) {
    if (*p) cudaFree(*p);
    *p = nullptr;
    cap_table().erase(p);
  }
}
static void free_all(sb_em_ctx* c) {
  void** ptrs[] = {(void**)&c->d_off, (void**)&c->d_tids, (void**)&c->d_aux, (void**)&c->d_counts,
                   (void**)&c->d_projected, (void**)&c->d_eff_in, (void**)&c->d_unique,
                   (void**)&c->d_efflens, (void**)&c->d_prior, (void**)&c->d_alpha0,
                   (void**)&c->d_alpha, (void**)&c->d_theta, (void**)&c->d_base, (void**)&c->d_cw,
                   (void**)&c->d_packed, (void**)&c->d_packed2, (void**)&c->d_packed_scan,
                   (void**)&c->d_valid, (void**)&c->d_scalars, (void**)&c->d_tcnt,
                   (void**)&c->d_tid_row, (void**)&c->m_off, (void**)&c->m_idx,
                   (void**)&c->m_idx_state, (void**)&c->m_w, (void**)&c->t_off, (void**)&c->t_idx,
                   (void**)&c->t_w, (void**)&c->d_cnt, (void**)&c->d_scale, (void**)&c->d_ent_cls,
                   (void**)&c->d_row_tid, (void**)&c->d_rank_tid, (void**)&c->d_rowperm,
                   (void**)&c->d_order, (void**)&c->d_sort_keys, (void**)&c->d_sort_vals,
                   (void**)&c->d_sort_keys2, (void**)&c->d_sort_vals2, (void**)&c->d_tmp,
                   (void**)&c->d_sum_partial, (void**)&c->d_flush, (void**)&c->d_part,
                   (void**)&c->d_part_red, (void**)&c->r_alpha, (void**)&c->r_theta,
                   (void**)&c->r_prior, (void**)&c->r_base, (void**)&c->r_alpha0,
                   (void**)&c->d_dbg, (void**)&c->d_cdf, (void**)&c->d_cls_map, (void**)&c->d_samp,
                   (void**)&c->d_valid_boot, (void**)&c->d_active, (void**)&c->d_gibbs_cnt,
                   (void**)&c->d_gibbs_mu, (void**)&c->d_gibbs_prior, (void**)&c->d_gibbs_out,
                   (void**)&c->ov_cnt, (void**)&c->ov_base_row, (void**)&c->ov_base_tid,
                   (void**)&c->ov_alpha0_row, (void**)&c->ov_alpha0_tid};
  for (void** p : ptrs) {
    if (*p) cudaFree(*p);
    *p = nullptr;
    cap_table().erase(p);
  }
  free_sell(c->cm);
  free_sell(c->tm);
}

extern "C" void sb_em_destroy(sb_em_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  for (void* p : c->x_opened) cudaIpcCloseMemHandle(p);
  cudaFree(c->x_block); cudaFree(c->d_peers); cudaFree(c->d_xfail);
  sb_em_comm_destroy(c);
  free_all(c);
  for (int i = 0; i < 4; ++i) cudaEventDestroy(c->ev[i]);
  cudaStreamDestroy(c->stream);
  delete c;
}

extern "C" int sb_em_set_option(sb_em_ctx* c, const char* key, int64_t value) {
  if (!c || !key) { set_error("null argument"); return SB_ERR_INVALID; }
  if (!strcmp(key, "variant")) c->variant = (int)value;
  else if (!strcmp(key, "blocks_per_sm")) { c->blocks_per_sm = (int)value; c->prepared = false; }
  else if (!strcmp(key, "config")) {
    if (value < 0 || value >= N_KERNEL_SETS) { set_error("config out of range"); return SB_ERR_INVALID; }
    c->config = (int)value;
    c->prepared = false;
  } else if (!strcmp(key, "lmax")) {
    if (value < 1 || value > 60000) { set_error("lmax out of range"); return SB_ERR_INVALID; }
    c->lmax = (int)value; c->prepared = false;
  } else if (!strcmp(key, "sell_group_cm") || !strcmp(key, "sell_group_tm")) {
    if (value < 32 || value > (1 << 20) || (value & (value - 1))) { set_error("sell_group must be a power of two >= 32"); return SB_ERR_INVALID; }
    (key[11] == 'c' ? c->sell_group_cm : c->sell_group_tm) = (int)value; c->prepared = false;
  } else if (!strcmp(key, "lwarp")) {
    if (value < 1 || value > 1000000) { set_error("lwarp out of range"); return SB_ERR_INVALID; }
    c->lwarp = (int)value; c->prepared = false;
  } else if (!strcmp(key, "balance_long")) { c->balance_long = (int)value; c->prepared = false;
  } else if (!strcmp(key, "l2_keep_cm")) { c->keep_cm = (int)value; }
  else if (!strcmp(key, "l2_keep_tm")) { c->keep_tm = (int)value; }
  else if (!strcmp(key, "push_pass")) { c->push_pass = (int)value; }
  else if (!strcmp(key, "sample_offset")) { c->sample_offset = (uint32_t)value; }
  else if (!strcmp(key, "rebalance")) { c->rebalance = (int)value; c->prepared = false; }
  else if (!strcmp(key, "rebalance_iters")) { c->rebalance_iters = (int)value; c->prepared = false; }
  else if (!strcmp(key, "overhead_p1")) { c->ovh_p1 = (int)value; c->prepared = false; }
  else if (!strcmp(key, "overhead_p2")) { c->ovh_p2 = (int)value; c->prepared = false; }
  else { set_error("unknown option '%s'", key); return SB_ERR_INVALID; }
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
  SB_TRY(dev_alloc(&c->d_off, C + 1));
  SB_TRY(dev_alloc(&c->d_tids, nnz));
  SB_TRY(dev_alloc(&c->d_aux, nnz));
  SB_TRY(dev_alloc(&c->d_counts, C));
  SB_TRY(dev_alloc(&c->d_projected, M));
  SB_TRY(dev_alloc(&c->d_eff_in, M));
  SB_TRY(dev_alloc(&c->d_unique, M));
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

// CSR (rows optionally permuted by rowperm) -> SELL-32 + long-row list + warp ranges
static int build_sell(sb_em_ctx* c, SellDev& m, uint32_t n_rows, const uint32_t* rowperm,
                      const uint32_t* csr_off, const uint32_t* csr_idx, const double* csr_w,
                      uint32_t pad_idx, uint32_t overhead, uint32_t n_warps) {
  cudaStream_t st = c->stream;
  m.n_rows = n_rows;
  m.n_slices = (n_rows + 31) / 32;
  m.csr_idx = csr_idx;
  m.csr_w = csr_w;
  SB_TRY(dev_alloc(&m.len, (size_t)n_rows));
  SB_TRY(dev_alloc(&m.width, (size_t)m.n_slices + 1));
  SB_TRY(dev_alloc(&m.slice_ptr, (size_t)m.n_slices + 1));
  SB_TRY(dev_alloc(&m.warp_begin, (size_t)n_warps + 1));
  uint32_t* d_nlong = (uint32_t*)(c->d_scalars + 8);
  SB_CUDA(cudaMemsetAsync(d_nlong, 0, 8, st));
  SB_CUDA(cudaMemsetAsync(m.width, 0, ((size_t)m.n_slices + 1) * 4, st));
  if (m.n_slices) {
    k_sell_widths<<<nblk(m.n_slices, 8), 256, 0, st>>>(n_rows, m.n_slices, (uint32_t)c->lmax, rowperm, csr_off, m.len,
                                                       m.width, d_nlong);
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
  SB_CUDA(cudaStreamSynchronize(st));
  m.n_cols = ncols;
  SB_TRY(dev_alloc(&m.idx, (size_t)ncols * 32 + 32));
  SB_TRY(dev_alloc(&m.w, (size_t)ncols * 32 + 32));
  SB_TRY(dev_alloc(&m.long_rows, (size_t)3 * m.n_long + 3));
  SB_CUDA(cudaMemsetAsync(m.idx, 0, ((size_t)ncols * 32 + 32) * 4, st));
  SB_CUDA(cudaMemsetAsync(m.w, 0, ((size_t)ncols * 32 + 32) * 8, st));
  if (m.n_slices) {
    k_sell_fill<<<nblk(m.n_slices, 8), 256, 0, st>>>(n_rows, m.n_slices, rowperm, csr_off, csr_idx,
                                                     csr_w, m.slice_ptr, m.len, pad_idx, m.idx,
                                                     m.w, m.long_rows, d_nlong + 1);
    c->launches++;
  }
  m.n_block = 0;
  std::vector<uint64_t> h_targets;
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
    for (uint32_t i = 0; i < m.n_long; ++i)
      if (h[3 * ord[i] + 2] - h[3 * ord[i] + 1] > (uint32_t)c->lwarp) m.n_block = i + 1;
    std::vector<uint32_t> h2(h.size());
    for (uint32_t i = 0; i < m.n_long; ++i)
      for (int k = 0; k < 3; ++k) h2[3 * i + k] = h[3 * ord[i] + k];
    SB_CUDA(cudaMemcpyAsync(m.long_rows, h2.data(), h2.size() * 4, cudaMemcpyHostToDevice, st));
    SB_CUDA(cudaStreamSynchronize(st));
    if (c->balance_long > 0 && n_warps > 0) {
      // The long rows are dealt to warps / blocks by position in the list; charge their cost (in slice columns,
      // balance_long = percent of one column per 32 entries) to the owner's share of the slice stream.
      const uint32_t wpb = EM_THREADS / 32, grid = n_warps / wpb;
      std::vector<double> extra(n_warps, 0.0);
      for (uint32_t i = 0; i < m.n_long; ++i) {
        const double L = (double)(h2[3 * i + 2] - h2[3 * i + 1]);
        if (i < m.n_block) {
          const uint32_t b = i % grid;
          for (uint32_t w = 0; w < wpb; ++w) extra[b * wpb + w] += L / EM_THREADS * c->balance_long / 100.0 + 8.0;
        } else {
          extra[(i - m.n_block) % n_warps] += L / 32.0 * c->balance_long / 100.0 + 4.0;
        }
      }
      const double total = (double)ncols + (double)overhead * m.n_slices;
      double sum_extra = 0.0;
      for (double e : extra) sum_extra += e;
      const double T = (total + sum_extra) / n_warps;
      double sum_share = 0.0;
      for (uint32_t w = 0; w < n_warps; ++w) sum_share += std::max(0.0, T - extra[w]);
      h_targets.resize(n_warps);
      double cum = 0.0;
      for (uint32_t w = 0; w < n_warps; ++w) {
        h_targets[w] = (uint64_t)(sum_share > 0.0 ? total * (cum / sum_share) : total * w / n_warps);
        cum += std::max(0.0, T - extra[w]);
      }
    }
  }
  uint64_t* d_targets = nullptr;
  if (!h_targets.empty()) {
    SB_TRY(dev_alloc(&m.targets, (size_t)n_warps));
    SB_CUDA(cudaMemcpyAsync(m.targets, h_targets.data(), h_targets.size() * 8, cudaMemcpyHostToDevice, st));
    d_targets = m.targets;
  }
  k_warp_ranges<<<nblk(n_warps + 1, 256), 256, 0, st>>>(m.n_slices, m.slice_ptr, overhead, n_warps, d_targets,
                                                        m.warp_begin);
  c->launches++;
  SB_CUDA(cudaStreamSynchronize(st));   // h_targets must outlive the copy
  return SB_OK;
}

static int em_rebalance(sb_em_ctx* c);

extern "C" int sb_em_prepare(sb_em_ctx* c, const sb_em_params* p, sb_em_stats* stats) {
  if (!c || !p) { set_error("null argument"); return SB_ERR_INVALID; }
  if (!c->uploaded) { set_error("sb_em_prepare before sb_em_upload"); return SB_ERR_STATE; }
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
  const KernelSet& ks = kernel_set(c->config);
  for (int v = 0; v < 2; ++v) {
    SB_CUDA(cudaFuncSetAttribute(ks.persistent[v], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ks.smem));
    SB_CUDA(cudaFuncSetAttribute((const void*)ks.p1[v], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ks.smem));
    SB_CUDA(cudaFuncSetAttribute((const void*)ks.p2[v], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ks.smem));
    SB_CUDA(cudaFuncSetAttribute((const void*)ks.p2_partial[v], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ks.smem));
    SB_CUDA(cudaFuncSetAttribute(ks.persistent_mgpu[v], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ks.smem));
  }
  const int vb = p->use_vbem ? 1 : 0;
  SB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, (c->nranks > 1 || c->fused_loopback) ? ks.persistent_mgpu[vb] : ks.persistent[vb],
                                                        EM_THREADS, ks.smem));
  if (occ < 1) { set_error("persistent EM kernel does not fit on an SM"); return SB_ERR_CUDA; }
  if (c->blocks_per_sm > 0) occ = std::min(occ, c->blocks_per_sm);
  c->grid = (uint32_t)(occ * c->n_sm);
  c->occ = occ;
  const uint32_t n_warps = c->grid * (EM_THREADS / 32);

  const uint64_t NP = std::max<uint64_t>(C, M) + 1;
  const uint64_t NS = std::max<uint64_t>(std::max<uint64_t>(C, nnz), (uint64_t)M) + 1;
  SB_TRY(dev_alloc(&c->d_efflens, M));
  SB_TRY(dev_alloc(&c->d_prior, M));
  SB_TRY(dev_alloc(&c->d_alpha0, M));
  SB_TRY(dev_alloc(&c->d_alpha, M));
  SB_TRY(dev_alloc(&c->d_theta, (size_t)M + 4));
  SB_CUDA(cudaMemsetAsync(c->d_theta, 0, ((size_t)M + 4) * 8, st));
  SB_TRY(dev_alloc(&c->d_base, M));
  SB_TRY(dev_alloc(&c->d_cw, nnz));
  SB_TRY(dev_alloc(&c->d_packed, NP));
  SB_TRY(dev_alloc(&c->d_packed2, NP));
  SB_TRY(dev_alloc(&c->d_packed_scan, NP));
  SB_TRY(dev_alloc(&c->d_valid, C));
  SB_TRY(dev_alloc(&c->d_cls_map, C));
  SB_TRY(dev_alloc(&c->d_scalars, 64));
  SB_TRY(dev_alloc(&c->d_tcnt, M));
  SB_TRY(dev_alloc(&c->d_tid_row, M));
  SB_TRY(dev_alloc(&c->d_sort_keys, NS));
  SB_TRY(dev_alloc(&c->d_sort_vals, NS));
  SB_TRY(dev_alloc(&c->d_sort_keys2, NS));
  SB_TRY(dev_alloc(&c->d_sort_vals2, NS));
  SB_TRY(dev_alloc(&c->d_order, NS));
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
    SB_TRY(dev_alloc((unsigned char**)&c->d_tmp, need));
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
  SB_TRY(dev_alloc(&c->m_off, (size_t)Cm + 1));
  SB_TRY(dev_alloc(&c->m_idx, (size_t)nnzm + 1));
  SB_TRY(dev_alloc(&c->m_idx_state, (size_t)nnzm + 1));
  SB_TRY(dev_alloc(&c->m_w, (size_t)nnzm + 1));
  SB_TRY(dev_alloc(&c->d_cnt, (size_t)Cm));
  SB_TRY(dev_alloc(&c->d_scale, (size_t)Cm + 4));
  SB_TRY(dev_alloc(&c->d_ent_cls, (size_t)nnzm));
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
  SB_TRY(dev_alloc(&c->t_off, (size_t)R + 1));
  SB_TRY(dev_alloc(&c->t_idx, (size_t)nnzm + 1));
  SB_TRY(dev_alloc(&c->t_w, (size_t)nnzm + 1));
  SB_TRY(dev_alloc(&c->d_rank_tid, (size_t)R + 1));
  SB_TRY(dev_alloc(&c->d_rowperm, (size_t)R + 1));
  SB_TRY(dev_alloc(&c->d_row_tid, (size_t)R + 1));
  SB_TRY(dev_alloc(&c->r_alpha, (size_t)R + 1));
  SB_TRY(dev_alloc(&c->r_theta, (size_t)R + 4));
  SB_CUDA(cudaMemsetAsync(c->r_theta, 0, ((size_t)R + 4) * 8, st));
  SB_TRY(dev_alloc(&c->r_prior, (size_t)R + 1));
  SB_TRY(dev_alloc(&c->r_base, (size_t)R + 1));
  SB_TRY(dev_alloc(&c->r_alpha0, (size_t)R + 1));
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
  SB_TRY(build_sell(c, c->cm, Cm, nullptr, c->m_off, c->m_idx_state, c->m_w, row_space ? R : M, (uint32_t)c->ovh_p1, n_warps));
  SB_TRY(build_sell(c, c->tm, R, c->d_rowperm, c->t_off, c->t_idx, c->t_w, Cm,
                    (uint32_t)(c->params.use_vbem ? c->ovh_p2 : c->ovh_p1), n_warps));

  // iteration-0 reductions
  double* d_sum0 = c->d_scalars + 16;
  double* d_inact = c->d_scalars + 17;
  k_sum1<<<1, 1024, 0, st>>>(M, c->d_alpha0, c->d_prior, c->d_tid_row, 0, d_sum0);
  k_sum1<<<1, 1024, 0, st>>>(M, c->d_base, c->d_prior, c->d_tid_row, 1, d_inact);
  c->launches += 2;
  SB_CUDA(cudaMemcpyAsync(&c->sum0, d_sum0, 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(&c->inactive_sum, d_inact, 8, cudaMemcpyDeviceToHost, st));
  SB_TRY(dev_alloc(&c->d_sum_partial, (size_t)2 * std::max<uint32_t>(c->grid, 4096)));
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
  s.slice_ptr = m.slice_ptr; s.len = m.len; s.idx = m.idx; s.w = m.w; s.warp_begin = m.warp_begin;
  s.long_rows = m.long_rows; s.csr_idx = m.csr_idx; s.csr_w = m.csr_w;
  s.n_rows = m.n_rows; s.n_slices = m.n_slices; s.n_long = m.n_long;
  s.n_block = m.n_block;
  s.keep_pct = 100;
  return s;
}

static void fill_args(sb_em_ctx* c, EmArgs& A, bool row_space) {
  memset(&A, 0, sizeof(A));
  A.cm = sell_view(c->cm);
  A.tm = sell_view(c->tm);
  A.cm.keep_pct = (uint32_t)c->keep_cm;
  A.tm.keep_pct = (uint32_t)c->keep_tm;
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
  size_t cap = 0;
};
extern "C" sb_comm* sb_comm_create(int rank, int nranks, const void* nccl_uid128, int device) {
  if (nranks < 1 || rank < 0 || rank >= nranks || (nranks > 1 && !nccl_uid128)) { set_error("sb_comm_create: bad arguments"); return nullptr; }
  sb_comm* cm = new sb_comm();
  cm->rank = rank; cm->nranks = nranks; cm->device = device;
  if (nranks == 1) return cm;
  if (nccl_load() != SB_OK) { delete cm; return nullptr; }
  if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreate(&cm->stream) != cudaSuccess) {
    set_error("sb_comm_create: cannot use device %d", device); delete cm; return nullptr;
  }
  NcclUid u;
  memcpy(u.b, nccl_uid128, 128);
  const int r = g_nccl.CommInitRank(&cm->nccl, nranks, u, rank);
  if (r != 0) {
    set_error("ncclCommInitRank -> %d (%s)", r, g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
    cudaStreamDestroy(cm->stream); delete cm; return nullptr;
  }
  return cm;
}
extern "C" void sb_comm_destroy(sb_comm* cm) {
  if (!cm) return;
  if (cm->nccl && g_nccl.CommDestroy) g_nccl.CommDestroy(cm->nccl);
  if (cm->d_buf) { cudaSetDevice(cm->device); cudaFree(cm->d_buf); }
  if (cm->stream) cudaStreamDestroy(cm->stream);
  delete cm;
}
extern "C" int sb_comm_rank(const sb_comm* cm) { return cm ? cm->rank : 0; }
extern "C" int sb_comm_size(const sb_comm* cm) { return cm ? cm->nranks : 1; }
static int comm_reserve(sb_comm* cm, size_t bytes) {
  if (bytes <= cm->cap) return SB_OK;
  SB_CUDA(cudaSetDevice(cm->device));
  if (cm->d_buf) cudaFree(cm->d_buf);
  cm->d_buf = nullptr; cm->cap = 0;
  SB_CUDA(cudaMalloc(&cm->d_buf, bytes + 256));
  cm->cap = bytes;
  return SB_OK;
}
// in place over host buffers; dtype: 0 = f64, 1 = u64; op: 0 sum, 2 max, 3 min (ncclRedOp_t)
extern "C" int sb_comm_allreduce(sb_comm* cm, void* buf, size_t n, int dtype, int op) {
  if (!cm || (n && !buf)) { set_error("null argument"); return SB_ERR_INVALID; }
  if (cm->nranks == 1 || n == 0) return SB_OK;
  SB_TRY(comm_reserve(cm, n * 8));
  SB_CUDA(cudaSetDevice(cm->device));
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
  SB_TRY(comm_reserve(cm, padded * (size_t)(cm->nranks + 1)));
  SB_CUDA(cudaSetDevice(cm->device));
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
  if (!c->x_block) {
    const size_t bytes = XchgLayout(max_txps, 64).bytes() + 64 * 8;   // G * ceil(M / G) <= M + 63 for every G <= 64
    SB_CUDA(cudaMalloc(&c->x_block, bytes));
    SB_CUDA(cudaMemset(c->x_block, 0, bytes));
    SB_CUDA(cudaMalloc(&c->d_xfail, 4));
    c->x_cap = max_txps;
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
  if (!c->d_peers) SB_CUDA(cudaMalloc(&c->d_peers, 64 * sizeof(unsigned char*)));
  SB_CUDA(cudaMemcpy(c->d_peers, ptrs.data(), (size_t)nranks * sizeof(unsigned char*), cudaMemcpyHostToDevice));
  c->rank = rank; c->nranks = nranks;
  c->peers_ready = true;
  c->fused_loopback = (nranks == 1);
  c->prepared = false;   // the index space of the class-major matrix depends on it
  return SB_OK;
}

// Fused path: one cooperative launch per run on every rank; the partial alpha' are pushed to their owners, the owners
// push theta back, all inside the kernel over the peers' exchange blocks (see k_em_persistent_mgpu).
static int em_run_multi_gpu_fused(sb_em_ctx* c, const KernelSet& ks, EmArgs& A, uint32_t* out,
                                  uint32_t* launches, uint32_t* loop_launches, float* loop_ms) {
  cudaStream_t st = c->stream;
  const uint32_t M = c->M;
  const int vb = c->params.use_vbem ? 1 : 0;
  const XchgLayout X(M, (uint32_t)c->nranks);
  SB_CUDA(cudaMemsetAsync(c->d_xfail, 0, 4, st));
  SB_TRY(dev_alloc(&c->d_part, (size_t)M));
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
  SB_CUDA(cudaLaunchCooperativeKernel(ks.persistent_mgpu[vb], dim3(c->grid), dim3(EM_THREADS), args, ks.smem, st));
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
static int em_run_multi_gpu(sb_em_ctx* c, const KernelSet& ks, EmArgs& A, uint32_t* out,
                            uint32_t* launches, uint32_t* loop_launches, float* loop_ms) {
  cudaStream_t st = c->stream;
  const uint32_t M = c->M;
  const int vb = c->params.use_vbem ? 1 : 0;
  if (!c->nccl_comm) { set_error("multi-GPU EM: neither peers (sb_em_peer_open) nor NCCL (sb_em_comm_init) are set up"); return SB_ERR_STATE; }
  SB_TRY(dev_alloc(&c->d_part, (size_t)M));
  SB_TRY(dev_alloc(&c->d_part_red, (size_t)M));
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
    ks.p1[vb]<<<c->grid, EM_THREADS, ks.smem, st>>>(A);
    ks.p2_partial[vb]<<<c->grid, EM_THREADS, ks.smem, st>>>(A);
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
  const KernelSet& ks = kernel_set(c->config);
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
    int r = fused ? em_run_multi_gpu_fused(c, ks, A, out, &launches, &loop_launches, &loop_ms)
                  : em_run_multi_gpu(c, ks, A, out, &launches, &loop_launches, &loop_ms);
    if (r != SB_OK) return r;
  } else if (c->variant == 1) {
    void* args[] = {(void*)&A};
    SB_CUDA(cudaEventRecord(c->ev[2], st));
    SB_CUDA(cudaLaunchCooperativeKernel(ks.persistent[vb], dim3(c->grid), dim3(EM_THREADS), args, ks.smem, st));
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
      ks.p1[vb]<<<c->grid, EM_THREADS, ks.smem, st>>>(A);
      ks.p2[vb]<<<c->grid, EM_THREADS, ks.smem, st>>>(A, it);
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
// at the two grid barriers for the slowest).  One short instrumented run of the persistent
// kernel accumulates, per warp, the duration of P1 and P2 and of their SELL parts (em_kernels.cuh: SB_ACC_*); the
// slice ranges are then re-cut so that   long-row time of the warp (fixed: those rows are dealt by list position)
// + sum over its slices of (measured time density of the warp that ran the slice x modelled slice cost)
// is equal for all warps (water-filling).  Deterministic given the measurements; the results of the iteration do not
// depend on the split (each row's sum is computed by one lane in a fixed order wherever the row lands).
// `unit` = warps that share one range: 1 (ring kernels: a warp owns its range) or 8 (direct kernel: a block's warps take
// slices from the block's range dynamically; the block's time is the mean of its warps').
static int em_recut(sb_em_ctx* c, sb::SellDev& m, uint32_t overhead, const std::vector<unsigned long long>& dbg_w,
                    int slot_total, int slot_sell, uint32_t n_warps_all, uint32_t unit) {
  const uint32_t n_warps = n_warps_all / unit;        // ranges
  if (m.n_slices == 0 || n_warps == 0) return SB_OK;
  std::vector<uint32_t> sp((size_t)m.n_slices + 1), wb_all((size_t)n_warps_all + 1), wb((size_t)n_warps + 1);
  SB_CUDA(cudaMemcpy(sp.data(), m.slice_ptr, sp.size() * 4, cudaMemcpyDeviceToHost));
  SB_CUDA(cudaMemcpy(wb_all.data(), m.warp_begin, wb_all.size() * 4, cudaMemcpyDeviceToHost));
  std::vector<unsigned long long> dbg((size_t)n_warps * 8, 0ull);
  for (uint32_t r = 0; r <= n_warps; ++r) wb[r] = wb_all[(size_t)r * unit];
  for (uint32_t r = 0; r < n_warps; ++r)
    for (int k = 0; k < 8; ++k) {
      unsigned long long a = 0;
      for (uint32_t u = 0; u < unit; ++u) a += dbg_w[((size_t)r * unit + u) * 8 + k];
      dbg[(size_t)r * 8 + k] = a / unit;
    }
  auto cost = [&](uint32_t s) { return (double)(sp[s + 1] - sp[s]) + (sp[s + 1] > sp[s] ? (double)overhead : 0.0); };
  std::vector<double> fixed(n_warps), dens(n_warps, 0.0);
  double sell_total = 0.0, dens_sum = 0.0, work_sum = 0.0;
  for (uint32_t w = 0; w < n_warps; ++w) {
    const double T = (double)dbg[(size_t)w * 8 + slot_total], Ts = std::min(T, (double)dbg[(size_t)w * 8 + slot_sell]);
    double W = 0.0;
    for (uint32_t s = wb[w]; s < wb[w + 1]; ++s) W += cost(s);
    fixed[w] = 0.0 * (T - Ts);   // the long rows are taken from a global queue: every warp's tail is filled, nothing is fixed
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
  // level L with sum_w max(0, L - fixed_w) = total
  double lo = 0.0, hi = total;
  for (double f : fixed) hi = std::max(hi, f + total);
  for (int it = 0; it < 100; ++it) {
    const double L = 0.5 * (lo + hi);
    double acc = 0.0;
    for (double f : fixed) acc += std::max(0.0, L - f);
    if (acc < total) lo = L; else hi = L;
  }
  const double L = hi;
  std::vector<uint32_t> nb((size_t)n_warps + 1);
  double cum = 0.0;
  uint32_t s = 0;
  for (uint32_t w = 0; w < n_warps; ++w) {
    nb[w] = s;
    cum += std::max(0.0, L - fixed[w]);
    while (s < m.n_slices && 0.5 * (F[s] + F[s + 1]) < cum) ++s;   // a slice goes to the warp that holds its midpoint
  }
  nb[n_warps] = m.n_slices;
  nb[0] = 0;
  std::vector<uint32_t> nb_all((size_t)n_warps_all + 1);
  for (uint32_t r = 0; r < n_warps; ++r)
    for (uint32_t u = 0; u < unit; ++u)    // inside a unit the cut points only matter to the ring kernels: even split
      nb_all[(size_t)r * unit + u] = nb[r] + (uint32_t)(((uint64_t)(nb[r + 1] - nb[r]) * u) / unit);
  nb_all[n_warps_all] = m.n_slices;
  SB_CUDA(cudaMemcpy(m.warp_begin, nb_all.data(), nb_all.size() * 4, cudaMemcpyHostToDevice));
  return SB_OK;
}

static int em_rebalance(sb_em_ctx* c) {
  const uint32_t n_warps = c->grid * (EM_THREADS / 32);
  SB_TRY(dev_alloc(&c->d_dbg, (size_t)n_warps * 8));
  SB_CUDA(cudaMemsetAsync(c->d_dbg, 0, (size_t)n_warps * 64, c->stream));
  const sb_em_params saved = c->params;
  const uint32_t saved_it = c->dbg_it;
  const bool saved_en = c->dbg_enabled;
  c->params.min_iter = c->params.max_iter = (uint32_t)std::max(2, c->rebalance_iters + 1);
  c->dbg_it = DBG_ACCUMULATE;
  c->dbg_enabled = true;
  int rc = sb_em_run(c, nullptr);
  c->params = saved; c->dbg_it = saved_it; c->dbg_enabled = saved_en;
  if (rc != SB_OK) return rc;
  std::vector<unsigned long long> dbg((size_t)n_warps * 8);
  SB_CUDA(cudaMemcpy(dbg.data(), c->d_dbg, dbg.size() * 8, cudaMemcpyDeviceToHost));
  const uint32_t unit = 1u;
  SB_TRY(em_recut(c, c->cm, (uint32_t)c->ovh_p1, dbg, 0, 3, n_warps, unit));
  SB_TRY(em_recut(c, c->tm, (uint32_t)(c->params.use_vbem ? c->ovh_p2 : c->ovh_p1), dbg, 1, 4, n_warps, unit));
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
  if (!c->d_flush || c->flush_bytes < bytes) {
    SB_TRY(dev_alloc((unsigned char**)&c->d_flush, bytes));
    c->flush_bytes = bytes;
  }
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

extern "C" int sb_em_debug_timeline(sb_em_ctx* c, uint64_t* out, uint32_t iteration) {
  if (!c) { set_error("null argument"); return SB_ERR_INVALID; }
  if (!c->prepared) { set_error("not prepared"); return SB_ERR_STATE; }
  SB_CUDA(cudaSetDevice(c->device));
  const uint32_t n_warps = c->grid * (EM_THREADS / 32);
  if (!out) {
    // arm: the next sb_em_run records iteration `iteration`
    SB_TRY(dev_alloc(&c->d_dbg, (size_t)n_warps * 8));
    SB_CUDA(cudaMemset(c->d_dbg, 0, (size_t)n_warps * 64));
    c->dbg_it = iteration;
    c->dbg_enabled = true;
    return (int)n_warps;
  }
  if (!c->d_dbg) { set_error("timeline not armed"); return SB_ERR_STATE; }
  SB_CUDA(cudaMemcpy(out, c->d_dbg, (size_t)n_warps * 64, cudaMemcpyDeviceToHost));
  return (int)n_warps;
}

#include "sampling.cuh"
