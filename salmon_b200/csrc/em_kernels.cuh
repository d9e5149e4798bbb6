// em_kernels.cuh -- the EM / VBEM iteration kernels (sm_90a).
//
// One iteration = two segmented reductions over the class<->transcript map held
// twice in HBM (class-major and transcript-major), no atomics on the data path,
// fixed summation order:
//   P1 (class-major):  denom_c = sum_i theta[t_i] * w_ci ;  scale_c = count_c / denom_c
//   P2 (txp-major):    alpha'_t = base_t + theta_t * sum_c w_ct * scale_c, convergence
//                      test, theta'_t (VBEM: exp(digamma(alpha'+prior) - logNorm))
// Reference arithmetic: src/inference/CollapsedEMOptimizer.cpp:178-234 (EMUpdate_),
// :241-328 (VBEMUpdate_), :945-957 (convergence + swap).
//
// Layout: sliced ELL, slice height 32 (SELL-32).  Rows are ordered for gather locality
// (classes by first transcript id, transcripts by id) and then bucketed by length inside
// groups of rows (SELL_GROUP by default), so the 32 rows of a slice have (nearly) equal length.  A
// warp owns a slice: lane = row, each lane accumulates its row sequentially in label order.
// A slice is exactly as wide as its longest row; an entry is a 16-bit index relative to the
// slice's base index + an 8-byte weight, 10 bytes (run_phase has the column order).  A slice
// whose indices span more than 16 bits hands its rows to the long-row path.  Slices are dealt to warps in contiguous
// ranges cut at prepare time -- first by a column count model, then re-cut from MEASURED per-warp phase times (em.cu:
// rebalance).  Rows longer than LMAX are reduced by a warp / a whole block from their CSR copy.
//
// Design points (a warp's time goes to waiting at the grid barriers, L2 gather latency and dependent FP64 chains):
//   * a warp streams its slice range through its ring, then takes long rows from the phase's work queue until it is
//     empty.  Every SELL row is summed by one lane in label order;
//   * inside a slice the gathers of two groups of 4 columns are issued before either is consumed, and the epilogue
//     operands of slice s+1 are loaded while slice s is reduced (gathers are not pipelined across slices);
//   * the VBEM epilogue is one branch-light function (em_math.h) instead of a Boost-style
//     digamma with data-dependent loops followed by exp();
//   * VBEM / EM are template parameters: the NaN guard of plain EM (:206) is compiled out of VBEM;
//   * the multi-GPU kernel reduce-scatters by PUSHING partials to the owner of each transcript
//     slice while P2 runs; the owner applies the update and pushes theta back (see below).
#pragma once
#include <cooperative_groups.h>
#include <float.h>

#include "common.cuh"
#include "em_math.h"

namespace sb {
namespace cg = cooperative_groups;

constexpr uint32_t LMAX = 96;                // rows longer than this leave the lane-per-row SELL path
constexpr uint32_t LWARP = 2048;             // ... and are reduced by one warp (<= LWARP) or one block
constexpr int EM_THREADS = 256;
// Warp ring (WarpRing): EM_CH columns per chunk, EM_RING chunks in flight per warp, EM_MIN_BLOCKS resident blocks per
// SM (__launch_bounds__).  DESIGN.md 3.4 has the H100 measurements of the other ring shapes.
constexpr int EM_CH = 8;
constexpr int EM_RING = 4;
constexpr int EM_MIN_BLOCKS = 2;
constexpr double DIGAMMA_MIN = 1e-10;        // CollapsedEMOptimizer.cpp:43
constexpr double MIN_EQ_W = DBL_MIN;         // :40
constexpr double ALPHA_CHECK_CUTOFF = 1e-2;  // :884
constexpr uint16_t LEN_LONG = 0xFFFFu;       // row handled by the warp / block path
constexpr uint16_t IDX_PAD = 0xFFFFu;        // SELL index of a padding entry: gathers the zero slot
constexpr uint32_t DBG_ACCUMULATE = 0xFFFFFFFFu;   // dbg_it value: accumulate phase durations over all iterations >= 1
constexpr uint32_t DBG_SLOTS = 16;                  // timeline slots per warp (see SB_DBG)

// One segmented matrix in SELL-32 form (+ CSR copy of the long rows only).
struct Sell {
  const uint32_t* slice_ptr;   // [n_slices+1] first column of each slice
  const uint32_t* base;        // [n_slices] smallest gather index of the slice's SELL rows
  const uint16_t* len;         // [n_rows] entries per row (LEN_LONG: long path)
  const uint16_t* idx;         // [n_cols*32] gather index - base of the slice (IDX_PAD: padding)
  const double* w;             // [n_cols*32]
  const uint32_t* warp_begin;  // [n_warps+1] slice range per warp, streamed through its ring
  // long rows: (row, first entry, end entry) triples into csr_idx / csr_w
  const uint32_t* long_rows;   // [3*n_long]
  const uint32_t* csr_idx;
  const double* csr_w;
  uint32_t n_rows, n_slices, n_long;
  uint32_t n_block;            // the first n_block long rows (longest first) take the block path
  uint32_t zero;               // gather slot that always holds 0.0 (what padding entries read)
};

struct EmArgs {
  Sell cm;                      // rows = kept multi-transcript classes; idx = state index
  Sell tm;                      // rows = active transcripts;           idx = class id
  const double* c_cnt;          // [classes] count as f64
  double* scale;                // [classes] count / denom
  // iteration state.  Single GPU: indexed by ROW of tm (cm.idx holds rows).  Multi GPU:
  // indexed by transcript id (cm.idx holds ids) and row_tid maps tm rows to ids.
  double* alpha; double* theta; const double* prior; const double* base;
  const uint32_t* row_tid;
  const uint32_t* tid_row;      // multi-GPU: row of a transcript id (0xffffffff: locally inactive)
  double* part_out;             // multi-GPU (NCCL path): this rank's alpha' share per transcript id
  // reductions
  double* sum_partial;          // [2][grid]
  unsigned long long* maxrel;   // [2] bit pattern of a non-negative double
  double inactive_sum; double sum0;
  double sum_scale;             // 2^s: unit of the fixed-point sum of (alpha' + prior), chosen at prepare (P2Acc)
  double tol;
  double min_eq_w;              // denominator guard: DBL_MIN (optimize) / denorm_min (serial EM)
  double first_bias;            // 1.0 for optimize's first plain-EM iteration (:812,:821), else 0
  uint32_t min_iter, max_iter;
  uint32_t* out;                // [0]=iters [1]=converged [2]=maxrel slot
  unsigned long long* dbg;      // optional [n_warps*DBG_SLOTS] phase timestamps (ns) of iteration dbg_it
  uint32_t dbg_it;
  unsigned int* lq;             // [2] long-row work queues of the persistent kernels (P1, P2)
  // multi-GPU, fused exchange over peer memory (k_em_persistent_mgpu): every rank owns one exchange block (layout:
  // XchgLayout) mapped into every peer (CUDA IPC, NVLink P2P)
  unsigned char* const* peers;  // [nranks] base pointers of the exchange blocks (peers[rank] = own)
  uint32_t rank, nranks, M;
  uint32_t push_pass;           // fused path: partials go to the owners in a coalesced pass (else from the row epilogues)
  unsigned long long epoch0;    // barrier epochs consumed by earlier launches
  uint32_t* xfail;              // set when a peer did not show up in time
};

// Exchange block of one rank (bytes from its base; S = ceil(M / G) transcripts per owner slice).  The per-iteration
// traffic travels as flagged 16-byte lines {lo32, epoch, hi32, epoch} (the NCCL "LL" idea: each 8-byte half carries its
// own flag and is written atomically, so the receiver polls the data itself and no fence or barrier orders it):
//   flags  [64] u64            end-of-run barrier: flags[q] = last epoch rank q has signalled to this rank
//   theta  [M + 4] f64         plain copy of the replicated state, what this rank's P1 gathers from
//   alpha  [M] f64             final alpha, all-gathered once after the loop
//   llth   [M] lines           theta' pushed by the owners of the other slices
//   llaux  [G][XAUX][2] lines  per source rank, per block: {sum(alpha'+prior), max rel diff} of its share of its slice
//   llrecv [G][S] lines        partial alpha' of this rank's slice, one row per source rank
constexpr uint32_t XAUX = 1024;   // blocks per rank the aux area has room for
struct XchgLayout {
  uint32_t M, G, S;
  __host__ __device__ XchgLayout(uint32_t m, uint32_t g) : M(m), G(g), S((m + g - 1) / g) {}
  __host__ __device__ size_t off_flags() const { return 0; }
  __host__ __device__ size_t off_theta() const { return 64 * 8; }
  __host__ __device__ size_t off_alpha() const { return off_theta() + ((size_t)M + 4) * 8; }
  __host__ __device__ size_t off_llth() const { return (off_alpha() + (size_t)M * 8 + 15) & ~(size_t)15; }
  __host__ __device__ size_t off_llaux() const { return off_llth() + (size_t)M * 16; }
  __host__ __device__ size_t off_llrecv() const { return off_llaux() + (size_t)G * XAUX * 2 * 16; }
  __host__ __device__ size_t bytes() const { return off_llrecv() + (size_t)G * S * 16; }
};

__device__ __forceinline__ unsigned long long gtime_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// sum of (alpha' + prior) over my rows, in units of 1 / A.sum_scale (2^-20 unless the table is large): integer
// additions commute, so the total -- and with it logNorm and every later bit of the run -- does not depend on which
// warp took which row (dynamic long-row queue) or on how the ranges were cut (measured re-balancing): runs are
// bit-reproducible.  (logNorm only has to be the same everywhere: any common factor of theta cancels in P1/P2.)
// sb_em_prepare picks the scale so that the grid's total stays below 2^62 (em.cu: sum_scale_log2).
struct P2Acc {
  long long isum;
  double maxrel;  // max rel diff over my rows
};
__device__ __forceinline__ long long warp_sum_ll(long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// all threads of the block; scratch: >= 32 doubles of shared memory; result valid in every thread
__device__ __forceinline__ long long block_sum_ll(long long v, double* scratch) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int nw = (blockDim.x + 31) >> 5;
  v = warp_sum_ll(v);
  __syncthreads();
  if (lane == 0) scratch[wid] = __longlong_as_double(v);
  __syncthreads();
  long long r = (lane < nw) ? __double_as_longlong(scratch[lane]) : 0ll;
  return warp_sum_ll(r);
}

// Per-warp TMA ring: each warp streams ITS contiguous column range of the SELL arrays
// through a private shared-memory ring with 1-D bulk copies (lane 0 is the producer, the
// warp is the consumer), so the index/weight stream is never a dependent load and no
// block-level barrier exists on the data path.
struct __align__(128) WarpRing {
  double w[EM_RING][EM_CH * 32];
  uint16_t idx[EM_RING][EM_CH * 32];
};
constexpr int EM_WARPS = EM_THREADS / 32;
// dynamic shared memory of every iteration kernel: the warps' rings, their mbarriers, the block scratch
constexpr size_t EM_SMEM = sizeof(WarpRing) * EM_WARPS + EM_WARPS * EM_RING * 8 + 40 * 8;

struct WarpCtx {
  WarpRing* ring;
  uint64_t* bars;        // [EM_RING]
  uint32_t phase_bits;   // mbarrier parity per stage
  double* scratch;       // block scratch (40 doubles)
  uint64_t pol_stream;   // L2 eviction policy of the bulk copies (evict_first: the layouts exceed the L2)
  unsigned long long* dbg;  // optional: the warp's timeline row (end of the home stream, queue items taken)
  unsigned long long* dbg_acc;   // optional: accumulates (end of the SELL part - t0)
  unsigned long long t0;
};

__device__ __forceinline__ void warp_setup(WarpCtx& W, unsigned char* smem) {
  const uint32_t wid = threadIdx.x >> 5;
  W.ring = reinterpret_cast<WarpRing*>(smem) + wid;
  W.bars = reinterpret_cast<uint64_t*>(smem + sizeof(WarpRing) * EM_WARPS) + wid * EM_RING;
  W.scratch = reinterpret_cast<double*>(smem + sizeof(WarpRing) * EM_WARPS + EM_WARPS * EM_RING * 8);
  W.phase_bits = 0;
  W.dbg = nullptr;
  W.dbg_acc = nullptr;
  W.t0 = 0;
  W.pol_stream = l2_policy_evict_first();
  if ((threadIdx.x & 31u) == 0) {
#pragma unroll
    for (int s = 0; s < EM_RING; ++s) mbar_init(&W.bars[s], 1);
    mbar_fence_init();
  }
  __syncthreads();
}

// operands of a row's epilogue, fetched while the row's columns stream
struct RowOps {
  double x0, x1, x2, x3;
  uint32_t len;
};
template <int PHASE>
__device__ __forceinline__ RowOps load_ops(const EmArgs& A, const Sell& S, uint32_t row) {
  RowOps o;
  o.x0 = o.x1 = o.x2 = o.x3 = 0.0;
  o.len = LEN_LONG;
  if (row < S.n_rows) {
    o.len = __ldg(&S.len[row]);
    if (PHASE == 1) {
      o.x0 = __ldg(&A.c_cnt[row]);
    } else if (PHASE == 2) {
      o.x0 = A.theta[row];
      o.x1 = __ldg(&A.prior[row]);
      o.x2 = __ldg(&A.base[row]);
      o.x3 = A.alpha[row];
    } else {
      const uint32_t t = __ldg(&A.row_tid[row]);
      o.x0 = A.theta[t];
      o.x2 = __ldg(&A.base[t]);
      o.x3 = __longlong_as_double((long long)t);   // the transcript id rides along
    }
  }
  return o;
}

// theta' of one transcript from its new alpha (both algorithms)
template <bool VBEM>
__device__ __forceinline__ double theta_of(double na, double ap, double logNorm) {
  if (VBEM) return (ap > DIGAMMA_MIN) ? exp_digamma_shifted(ap, logNorm) : 0.0;
  return na;
}

// PHASE 1: scale of a class.  PHASE 2: single-GPU update of a transcript.  PHASE 3: multi-GPU partial alpha' of a
// transcript, delivered by `deliver(t, value)` (NCCL path: into part_out; fused path: pushed to the owner's recv row).
template <int PHASE, bool VBEM, class Deliver>
__device__ __forceinline__ void row_finish(const EmArgs& A, uint32_t row, const RowOps& o, double acc,
                                           double logNorm, double bias, P2Acc& pa, Deliver&& deliver) {
  if (o.len == LEN_LONG) return;  // beyond the last row, or a long row (other path)
  if (PHASE == 1) {
    A.scale[row] = (acc <= A.min_eq_w) ? 0.0 : o.x0 / acc;
  } else if (PHASE == 2) {
    const double th = o.x0, pr = o.x1;
    double na = o.x2 + bias;
    if (th > 0.0) na = fma(th, acc, na);
    if (na > ALPHA_CHECK_CUTOFF) pa.maxrel = fmax(pa.maxrel, fabs(o.x3 - na) / na);
    A.alpha[row] = na;
    const double ap = na + pr;
    pa.isum += __double2ll_rn(ap * A.sum_scale);
    A.theta[row] = theta_of<VBEM>(na, ap, logNorm);
  } else {
    const uint32_t t = (uint32_t)__double_as_longlong(o.x3);
    double na = o.x2;
    if (o.x0 > 0.0) na = fma(o.x0, acc, na);
    deliver(t, na);
  }
}

// static home stream range of one warp in one matrix (the matrices never change)
struct WarpRange {
  uint32_t s0, s1, cbeg, cend;
};
__device__ __forceinline__ WarpRange load_range(const Sell& S, uint32_t gwarp) {
  WarpRange r;
  r.s0 = __ldg(&S.warp_begin[gwarp]);
  r.s1 = __ldg(&S.warp_begin[gwarp + 1]);
  r.cbeg = __ldg(&S.slice_ptr[r.s0]);
  r.cend = __ldg(&S.slice_ptr[r.s1]);
  return r;
}
__device__ __forceinline__ void ring_issue(const Sell& S, WarpCtx& W, const WarpRange& R, uint32_t k) {
  if ((threadIdx.x & 31u) == 0) {
    const uint32_t c = R.cbeg + k * EM_CH;
    const uint32_t cols = min((uint32_t)EM_CH, R.cend - c);
    const int st = k % EM_RING;
    mbar_arrive_expect_tx(&W.bars[st], cols * 320u);
    bulk_g2s_hint(W.ring->w[st], S.w + (size_t)c * 32u, cols * 256u, &W.bars[st], W.pol_stream);
    bulk_g2s_hint(W.ring->idx[st], S.idx + (size_t)c * 32u, cols * 64u, &W.bars[st], W.pol_stream);
  }
}
// fill the ring with the first chunks of a phase.  The matrices are read-only, so this
// may run BEFORE the grid barrier that precedes the phase: the stream then lands while
// the grid synchronises and is never on the critical path.
__device__ __forceinline__ void ring_prefetch(const Sell& S, WarpCtx& W, const WarpRange& R) {
  const uint32_t nchunks = (R.cend - R.cbeg + EM_CH - 1) / EM_CH;
#pragma unroll
  for (int k = 0; k < EM_RING; ++k)
    if ((uint32_t)k < nchunks) ring_issue(S, W, R, k);
}
// wait for the chunks a speculative ring_prefetch put in flight (before the block retires)
__device__ __forceinline__ void ring_drain(WarpCtx& W, const WarpRange& R) {
  const uint32_t nchunks = (R.cend - R.cbeg + EM_CH - 1) / EM_CH;
#pragma unroll
  for (int k = 0; k < EM_RING; ++k)
    if ((uint32_t)k < nchunks) mbar_wait(&W.bars[k], (W.phase_bits >> k) & 1u);
}

// Where sell_rows reads the entries of column c, counted from the first column of the warp's range.  A slice of
// width W = its longest row has W / 4 GROUPS of 4 columns and then W % 4 remainder columns.  Inside a group the layout
// is lane-major,
//   idx[(group * 32 + lane) * 4 + j],  w[(group * 32 + lane) * 4 + j]        j = 0..3,
// so a lane reads its four indices with ONE 8-byte load and its four weights with two 16-byte loads and issues the
// four gathers together; a remainder column is plain column-major (idx[col * 32 + lane]).
//
// The range streams through the warp's TMA ring, a circular buffer of EM_CH * EM_RING columns: column c sits at ring
// column c % (EM_CH * EM_RING), so a group that straddles two chunks is read in place (each lane's four entries are in
// one chunk: a chunk boundary falls on a multiple of 32 entries) and a chunk is handed back once the stream has passed
// its last column.
struct RingCols {
  static constexpr uint32_t RC = (uint32_t)(EM_CH * EM_RING);   // ring capacity in columns
  const Sell& S;
  WarpCtx& W;
  const WarpRange& R;
  uint32_t lane, nchunks;
  uint32_t done = 0, ready = 0;             // chunks handed back to the producer / waited for
  // columns [c0, c1) resident: hand back the chunks wholly before c0, wait for those up to column c1 - 1
  __device__ __forceinline__ void need(uint32_t c0, uint32_t c1) {
    for (; (done + 1u) * EM_CH <= c0; ++done) {
      __syncwarp();
      if (done + EM_RING < nchunks) ring_issue(S, W, R, done + EM_RING);
    }
    for (; ready * EM_CH < c1; ++ready) {
      const int st = ready % EM_RING;
      mbar_wait(&W.bars[st], (W.phase_bits >> st) & 1u);
      W.phase_bits ^= (1u << st);
    }
  }
  // ring entry of this lane's first entry in the group that starts at column c
  __device__ __forceinline__ uint32_t group_at(uint32_t c) const {
    const uint32_t p = (c % RC) * 32u + lane * 4u;
    return p >= RC * 32u ? p - RC * 32u : p;
  }
  __device__ __forceinline__ uint2 idx4(uint32_t c) const {
    return *reinterpret_cast<const uint2*>(&W.ring->idx[0][0] + group_at(c));
  }
  __device__ __forceinline__ double2 w4(uint32_t c, uint32_t j) const {
    return *reinterpret_cast<const double2*>(&W.ring->w[0][0] + group_at(c) + j);
  }
  __device__ __forceinline__ uint32_t idx1(uint32_t c) const { return (&W.ring->idx[0][0])[(c % RC) * 32u + lane]; }
  __device__ __forceinline__ double w1(uint32_t c) const { return (&W.ring->w[0][0])[(c % RC) * 32u + lane]; }
};
// The rows of slices [s0, s1), whose columns are [cbeg, cend) of the layout, read through the ring `cols`.  Every row
// is summed by one lane in label order -- pairs of groups (8 gathers in flight), then a single group, then the
// remainder columns -- and finished (row_finish) with operands loaded one slice ahead.  The remainder is the same for
// the 32 lanes, so it is a warp-uniform branch, not a per-lane predicate.  Padding entries (a row shorter than its
// slice) have weight 0 and gather a slot that always holds 0.0, so a row's sum is its label-order sum.
template <int PHASE, bool VBEM, class Deliver>
__device__ __forceinline__ void sell_rows(const EmArgs& A, const Sell& S, RingCols& cols, uint32_t s0,
                                          uint32_t s1, uint32_t cbeg, uint32_t cend, double logNorm, double bias,
                                          P2Acc& pa, Deliver&& deliver) {
  // theta / scale are rewritten by other blocks inside the persistent kernel: plain
  // coherent loads only, never ld.global.nc.
  const double* gsrc = (PHASE == 1) ? A.theta : A.scale;
  constexpr bool GUARD = (PHASE == 1) && !VBEM;   // plain EM skips NaN products (:206)
  const uint32_t lane = threadIdx.x & 31u;
  auto slot = [&](uint32_t base, uint32_t u) { return u == IDX_PAD ? S.zero : base + u; };
  auto fma1 = [&](double& acc, double g, double w) {
    if (GUARD) {
      const double v = g * w;
      if (!isnan(v)) acc += v;
    } else {
      acc = fma(g, w, acc);
    }
  };
  // one group of four columns: the gathers of the group are issued before any of them is consumed
  struct Group {
    double g0, g1, g2, g3;
    double2 wa, wb;
  };
  auto group_load = [&](uint32_t c, uint32_t base) {
    const uint2 i2 = cols.idx4(c);
    Group q;
    q.g0 = gsrc[slot(base, i2.x & 0xFFFFu)];
    q.g1 = gsrc[slot(base, i2.x >> 16)];
    q.g2 = gsrc[slot(base, i2.y & 0xFFFFu)];
    q.g3 = gsrc[slot(base, i2.y >> 16)];
    q.wa = cols.w4(c, 0u);
    q.wb = cols.w4(c, 2u);
    return q;
  };
  auto group_fma = [&](double& acc, const Group& q) {
    fma1(acc, q.g0, q.wa.x); fma1(acc, q.g1, q.wa.y); fma1(acc, q.g2, q.wb.x); fma1(acc, q.g3, q.wb.y);
  };
  uint32_t sbase = s0;
  uint32_t sp = (s0 + lane < s1) ? __ldg(&S.slice_ptr[s0 + lane + 1]) : cend;   // end columns of 32 slices
  uint32_t sb = (s0 + lane < s1) ? __ldg(&S.base[s0 + lane]) : 0u;              // and their base indices
  uint32_t c = 0;                           // column, counted from cbeg
  RowOps ops_next = load_ops<PHASE>(A, S, s0 * 32u + lane);
  for (uint32_t s = s0; s < s1; ++s) {
    if (s - sbase == 32u) {
      sbase = s;
      sp = (s + lane < s1) ? __ldg(&S.slice_ptr[s + lane + 1]) : cend;
      sb = (s + lane < s1) ? __ldg(&S.base[s + lane]) : 0u;
    }
    const uint32_t slice_end = __shfl_sync(0xffffffffu, sp, (int)(s - sbase)) - cbeg;
    const uint32_t base = __shfl_sync(0xffffffffu, sb, (int)(s - sbase));
    uint32_t ng = (slice_end - c) >> 2;
    const uint32_t rem = (slice_end - c) & 3u;
    // epilogue operands one slice ahead: the loads of slice s+1 are in flight while slice s is reduced and finished
    const RowOps ops = ops_next;
    if (s + 1u < s1) ops_next = load_ops<PHASE>(A, S, (s + 1u) * 32u + lane);
    if (slice_end == c) continue;           // only long / absent rows
    double acc = 0.0;
    for (; ng >= 2; ng -= 2, c += 8) {      // two groups: 8 gathers in flight
      cols.need(c, c + 8);
      const Group qa = group_load(c, base);
      const Group qb = group_load(c + 4, base);
      group_fma(acc, qa);
      group_fma(acc, qb);
    }
    if (ng) {
      cols.need(c, c + 4);
      group_fma(acc, group_load(c, base));
      c += 4;
    }
    if (rem) {                              // 1-3 remainder columns, column-major
      cols.need(c, c + rem);
      const double g0 = gsrc[slot(base, cols.idx1(c))];
      if (rem == 1) {
        fma1(acc, g0, cols.w1(c));
      } else if (rem == 2) {
        const double g1 = gsrc[slot(base, cols.idx1(c + 1))];
        fma1(acc, g0, cols.w1(c)); fma1(acc, g1, cols.w1(c + 1));
      } else {
        const double g1 = gsrc[slot(base, cols.idx1(c + 1))], g2 = gsrc[slot(base, cols.idx1(c + 2))];
        fma1(acc, g0, cols.w1(c)); fma1(acc, g1, cols.w1(c + 1)); fma1(acc, g2, cols.w1(c + 2));
      }
      c += rem;
    }
    row_finish<PHASE, VBEM>(A, s * 32u + lane, ops, acc, logNorm, bias, pa, deliver);
  }
}

struct Nothing {
  __device__ __forceinline__ void operator()() const {}
};

// One phase of a warp: its home range through the ring, then `after_home` (the ring is idle from there on: the caller
// hands it to the next phase's home range), then the block-path rows, then the phase's work queue: items [0, n_mid)
// are the warp-path long rows (LMAX < len <= LWARP), longest first, so the short ones fill the end of the phase.
template <int PHASE, bool VBEM, bool DYNQ, class AfterHome, class Deliver>
__device__ __forceinline__ void run_phase(const EmArgs& A, WarpCtx& W, const WarpRange& R,
                                          uint32_t bid, uint32_t nblk, double logNorm, double bias,
                                          P2Acc& pa, AfterHome&& after_home, Deliver&& deliver) {
  static_assert(EM_CH >= 8 && EM_RING >= 2, "two groups in flight span at most two resident chunks");
  const Sell& S = (PHASE == 1) ? A.cm : A.tm;
  const double* gsrc = (PHASE == 1) ? A.theta : A.scale;
  constexpr bool GUARD = (PHASE == 1) && !VBEM;   // plain EM skips NaN products (:206)
  const uint32_t lane = threadIdx.x & 31u;
  if (R.s1 > R.s0 && R.cend > R.cbeg) {
    RingCols rc{S, W, R, lane, (R.cend - R.cbeg + EM_CH - 1) / EM_CH};
    sell_rows<PHASE, VBEM>(A, S, rc, R.s0, R.s1, R.cbeg, R.cend, logNorm, bias, pa, deliver);
    // the chunks still held are not handed back: nothing more to stream in this phase
  }
  unsigned long long* const dbg = W.dbg;
  if (dbg && lane == 0) dbg[PHASE == 1 ? 8 : 7] = gtime_ns();
  if (W.dbg_acc && lane == 0) *W.dbg_acc += gtime_ns() - W.t0;
  __syncwarp();   // every lane has read its last ring entry before lane 0 refills the ring
  after_home();
  // very long rows: whole block per row, fixed-order tree reduction
  for (uint32_t li = bid; li < S.n_block; li += nblk) {
    const uint32_t r = __ldg(&S.long_rows[3 * li]);
    const uint32_t b = __ldg(&S.long_rows[3 * li + 1]);
    const uint32_t e = __ldg(&S.long_rows[3 * li + 2]);
    double a0 = 0.0, a1 = 0.0;
    uint32_t k = b + threadIdx.x;
    for (; k + EM_THREADS < e; k += 2 * EM_THREADS) {
      const uint32_t i0 = __ldg(&S.csr_idx[k]), i1 = __ldg(&S.csr_idx[k + EM_THREADS]);
      double v0 = gsrc[i0] * __ldg(&S.csr_w[k]);
      double v1 = gsrc[i1] * __ldg(&S.csr_w[k + EM_THREADS]);
      if (GUARD) {
        if (isnan(v0)) v0 = 0.0;
        if (isnan(v1)) v1 = 0.0;
      }
      a0 += v0;
      a1 += v1;
    }
    if (k < e) {
      double v = gsrc[__ldg(&S.csr_idx[k])] * __ldg(&S.csr_w[k]);
      if (GUARD && isnan(v)) v = 0.0;
      a0 += v;
    }
    const double acc = block_reduce<false>(a0 + a1, W.scratch);
    if (threadIdx.x == 0) {
      RowOps o = load_ops<PHASE>(A, S, r);
      o.len = 0;  // force the epilogue for this long row
      row_finish<PHASE, VBEM>(A, r, o, acc, logNorm, bias, pa, deliver);
    }
    __syncthreads();
  }
  // The work queue.  Persistent kernels (DYNQ): items are taken one at a time from a global queue by whichever warp is
  // free (the next claim is in flight while an item is reduced), so the tail of a phase is filled evenly -- dealt
  // statically, the warp that draws the longest row ends the phase well after the others.  Claiming two ahead measured
  // slower: the first free warp took the two longest rows.  Per-phase launches: dealt round-robin over the warps.
  {
    const uint32_t gw = bid * EM_WARPS + (threadIdx.x >> 5);
    const uint32_t nw = nblk * EM_WARPS;
    const uint32_t n_mid = S.n_long - S.n_block;
    unsigned int* queue = A.lq + ((PHASE == 1) ? 0 : 1);
    // lane k keeps the sum of the k-th long row this warp reduced; the epilogues (digamma, exp)
    // then run lane-parallel, 32 rows at a time.
    uint32_t cnt = 0, myrow = 0xffffffffu;
    double myacc = 0.0;
    auto flush = [&]() {
      if (myrow != 0xffffffffu) {
        RowOps o = load_ops<PHASE>(A, S, myrow);
        o.len = 0;  // force the epilogue for a long row
        row_finish<PHASE, VBEM>(A, myrow, o, myacc, logNorm, bias, pa, deliver);
      }
      myrow = 0xffffffffu;
      cnt = 0;
    };
    auto claim = [&]() -> uint32_t {
      uint32_t q = 0;
      if (lane == 0) q = atomicAdd(queue, 1u);
      return q;               // lane 0's value is broadcast when it is consumed
    };
    uint32_t q_next;
    if (DYNQ) q_next = n_mid ? claim() : 0u; else q_next = gw;
    // timeline: what this warp took from the queue (slots zeroed when the timeline is armed)
    unsigned long long* const qs = (dbg && lane == 0) ? dbg + (PHASE == 1 ? 9 : 11) : nullptr;
    for (;;) {
      const uint32_t q = DYNQ ? __shfl_sync(0xffffffffu, q_next, 0) : q_next;
      if (q >= n_mid) break;
      if (DYNQ) q_next = claim(); else q_next = q + nw;
      // one warp per row, lanes stride the CSR copy with four independent gathers in flight, fixed shuffle tree.
      // The CSR loads of step k + 128 are issued before the gathers of step k are consumed.
      const uint32_t li = S.n_block + q;
      const uint32_t r = __ldg(&S.long_rows[3 * li]);
      const uint32_t b = __ldg(&S.long_rows[3 * li + 1]);
      const uint32_t e = __ldg(&S.long_rows[3 * li + 2]);
      double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
      uint32_t k = b + lane;
      uint32_t i0 = 0u, i1 = 0u, i2 = 0u, i3 = 0u;
      double w0 = 0.0, w1 = 0.0, w2 = 0.0, w3 = 0.0;
      if (k + 96 < e) {
        i0 = __ldg(&S.csr_idx[k]); i1 = __ldg(&S.csr_idx[k + 32]);
        i2 = __ldg(&S.csr_idx[k + 64]); i3 = __ldg(&S.csr_idx[k + 96]);
        w0 = __ldg(&S.csr_w[k]); w1 = __ldg(&S.csr_w[k + 32]);
        w2 = __ldg(&S.csr_w[k + 64]); w3 = __ldg(&S.csr_w[k + 96]);
      }
      for (; k + 96 < e; k += 128) {
        const double g0 = gsrc[i0], g1 = gsrc[i1], g2 = gsrc[i2], g3 = gsrc[i3];
        const double x0 = w0, x1 = w1, x2 = w2, x3 = w3;
        // no branch around the next step's loads (a last step reloads its own entries), so that they can be issued
        // ahead of this step's FMAs
        const uint32_t kn = (k + 224 < e) ? k + 128 : k;
        i0 = __ldg(&S.csr_idx[kn]); i1 = __ldg(&S.csr_idx[kn + 32]);
        i2 = __ldg(&S.csr_idx[kn + 64]); i3 = __ldg(&S.csr_idx[kn + 96]);
        w0 = __ldg(&S.csr_w[kn]); w1 = __ldg(&S.csr_w[kn + 32]);
        w2 = __ldg(&S.csr_w[kn + 64]); w3 = __ldg(&S.csr_w[kn + 96]);
        double v0 = g0 * x0, v1 = g1 * x1;
        double v2 = g2 * x2, v3 = g3 * x3;
        if (GUARD) {
          if (isnan(v0)) v0 = 0.0;
          if (isnan(v1)) v1 = 0.0;
          if (isnan(v2)) v2 = 0.0;
          if (isnan(v3)) v3 = 0.0;
        }
        a0 += v0; a1 += v1; a2 += v2; a3 += v3;
      }
      {
        // tail: up to three more strides, issued together
        const uint32_t j0 = (k < e) ? __ldg(&S.csr_idx[k]) : 0u;
        const uint32_t j1 = (k + 32 < e) ? __ldg(&S.csr_idx[k + 32]) : 0u;
        const uint32_t j2 = (k + 64 < e) ? __ldg(&S.csr_idx[k + 64]) : 0u;
        double v0 = (k < e) ? gsrc[j0] * __ldg(&S.csr_w[k]) : 0.0;
        double v1 = (k + 32 < e) ? gsrc[j1] * __ldg(&S.csr_w[k + 32]) : 0.0;
        double v2 = (k + 64 < e) ? gsrc[j2] * __ldg(&S.csr_w[k + 64]) : 0.0;
        if (GUARD) {
          if (isnan(v0)) v0 = 0.0;
          if (isnan(v1)) v1 = 0.0;
          if (isnan(v2)) v2 = 0.0;
        }
        a0 += v0; a1 += v1; a2 += v2;
      }
      const double acc = warp_sum((a0 + a1) + (a2 + a3));
      if (lane == cnt) { myacc = acc; myrow = r; }
      if (++cnt == 32) flush();
      if (qs) { qs[0] += (1ull << 32) | (e - b); qs[1] = max(qs[1], (unsigned long long)(e - b)); }
    }
    flush();
  }
}

struct NoDeliver {
  __device__ __forceinline__ void operator()(uint32_t, double) const {}
};
struct DeliverLocal {          // NCCL path: this rank's share of alpha' per transcript id
  double* part;
  __device__ __forceinline__ void operator()(uint32_t t, double v) const { part[t] = v; }
};

// alphaSum of the iteration input, from the per-block partials of the previous P2
__device__ __forceinline__ double sum_partials(const double* part, uint32_t n, double extra,
                                               double* scratch) {
  double acc = 0.0;
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) acc += __ldcg(&part[i]);
  acc = block_reduce<false>(acc, scratch);
  return acc + extra;
}

// lagged logNorm: alphaSum of THIS iteration's input = the per-block partials written by
// the previous P2 (complete since the last grid barrier / kernel boundary).  Any common
// factor in theta cancels in P1/P2 (DESIGN.md).  One whole warp; result in scratch[33].
__device__ __forceinline__ void lag_lognorm_warp(const EmArgs& A, uint32_t par, uint32_t nblk, double* scratch) {
  const uint32_t lane = threadIdx.x & 31u;
  const double* part = A.sum_partial + (size_t)(par ^ 1u) * nblk;
  long long acc = 0;
  for (uint32_t i = lane; i < nblk; i += 32) acc += __double_as_longlong(__ldcg(&part[i]));
  acc = warp_sum_ll(acc);
  if (lane == 0) scratch[33] = digamma_pos((double)acc / A.sum_scale + A.inactive_sum);
}
// Persistent kernel: the first warp of the block to finish its P1 home range computes the lagged logNorm (claim in
// scratch[34], cleared after the grid barrier that follows P1).  That warp has time to spare before the barrier,
// while a fixed warp that did it before its home range started P1 about 2.5 us after the others.
__device__ __forceinline__ void lag_lognorm_first_warp(const EmArgs& A, uint32_t par, uint32_t nblk,
                                                       double* scratch) {
  uint32_t first = 0;
  if ((threadIdx.x & 31u) == 0) first = atomicAdd(reinterpret_cast<unsigned int*>(&scratch[34]), 1u) == 0u;
  if (__shfl_sync(0xffffffffu, first, 0)) lag_lognorm_warp(A, par, nblk, scratch);
}

__device__ __forceinline__ void p2_finish(const EmArgs& A, double* scratch, P2Acc& pa,
                                          uint32_t par) {
  const long long bs = block_sum_ll(pa.isum, scratch);
  double bm = block_reduce<true>(pa.maxrel, scratch);
  if (threadIdx.x == 0) {
    A.sum_partial[(size_t)par * gridDim.x + blockIdx.x] = __longlong_as_double(bs);   // fixed point, bit pattern
    if (bm > 0.0) atomicMax(&A.maxrel[par], (unsigned long long)__double_as_longlong(bm));
  }
}

// timeline taps: one iteration's timestamps (dbg_it = that iteration), or phase durations accumulated over the
// iterations >= 1 of a run (dbg_it = DBG_ACCUMULATE; slot 0 = P1, slot 1 = P2, slot 2 = iterations) -- the input of
// the measured re-balancing in em.cu (slots 3 / 4: the home stream of P1 / P2 alone).  One iteration's row of the
// persistent kernel: 0 P1 start, 1 P1 end, 2 end of barrier 1, 3 P2 start, 4 P2 end, 5 reduction end, 6 end of
// barrier 2, 7 / 8 end of the P2 / P1 home stream, 9-10 / 11-12 what the warp took from the P1 / P2 queue:
// (long rows << 32 | their entries), longest row taken (run_phase)
#define SB_DBG(slot)                                                        \
  if (A.dbg && it == A.dbg_it && (threadIdx.x & 31u) == 0) A.dbg[(size_t)gwarp * DBG_SLOTS + (slot)] = gtime_ns();
#define SB_ACC_BEGIN(var, sell_slot) \
  unsigned long long var = 0; \
  if (dbg_acc) { var = gtime_ns(); W.t0 = var; W.dbg_acc = &A.dbg[(size_t)gwarp * DBG_SLOTS + (sell_slot)]; }
#define SB_ACC_END(var, slot) \
  W.dbg_acc = nullptr; \
  if (dbg_acc && (threadIdx.x & 31u) == 0) A.dbg[(size_t)gwarp * DBG_SLOTS + (slot)] += gtime_ns() - var;

// ---- persistent cooperative kernel: the whole iteration loop, two grid barriers/iter
template <bool VBEM>
__global__ void __launch_bounds__(EM_THREADS, EM_MIN_BLOCKS) k_em_persistent(const __grid_constant__ EmArgs A) {
  extern __shared__ __align__(128) unsigned char smem[];
  WarpCtx W;
  warp_setup(W, smem);
  double* scratch = W.scratch;
  cg::grid_group grid = cg::this_grid();
  const uint32_t bid = blockIdx.x, nblk = gridDim.x;
  const uint32_t gwarp = bid * (EM_THREADS / 32) + (threadIdx.x >> 5);
  const WarpRange R1 = load_range(A.cm, gwarp);
  const WarpRange R2 = load_range(A.tm, gwarp);
  uint32_t it = 0;
  bool converged = false;
  double logNorm = VBEM ? digamma_pos(A.sum0) : 0.0;
  ring_prefetch(A.cm, W, R1);
  while (it < A.min_iter || (it < A.max_iter && !converged)) {
    const uint32_t par = it & 1u;
    const bool dbg_acc = A.dbg && A.dbg_it == DBG_ACCUMULATE && it > 0;
    if (bid == 0 && threadIdx.x == 0) A.maxrel[par] = 0ull;
    P2Acc pa{0ll, 0.0};
    SB_DBG(0)
    SB_ACC_BEGIN(t1, 3)
    W.dbg = (A.dbg && it == A.dbg_it) ? &A.dbg[(size_t)gwarp * DBG_SLOTS] : nullptr;
    // P2's home stream lands while this warp takes queue items and during the grid barrier; the logNorm P2 uses is
    // computed by the block's first warp to get here (consumed after the next barrier)
    run_phase<1, VBEM, true>(A, W, R1, bid, nblk, 0.0, 0.0, pa, [&] {
      ring_prefetch(A.tm, W, R2);
      if (VBEM && it > 0) lag_lognorm_first_warp(A, par, nblk, scratch);
    }, NoDeliver{});
    SB_ACC_END(t1, 0)
    SB_DBG(1)
    grid.sync();
    SB_DBG(2)
    if (bid == 0 && threadIdx.x == 0) A.lq[0] = 0u;   // P1's work queue: idle until the next iteration
    if (VBEM && it > 0) logNorm = scratch[33];   // written before the grid barrier above
    if (threadIdx.x == 0) *reinterpret_cast<unsigned int*>(&scratch[34]) = 0u;   // the next iteration's claim
    const double bias = (it == 0) ? A.first_bias : 0.0;  // alphasPrime starts at 1.0 (:812,:821)
    SB_DBG(3)
    SB_ACC_BEGIN(t2, 4)
    // next iteration's P1 home stream (harmless if the loop ends)
    run_phase<2, VBEM, true>(A, W, R2, bid, nblk, logNorm, bias, pa, [&] { ring_prefetch(A.cm, W, R1); }, NoDeliver{});
    W.dbg = nullptr;
    SB_ACC_END(t2, 1)
    SB_DBG(4)
    p2_finish(A, scratch, pa, par);
    SB_DBG(5)
    grid.sync();
    SB_DBG(6)
    if (bid == 0 && threadIdx.x == 0) A.lq[1] = 0u;   // P2's work queue
    if (dbg_acc && (threadIdx.x & 31u) == 0) A.dbg[(size_t)gwarp * DBG_SLOTS + 2] += 1ull;
    const double mr = __longlong_as_double((long long)__ldcg(&A.maxrel[par]));
    converged = !(mr > A.tol);
    ++it;
  }
  if (bid == 0 && threadIdx.x == 0) {
    A.out[0] = it;
    A.out[1] = converged ? 1u : 0u;
    A.out[2] = (it - 1) & 1u;
  }
  ring_drain(W, R1);   // the speculative prefetch must land before the block (and its shared memory) retires
}

// ---- multi-GPU persistent kernel --------------------------------------------------------------------------------------
// Classes stay sharded per rank; the state (theta) is replicated; transcript t is OWNED by rank t / S (S = ceil(M/G)).
// One iteration (three grid barriers; NO exchange barrier and no system-scope fence):
//   P1 (local classes, local plain copy of theta)                                                    -> grid barrier
//   P2-partial: every transcript's local share of alpha' (locally inactive ones: their constant folded singleton mass)
//     into a local buffer                                                                              -> grid barrier
//   push: the buffer goes to the owners as flagged lines, row `rank` of the owner's llrecv, in transcript order
//   owner phase: rank r polls the G lines of each transcript of its slice (they arrive as the peers' P2 proceeds), sums
//     them in rank order, applies the update (convergence terms, digamma / exp) for M/G transcripts only, keeps alpha,
//     writes theta' into its own plain copy and pushes it as a flagged line into every peer's llth; every block pushes
//     its {sum(alpha'+prior), max rel diff} into every rank's llaux
//   unpack: every rank polls the llth lines of the other slices into its plain theta; block 0 polls the G x grid aux
//     pairs and reduces them in (rank, block) order -> identical logNorm / convergence decision everywhere  -> grid barrier
// Pushing flagged lines replaces pulling the partials with remote loads between two exchange barriers (system fence +
// grid barrier + flag round trip + grid barrier, every thread fencing at system scope), which costs per iteration.
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_sys_f64(double* p, double v) {
  asm volatile("st.relaxed.sys.global.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
// flagged line: {lo32, epoch, hi32, epoch}; each 8-byte half is single-copy atomic
__device__ __forceinline__ void ll_store(uint4* line, double v, uint32_t epoch) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(v);
  asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(line), "r"((uint32_t)b), "r"(epoch),
               "r"((uint32_t)(b >> 32)), "r"(epoch)
               : "memory");
}
__device__ __forceinline__ bool ll_try_load(const uint4* line, uint32_t epoch, double& v) {
  uint4 q;
  asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(q.x), "=r"(q.y), "=r"(q.z), "=r"(q.w) : "l"(line) : "memory");
  v = __longlong_as_double((long long)(((unsigned long long)q.z << 32) | q.x));
  return q.y == epoch && q.w == epoch;
}
__device__ __forceinline__ double ll_wait(const uint4* line, uint32_t epoch, uint32_t* fail);
__device__ __forceinline__ uint4 ll_load_raw(const uint4* line) {
  uint4 q;
  asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(q.x), "=r"(q.y), "=r"(q.z), "=r"(q.w) : "l"(line) : "memory");
  return q;
}
// value of a line whose first copy `q` is already in registers (so that a thread can put several polls in flight
// before it looks at any of them); re-polls while the flags are stale
__device__ __forceinline__ double ll_finish(const uint4* line, uint4 q, uint32_t epoch, uint32_t* fail) {
  if (q.y != epoch || q.w != epoch) return ll_wait(line, epoch, fail);
  return __longlong_as_double((long long)(((unsigned long long)q.z << 32) | q.x));
}

__device__ __forceinline__ double ll_wait(const uint4* line, uint32_t epoch, uint32_t* fail) {
  double v;
  if (ll_try_load(line, epoch, v)) return v;
  const unsigned long long t0 = gtime_ns();
  for (uint32_t spins = 0;; ++spins) {
    __nanosleep(spins < 4 ? 100u : 400u);    // thousands of pollers: leave the L2 to the lines that are still arriving
    if (ll_try_load(line, epoch, v)) return v;
    if ((spins & 63u) == 63u) {
      if (*reinterpret_cast<volatile uint32_t*>(fail)) return 0.0;
      if (gtime_ns() - t0 > 20000000000ull) { *fail = 1u; return 0.0; }
    }
  }
}
// end-of-run barrier over all GPUs.  Only the signalling threads fence at system scope (st.release.sys): the other
// threads' remote stores happen-before it through the gpu-scope grid barrier, and release is cumulative.
__device__ __forceinline__ void xgpu_barrier(cg::grid_group& grid, const EmArgs& A, unsigned long long epoch) {
  grid.sync();
  if (blockIdx.x == 0 && threadIdx.x < A.nranks) {
    const uint32_t q = threadIdx.x;
    st_release_sys(reinterpret_cast<unsigned long long*>(A.peers[q]) + A.rank, epoch);
    const unsigned long long* mine = reinterpret_cast<const unsigned long long*>(A.peers[A.rank]) + q;
    const unsigned long long t0 = gtime_ns();
    while (ld_acquire_sys(mine) < epoch) {
      if (gtime_ns() - t0 > 20000000000ull) { *A.xfail = 1u; break; }   // a peer is missing: give up, report
    }
  }
  grid.sync();
}

struct DeliverPush {           // fused path: a flagged line into row `rank` of the owner's llrecv
  unsigned char* const* peers;
  size_t off_llrecv;
  uint32_t S, rank, epoch;
  __device__ __forceinline__ void operator()(uint32_t t, double v) const {
    const uint32_t owner = t / S;
    uint4* dst = reinterpret_cast<uint4*>(peers[owner] + off_llrecv) + (size_t)rank * S + (t - owner * S);
    ll_store(dst, v, epoch);
  }
};

template <bool VBEM>
__global__ void __launch_bounds__(EM_THREADS, EM_MIN_BLOCKS) k_em_persistent_mgpu(const __grid_constant__ EmArgs A) {
  extern __shared__ __align__(128) unsigned char smem[];
  WarpCtx W;
  warp_setup(W, smem);
  double* scratch = W.scratch;
  cg::grid_group grid = cg::this_grid();
  const uint32_t bid = blockIdx.x, nblk = gridDim.x;
  const uint32_t gwarp = bid * (EM_THREADS / 32) + (threadIdx.x >> 5);
  const uint32_t gtid = bid * EM_THREADS + threadIdx.x, gthreads = nblk * EM_THREADS;
  const WarpRange R1 = load_range(A.cm, gwarp);
  const WarpRange R2 = load_range(A.tm, gwarp);
  const uint32_t M = A.M, G = A.nranks;
  const XchgLayout X(M, G);
  const uint32_t S = X.S, lo = min(A.rank * S, M), hi = min(lo + S, M);
  unsigned char* const own = A.peers[A.rank];
  const uint4* my_recv = reinterpret_cast<const uint4*>(own + X.off_llrecv());
  const uint4* my_llth = reinterpret_cast<const uint4*>(own + X.off_llth());
  const uint4* my_aux = reinterpret_cast<const uint4*>(own + X.off_llaux());
  double* theta = A.theta;                   // = own + off_theta: the plain copy P1 gathers from
  uint32_t it = 0;
  bool converged = false;
  double logNorm = VBEM ? digamma_pos(A.sum0) : 0.0;
  ring_prefetch(A.cm, W, R1);
  while (it < A.min_iter || (it < A.max_iter && !converged)) {
    const uint32_t par = it & 1u;
    const uint32_t epoch = (uint32_t)(A.epoch0 + it + 1ull);
    const DeliverPush push{A.peers, X.off_llrecv(), S, A.rank, epoch};
    const bool dbg_acc = A.dbg && A.dbg_it == DBG_ACCUMULATE && it > 0;
    P2Acc pa{0ll, 0.0};
    SB_DBG(0)
    SB_ACC_BEGIN(t1, 3)
    run_phase<1, VBEM, true>(A, W, R1, bid, nblk, 0.0, 0.0, pa, [&] { ring_prefetch(A.tm, W, R2); }, NoDeliver{});
    SB_ACC_END(t1, 0)
    SB_DBG(1)
    grid.sync();
    SB_DBG(2)
    if (bid == 0 && threadIdx.x == 0) A.lq[0] = 0u;
    SB_ACC_BEGIN(t2, 4)
    if (A.push_pass) {
      // this rank's share of alpha' per transcript id into the local buffer (locally inactive transcripts keep their
      // constant folded singleton mass, written once per run by the host) ...
      run_phase<3, VBEM, true>(A, W, R2, bid, nblk, 0.0, 0.0, pa, [&] { ring_prefetch(A.cm, W, R1); },
                               DeliverLocal{A.part_out});
      SB_ACC_END(t2, 1)
      SB_DBG(3)
      __threadfence();
      grid.sync();
      if (bid == 0 && threadIdx.x == 0) A.lq[1] = 0u;
      // ... and from there to the owners in transcript order: consecutive threads write consecutive 16-byte lines,
      // i.e. whole 512-byte runs per warp over NVLink, instead of the row epilogues' pushes below (32 scattered
      // remote stores per warp instruction).  With one destination (N=2) the epilogue pushes overlap P2 and the extra
      // pass does not pay, so the host picks the pass for more than two ranks (scripts/timeline_mgpu.py times both;
      // not measured on H100).
      for (uint32_t t = gtid; t < M; t += gthreads) push(t, __ldcg(&A.part_out[t]));
    } else {
      // straight from the row epilogues; locally inactive transcripts (constant share) first
      for (uint32_t t = gtid; t < M; t += gthreads)
        if (__ldg(&A.tid_row[t]) == 0xffffffffu) push(t, __ldg(&A.base[t]));
      run_phase<3, VBEM, true>(A, W, R2, bid, nblk, 0.0, 0.0, pa, [&] { ring_prefetch(A.cm, W, R1); }, push);
      SB_ACC_END(t2, 1)
      SB_DBG(3)
    }
    // ---- owner phase: my slice [lo, hi); the lines are polled as they arrive
    const double bias = (it == 0) ? A.first_bias : 0.0;
    double sum = 0.0, mx = 0.0;
    for (uint32_t t = lo + gtid; t < hi; t += gthreads) {
      double na = bias;
      for (uint32_t q0 = 0; q0 < G; q0 += 8) {                 // up to 8 polls in flight, summed in rank order
        uint4 ln[8];
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (q0 + j < G) ln[j] = ll_load_raw(&my_recv[(size_t)(q0 + j) * S + (t - lo)]);
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (q0 + j < G) na += ll_finish(&my_recv[(size_t)(q0 + j) * S + (t - lo)], ln[j], epoch, A.xfail);
      }
      const double old = A.alpha[t];
      if (na > ALPHA_CHECK_CUTOFF) mx = fmax(mx, fabs(old - na) / na);
      A.alpha[t] = na;
      const double ap = na + A.prior[t];
      sum += ap;
      const double th = theta_of<VBEM>(na, ap, logNorm);
      theta[t] = th;
      for (uint32_t q = 0; q < G; ++q)
        if (q != A.rank) ll_store(reinterpret_cast<uint4*>(A.peers[q] + X.off_llth()) + t, th, epoch);
    }
    SB_DBG(4)
    {
      const double bs = block_reduce<false>(sum, scratch);
      const double bm = block_reduce<true>(mx, scratch);
      if (threadIdx.x < G) {                                   // this block's pair -> every rank's aux area
        uint4* aux = reinterpret_cast<uint4*>(A.peers[threadIdx.x] + X.off_llaux()) + ((size_t)A.rank * XAUX + bid) * 2;
        ll_store(aux, bs, epoch);
        ll_store(aux + 1, fmax(bm, 0.0), epoch);
      }
    }
    // ---- unpack: the other slices' theta into my plain copy
    for (uint32_t t0 = gtid; t0 < M; t0 += 4 * gthreads) {       // four polls in flight per thread
      uint4 ln[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t t = t0 + j * gthreads;
        if (t < M && (t < lo || t >= hi)) ln[j] = ll_load_raw(&my_llth[t]);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t t = t0 + j * gthreads;
        if (t < M && (t < lo || t >= hi)) theta[t] = ll_finish(&my_llth[t], ln[j], epoch, A.xfail);
      }
    }
    SB_DBG(5)
    if (bid == 0) {                                            // (rank, block) order: identical on every rank
      double s2 = 0.0, m2 = 0.0;
      for (uint32_t i0 = threadIdx.x; i0 < G * nblk; i0 += 4 * EM_THREADS) {   // four pairs in flight per thread
        uint4 ls[4], lm[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t i = i0 + j * EM_THREADS;
          if (i < G * nblk) {
            const uint32_t q = i / nblk, b = i - q * nblk;
            ls[j] = ll_load_raw(&my_aux[((size_t)q * XAUX + b) * 2]);
            lm[j] = ll_load_raw(&my_aux[((size_t)q * XAUX + b) * 2 + 1]);
          }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t i = i0 + j * EM_THREADS;
          if (i < G * nblk) {
            const uint32_t q = i / nblk, b = i - q * nblk;
            s2 += ll_finish(&my_aux[((size_t)q * XAUX + b) * 2], ls[j], epoch, A.xfail);
            m2 = fmax(m2, ll_finish(&my_aux[((size_t)q * XAUX + b) * 2 + 1], lm[j], epoch, A.xfail));
          }
        }
      }
      s2 = block_reduce<false>(s2, scratch);
      m2 = block_reduce<true>(m2, scratch);
      if (threadIdx.x == 0) {
        A.sum_partial[par] = s2;
        A.maxrel[par] = (unsigned long long)__double_as_longlong(m2);
      }
    }
    __threadfence();
    grid.sync();
    SB_DBG(6)
    if (!A.push_pass && bid == 0 && threadIdx.x == 0) A.lq[1] = 0u;
    if (*reinterpret_cast<volatile uint32_t*>(A.xfail)) break;
    {
      const double mr = __longlong_as_double((long long)__ldcg(&A.maxrel[par]));
      converged = !(mr > A.tol);
      if (VBEM) logNorm = digamma_pos(__ldcg(&A.sum_partial[par]));
    }
    SB_DBG(7)
    if (dbg_acc && (threadIdx.x & 31u) == 0) A.dbg[(size_t)gwarp * DBG_SLOTS + 2] += 1ull;
    ++it;
  }
  // all-gather of the final alpha: every owner pushes its slice into every rank's alpha region
  for (uint32_t t = lo + gtid; t < hi; t += gthreads) {
    const double a = A.alpha[t];
    for (uint32_t q = 0; q < G; ++q) st_relaxed_sys_f64(reinterpret_cast<double*>(A.peers[q] + X.off_alpha()) + t, a);
  }
  xgpu_barrier(grid, A, A.epoch0 + it + 1ull);
  if (bid == 0 && threadIdx.x == 0) {
    A.out[0] = it;
    A.out[1] = converged ? 1u : 0u;
    A.out[2] = (it - 1) & 1u;
    A.out[3] = it + 2u;                       // epochs consumed
  }
  ring_drain(W, R1);
}

// ---- one launch per phase (baseline variant; also the NCCL multi-GPU building blocks)
template <bool VBEM>
__global__ void __launch_bounds__(EM_THREADS, EM_MIN_BLOCKS) k_em_p1(const __grid_constant__ EmArgs A) {
  extern __shared__ __align__(128) unsigned char smem[];
  WarpCtx W;
  warp_setup(W, smem);
  P2Acc pa{0ll, 0.0};
  const WarpRange R = load_range(A.cm, blockIdx.x * (EM_THREADS / 32) + (threadIdx.x >> 5));
  ring_prefetch(A.cm, W, R);
  run_phase<1, VBEM, false>(A, W, R, blockIdx.x, gridDim.x, 0.0, 0.0, pa, Nothing{}, NoDeliver{});
}
template <bool VBEM>
__global__ void __launch_bounds__(EM_THREADS, EM_MIN_BLOCKS) k_em_p2(const __grid_constant__ EmArgs A, uint32_t it) {
  extern __shared__ __align__(128) unsigned char smem[];
  WarpCtx W;
  warp_setup(W, smem);
  double* scratch = W.scratch;
  const uint32_t par = it & 1u;
  double logNorm = 0.0;
  if (VBEM) {
    if (it == 0) {
      logNorm = digamma_pos(A.sum0);
    } else {
      if (threadIdx.x < 32) lag_lognorm_warp(A, par, gridDim.x, scratch);
      __syncthreads();
      logNorm = scratch[33];
    }
  }
  const double bias = (it == 0) ? A.first_bias : 0.0;
  P2Acc pa{0ll, 0.0};
  const WarpRange R = load_range(A.tm, blockIdx.x * (EM_THREADS / 32) + (threadIdx.x >> 5));
  ring_prefetch(A.tm, W, R);
  run_phase<2, VBEM, false>(A, W, R, blockIdx.x, gridDim.x, logNorm, bias, pa, Nothing{}, NoDeliver{});
  p2_finish(A, scratch, pa, par);
}
template <bool VBEM>
__global__ void __launch_bounds__(EM_THREADS, EM_MIN_BLOCKS) k_em_p2_partial(const __grid_constant__ EmArgs A) {
  extern __shared__ __align__(128) unsigned char smem[];
  WarpCtx W;
  warp_setup(W, smem);
  P2Acc pa{0ll, 0.0};
  const WarpRange R = load_range(A.tm, blockIdx.x * (EM_THREADS / 32) + (threadIdx.x >> 5));
  ring_prefetch(A.tm, W, R);
  run_phase<3, VBEM, false>(A, W, R, blockIdx.x, gridDim.x, 0.0, 0.0, pa, Nothing{}, DeliverLocal{A.part_out});
}

}  // namespace sb
