// em_internal.h -- host-side state of the Stage-B optimiser context.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

#include "../../include/salmon_b200.h"
#include "resources.h"

namespace sb {

constexpr int SELL_GROUP = 1024;    // default rows per length-bucketing group (options sell_group_cm / sell_group_tm)

// Device-side owner of one SELL-32 matrix (see em_kernels.cuh: struct Sell).
struct SellDev {
  uint32_t n_rows = 0, n_slices = 0, n_cols = 0, n_long = 0, n_block = 0;
  uint32_t n_fallback = 0;            // rows sent to the long-row path because their slice spans > 16-bit indices
  uint64_t long_entries = 0;          // entries of all long rows (their CSR copy is what the long-row path reads)
  uint32_t zero = 0;                  // gather slot holding 0.0 (padding entries)
  uint32_t* slice_ptr = nullptr;
  uint32_t* width = nullptr;
  uint32_t* base = nullptr;           // per slice: smallest gather index (the 16-bit indices are relative to it)
  uint16_t* len = nullptr;
  uint16_t* idx = nullptr;
  double* w = nullptr;
  uint32_t* warp_begin = nullptr;
  uint32_t* long_rows = nullptr;
  const uint32_t* csr_idx = nullptr;  // not owned
  const double* csr_w = nullptr;      // not owned
};

}  // namespace sb

struct sb_em_ctx {
  int device = 0;
  sb::Resources res;              // every device buffer, the stream and the events below
  explicit sb_em_ctx(int dev) : device(dev), res(dev) {}
  int n_sm = 0;
  size_t l2_bytes = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};

  // options
  int variant = 1;        // 1 = persistent cooperative kernel, 0 = one launch per phase
  int blocks_per_sm = 0;  // 0 = as many as fit
  int rebalance = 1;      // rounds of measured re-cutting of the warp ranges at prepare (0 = column-count model only)
  int occ = 0;
  // rows per length-bucketing group (locality window of the gathers)
  int sell_group_cm = sb::SELL_GROUP, sell_group_tm = sb::SELL_GROUP;

  // problem
  uint64_t C = 0, nnz = 0;
  uint32_t M = 0;
  double total_weight = 0.0;
  double count_sum = 0.0, eff_abs_sum = 0.0;   // sum of the class counts, of |effective length|
  int sum_scale_log2 = 20;                     // the fixed-point sum of (alpha' + prior) counts units of 2^-s
  size_t h2d_bytes = 0;
  bool uploaded = false, prepared = false;
  sb_em_params params{};

  // uploaded inputs
  uint64_t* d_off = nullptr;
  uint32_t* d_tids = nullptr;
  double* d_aux = nullptr;
  uint64_t* d_counts = nullptr;
  double* d_projected = nullptr;
  double* d_eff_in = nullptr;
  uint64_t* d_unique = nullptr;

  // per transcript
  double* d_efflens = nullptr;
  double* d_prior = nullptr;
  double* d_alpha0 = nullptr;
  double* d_alpha = nullptr;
  double* d_theta = nullptr;
  double* d_base = nullptr;       // folded singleton classes
  uint32_t* d_tcnt = nullptr;
  uint32_t* d_tid_row = nullptr;
  uint32_t* d_row_tid = nullptr;
  // row-space (active transcripts) iteration state, single-GPU path
  double *r_alpha = nullptr, *r_theta = nullptr, *r_prior = nullptr, *r_base = nullptr,
         *r_alpha0 = nullptr;

  // per class / entry
  double* d_cw = nullptr;         // combinedWeights in input order
  uint64_t* d_packed = nullptr;
  uint64_t* d_packed2 = nullptr;
  uint64_t* d_packed_scan = nullptr;
  uint8_t* d_valid = nullptr;
  double* d_cnt = nullptr;        // counts of compact classes (as f64)
  double* d_scale = nullptr;      // count/denom per compact class
  uint32_t* d_ent_cls = nullptr;
  uint32_t *d_sort_keys = nullptr, *d_sort_vals = nullptr, *d_sort_keys2 = nullptr,
           *d_sort_vals2 = nullptr;
  void* d_tmp = nullptr;
  size_t tmp_bytes = 0;

  // compact CSR copies (final class order / rank order) + SELL-32 matrices
  uint32_t n_cls = 0, nnzm = 0, n_rows = 0;
  uint32_t *m_off = nullptr, *m_idx = nullptr, *m_idx_state = nullptr;
  double* m_w = nullptr;
  uint32_t *t_off = nullptr, *t_idx = nullptr;
  double* t_w = nullptr;
  uint32_t *d_rank_tid = nullptr, *d_rowperm = nullptr, *d_order = nullptr;
  sb::SellDev cm, tm;

  double* d_scalars = nullptr;    // 64 doubles of misc device scalars
  double* d_sum_partial = nullptr;
  uint32_t grid = 0;
  double sum0 = 0.0, inactive_sum = 0.0;

  // multi-GPU
  int rank = 0, nranks = 1;
  void* nccl_comm = nullptr;
  double* d_part = nullptr;       // per-transcript partial alpha' (send)
  double* d_part_red = nullptr;   // all-reduced (recv)
  // fused path: exchange block [part M | red M | flags 64] shared with the peers through CUDA IPC
  unsigned char* x_block = nullptr;
  uint32_t x_cap = 0;
  unsigned char** d_peers = nullptr;
  uint32_t sample_offset = 0;     // index of the first sample of this call within the whole run (samples split over GPUs)
  int push_pass = -1;             // fused path: -1 = by rank count, 0 = push from the row epilogues, 1 = coalesced pass
  bool fused_loopback = false;    // one rank that is its own peer: the fused exchange logic on one GPU (tests)
  std::vector<void*> x_opened;
  bool peers_ready = false;
  unsigned long long x_epoch = 0;
  uint32_t* d_xfail = nullptr;

  // overrides used by the bootstrap driver (sampling.cuh): resampled counts, uniform init
  bool ov_active = false;
  double* ov_cnt = nullptr;
  double* ov_base_row = nullptr;
  double* ov_base_tid = nullptr;
  double* ov_alpha0_row = nullptr;
  double* ov_alpha0_tid = nullptr;
  double ov_sum0 = 0.0, ov_inactive_sum = 0.0, ov_min_eq_w = 0.0;
  // --bootstrapReproject: the original counts of the classes the replicates resample, in the overlay's layout
  double* rp_cnt = nullptr;
  double* rp_base_row = nullptr;
  double* rp_base_tid = nullptr;
  // sampling scratch
  uint64_t* d_cdf = nullptr;
  uint32_t* d_cls_map = nullptr;
  unsigned long long* d_samp = nullptr;
  uint8_t* d_valid_boot = nullptr;
  uint8_t* d_active = nullptr;
  double *d_gibbs_cnt = nullptr, *d_gibbs_mu = nullptr, *d_gibbs_prior = nullptr, *d_gibbs_out = nullptr;
  uint32_t gibbs_m = 0;           // transcripts of the last sb_gibbs run (0: none has run); read by sb_gibbs_last_state

  // debug timeline
  unsigned long long* d_dbg = nullptr;
  uint32_t dbg_it = 0;
  bool dbg_enabled = false;
  int rebalance_rounds_done = 0;

  // L2 flush
  void* d_flush = nullptr;
  uint32_t flush_ctr = 0;

  // results
  uint32_t iters = 0, converged = 0, launches = 0;
  double max_rel_diff = 0.0;
  uint64_t n_degenerate = 0;
  float prepare_ms = 0, run_ms = 0;
};
