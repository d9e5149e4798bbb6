// sampling.cuh -- bootstrap resampling and Gibbs sampling on the device (included by em.cu).
//
// Replaces CollapsedEMOptimizer::gatherBootstraps / doBootstrap
// (src/inference/CollapsedEMOptimizer.cpp:554-690 / :398-552) and
// CollapsedGibbsSampler::sample / sampleRoundNonCollapsedMultithreaded_
// (src/inference/CollapsedGibbsSampler.cpp:317-508 / :92-278).
//
// The reference draws from random_device-seeded mt19937 / pcg32, so its samples are not
// reproducible; here every draw is a pure function of (seed, stream, indices) through
// Philox-4x32-10, the stream layout being the one oracle/em_oracle.c fixes:
//   bootstrap: fragment f of replicate b  -> philox(f_lo, f_hi, b, 0)      class = CDF^-1(mulhi(r64, total))
//   gibbs    : draw s of class c, round r -> philox(c, s, r, 1|hi bits)    category by cumulative scan
//              gamma for transcript i      -> philox(i, attempt, r, 2)      Marsaglia-Tsang
#pragma once

using namespace sb;

namespace sb {

__device__ __forceinline__ void philox4x32(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                           uint32_t k0, uint32_t k1, uint32_t* out) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t h0 = __umulhi(0xD2511F53u, c0), l0 = 0xD2511F53u * c0;
    const uint32_t h1 = __umulhi(0xCD9E8D57u, c2), l1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = h1 ^ c1 ^ k0, n1 = l1, n2 = h0 ^ c3 ^ k1, n3 = l0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
__device__ __forceinline__ double u53(uint32_t hi, uint32_t lo) {
  const uint64_t x = ((uint64_t)hi << 32) | lo;
  return (double)(x >> 11) * (1.0 / 9007199254740992.0);
}

// ---- shared helpers ---------------------------------------------------------------
__global__ void k_mark_members(uint64_t C, const uint64_t* __restrict__ off,
                               const uint32_t* __restrict__ tids, const uint8_t* __restrict__ valid,
                               int only_valid, uint8_t* __restrict__ flag) {
  uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  if (only_valid && !valid[c]) return;
  for (uint64_t j = off[c]; j < off[c + 1]; ++j) flag[tids[j]] = 1;
}
__global__ void k_count_flags(uint32_t M, const uint8_t* __restrict__ flag, unsigned long long* out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned v = (i < M && flag[i]) ? 1u : 0u;
  v = __reduce_add_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0 && v) atomicAdd(out, (unsigned long long)v);
}
// gatherBootstraps' markDegenerateClasses with the uniform start (:620-621)
__global__ void k_boot_valid(uint64_t C, const uint64_t* __restrict__ off,
                             const uint32_t* __restrict__ tids, const double* __restrict__ cw,
                             const uint8_t* __restrict__ valid, const uint8_t* __restrict__ active,
                             double unif, uint8_t* __restrict__ valid_boot) {
  uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double denom = 0.0;
  for (uint64_t j = off[c]; j < off[c + 1]; ++j) {
    double v = __dmul_rn(active[tids[j]] ? unif : 0.0, cw[j]);
    if (!isnan(v)) denom = __dadd_rn(denom, v);
  }
  valid_boot[c] = (valid[c] && !(denom <= DBL_MIN)) ? 1 : 0;
}
// weights of the class CDF: mode 0 = all valid classes, mode 1 = valid classes with > 1 transcript
__global__ void k_cdf_weights(uint64_t C, const uint64_t* __restrict__ off,
                              const uint64_t* __restrict__ counts, const uint8_t* __restrict__ valid,
                              int mode, uint64_t* __restrict__ w) {
  uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  bool ok = valid[c] != 0;
  if (mode == 1 && off[c + 1] - off[c] < 2) ok = false;
  w[c] = ok ? counts[c] : 0ull;
}
__device__ __forceinline__ uint64_t cdf_search(const uint64_t* __restrict__ cdf, uint64_t C, uint64_t x) {
  uint64_t lo = 0, hi = C;  // first class with inclusive cdf > x
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if (__ldg(&cdf[mid]) > x) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// ---- bootstrap --------------------------------------------------------------------
__global__ void k_boot_sample(uint64_t total, uint32_t b, uint32_t k0, uint32_t k1,
                              const uint64_t* __restrict__ cdf, uint64_t C,
                              const uint32_t* __restrict__ cls_map,
                              unsigned long long* __restrict__ samp_multi,
                              unsigned long long* __restrict__ samp_single) {
  for (uint64_t f = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; f < total;
       f += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t r[4];
    philox4x32((uint32_t)f, (uint32_t)(f >> 32), b, 0u, k0, k1, r);
    const uint64_t x = __umul64hi(((uint64_t)r[1] << 32) | r[0], total);
    const uint64_t c = cdf_search(cdf, C, x);
    const uint32_t m = __ldg(&cls_map[c]);
    if (m & 0x80000000u) atomicAdd(&samp_single[m & 0x7fffffffu], 1ull);
    else atomicAdd(&samp_multi[m], 1ull);
  }
}
__global__ void k_u64_to_f64(uint64_t n, const unsigned long long* __restrict__ a, double* __restrict__ o) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) o[i] = (double)a[i];
}
__global__ void k_boot_rows(uint32_t R, const uint32_t* __restrict__ row_tid,
                            const double* __restrict__ base_tid, double unif,
                            double* __restrict__ base_row, double* __restrict__ alpha0_row) {
  uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  base_row[r] = base_tid[row_tid[r]];
  alpha0_row[r] = unif;  // every row is a member of some class, hence active
}
__global__ void k_fill_active(uint32_t M, const uint8_t* __restrict__ active, double unif,
                              double* __restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < M) out[i] = active[i] ? unif : 0.0;
}
// per original class: the count the last replicate drew (parity tap)
__global__ void k_boot_counts_out(uint64_t C, const uint32_t* __restrict__ cls_map,
                                  const uint8_t* __restrict__ valid_boot,
                                  const unsigned long long* __restrict__ samp_multi,
                                  const unsigned long long* __restrict__ samp_single,
                                  const uint64_t* __restrict__ off, uint64_t* __restrict__ out) {
  uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  uint64_t v = 0;
  const uint32_t m = cls_map[c];
  if (valid_boot[c] && m != 0xffffffffu) {
    // several single-transcript classes on the same transcript share one accumulator, and each
    // of them reports it: the value is what all of them drew together.
    v = (m & 0x80000000u) ? samp_single[m & 0x7fffffffu] : samp_multi[m];
  }
  out[c] = v;
}

// ---- Gibbs ------------------------------------------------------------------------
__device__ double gamma_mt(double shape, double scale, uint32_t i, uint32_t round, uint32_t k0,
                           uint32_t k1) {
  // a shape that is not a positive finite number has no gamma distribution, and the rejection
  // loop below would never accept: return NaN so the sample shows it instead of hanging the kernel
  if (!(shape > 0.0) || isinf(shape)) return nan("");
  double a = shape, boost = 1.0;
  uint32_t r[4];
  if (a < 1.0) {
    philox4x32(i, 0xFFFFFFFFu, round, 2u, k0, k1, r);
    double u = u53(r[1], r[0]);
    if (u <= 0.0) u = 1.0 / 9007199254740992.0;
    boost = pow(u, 1.0 / a);
    a += 1.0;
  }
  const double d = a - 1.0 / 3.0;
  const double c = 1.0 / sqrt(9.0 * d);
  for (uint32_t attempt = 0;; ++attempt) {
    philox4x32(i, attempt, round, 2u, k0, k1, r);
    const double u1 = ((double)r[0] + 0.5) * (1.0 / 4294967296.0);
    const double u2 = ((double)r[1] + 0.5) * (1.0 / 4294967296.0);
    const double x = sqrt(-2.0 * log(u1)) * cos(2.0 * 3.14159265358979323846 * u2);
    double v = 1.0 + c * x;
    if (v <= 0.0) continue;
    v = v * v * v;
    double u = u53(r[3], r[2]);
    if (u <= 0.0) u = 1.0 / 9007199254740992.0;
    if (log(u) < 0.5 * x * x + d - d * v + d * log(v)) return d * v * boost * scale;
  }
}
__global__ void k_gibbs_init(uint32_t M, const uint8_t* __restrict__ active,
                             const double* __restrict__ effLens, const double* __restrict__ init,
                             int per_txp, double prior, double* __restrict__ priorA,
                             double* __restrict__ cnt, double* __restrict__ mu) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const double ml = effLens[i] > 1.0 ? effLens[i] : 1.0;
  priorA[i] = per_txp ? prior : prior * ml;          // CollapsedGibbsSampler.cpp:296-315
  cnt[i] = active[i] ? init[i] : 0.0;                // :350-352, :404-410
  mu[i] = 0.0;
}
__global__ void k_gibbs_mu(uint32_t M, const uint8_t* __restrict__ active,
                           const double* __restrict__ effLens, const double* __restrict__ priorA,
                           int no_gamma, uint32_t round, uint32_t k0, uint32_t k1,
                           double* __restrict__ cnt, double* __restrict__ mu) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M || !active[i]) return;
  const double ci = cnt[i] + priorA[i];                         // :131 / :146
  mu[i] = no_gamma ? ci / effLens[i] : gamma_mt(ci, 1.0 / (0.1 + effLens[i]), i, round, k0, k1);
  cnt[i] = 0.0;
}
__global__ void k_gibbs_singles(uint64_t C, const uint64_t* __restrict__ off,
                                const uint32_t* __restrict__ tids, const uint64_t* __restrict__ counts,
                                const uint8_t* __restrict__ valid, double* __restrict__ cnt) {
  uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C || !valid[c]) return;
  if (off[c + 1] - off[c] == 1) atomicAdd(&cnt[tids[off[c]]], (double)(int)counts[c]);   // :262-265
}
// one thread per draw of a multi-transcript class (:188-260)
__global__ void k_gibbs_draw(uint64_t total, uint32_t round, uint32_t k0, uint32_t k1,
                             const uint64_t* __restrict__ cdf, uint64_t C,
                             const uint64_t* __restrict__ off, const uint32_t* __restrict__ tids,
                             const double* __restrict__ weights, const double* __restrict__ mu,
                             const double* __restrict__ effLens, double* __restrict__ cnt) {
  const double DENORM_MIN = 4.9406564584124654e-324;
  for (uint64_t d = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; d < total;
       d += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t c = cdf_search(cdf, C, d);
    const uint64_t s = d - (c ? __ldg(&cdf[c - 1]) : 0ull);
    const uint64_t b = __ldg(&off[c]), n = __ldg(&off[c + 1]) - b;
    int mode = 0;   // 0: mu*w   1: 1/effLen   2: uniform
    double denom = 0.0;
    for (uint64_t i = 0; i < n; ++i)
      denom = __dadd_rn(denom, __dmul_rn(__dmul_rn(1000.0, mu[__ldg(&tids[b + i])]), __ldg(&weights[b + i])));
    if (denom <= DENORM_MIN) {
      mode = 1;
      denom = 0.0;
      for (uint64_t i = 0; i < n; ++i) denom = __dadd_rn(denom, 1.0 / effLens[__ldg(&tids[b + i])]);
      if (denom <= DENORM_MIN) { mode = 2; denom = (double)n; }
    }
    uint32_t r[4];
    philox4x32((uint32_t)c, (uint32_t)s, round, 1u | ((uint32_t)(c >> 32) << 8) | ((uint32_t)(s >> 32) << 16),
               k0, k1, r);
    const double target = __dmul_rn(u53(r[1], r[0]), denom);
    double cum = 0.0;
    uint64_t pick = n - 1;
    for (uint64_t i = 0; i < n; ++i) {
      const uint32_t t = __ldg(&tids[b + i]);
      const double p = mode == 0 ? __dmul_rn(__dmul_rn(1000.0, mu[t]), __ldg(&weights[b + i]))
                                 : (mode == 1 ? 1.0 / effLens[t] : 1.0);
      cum = __dadd_rn(cum, p);
      if (cum > target) { pick = i; break; }
    }
    atomicAdd(&cnt[__ldg(&tids[b + pick])], 1.0);   // integer-valued: order independent
  }
}
__global__ void k_gibbs_dot(uint32_t M, const double* __restrict__ mu, const double* __restrict__ effLens,
                            double* __restrict__ out) {
  __shared__ double scratch[32];
  double acc = 0.0;
  for (uint32_t i = threadIdx.x; i < M; i += blockDim.x) acc += mu[i] * effLens[i];
  acc = block_reduce<false>(acc, scratch);
  if (threadIdx.x == 0) out[0] = acc;
}
__global__ void k_gibbs_out(uint32_t M, const double* __restrict__ mu, const double* __restrict__ effLens,
                            const double* __restrict__ denom, double nmapped, double* __restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const double scale = nmapped / denom[0];
  const double a = __dmul_rn(__dmul_rn(mu[i], effLens[i]), scale);      // :497-500
  out[i] = (a > 1e-8) ? a : 0.0;
}

}  // namespace sb

static int build_cdf(sb_em_ctx* c, const uint8_t* valid, int mode, uint64_t* total_out) {
  cudaStream_t st = c->stream;
  const uint64_t C = c->C;
  SB_TRY(dev_alloc(&c->d_cdf, C + 1));
  if (C) {
    k_cdf_weights<<<nblk(C, 256), 256, 0, st>>>(C, c->d_off, c->d_counts, valid, mode, c->d_packed);
    size_t tb = c->tmp_bytes;
    SB_CUDA(cub::DeviceScan::InclusiveSum(c->d_tmp, tb, c->d_packed, c->d_cdf, (int)C, st));
    SB_CUDA(cudaMemcpyAsync(total_out, c->d_cdf + (C - 1), 8, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
  } else {
    *total_out = 0;
  }
  return SB_OK;
}

extern "C" int sb_bootstrap(sb_em_ctx* c, const sb_em_params* p, double num_mapped_frags,
                            uint32_t n_boot, uint64_t seed, sb_sample_cb cb, void* user) {
  if (!c || !p || !cb) { set_error("null argument"); return SB_ERR_INVALID; }
  if (!c->prepared) { set_error("sb_bootstrap needs a prepared context (run sb_em_optimize first)"); return SB_ERR_STATE; }
  if (c->nranks > 1) { set_error("sb_bootstrap: replicates are independent; run them per rank on a full table"); return SB_ERR_STATE; }
  SB_CUDA(cudaSetDevice(c->device));
  cudaStream_t st = c->stream;
  const uint64_t C = c->C;
  const uint32_t M = c->M, R = c->n_rows, Cm = c->n_cls;
  SB_TRY(dev_alloc(&c->d_active, (size_t)M));
  SB_TRY(dev_alloc(&c->d_valid_boot, C));
  SB_TRY(dev_alloc(&c->d_samp, (size_t)Cm + M + 1));
  SB_TRY(dev_alloc(&c->ov_cnt, (size_t)Cm + 1));
  SB_TRY(dev_alloc(&c->ov_base_tid, (size_t)M));
  SB_TRY(dev_alloc(&c->ov_base_row, (size_t)R + 1));
  SB_TRY(dev_alloc(&c->ov_alpha0_row, (size_t)R + 1));
  SB_TRY(dev_alloc(&c->ov_alpha0_tid, (size_t)M));
  // active transcripts: members of ANY class (:582-590)
  SB_CUDA(cudaMemsetAsync(c->d_active, 0, M, st));
  unsigned long long* d_nact = (unsigned long long*)(c->d_scalars + 40);
  SB_CUDA(cudaMemsetAsync(d_nact, 0, 8, st));
  if (C) k_mark_members<<<nblk(C, 256), 256, 0, st>>>(C, c->d_off, c->d_tids, c->d_valid, 0, c->d_active);
  k_count_flags<<<nblk(M, 256), 256, 0, st>>>(M, c->d_active, d_nact);
  unsigned long long nact = 0;
  SB_CUDA(cudaMemcpyAsync(&nact, d_nact, 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  if (nact == 0) { set_error("no transcripts are expressed"); return SB_ERR_INVALID; }   // :601-605
  const double scale = 1.0 / (double)nact;                                           // :607
  // degenerate marking with the uniform start over numMappedFrags (:600,:608-621)
  if (C)
    k_boot_valid<<<nblk(C, 128), 128, 0, st>>>(C, c->d_off, c->d_tids, c->d_cw, c->d_valid, c->d_active,
                                               scale * num_mapped_frags, c->d_valid_boot);
  uint64_t total = 0;
  SB_TRY(build_cdf(c, c->d_valid_boot, 0, &total));
  if (total == 0) { set_error("no fragments to resample"); return SB_ERR_INVALID; }
  const double unif = scale * (double)total;                                         // :450-453, :681
  // restores the context on EVERY exit path (the SB_CUDA macros below return early on a CUDA error)
  struct Restore {
    sb_em_ctx* c; sb_em_params saved;
    ~Restore() { c->params = saved; c->ov_active = false; }
  } restore{c, c->params};
  c->params = *p;
  std::vector<double> alpha(M);
  int rc_out = SB_OK;
  const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  for (uint32_t b = 0; b < n_boot && rc_out == SB_OK; ++b) {
    SB_CUDA(cudaMemsetAsync(c->d_samp, 0, ((size_t)Cm + M + 1) * 8, st));
    k_boot_sample<<<c->n_sm * 8, 256, 0, st>>>(total, b + c->sample_offset, k0, k1, c->d_cdf, C, c->d_cls_map, c->d_samp,
                                                c->d_samp + Cm);
    if (Cm) k_u64_to_f64<<<nblk(Cm, 256), 256, 0, st>>>(Cm, c->d_samp, c->ov_cnt);
    k_u64_to_f64<<<nblk(M, 256), 256, 0, st>>>(M, c->d_samp + Cm, c->ov_base_tid);
    if (R) k_boot_rows<<<nblk(R, 256), 256, 0, st>>>(R, c->d_row_tid, c->ov_base_tid, unif, c->ov_base_row,
                                                      c->ov_alpha0_row);
    k_fill_active<<<nblk(M, 256), 256, 0, st>>>(M, c->d_active, unif, c->ov_alpha0_tid);
    k_sum1<<<1, 1024, 0, st>>>(M, c->ov_alpha0_tid, c->d_prior, c->d_tid_row, 0, c->d_scalars + 18);
    k_sum1<<<1, 1024, 0, st>>>(M, c->ov_base_tid, c->d_prior, c->d_tid_row, 1, c->d_scalars + 19);
    double sums[2];
    SB_CUDA(cudaMemcpyAsync(sums, c->d_scalars + 18, 16, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    c->ov_active = true;
    c->ov_sum0 = sums[0];
    c->ov_inactive_sum = sums[1];
    c->ov_min_eq_w = p->use_vbem ? DBL_MIN : 4.9406564584124654e-324;   // :153 vs EMUtils.cpp:36
    sb_em_stats stt;
    int rc = sb_em_run(c, &stt);
    c->ov_active = false;
    if (rc != SB_OK) { rc_out = rc; break; }
    rc = sb_em_download(c, alpha.data(), &stt);
    if (rc < 0) { rc_out = rc; break; }
    if (rc == 1) { rc_out = 1; break; }                                  // :521-525
    if (cb(alpha.data(), M, user) != 0) break;
  }
  return rc_out;
}

extern "C" int sb_bootstrap_last_counts(sb_em_ctx* c, uint64_t* counts_out) {
  if (!c || !counts_out) { set_error("null argument"); return SB_ERR_INVALID; }
  if (!c->d_samp || !c->d_valid_boot) { set_error("no bootstrap has run"); return SB_ERR_STATE; }
  SB_CUDA(cudaSetDevice(c->device));
  const uint64_t C = c->C;
  if (!C) return SB_OK;
  k_boot_counts_out<<<nblk(C, 256), 256, 0, c->stream>>>(C, c->d_cls_map, c->d_valid_boot, c->d_samp,
                                                          c->d_samp + c->n_cls, c->d_off,
                                                          (uint64_t*)c->d_packed);
  SB_CUDA(cudaMemcpyAsync(counts_out, c->d_packed, C * 8, cudaMemcpyDeviceToHost, c->stream));
  SB_CUDA(cudaStreamSynchronize(c->stream));
  return SB_OK;
}

extern "C" int sb_gibbs(sb_em_ctx* c, const double* alphas_init, int use_vbem, int per_txp_prior,
                        double vb_prior, uint32_t n_samples, uint32_t thinning, int no_gamma_draw,
                        double num_mapped_frags, uint64_t seed, sb_sample_cb cb, void* user) {
  if (!c || !alphas_init || !cb) { set_error("null argument"); return SB_ERR_INVALID; }
  if (!c->prepared) { set_error("sb_gibbs needs a prepared context (run sb_em_optimize first)"); return SB_ERR_STATE; }
  SB_CUDA(cudaSetDevice(c->device));
  cudaStream_t st = c->stream;
  const uint64_t C = c->C;
  const uint32_t M = c->M;
  // :357-371
  const int perTxp = use_vbem ? per_txp_prior : 1;
  double prior = 1e-3;
  if (use_vbem) prior = perTxp ? (vb_prior < 1.0 ? 1.0 : vb_prior) : (vb_prior < 1e-3 ? 1e-3 : vb_prior);
  SB_TRY(dev_alloc(&c->d_active, (size_t)M));
  SB_TRY(dev_alloc(&c->d_gibbs_cnt, (size_t)M));
  SB_TRY(dev_alloc(&c->d_gibbs_mu, (size_t)M));
  SB_TRY(dev_alloc(&c->d_gibbs_prior, (size_t)M));
  SB_TRY(dev_alloc(&c->d_gibbs_out, (size_t)2 * M));   // [init | out]
  double* d_init = c->d_gibbs_out;
  double* d_out = c->d_gibbs_out + M;
  SB_CUDA(cudaMemcpyAsync(d_init, alphas_init, (size_t)M * 8, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemsetAsync(c->d_active, 0, M, st));
  if (C) k_mark_members<<<nblk(C, 256), 256, 0, st>>>(C, c->d_off, c->d_tids, c->d_valid, 1, c->d_active);  // :382-398
  uint64_t total = 0;
  SB_TRY(build_cdf(c, c->d_valid, 1, &total));
  // :425-442
  uint32_t nchains = 1;
  if (n_samples >= 50) nchains = 2;
  if (n_samples >= 100) nchains = 4;
  if (n_samples >= 200) nchains = 8;
  const uint32_t step = n_samples / nchains;
  const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  k_gibbs_init<<<nblk(M, 256), 256, 0, st>>>(M, c->d_active, c->d_efflens, d_init, perTxp, prior,
                                              c->d_gibbs_prior, c->d_gibbs_cnt, c->d_gibbs_mu);
  c->gibbs_m = M;
  std::vector<double> out(M);
  uint32_t round = c->sample_offset * thinning;   // a rank's share of a split run draws from its own rounds
  for (uint32_t sid = 0; sid < n_samples; ++sid) {
    if (nchains > 1 && sid > 0 && sid % step == 0 && sid / step < nchains)   // :457-461
      k_gibbs_init<<<nblk(M, 256), 256, 0, st>>>(M, c->d_active, c->d_efflens, d_init, perTxp, prior,
                                                  c->d_gibbs_prior, c->d_gibbs_cnt, c->d_gibbs_mu + 0);
    for (uint32_t r = 0; r < thinning; ++r, ++round) {
      k_gibbs_mu<<<nblk(M, 256), 256, 0, st>>>(M, c->d_active, c->d_efflens, c->d_gibbs_prior,
                                                no_gamma_draw, round, k0, k1, c->d_gibbs_cnt, c->d_gibbs_mu);
      if (C) k_gibbs_singles<<<nblk(C, 256), 256, 0, st>>>(C, c->d_off, c->d_tids, c->d_counts, c->d_valid,
                                                            c->d_gibbs_cnt);
      if (total)
        k_gibbs_draw<<<c->n_sm * 16, 256, 0, st>>>(total, round, k0, k1, c->d_cdf, C, c->d_off, c->d_tids,
                                                    c->d_aux, c->d_gibbs_mu, c->d_efflens, c->d_gibbs_cnt);
    }
    k_gibbs_dot<<<1, 1024, 0, st>>>(M, c->d_gibbs_mu, c->d_efflens, c->d_scalars + 41);
    k_gibbs_out<<<nblk(M, 256), 256, 0, st>>>(M, c->d_gibbs_mu, c->d_efflens, c->d_scalars + 41,
                                               num_mapped_frags, d_out);
    SB_CUDA(cudaMemcpyAsync(out.data(), d_out, (size_t)M * 8, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    if (cb(out.data(), M, user) != 0) break;
  }
  return SB_OK;
}

extern "C" int sb_gibbs_last_state(sb_em_ctx* c, double* mu_out, double* cnt_out) {
  if (!c || !mu_out || !cnt_out) { set_error("null argument"); return SB_ERR_INVALID; }
  if (!c->gibbs_m || c->gibbs_m != c->M) { set_error("no Gibbs run on the current table"); return SB_ERR_STATE; }
  SB_CUDA(cudaSetDevice(c->device));
  const size_t bytes = (size_t)c->M * 8;
  SB_CUDA(cudaMemcpyAsync(mu_out, c->d_gibbs_mu, bytes, cudaMemcpyDeviceToHost, c->stream));
  SB_CUDA(cudaMemcpyAsync(cnt_out, c->d_gibbs_cnt, bytes, cudaMemcpyDeviceToHost, c->stream));
  SB_CUDA(cudaStreamSynchronize(c->stream));
  return SB_OK;
}
