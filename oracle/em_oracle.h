/*
 * oracle/em_oracle.h -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement (plain C) of Salmon's offline inference path ("Stage B",
 * SURVEY.md section 8 rows a9-a14).  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may load this library; the
 * product (libsalmon_b200.so) never links, loads or calls it.
 *
 * Every function cites the reference file:line (relative to the salmon
 * source tree, v1.11.4 @ aac21be4) whose arithmetic it restates.
 *
 * Pinning status (see DESIGN.md "Oracle"):
 *   - digamma: Boost.Math 1.84 is NOT vendored in the reference tree; its
 *     published 53-bit algorithm is restated here and pinned against
 *     high-precision mpmath values (tests/golden/digamma_golden.json).
 *   - EMUpdate_/truncateCountVector (serial): pinned against the reference's
 *     own src/inference/EMUtils.cpp compiled into oracle/_ref (see
 *     oracle/build_ref.sh) from a salmon source tree.
 *   - the reference ships no golden vectors / KATs for this path
 *     (SURVEY.md section 4), so the remaining functions are pinned only by
 *     hand-derived tiny cases in tests/golden/.
 */
#ifndef SB_EM_ORACLE_H
#define SB_EM_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Options of CollapsedEMOptimizer::optimize that reach the arithmetic
 * (SalmonOpts fields; defaults from include/salmon/internal/config/SalmonDefaults.hpp). */
typedef struct orc_em_params {
  int32_t use_vbem;           /* sopt.useVBOpt            (default true)  */
  int32_t per_txp_prior;      /* sopt.perTranscriptPrior  (default true)  */
  int32_t init_uniform;       /* sopt.initUniform                        */
  int32_t eq_class_mode;      /* sopt.eqClassMode (--eqclasses entry)    */
  int32_t no_rich_eq;         /* sopt.noRichEqClasses                    */
  int32_t no_length_correction; /* sopt.noLengthCorrection (effLen=100)  */
  int32_t alt_init;           /* sopt.meta || sopt.alternativeInitMode   */
  int32_t n_threads;          /* only used by the *_mt entry points       */
  double vb_prior;            /* sopt.vbPrior (1e-2)                      */
  double tol;                 /* relDiffTolerance (0.01)                  */
  double num_required_frags;  /* sopt.numRequiredFragments (5e7)          */
  uint32_t min_iter;          /* 100 in optimize, 50 in doBootstrap       */
  uint32_t max_iter;          /* 10000 (caller MappingPipelineStages.cpp:49) */
} orc_em_params;

typedef struct orc_em_stats {
  uint32_t iters;
  uint32_t converged;
  double max_rel_diff;
  double alpha_sum;
  uint64_t n_degenerate;
  int32_t ok;                 /* 0 <=> optimize returned false            */
} orc_em_stats;

double orc_digamma(double x);

/* CollapsedEMOptimizer::optimize, single-threaded, deterministic order.
 * CSR inputs: off[C+1], tids[nnz], aux[nnz] (TGValue::weights after finish()),
 * counts[C].  Per transcript: projected (Transcript::projectedCounts),
 * eff_len (exp(cachedLogEffectiveLength) or RefLength), unique (uniqueCount()).
 * Outputs: alpha_out[M]; optional combined_out[nnz], valid_out[C], eff_len_out[M]. */
int orc_em_optimize(uint64_t C, uint32_t M, const uint64_t* off,
                    const uint32_t* tids, const double* aux,
                    const uint64_t* counts, const double* projected,
                    const double* eff_len, const uint64_t* unique,
                    const orc_em_params* p, double* alpha_out,
                    double* combined_out, uint8_t* valid_out,
                    double* eff_len_out, orc_em_stats* st);

/* Same arithmetic, parallelised the way the reference is: static partition of
 * classes over threads with CAS f64 accumulation (CollapsedEMOptimizer.cpp:178-328;
 * incLoop SalmonUtils.hpp:166-172).  OpenMP stands in for oneTBB.  This is the
 * "port" CPU baseline bench.py times. */
int orc_em_optimize_mt(uint64_t C, uint32_t M, const uint64_t* off,
                       const uint32_t* tids, const double* aux,
                       const uint64_t* counts, const double* projected,
                       const double* eff_len, const uint64_t* unique,
                       const orc_em_params* p, double* alpha_out,
                       orc_em_stats* st);

/* One serial update step on explicit state (for per-iteration parity tests).
 * vbem=0: EMUtils.cpp:7-53 (denorm_min guard);  vbem=1: CollapsedEMOptimizer.cpp:104-171.
 * valid may be NULL (all valid). */
void orc_em_step_serial(uint64_t C, uint32_t M, const uint64_t* off,
                        const uint32_t* tids, const double* cw,
                        const uint64_t* counts, const uint8_t* valid,
                        const double* prior, const double* alpha_in,
                        double* alpha_out, double* exp_theta, int vbem);

/* One parallel-semantics update step (CollapsedEMOptimizer.cpp:178-234 / 241-328:
 * DBL_MIN guard, valid flags) executed serially. */
void orc_em_step(uint64_t C, uint32_t M, const uint64_t* off,
                 const uint32_t* tids, const double* cw, const uint64_t* counts,
                 const uint8_t* valid, const double* prior,
                 const double* alpha_in, double* alpha_out, double* exp_theta,
                 int vbem);

/* TPM as GZipWriter::writeAbundances computes it (GZipWriter.cpp:719-736). */
void orc_tpm(uint32_t M, const double* alpha, const double* eff_len, double* tpm);

/* Philox-4x32-10 counter RNG shared (by specification, not by code) with the
 * CUDA path so that sampling parity can be bit-exact.  out[4]. */
void orc_philox4x32(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                    uint32_t k0, uint32_t k1, uint32_t* out);

/* Bootstrap (CollapsedEMOptimizer.cpp:398-552).  The reference draws from a
 * random_device-seeded mt19937, so its samples are not reproducible; the
 * restatement keeps the arithmetic and substitutes the counter RNG above:
 * fragment f of bootstrap b picks the class with inverse-CDF on
 * u = philox(f, b, 0, 0; seed).  samp_counts_out may be NULL. */
int orc_bootstrap(uint64_t C, uint32_t M, const uint64_t* off,
                  const uint32_t* tids, const double* cw, const uint64_t* counts,
                  const uint8_t* valid, const double* prior,
                  const uint8_t* active, const orc_em_params* p,
                  uint32_t n_boot, uint64_t seed, double* alphas_out /* n_boot*M */,
                  uint64_t* samp_counts_out /* n_boot*C or NULL */);

/* Gibbs (CollapsedGibbsSampler.cpp:92-278, 317-508).  no_gamma_draw=1 is the
 * reference's --noGammaDraw mode (mu = (count+prior)/effLen).  With gamma
 * draws, Marsaglia-Tsang on the counter RNG replaces std::gamma_distribution.
 * weights = TGValue::weights (NOT combinedWeights; :209,220). */
int orc_gibbs(uint64_t C, uint32_t M, const uint64_t* off, const uint32_t* tids,
              const double* weights, const uint64_t* counts,
              const uint8_t* valid, const double* eff_len,
              const double* alphas_init, int use_vbem, int per_txp_prior,
              double vb_prior, uint32_t n_samples, uint32_t thinning,
              int no_gamma_draw, double num_mapped_frags, uint64_t seed,
              double* samples_out /* n_samples*M */);

/* orc_gibbs with two additions.  round0: the global round of the first draw, so that a
 * call with round0 = k*thinning draws samples k, k+1, ... of a longer run started at
 * round 0 (a split run's share; its chains restart from alphas_init as in orc_gibbs).
 * last_mu / last_cnt (M each, may be NULL): mu and the drawn counts as the last round
 * left them.  orc_gibbs is orc_gibbs_ex with round0 = 0 and no state outputs. */
int orc_gibbs_ex(uint64_t C, uint32_t M, const uint64_t* off, const uint32_t* tids,
                 const double* weights, const uint64_t* counts,
                 const uint8_t* valid, const double* eff_len,
                 const double* alphas_init, int use_vbem, int per_txp_prior,
                 double vb_prior, uint32_t n_samples, uint32_t thinning,
                 int no_gamma_draw, double num_mapped_frags, uint64_t seed,
                 uint32_t round0, double* samples_out /* n_samples*M */,
                 double* last_mu, double* last_cnt);

/* One gamma draw of the Gibbs sampler (Marsaglia-Tsang with the shape < 1 boost): the
 * draw for transcript i in global round `round` under the key (k0, k1).  Exposed so the
 * draws can be checked against the gamma distribution and against the device. */
double orc_gamma_draw(double shape, double scale, uint32_t i, uint32_t round,
                      uint32_t k0, uint32_t k1);

#ifdef __cplusplus
}
#endif
#endif
