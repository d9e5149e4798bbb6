/*
 * oracle/em_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE (see em_oracle.h).
 *
 * Plain-C restatement of Salmon's Stage-B inference arithmetic.  Reference
 * citations are file:line in COMBINE-lab/salmon v1.11.4 (aac21be4).
 * Compile with -ffp-contract=off so the sums round the way the reference's
 * x86-64 build does.
 */
#include "em_oracle.h"

#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* CollapsedEMOptimizer.cpp:40-43 */
#define MIN_EQ_CLASS_WEIGHT DBL_MIN
#define MIN_WEIGHT DBL_MIN
#define DIGAMMA_MIN 1e-10
/* EMUtils.cpp:36, CollapsedGibbsSampler.cpp:46-47 */
#define DENORM_MIN 4.9406564584124654e-324

/* ------------------------------------------------------------------------
 * digamma.  The reference calls boost::math::digamma (CollapsedEMOptimizer.cpp:
 * 119,127,256,269); Boost 1.84.0 is fetched at configure time
 * (cmake/SalmonDependencies.cmake:182-190) and is not in the reference tree.
 * This restates Boost.Math's published double-precision (53-bit) algorithm:
 * reflection for x<=-1, asymptotic series for x>=10, otherwise recurrence into
 * [1,2] and a rational minimax approximation around the positive root.
 * Pinned against mpmath (tests/golden/digamma_golden.json).
 * ---------------------------------------------------------------------- */
static double digamma_large(double x) {
  static const double P[] = {
      0.083333333333333333333333333333333333333333333333333,
      -0.0083333333333333333333333333333333333333333333333333,
      0.003968253968253968253968253968253968253968253968254,
      -0.0041666666666666666666666666666666666666666666666667,
      0.0075757575757575757575757575757575757575757575757576,
      -0.021092796092796092796092796092796092796092796092796,
      0.083333333333333333333333333333333333333333333333333,
      -0.44325980392156862745098039215686274509803921568627};
  x -= 1.0;
  double result = log(x);
  result += 1.0 / (2.0 * x);
  double z = 1.0 / (x * x);
  double poly = P[7];
  for (int i = 6; i >= 0; --i) poly = poly * z + P[i];
  result -= z * poly;
  return result;
}

static double digamma_1_2(double x) {
  static const float Y = 0.99558162689208984F;
  static const double root1 = 1569415565.0 / 1073741824.0;
  static const double root2 = (381566830.0 / 1073741824.0) / 1073741824.0;
  static const double root3 = 0.9016312093258695918615325266959189453125e-19;
  static const double P[] = {0.25479851061131551,   -0.32555031186804491,
                             -0.65031853770896507,  -0.28919126444774784,
                             -0.045251321448739056, -0.0020713321167745952};
  static const double Q[] = {1.0,
                             2.0767117023730469,
                             1.4606242909763515,
                             0.43593529692665969,
                             0.054151797245674225,
                             0.0021284987017821144,
                             -0.55789841321675513e-6};
  double g = x - root1;
  g -= root2;
  g -= root3;
  double z = x - 1.0;
  double p = P[5];
  for (int i = 4; i >= 0; --i) p = p * z + P[i];
  double q = Q[6];
  for (int i = 5; i >= 0; --i) q = q * z + Q[i];
  double r = p / q;
  return g * (double)Y + g * r;
}

double orc_digamma(double x) {
  double result = 0.0;
  if (x <= -1.0) {
    /* reflect */
    x = 1.0 - x;
    double rem = x - floor(x);
    if (rem > 0.5) rem -= 1.0;
    if (rem == 0.0) return NAN; /* pole */
    result = M_PI / tan(M_PI * rem);
  }
  if (x == 0.0) return NAN; /* pole */
  if (x >= 10.0) {
    result += digamma_large(x);
  } else {
    while (x > 2.0) {
      x -= 1.0;
      result += 1.0 / x;
    }
    while (x < 1.0) {
      result -= 1.0 / x;
      x += 1.0;
    }
    result += digamma_1_2(x);
  }
  return result;
}

/* ------------------------------------------------------------------------
 * Update steps.
 * ---------------------------------------------------------------------- */

/* Serial steps used by bootstrapping.
 * EM:   src/inference/EMUtils.cpp:7-53   (guard: denorm_min, NaN skip)
 * VBEM: src/inference/CollapsedEMOptimizer.cpp:104-171 (guard: DBL_MIN, expTheta>0) */
void orc_em_step_serial(uint64_t C, uint32_t M, const uint64_t* off,
                        const uint32_t* tids, const double* cw,
                        const uint64_t* counts, const uint8_t* valid,
                        const double* prior, const double* alpha_in,
                        double* alpha_out, double* exp_theta, int vbem) {
  if (vbem) {
    double alphaSum = 0.0;
    for (uint32_t i = 0; i < M; ++i) alphaSum += alpha_in[i] + prior[i];
    double logNorm = orc_digamma(alphaSum);
    for (uint32_t i = 0; i < M; ++i) {
      double ap = alpha_in[i] + prior[i];
      exp_theta[i] = (ap > DIGAMMA_MIN) ? exp(orc_digamma(ap) - logNorm) : 0.0;
      alpha_out[i] = 0.0;
    }
  }
  for (uint64_t c = 0; c < C; ++c) {
    if (valid && !valid[c]) continue; /* doBootstrap only receives valid classes (:641) */
    uint64_t b = off[c], e = off[c + 1];
    uint64_t n = e - b;
    double count = (double)counts[c];
    if (n > 1) {
      double denom = 0.0;
      if (vbem) {
        for (uint64_t j = b; j < e; ++j) {
          double th = exp_theta[tids[j]];
          if (th > 0.0) denom += th * cw[j];
        }
        if (denom <= MIN_EQ_CLASS_WEIGHT) continue;
        double invDenom = count / denom;
        for (uint64_t j = b; j < e; ++j) {
          double th = exp_theta[tids[j]];
          if (th > 0.0) alpha_out[tids[j]] += (th * cw[j]) * invDenom;
        }
      } else {
        for (uint64_t j = b; j < e; ++j) denom += alpha_in[tids[j]] * cw[j];
        if (denom <= DENORM_MIN) continue;
        double invDenom = count / denom;
        for (uint64_t j = b; j < e; ++j) {
          double v = alpha_in[tids[j]] * cw[j];
          if (!isnan(v)) alpha_out[tids[j]] += v * invDenom;
        }
      }
    } else if (n == 1) {
      alpha_out[tids[b]] += count;
    }
  }
}

/* Parallel-version semantics (CollapsedEMOptimizer.cpp:178-234 EM, :241-328 VBEM),
 * executed in class order.  alpha_out must be zeroed by the caller for EM
 * (optimize zeroes alphasPrime after each swap, :956); VBEM zeroes it itself (:274). */
void orc_em_step(uint64_t C, uint32_t M, const uint64_t* off,
                 const uint32_t* tids, const double* cw, const uint64_t* counts,
                 const uint8_t* valid, const double* prior,
                 const double* alpha_in, double* alpha_out, double* exp_theta,
                 int vbem) {
  const double* theta = alpha_in;
  if (vbem) {
    double alphaSum = 0.0;
    for (uint32_t i = 0; i < M; ++i) alphaSum += alpha_in[i] + prior[i];
    double logNorm = orc_digamma(alphaSum);
    for (uint32_t i = 0; i < M; ++i) {
      double ap = alpha_in[i] + prior[i];
      exp_theta[i] = (ap > DIGAMMA_MIN) ? exp(orc_digamma(ap) - logNorm) : 0.0;
      alpha_out[i] = 0.0;
    }
    theta = exp_theta;
  }
  for (uint64_t c = 0; c < C; ++c) {
    if (valid && !valid[c]) continue;
    uint64_t b = off[c], e = off[c + 1];
    uint64_t n = e - b;
    double count = (double)counts[c];
    if (n > 1) {
      double denom = 0.0;
      if (vbem) {
        for (uint64_t j = b; j < e; ++j) {
          double th = theta[tids[j]];
          if (th > 0.0) denom += th * cw[j];
        }
      } else {
        for (uint64_t j = b; j < e; ++j) denom += theta[tids[j]] * cw[j];
      }
      if (denom <= MIN_EQ_CLASS_WEIGHT) continue;
      double invDenom = count / denom;
      for (uint64_t j = b; j < e; ++j) {
        double th = theta[tids[j]];
        double v = th * cw[j];
        if (vbem ? (th > 0.0) : !isnan(v)) alpha_out[tids[j]] += v * invDenom;
      }
    } else if (n == 1) {
      alpha_out[tids[b]] += count;
    }
  }
}

/* ------------------------------------------------------------------------
 * optimize: shared setup (CollapsedEMOptimizer.cpp:778-878)
 * ---------------------------------------------------------------------- */
typedef struct {
  double* alphas;
  double* alphasPrime;
  double* expTheta;
  double* effLens;
  double* prior;
  double* cw;
  uint8_t* valid;
  uint64_t n_degenerate;
} em_state;

static int em_setup(uint64_t C, uint32_t M, const uint64_t* off,
                    const uint32_t* tids, const double* aux,
                    const uint64_t* counts, const double* projected,
                    const double* eff_len, const uint64_t* unique,
                    const orc_em_params* p, em_state* s) {
  uint64_t nnz = off[C];
  s->alphas = (double*)calloc(M ? M : 1, sizeof(double));
  s->alphasPrime = (double*)calloc(M ? M : 1, sizeof(double));
  s->expTheta = (double*)calloc(M ? M : 1, sizeof(double));
  s->effLens = (double*)calloc(M ? M : 1, sizeof(double));
  s->prior = (double*)calloc(M ? M : 1, sizeof(double));
  s->cw = (double*)calloc(nnz ? nnz : 1, sizeof(double));
  s->valid = (uint8_t*)calloc(C ? C : 1, 1);
  if (!s->alphas || !s->alphasPrime || !s->expTheta || !s->effLens ||
      !s->prior || !s->cw || !s->valid)
    return -1;

  /* :778-794 */
  double totalWeight = 0.0;
  int64_t numActive = 0;
  for (uint32_t i = 0; i < M; ++i) {
    s->alphas[i] = projected[i];
    totalWeight += s->alphas[i];
    s->effLens[i] = eff_len[i];
    if (p->no_length_correction) s->effLens[i] = 100.0;
    double uniqueCount = (double)unique[i] + 0.5; /* static_cast<double>(uniqueCount()+0.5) */
    double wi = p->init_uniform ? 100.0 : (uniqueCount * 1e-3 * s->effLens[i]);
    s->alphasPrime[i] = wi;
    ++numActive;
  }
  /* :797-798, :82-99 */
  for (uint32_t i = 0; i < M; ++i)
    s->prior[i] = p->per_txp_prior ? p->vb_prior : p->vb_prior * s->effLens[i];
  /* :803-823 */
  double uniformPrior = totalWeight / (double)numActive;
  double maxFrac = 0.999;
  double fracObserved = totalWeight / p->num_required_frags;
  if (maxFrac < fracObserved) fracObserved = maxFrac;
  if (p->init_uniform) {
    for (uint32_t i = 0; i < M; ++i) {
      s->alphas[i] = s->alphasPrime[i];
      s->alphasPrime[i] = 1.0;
    }
  } else {
    for (uint32_t i = 0; i < M; ++i) {
      double uniAbund = p->alt_init ? s->alphasPrime[i] : uniformPrior;
      s->alphas[i] = (s->alphas[i] * fracObserved) + (uniAbund * (1.0 - fracObserved));
      s->alphasPrime[i] = 1.0;
    }
  }
  /* :830-873 combined weights */
  for (uint64_t c = 0; c < C; ++c) {
    double wsum = 0.0;
    double count = (double)counts[c];
    for (uint64_t j = off[c]; j < off[c + 1]; ++j) {
      double el = s->effLens[tids[j]];
      if (el <= 1.0) el = 1.0;
      double w = p->no_rich_eq ? 1.0 : aux[j];
      double probStartPos = 1.0 / el;
      double wt = p->eq_class_mode ? w : count * w * probStartPos;
      s->cw[j] = wt;
      wsum += wt;
    }
    double wnorm = 1.0 / wsum;
    for (uint64_t j = off[c]; j < off[c + 1]; ++j) s->cw[j] = s->cw[j] * wnorm;
  }
  /* :330-394 markDegenerateClasses */
  s->n_degenerate = 0;
  for (uint64_t c = 0; c < C; ++c) {
    double denom = 0.0;
    for (uint64_t j = off[c]; j < off[c + 1]; ++j) {
      double v = s->alphas[tids[j]] * s->cw[j];
      if (!isnan(v)) denom += v;
    }
    if (denom <= MIN_EQ_CLASS_WEIGHT) {
      ++s->n_degenerate;
      s->valid[c] = 0;
    } else {
      s->valid[c] = 1;
    }
  }
  /* the loop enters with alphasPrime zeroed?  No: alphasPrime is 1.0 here (:812,821)
   * and VBEMUpdate_ zeroes alphaOut itself (:274) while EMUpdate_ ACCUMULATES into it
   * (:223,228).  So in EM mode the first iteration's output carries +1.0 per
   * transcript.  Restated faithfully below (the caller does not reset it). */
  return 0;
}

static void em_free(em_state* s) {
  free(s->alphas);
  free(s->alphasPrime);
  free(s->expTheta);
  free(s->effLens);
  free(s->prior);
  free(s->cw);
  free(s->valid);
}

/* :945-957 */
static int em_converge_swap(uint32_t M, double* alphas, double* alphasPrime,
                            double tol, double* maxRelDiffOut) {
  int converged = 1;
  double maxRelDiff = -DBL_MAX;
  const double alphaCheckCutoff = 1e-2;
  for (uint32_t i = 0; i < M; ++i) {
    if (alphasPrime[i] > alphaCheckCutoff) {
      double relDiff = fabs(alphas[i] - alphasPrime[i]) / alphasPrime[i];
      maxRelDiff = (relDiff > maxRelDiff) ? relDiff : maxRelDiff;
      if (relDiff > tol) converged = 0;
    }
    alphas[i] = alphasPrime[i];
    alphasPrime[i] = 0.0;
  }
  *maxRelDiffOut = maxRelDiff;
  return converged;
}

/* :1004-1020 (+ EMUtils.cpp:55-67) */
static double em_truncate(uint32_t M, double* alphas) {
  const double minAlpha = 1e-8;
  double alphaSum = 0.0;
  for (uint32_t i = 0; i < M; ++i) {
    if (alphas[i] <= minAlpha) alphas[i] = 0.0;
    alphaSum += alphas[i];
  }
  return alphaSum;
}

int orc_em_optimize(uint64_t C, uint32_t M, const uint64_t* off,
                    const uint32_t* tids, const double* aux,
                    const uint64_t* counts, const double* projected,
                    const double* eff_len, const uint64_t* unique,
                    const orc_em_params* p, double* alpha_out,
                    double* combined_out, uint8_t* valid_out,
                    double* eff_len_out, orc_em_stats* st) {
  em_state s;
  memset(&s, 0, sizeof(s));
  if (em_setup(C, M, off, tids, aux, counts, projected, eff_len, unique, p, &s)) {
    em_free(&s);
    return -1;
  }
  uint32_t itNum = 0;
  int converged = 0;
  double maxRelDiff = -DBL_MAX;
  /* :900 (no bias correction in scope) */
  while (itNum < p->min_iter || (itNum < p->max_iter && !converged)) {
    orc_em_step(C, M, off, tids, s.cw, counts, s.valid, s.prior, s.alphas,
                s.alphasPrime, s.expTheta, p->use_vbem);
    converged = em_converge_swap(M, s.alphas, s.alphasPrime, p->tol, &maxRelDiff);
    ++itNum;
  }
  double alphaSum = em_truncate(M, s.alphas);
  memcpy(alpha_out, s.alphas, (size_t)M * sizeof(double));
  if (combined_out) memcpy(combined_out, s.cw, (size_t)off[C] * sizeof(double));
  if (valid_out) memcpy(valid_out, s.valid, (size_t)C);
  if (eff_len_out) memcpy(eff_len_out, s.effLens, (size_t)M * sizeof(double));
  if (st) {
    st->iters = itNum;
    st->converged = (uint32_t)converged;
    st->max_rel_diff = maxRelDiff;
    st->alpha_sum = alphaSum;
    st->n_degenerate = s.n_degenerate;
    st->ok = !(alphaSum < MIN_WEIGHT);
  }
  em_free(&s);
  return 0;
}

/* ------------------------------------------------------------------------
 * Multi-threaded port: same decomposition as the reference (parallel_for over
 * classes, CAS accumulation, serial O(M) scans between).  OpenMP for oneTBB.
 * ---------------------------------------------------------------------- */
static inline void inc_loop(double* val, double inc) {
  /* salmon::utils::incLoop (SalmonUtils.hpp:166-172) */
  uint64_t* p = (uint64_t*)val;
  uint64_t oldb = __atomic_load_n(p, __ATOMIC_RELAXED);
  for (;;) {
    double oldv, newv;
    memcpy(&oldv, &oldb, 8);
    newv = oldv + inc;
    uint64_t newb;
    memcpy(&newb, &newv, 8);
    if (__atomic_compare_exchange_n(p, &oldb, newb, 0, __ATOMIC_SEQ_CST,
                                    __ATOMIC_RELAXED))
      break;
  }
}

static void em_step_mt(uint64_t C, uint32_t M, const uint64_t* off,
                       const uint32_t* tids, const double* cw,
                       const uint64_t* counts, const uint8_t* valid,
                       const double* prior, const double* alpha_in,
                       double* alpha_out, double* exp_theta, int vbem) {
  const double* theta = alpha_in;
  if (vbem) {
    double alphaSum = 0.0;
    for (uint32_t i = 0; i < M; ++i) alphaSum += alpha_in[i] + prior[i]; /* serial, :251-254 */
    double logNorm = orc_digamma(alphaSum);
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)M; ++i) {
      double ap = alpha_in[i] + prior[i];
      exp_theta[i] = (ap > DIGAMMA_MIN) ? exp(orc_digamma(ap) - logNorm) : 0.0;
      alpha_out[i] = 0.0;
    }
    theta = exp_theta;
  }
#pragma omp parallel for schedule(dynamic, 1024)
  for (int64_t c = 0; c < (int64_t)C; ++c) {
    if (!valid[c]) continue;
    uint64_t b = off[c], e = off[c + 1];
    uint64_t n = e - b;
    double count = (double)counts[c];
    if (n > 1) {
      double denom = 0.0;
      if (vbem) {
        for (uint64_t j = b; j < e; ++j) {
          double th = theta[tids[j]];
          if (th > 0.0) denom += th * cw[j];
        }
      } else {
        for (uint64_t j = b; j < e; ++j) denom += theta[tids[j]] * cw[j];
      }
      if (denom <= MIN_EQ_CLASS_WEIGHT) continue;
      double invDenom = count / denom;
      for (uint64_t j = b; j < e; ++j) {
        double th = theta[tids[j]];
        double v = th * cw[j];
        if (vbem ? (th > 0.0) : !isnan(v)) inc_loop(&alpha_out[tids[j]], v * invDenom);
      }
    } else if (n == 1) {
      inc_loop(&alpha_out[tids[b]], count);
    }
  }
}

int orc_em_optimize_mt(uint64_t C, uint32_t M, const uint64_t* off,
                       const uint32_t* tids, const double* aux,
                       const uint64_t* counts, const double* projected,
                       const double* eff_len, const uint64_t* unique,
                       const orc_em_params* p, double* alpha_out,
                       orc_em_stats* st) {
#ifdef _OPENMP
  if (p->n_threads > 0) omp_set_num_threads(p->n_threads);
#endif
  em_state s;
  memset(&s, 0, sizeof(s));
  if (em_setup(C, M, off, tids, aux, counts, projected, eff_len, unique, p, &s)) {
    em_free(&s);
    return -1;
  }
  uint32_t itNum = 0;
  int converged = 0;
  double maxRelDiff = -DBL_MAX;
  while (itNum < p->min_iter || (itNum < p->max_iter && !converged)) {
    em_step_mt(C, M, off, tids, s.cw, counts, s.valid, s.prior, s.alphas,
               s.alphasPrime, s.expTheta, p->use_vbem);
    converged = em_converge_swap(M, s.alphas, s.alphasPrime, p->tol, &maxRelDiff);
    ++itNum;
  }
  double alphaSum = em_truncate(M, s.alphas);
  memcpy(alpha_out, s.alphas, (size_t)M * sizeof(double));
  if (st) {
    st->iters = itNum;
    st->converged = (uint32_t)converged;
    st->max_rel_diff = maxRelDiff;
    st->alpha_sum = alphaSum;
    st->n_degenerate = s.n_degenerate;
    st->ok = !(alphaSum < MIN_WEIGHT);
  }
  em_free(&s);
  return 0;
}

/* GZipWriter.cpp:719-736 (numMappedFrags cancels; kept for rounding fidelity
 * with explicitSum=true, i.e. numMappedFrags = sum of sharedCount). */
void orc_tpm(uint32_t M, const double* alpha, const double* eff_len, double* tpm) {
  double numMappedFrags = 0.0;
  for (uint32_t i = 0; i < M; ++i) numMappedFrags += alpha[i];
  double tfracDenom = 0.0;
  for (uint32_t i = 0; i < M; ++i) tfracDenom += (alpha[i] / numMappedFrags) / eff_len[i];
  for (uint32_t i = 0; i < M; ++i) {
    double npm = alpha[i] / numMappedFrags;
    double tfrac = (npm / eff_len[i]) / tfracDenom;
    tpm[i] = tfrac * 1000000.0;
  }
}

/* ------------------------------------------------------------------------
 * Counter RNG (Philox-4x32-10, Salmon et al. SC'11 -- public algorithm).
 * ---------------------------------------------------------------------- */
void orc_philox4x32(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                    uint32_t k0, uint32_t k1, uint32_t* out) {
  for (int r = 0; r < 10; ++r) {
    uint64_t p0 = (uint64_t)0xD2511F53u * c0;
    uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
    uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
    uint32_t n1 = (uint32_t)p1;
    uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
    uint32_t n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

static inline uint64_t mulhi64(uint64_t a, uint64_t b) {
  return (uint64_t)(((unsigned __int128)a * b) >> 64);
}
static inline double u53(uint32_t hi, uint32_t lo) {
  uint64_t x = ((uint64_t)hi << 32) | lo;
  return (double)(x >> 11) * (1.0 / 9007199254740992.0);
}

/* ------------------------------------------------------------------------
 * Bootstrap: CollapsedEMOptimizer.cpp:398-552 (doBootstrap) with the class
 * list/weights prepared as in gatherBootstraps (:635-668).
 * Stream ids: c3 = 0 bootstrap resampling.
 * ---------------------------------------------------------------------- */
int orc_bootstrap(uint64_t C, uint32_t M, const uint64_t* off,
                  const uint32_t* tids, const double* cw, const uint64_t* counts,
                  const uint8_t* valid, const double* prior,
                  const uint8_t* active, const orc_em_params* p,
                  uint32_t n_boot, uint64_t seed, double* alphas_out,
                  uint64_t* samp_counts_out) {
  /* valid classes only (:641); integer CDF of origCounts */
  uint64_t* cdf = (uint64_t*)malloc((C ? C : 1) * sizeof(uint64_t));
  uint64_t* samp = (uint64_t*)malloc((C ? C : 1) * sizeof(uint64_t));
  double* alphas = (double*)malloc((size_t)(M ? M : 1) * sizeof(double));
  double* alphasPrime = (double*)malloc((size_t)(M ? M : 1) * sizeof(double));
  double* expTheta = (double*)malloc((size_t)(M ? M : 1) * sizeof(double));
  if (!cdf || !samp || !alphas || !alphasPrime || !expTheta) return -1;
  uint64_t total = 0;
  for (uint64_t c = 0; c < C; ++c) {
    if (!valid || valid[c]) total += counts[c];
    cdf[c] = total; /* inclusive */
  }
  uint64_t nActive = 0;
  for (uint32_t i = 0; i < M; ++i) nActive += active[i] ? 1 : 0;
  double scale = 1.0 / (double)nActive;          /* :607 */
  double totalNumFrags = (double)total;           /* totalCount passed as totalNumFrags (:681) */
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  for (uint32_t b = 0; b < n_boot; ++b) {
    memset(samp, 0, (C ? C : 1) * sizeof(uint64_t));
    for (uint64_t f = 0; f < total; ++f) {      /* :443-445 */
      uint32_t r[4];
      orc_philox4x32((uint32_t)f, (uint32_t)(f >> 32), b, 0u, k0, k1, r);
      uint64_t x = mulhi64(((uint64_t)r[1] << 32) | r[0], total);
      /* first class with cdf > x */
      uint64_t lo = 0, hi = C;
      while (lo < hi) {
        uint64_t mid = (lo + hi) >> 1;
        if (cdf[mid] > x) hi = mid; else lo = mid + 1;
      }
      ++samp[lo];
    }
    for (uint32_t i = 0; i < M; ++i) {           /* :450-453 */
      alphas[i] = active[i] ? scale * totalNumFrags : 0.0;
      alphasPrime[i] = 0.0;
    }
    int converged = 0;
    double maxRelDiff = -DBL_MAX;
    uint32_t itNum = 0;
    while (itNum < p->min_iter || (itNum < p->max_iter && !converged)) { /* :467 */
      orc_em_step_serial(C, M, off, tids, cw, samp, valid, prior, alphas,
                         alphasPrime, expTheta, p->use_vbem);
      converged = em_converge_swap(M, alphas, alphasPrime, p->tol, &maxRelDiff);
      ++itNum;
    }
    double alphaSum = em_truncate(M, alphas);   /* :507-519 */
    if (alphaSum < MIN_WEIGHT) return 1;        /* :521-525 */
    /* useScaledCounts is false for quasi-mapping (:414) */
    memcpy(alphas_out + (size_t)b * M, alphas, (size_t)M * sizeof(double));
    if (samp_counts_out) memcpy(samp_counts_out + (size_t)b * C, samp, C * sizeof(uint64_t));
  }
  free(cdf); free(samp); free(alphas); free(alphasPrime); free(expTheta);
  return 0;
}

/* ------------------------------------------------------------------------
 * Gibbs: CollapsedGibbsSampler.cpp:92-278 (round), :317-508 (driver).
 * Stream ids: c3 = 1 multinomial draws, c3 = 2 gamma draws.
 * ---------------------------------------------------------------------- */
static double gamma_mt(double shape, double scale, uint32_t i, uint32_t round,
                       uint32_t k0, uint32_t k1) {
  /* Marsaglia & Tsang (2000) on the counter RNG; replaces
   * std::gamma_distribution<double> d(ci, 1/(beta+effLen)) (:146-147). */
  double a = shape, boost = 1.0;
  uint32_t attempt = 0;
  uint32_t r[4];
  /* no gamma distribution, and the loop below would never accept (the device returns NaN too) */
  if (!(shape > 0.0) || isinf(shape)) return NAN;
  if (a < 1.0) {
    orc_philox4x32(i, 0xFFFFFFFFu, round, 2u, k0, k1, r);
    double u = u53(r[1], r[0]);
    if (u <= 0.0) u = 1.0 / 9007199254740992.0;
    boost = pow(u, 1.0 / a);
    a += 1.0;
  }
  double d = a - 1.0 / 3.0;
  double c = 1.0 / sqrt(9.0 * d);
  for (;; ++attempt) {
    orc_philox4x32(i, attempt, round, 2u, k0, k1, r);
    double u1 = ((double)r[0] + 0.5) * (1.0 / 4294967296.0);
    double u2 = ((double)r[1] + 0.5) * (1.0 / 4294967296.0);
    double x = sqrt(-2.0 * log(u1)) * cos(2.0 * M_PI * u2);
    double v = 1.0 + c * x;
    if (v <= 0.0) continue;
    v = v * v * v;
    double u = u53(r[3], r[2]);
    if (u <= 0.0) u = 1.0 / 9007199254740992.0;
    if (log(u) < 0.5 * x * x + d - d * v + d * log(v)) return d * v * boost * scale;
  }
}

double orc_gamma_draw(double shape, double scale, uint32_t i, uint32_t round,
                      uint32_t k0, uint32_t k1) {
  return gamma_mt(shape, scale, i, round, k0, k1);
}

int orc_gibbs(uint64_t C, uint32_t M, const uint64_t* off, const uint32_t* tids,
              const double* weights, const uint64_t* counts,
              const uint8_t* valid, const double* eff_len,
              const double* alphas_init, int use_vbem, int per_txp_prior_in,
              double vb_prior, uint32_t n_samples, uint32_t thinning,
              int no_gamma_draw, double num_mapped_frags, uint64_t seed,
              double* samples_out) {
  return orc_gibbs_ex(C, M, off, tids, weights, counts, valid, eff_len, alphas_init,
                      use_vbem, per_txp_prior_in, vb_prior, n_samples, thinning,
                      no_gamma_draw, num_mapped_frags, seed, 0, samples_out, NULL, NULL);
}

int orc_gibbs_ex(uint64_t C, uint32_t M, const uint64_t* off, const uint32_t* tids,
                 const double* weights, const uint64_t* counts,
                 const uint8_t* valid, const double* eff_len,
                 const double* alphas_init, int use_vbem, int per_txp_prior_in,
                 double vb_prior, uint32_t n_samples, uint32_t thinning,
                 int no_gamma_draw, double num_mapped_frags, uint64_t seed,
                 uint32_t round0, double* samples_out, double* last_mu,
                 double* last_cnt) {
  const double beta = 0.1;
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  /* :357-371, :296-315 */
  int perTxp = use_vbem ? per_txp_prior_in : 1;
  double prior = 1e-3;
  if (use_vbem) {
    if (perTxp) prior = (vb_prior < 1.0) ? 1.0 : vb_prior;
    else prior = (vb_prior < 1e-3) ? 1e-3 : vb_prior;
  }
  double* priorAlphas = (double*)malloc((size_t)(M ? M : 1) * sizeof(double));
  double* alphasIn = (double*)malloc((size_t)(M ? M : 1) * sizeof(double));
  double* alphasInit = (double*)malloc((size_t)(M ? M : 1) * sizeof(double));
  double* mu = (double*)calloc((size_t)(M ? M : 1), sizeof(double));
  uint8_t* active = (uint8_t*)calloc((size_t)(M ? M : 1), 1);
  uint64_t maxLen = 1;
  for (uint64_t c = 0; c < C; ++c) if (off[c + 1] - off[c] > maxLen) maxLen = off[c + 1] - off[c];
  double* prob = (double*)malloc(maxLen * sizeof(double));
  if (!priorAlphas || !alphasIn || !alphasInit || !mu || !active || !prob) return -1;
  for (uint32_t i = 0; i < M; ++i) {
    double ml = eff_len[i] > 1.0 ? eff_len[i] : 1.0;
    priorAlphas[i] = perTxp ? prior : prior * ml;
    alphasIn[i] = alphasInit[i] = alphas_init[i];
  }
  /* :382-410 */
  for (uint64_t c = 0; c < C; ++c)
    if (!valid || valid[c])
      for (uint64_t j = off[c]; j < off[c + 1]; ++j) active[tids[j]] = 1;
  for (uint32_t i = 0; i < M; ++i)
    if (!active[i]) alphasIn[i] = alphasInit[i] = 0.0;
  /* :425-442 */
  uint32_t nchains = 1;
  if (n_samples >= 50) nchains = 2;
  if (n_samples >= 100) nchains = 4;
  if (n_samples >= 200) nchains = 8;
  uint32_t step = n_samples / nchains;
  uint32_t round_global = round0;
  for (uint32_t sampleID = 0; sampleID < n_samples; ++sampleID) {
    /* :457-461 chain restarts at i*step, i>=1 */
    if (nchains > 1 && sampleID > 0 && sampleID % step == 0 && sampleID / step < nchains)
      memcpy(alphasIn, alphasInit, (size_t)M * sizeof(double));
    for (uint32_t rnd = 0; rnd < thinning; ++rnd, ++round_global) {
      /* :123-162 */
      for (uint32_t i = 0; i < M; ++i) {
        if (!active[i]) continue;
        double ci = alphasIn[i] + priorAlphas[i];
        if (no_gamma_draw) mu[i] = ci / eff_len[i];
        else mu[i] = gamma_mt(ci, 1.0 / (beta + eff_len[i]), i, round_global, k0, k1);
        alphasIn[i] = 0.0;
      }
      /* :188-270 */
      for (uint64_t c = 0; c < C; ++c) {
        if (valid && !valid[c]) continue;
        uint64_t b = off[c], n = off[c + 1] - off[c];
        uint64_t classCount = counts[c];
        if (n > 1) {
          double denom = 0.0;
          for (uint64_t i = 0; i < n; ++i) {
            prob[i] = (1000.0 * mu[tids[b + i]]) * weights[b + i];
            denom += prob[i];
          }
          if (denom <= DENORM_MIN) {
            denom = 0.0;
            for (uint64_t i = 0; i < n; ++i) {
              prob[i] = 1.0 / eff_len[tids[b + i]];
              denom += prob[i];
            }
            if (denom <= DENORM_MIN) {
              for (uint64_t i = 0; i < n; ++i) prob[i] = 1.0;
              denom = (double)n;
            }
          }
          if (denom > DENORM_MIN) {
            /* std::discrete_distribution draw == inverse CDF on the normalised
             * weights; here: first i with cumsum_i > u*denom (last index on tie). */
            for (uint64_t s = 0; s < classCount; ++s) {
              uint32_t r[4];
              orc_philox4x32((uint32_t)c, (uint32_t)s,
                             round_global, 1u | ((uint32_t)(c >> 32) << 8) | ((uint32_t)(s >> 32) << 16),
                             k0, k1, r);
              double target = u53(r[1], r[0]) * denom;
              double cum = 0.0;
              uint64_t pick = n - 1;
              for (uint64_t i = 0; i < n; ++i) {
                cum += prob[i];
                if (cum > target) { pick = i; break; }
              }
              alphasIn[tids[b + pick]] += 1.0;
            }
          }
        } else if (n == 1) {
          alphasIn[tids[b]] += (double)(int)classCount;
        }
      }
    }
    /* :489-503 (dontExtrapolateCounts=false) */
    double denom = 0.0;
    for (uint32_t t = 0; t < M; ++t) denom += mu[t] * eff_len[t];
    double scale = num_mapped_frags / denom;
    double* out = samples_out + (size_t)sampleID * M;
    for (uint32_t t = 0; t < M; ++t) {
      double a = (mu[t] * eff_len[t]) * scale;
      out[t] = (a > 1e-8) ? a : 0.0;
    }
  }
  if (last_mu) memcpy(last_mu, mu, (size_t)M * sizeof(double));
  if (last_cnt) memcpy(last_cnt, alphasIn, (size_t)M * sizeof(double));
  free(priorAlphas); free(alphasIn); free(alphasInit); free(mu); free(active); free(prob);
  return 0;
}
