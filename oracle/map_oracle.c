/*
 * oracle/map_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE (see map_oracle.h).
 * Straightforward, allocation-happy, sort-based statement of Stage A ("MAPSPEC" in DESIGN.md).
 */
#include "map_oracle.h"
#include "em_oracle.h"
#include "orc_math.h"

#include <limits.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define LOG_0 HUGE_VAL
#define LOG_1 0.0
#define EPSILON_ 0.375e-10
#define MAXSEEDS 2048
#define MAXCAND 64
#define NEG_SCORE (-(1 << 28))

/* include/salmon/internal/util/SalmonMath.hpp:54-66 */
static double logAdd(double x, double y) {
  if (fabs(x) == LOG_0) return y;
  if (fabs(y) == LOG_0) return x;
  if (y > x) { double t = x; x = y; y = t; }
  return x + log(1 + exp(y - x));
}

int orc_math_mode_ = ORC_MATH_LIBM;
void orc_set_math_mode(int mode) { orc_math_mode_ = mode ? ORC_MATH_FDLIBM : ORC_MATH_LIBM; }
int orc_get_math_mode(void) { return orc_math_mode_; }
/* test tap: exp over x[], log over y[] in the given mode */
void orc_math_probe(int mode, uint64_t nx, const double* x, double* ex, uint64_t ny, const double* y, double* ly) {
  for (uint64_t i = 0; i < nx; ++i) ex[i] = mode ? orc_fd_exp(x[i]) : exp(x[i]);
  for (uint64_t i = 0; i < ny; ++i) ly[i] = mode ? orc_fd_log(y[i]) : log(y[i]);
}

/* the same function on the mode's exp/log (per-alignment arithmetic, see orc_math.h) */
static double logAddDet(double x, double y) {
  if (fabs(x) == LOG_0) return y;
  if (fabs(y) == LOG_0) return x;
  if (y > x) { double t = x; x = y; y = t; }
  return x + m_log(1 + m_exp(y - x));
}

/* ---------------------------------------------------------------- FLD tables
 * FragmentLengthDistribution ctor (FragmentLengthDistribution.cpp:22-78) with alpha=1,
 * bin_size=1; pmf (:122-132), cmf (:146-161); after burn-in the cached, renormalised
 * tables (getLockedPMF :163-175, cmf(vector) :190-201).  boost::math::normal cdf =
 * 0.5*erfc(-(x-mu)/(sd*sqrt(2))). */
static double norm_cdf(double x, double mu, double sd) { return 0.5 * erfc(-(x - mu) / (sd * sqrt(2.0))); }

typedef struct {
  uint32_t max_val;
  double* hist;      /* log mass */
  double tot;        /* log total mass */
  double* pmf_live;  /* hist - tot */
  double* cmf_live;
  double* pmf_cached;
  double* cmf_cached;
  double* cmf_quirk; /* LogCMFCache before burn-in: cmf of a constant LOG_EPSILON pmf */
} fld_t;

static void fld_init(fld_t* f, double mean, double sd, uint32_t max_val) {
  const double LOG_EPSILON = log(EPSILON_);
  uint32_t n = max_val + 1;
  f->max_val = max_val;
  f->hist = (double*)malloc(n * sizeof(double));
  f->pmf_live = (double*)malloc(n * sizeof(double));
  f->cmf_live = (double*)malloc(n * sizeof(double));
  f->pmf_cached = (double*)malloc(n * sizeof(double));
  f->cmf_cached = (double*)malloc(n * sizeof(double));
  f->cmf_quirk = (double*)malloc(n * sizeof(double));
  f->tot = LOG_0;
  for (uint32_t i = 0; i < n; ++i) {
    double nm = norm_cdf(i + 0.5, mean, sd) - norm_cdf(i - 0.5, mean, sd);
    double mass = LOG_EPSILON;
    if (nm != 0) mass = 0.0 + log(nm);
    f->hist[i] = mass;
    f->tot = logAdd(f->tot, mass);
  }
  double cum = LOG_0, tm = LOG_0;
  for (uint32_t i = 0; i < n; ++i) {
    f->pmf_live[i] = f->hist[i] - f->tot;
    cum = logAdd(cum, f->hist[i]);
    f->cmf_live[i] = cum - f->tot;
    tm = logAdd(tm, f->pmf_live[i]);
  }
  cum = LOG_0;
  double cq = LOG_0;
  for (uint32_t i = 0; i < n; ++i) {
    f->pmf_cached[i] = f->pmf_live[i] - tm;
    cum = logAdd(cum, f->pmf_cached[i]);
    f->cmf_cached[i] = cum;
    cq = logAdd(cq, LOG_EPSILON);   /* DistributionUtils.cpp:103-116 (logPMF stays LOG_EPSILON) */
    f->cmf_quirk[i] = cq;
  }
}
static void fld_free(fld_t* f) {
  free(f->hist); free(f->pmf_live); free(f->cmf_live); free(f->pmf_cached); free(f->cmf_cached);
  free(f->cmf_quirk);
}
static double tab(const double* t, uint32_t max_val, uint64_t len) { return t[len > max_val ? max_val : len]; }

void orc_fld_tables(double mean, double sd, uint32_t max_val, double* log_pmf, double* log_cmf) {
  fld_t f;
  fld_init(&f, mean, sd, max_val);
  memcpy(log_pmf, f.pmf_live, (max_val + 1) * sizeof(double));
  memcpy(log_cmf, f.cmf_live, (max_val + 1) * sizeof(double));
  fld_free(&f);
}

/* ---------------------------------------------------------------- index (sorted arrays) */
struct orc_index {
  uint32_t n_txps, k;
  uint64_t total;
  uint64_t* off;      /* [n+1] */
  uint8_t* codes;     /* [total] */
  uint64_t n_kmers;
  uint64_t* kmers;    /* sorted distinct canonical k-mers */
  uint64_t* post_off; /* [n_kmers+1] */
  uint32_t* post;     /* global positions, ascending per k-mer */
};

typedef struct { uint64_t km; uint32_t pos; } kp_t;
static int cmp_kp(const void* a, const void* b) {
  const kp_t* x = (const kp_t*)a; const kp_t* y = (const kp_t*)b;
  if (x->km != y->km) return x->km < y->km ? -1 : 1;
  return x->pos < y->pos ? -1 : (x->pos > y->pos);
}
static uint64_t rc_kmer(uint64_t km, uint32_t k) {
  uint64_t r = 0;
  for (uint32_t i = 0; i < k; ++i) { r = (r << 2) | (3 - (km & 3)); km >>= 2; }
  return r;
}

orc_index* orc_index_build(uint32_t n, const uint64_t* seq_off, const uint8_t* codes, uint32_t k) {
  orc_index* ix = (orc_index*)calloc(1, sizeof(orc_index));
  ix->n_txps = n; ix->k = k; ix->total = seq_off[n];
  ix->off = (uint64_t*)malloc((n + 1) * sizeof(uint64_t));
  memcpy(ix->off, seq_off, (n + 1) * sizeof(uint64_t));
  ix->codes = (uint8_t*)malloc(ix->total ? ix->total : 1);
  memcpy(ix->codes, codes, ix->total);
  uint64_t cap = 0;
  for (uint32_t t = 0; t < n; ++t) { uint64_t L = seq_off[t + 1] - seq_off[t]; if (L >= k) cap += L - k + 1; }
  kp_t* kp = (kp_t*)malloc((cap ? cap : 1) * sizeof(kp_t));
  uint64_t m = 0;
  for (uint32_t t = 0; t < n; ++t) {
    uint64_t b = seq_off[t], e = seq_off[t + 1];
    for (uint64_t p = b; p + k <= e; ++p) {
      uint64_t km = 0; int bad = 0;
      for (uint32_t i = 0; i < k; ++i) { uint8_t c = codes[p + i]; if (c > 3) { bad = 1; break; } km = (km << 2) | c; }
      if (bad) continue;
      uint64_t rc = rc_kmer(km, k);
      kp[m].km = km < rc ? km : rc; kp[m].pos = (uint32_t)p; ++m;
    }
  }
  qsort(kp, m, sizeof(kp_t), cmp_kp);
  uint64_t nk = 0;
  for (uint64_t i = 0; i < m; ++i) if (i == 0 || kp[i].km != kp[i - 1].km) ++nk;
  ix->n_kmers = nk;
  ix->kmers = (uint64_t*)malloc((nk ? nk : 1) * sizeof(uint64_t));
  ix->post_off = (uint64_t*)malloc((nk + 1) * sizeof(uint64_t));
  ix->post = (uint32_t*)malloc((m ? m : 1) * sizeof(uint32_t));
  uint64_t j = 0;
  for (uint64_t i = 0; i < m; ++i) {
    if (i == 0 || kp[i].km != kp[i - 1].km) { ix->kmers[j] = kp[i].km; ix->post_off[j] = i; ++j; }
    ix->post[i] = kp[i].pos;
  }
  ix->post_off[nk] = m;
  free(kp);
  return ix;
}
void orc_index_free(orc_index* ix) {
  if (!ix) return;
  free(ix->off); free(ix->codes); free(ix->kmers); free(ix->post_off); free(ix->post); free(ix);
}
uint64_t orc_index_n_kmers(const orc_index* ix) { return ix->n_kmers; }

static int64_t idx_find(const orc_index* ix, uint64_t km) {
  uint64_t lo = 0, hi = ix->n_kmers;
  while (lo < hi) { uint64_t mid = (lo + hi) >> 1; if (ix->kmers[mid] < km) lo = mid + 1; else hi = mid; }
  return (lo < ix->n_kmers && ix->kmers[lo] == km) ? (int64_t)lo : -1;
}
static uint32_t txp_of(const orc_index* ix, uint64_t pos) {
  uint32_t lo = 0, hi = ix->n_txps;  /* last t with off[t] <= pos */
  while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (ix->off[mid] <= pos) lo = mid; else hi = mid; }
  return lo;
}

/* ---------------------------------------------------------------- per-mate seeding + chaining */
typedef struct { uint32_t tid; uint32_t ori; int32_t diag; int32_t qpos; } seed_t;
typedef struct { uint32_t tid; uint32_t ori; int32_t dmin, dmax, diag_c; uint32_t cov; } cand_t;

static int cmp_seed(const void* a, const void* b) {
  const seed_t* x = (const seed_t*)a; const seed_t* y = (const seed_t*)b;
  if (x->tid != y->tid) return x->tid < y->tid ? -1 : 1;
  if (x->ori != y->ori) return x->ori < y->ori ? -1 : 1;
  if (x->diag != y->diag) return x->diag < y->diag ? -1 : 1;
  return x->qpos < y->qpos ? -1 : (x->qpos > y->qpos);
}
static int cmp_cand_cov(const void* a, const void* b) {
  const cand_t* x = (const cand_t*)a; const cand_t* y = (const cand_t*)b;
  if (x->cov != y->cov) return x->cov > y->cov ? -1 : 1;
  if (x->tid != y->tid) return x->tid < y->tid ? -1 : 1;
  if (x->ori != y->ori) return x->ori < y->ori ? -1 : 1;
  return x->diag_c < y->diag_c ? -1 : (x->diag_c > y->diag_c);
}
static int cmp_cand_pos(const void* a, const void* b) {
  const cand_t* x = (const cand_t*)a; const cand_t* y = (const cand_t*)b;
  if (x->tid != y->tid) return x->tid < y->tid ? -1 : 1;
  if (x->ori != y->ori) return x->ori < y->ori ? -1 : 1;
  return x->diag_c < y->diag_c ? -1 : (x->diag_c > y->diag_c);
}

/* info (may be NULL): what the mate's seeds look like, see orc_mate_candidates */
static uint32_t mate_candidates_info(const orc_index* ix, const orc_map_params* p, const uint8_t* read,
                                     uint32_t L, cand_t* out, orc_map_counters* ctr, orc_mate_info* info) {
  const uint32_t K = p->k;
  if (info) memset(info, 0, sizeof(*info));
  if (L < K) return 0;
  seed_t* seeds = (seed_t*)malloc(MAXSEEDS * sizeof(seed_t));
  uint32_t ns = 0;
  /* sample positions 0, S, 2S, ... and the last k-mer */
  for (uint32_t i = 0, pi = 0;; i += p->stride, ++pi) {
    uint32_t pos_i = i;
    int last = 0;
    if (i > L - K) { if ((L - K) % p->stride == 0) break; pos_i = L - K; last = 1; }
    uint64_t fw = 0; int bad = 0;
    for (uint32_t j = 0; j < K; ++j) { uint8_t c = read[pos_i + j]; if (c > 3) { bad = 1; break; } fw = (fw << 2) | c; }
    if (!bad) {
      uint64_t rc = rc_kmer(fw, K);
      uint64_t canon = fw < rc ? fw : rc;
      ctr->lookups++;
      int64_t h = idx_find(ix, canon);
      if (h >= 0) {
        uint64_t b = ix->post_off[h], e = ix->post_off[h + 1];
        if (e - b <= p->max_occs_per_hit) {
          if (info) {
            if (!info->cut_round && ns + (e - b) > MAXSEEDS) info->cut_round = 1 + pi / 32;
            info->postings_all += (uint32_t)(e - b);
          }
          for (uint64_t q = b; q < e && ns < MAXSEEDS; ++q) {
            ctr->postings++;
            uint64_t gp = ix->post[q];
            uint64_t rf = 0;
            for (uint32_t j = 0; j < K; ++j) rf = (rf << 2) | ix->codes[gp + j];
            uint32_t tid = txp_of(ix, gp);
            int32_t tpos = (int32_t)(gp - ix->off[tid]);
            seed_t s;
            s.tid = tid;
            if (rf == fw) { s.ori = 0; s.qpos = (int32_t)pos_i; }
            else { s.ori = 1; s.qpos = (int32_t)(L - K - pos_i); }
            s.diag = tpos - s.qpos;
            seeds[ns++] = s;
          }
        }
      }
    }
    if (last) break;
  }
  if (info) {
    info->lookups = (uint32_t)ctr->lookups;   /* the caller passes fresh counters */
    info->seeds = ns;
  }
  ctr->seeds += ns;
  qsort(seeds, ns, sizeof(seed_t), cmp_seed);
  /* chains: same (tid, ori), consecutive diagonals at most chain_gap apart */
  cand_t* all = (cand_t*)malloc((ns ? ns : 1) * sizeof(cand_t));
  uint32_t nc = 0;
  uint32_t i = 0;
  while (i < ns) {
    uint32_t j = i + 1;
    while (j < ns && seeds[j].tid == seeds[i].tid && seeds[j].ori == seeds[i].ori &&
           seeds[j].diag - seeds[j - 1].diag <= (int32_t)p->chain_gap) ++j;
    uint8_t covered[256];
    memset(covered, 0, sizeof(covered));
    for (uint32_t s = i; s < j; ++s)
      for (uint32_t b = 0; b < K; ++b) { int32_t q = seeds[s].qpos + (int32_t)b; if (q >= 0 && q < 256) covered[q] = 1; }
    uint32_t cov = 0;
    for (uint32_t b = 0; b < 256; ++b) cov += covered[b];
    if (info) {   /* the chain spans seeds i..j-1: does it cross a 32-key chunk of the seed array / of the array of
                   * distinct (tid, ori, diag) keys? */
      uint32_t d0 = info->distinct;
      for (uint32_t s = i; s < j; ++s)
        if (s == i || seeds[s].diag != seeds[s - 1].diag) ++info->distinct;
      info->straddle_seeds += (i / 32 != (j - 1) / 32);
      info->straddle_distinct += (d0 / 32 != (info->distinct - 1) / 32);
    }
    cand_t c;
    c.tid = seeds[i].tid; c.ori = seeds[i].ori; c.dmin = seeds[i].diag; c.dmax = seeds[j - 1].diag;
    c.diag_c = c.dmin + (c.dmax - c.dmin) / 2; c.cov = cov;
    all[nc++] = c;
    i = j;
  }
  uint32_t best = 0;
  for (uint32_t c = 0; c < nc; ++c) if (all[c].cov > best) best = all[c].cov;
  uint32_t nk = 0;
  for (uint32_t c = 0; c < nc; ++c)
    if ((double)all[c].cov >= p->consensus_frac * (double)best) all[nk++] = all[c];
  if (info) { info->chains = nc; info->survivors = nk; }
  if (nk > MAXCAND) { qsort(all, nk, sizeof(cand_t), cmp_cand_cov); nk = MAXCAND; }
  qsort(all, nk, sizeof(cand_t), cmp_cand_pos);
  memcpy(out, all, nk * sizeof(cand_t));
  free(all); free(seeds);
  return nk;
}

static uint32_t mate_candidates(const orc_index* ix, const orc_map_params* p, const uint8_t* read,
                                uint32_t L, cand_t* out, orc_map_counters* ctr) {
  return mate_candidates_info(ix, p, read, L, out, ctr, NULL);
}

/* test hook: the candidates of one mate in (tid, ori, diag_c) order, as orc_map_reads derives them */
uint32_t orc_mate_candidates(const orc_index* ix, const orc_map_params* p, const uint8_t* read, uint32_t L,
                             orc_cand* out, orc_mate_info* info) {
  cand_t c[MAXCAND];
  orc_map_counters ctr;
  memset(&ctr, 0, sizeof ctr);
  const uint32_t n = mate_candidates_info(ix, p, read, L, c, &ctr, info);
  for (uint32_t a = 0; a < n; ++a) {
    out[a].tid = c[a].tid; out[a].ori = c[a].ori; out[a].diag_c = c[a].diag_c; out[a].cov = c[a].cov;
  }
  return n;
}

/* ---------------------------------------------------------------- banded affine glocal DP */
static int32_t dp_score(const orc_index* ix, const orc_map_params* p, const uint8_t* read, uint32_t L,
                        uint32_t ori, uint32_t tid, int32_t diag_c) {
  const int32_t B = (int32_t)p->band, W = 2 * B + 1;
  const int64_t tlen = (int64_t)(ix->off[tid + 1] - ix->off[tid]);
  const uint8_t* ref = ix->codes + ix->off[tid];
  int32_t Hp[128], Ep[128], Hc[128], Ec[128];
  for (int32_t j = 0; j < W; ++j) { Hp[j] = 0; Ep[j] = NEG_SCORE; }
  for (uint32_t i = 0; i < L; ++i) {
    uint8_t rb = ori ? (uint8_t)(read[L - 1 - i] > 3 ? 4 : 3 - read[L - 1 - i]) : read[i];
    int32_t Fprev = NEG_SCORE, Hleft = NEG_SCORE;
    for (int32_t j = 0; j < W; ++j) {
      int64_t r = (int64_t)diag_c + (int64_t)i + (j - B);
      int32_t h = NEG_SCORE, e = NEG_SCORE, f = NEG_SCORE;
      if (r >= 0 && r < tlen) {
        int32_t s = (rb < 4 && rb == ref[r]) ? p->ma : p->mp;
        int32_t m = Hp[j] + s;
        if (j + 1 < W) {
          int32_t a = Hp[j + 1] - p->go - p->ge, b = Ep[j + 1] - p->ge;
          e = a > b ? a : b;
        }
        if (j > 0) {
          int32_t a = Hleft - p->go - p->ge, b = Fprev - p->ge;
          f = a > b ? a : b;
        }
        h = m;
        if (e > h) h = e;
        if (f > h) h = f;
        if (h < NEG_SCORE) h = NEG_SCORE;
        if (e < NEG_SCORE) e = NEG_SCORE;
        if (f < NEG_SCORE) f = NEG_SCORE;
      }
      Hc[j] = h; Ec[j] = e;
      Hleft = h; Fprev = f;
    }
    memcpy(Hp, Hc, W * sizeof(int32_t));
    memcpy(Ep, Ec, W * sizeof(int32_t));
  }
  int32_t best = NEG_SCORE;
  for (int32_t j = 0; j < W; ++j) if (Hp[j] > best) best = Hp[j];
  return best;
}

/* test hook: the DP score of one read against one reference of an index (tests/test_dp_vs_edlib.py pins the recurrence
 * against the reference tree's own edlib build, oracle/_ref/libedlib_ref.so) */
int32_t orc_dp_score(const orc_index* ix, const orc_map_params* p, const uint8_t* read, uint32_t L, uint32_t ori,
                     uint32_t tid, int32_t diag_c) {
  return dp_score(ix, p, read, L, ori, tid, diag_c);
}

/* ---------------------------------------------------------------- joint hits */
typedef struct {
  uint32_t tid; int32_t li, ri;   /* candidate indices, -1 if absent */
  int32_t frag_len; uint32_t status; /* 0 paired, 1 left orphan, 2 right orphan */
} joint_t;

typedef struct { int32_t idx; int32_t tid; } perm_t;
static int cmp_perm(const void* a, const void* b) {
  const perm_t* x = (const perm_t*)a; const perm_t* y = (const perm_t*)b;
  return x->tid < y->tid ? -1 : (x->tid > y->tid);
}

struct orc_online;
static void online_fragment(struct orc_online* on, uint32_t r, uint32_t L, uint32_t na, const uint32_t* tid,
                            const int32_t* pos, const int32_t* mate_pos, const uint8_t* flags, const int32_t* flen,
                            const double* aux);

static int map_reads_core(const orc_index* ix, const orc_map_params* p, const fld_t* fldp, int useAux, int burnedIn,
                          struct orc_online* on, const uint8_t* left,
                  const uint8_t* right, uint32_t n, uint32_t L,
                  uint32_t* n_aln, uint32_t* aln_tid, int32_t* aln_score, double* aln_prob,
                  int32_t* aln_pos, int32_t* aln_mate_pos, uint8_t* aln_flags, int32_t* aln_flen,
                  uint32_t* label, double* weight, orc_map_counters* ctr) {
  const double LOG_EPSILON = log(EPSILON_);
  const uint32_t cap = p->max_read_occ;
  const fld_t fld = *fldp;   /* tables of the state the batch starts from (frozen for the batch) */
  orc_map_counters local;
  memset(&local, 0, sizeof(local));
  cand_t* lc = (cand_t*)malloc(MAXCAND * sizeof(cand_t));
  cand_t* rcand = (cand_t*)malloc(MAXCAND * sizeof(cand_t));
  joint_t* jh = (joint_t*)malloc((size_t)(MAXCAND * MAXCAND + 2 * MAXCAND) * sizeof(joint_t));
  int32_t* scores = (int32_t*)malloc((size_t)(MAXCAND * MAXCAND + 2 * MAXCAND) * sizeof(int32_t));
  perm_t* perm = (perm_t*)malloc((size_t)(MAXCAND * MAXCAND + 2 * MAXCAND) * sizeof(perm_t));
  /* best score per transcript: small open list (reads hit few transcripts) */
  int32_t* bs_tid = (int32_t*)malloc((size_t)(MAXCAND * MAXCAND + 2 * MAXCAND) * sizeof(int32_t));
  int32_t* bs_score = (int32_t*)malloc((size_t)(MAXCAND * MAXCAND + 2 * MAXCAND) * sizeof(int32_t));
  int32_t* bs_idx = (int32_t*)malloc((size_t)(MAXCAND * MAXCAND + 2 * MAXCAND) * sizeof(int32_t));

  for (uint32_t r = 0; r < n; ++r) {
    const uint8_t* rl = left + (size_t)r * L;
    const uint8_t* rr = right + (size_t)r * L;
    n_aln[r] = 0;
    uint32_t nl = mate_candidates(ix, p, rl, L, lc, &local);
    uint32_t nr = mate_candidates(ix, p, rr, L, rcand, &local);
    /* ---- join (inward pairs; single-end libraries arrive with an all-N second mate, i.e. left orphans only, and the
     *      orphan threshold does not apply to them: joinReadsAndFilterSingle) with the constraint policy salmon sets
     *      (SalmonMappingUtils.hpp:208-220; ProgramOptionsGenerator.cpp:111-137,198-201; MAPSPEC step 4):
     *      pre-merge filter per mate and transcript, concordant pairs, post-merge filter per transcript, pair consensus
     *      over the read, else orphans above the orphan threshold */
    uint32_t nj = 0;
    {
      uint8_t okl[MAXCAND], okr[MAXCAND];
      for (uint32_t a = 0; a < nl; ++a) {                 /* best chain of this mate on the transcript of chain a */
        uint32_t best = 0;
        for (uint32_t q = 0; q < nl; ++q) if (lc[q].tid == lc[a].tid && lc[q].cov > best) best = lc[q].cov;
        okl[a] = (double)lc[a].cov >= p->pre_merge_thresh * (double)best;
      }
      for (uint32_t b = 0; b < nr; ++b) {
        uint32_t best = 0;
        for (uint32_t q = 0; q < nr; ++q) if (rcand[q].tid == rcand[b].tid && rcand[q].cov > best) best = rcand[q].cov;
        okr[b] = (double)rcand[b].cov >= p->pre_merge_thresh * (double)best;
      }
      /* all geometrically valid pairs, left-major */
      uint32_t npair = 0, best_all = 0;
      for (uint32_t a = 0; a < nl; ++a)
        for (uint32_t b = 0; b < nr; ++b) {
          if (!okl[a] || !okr[b] || lc[a].tid != rcand[b].tid || lc[a].ori == rcand[b].ori) continue;
          const cand_t* fw = lc[a].ori == 0 ? &lc[a] : &rcand[b];
          const cand_t* rv = lc[a].ori == 0 ? &rcand[b] : &lc[a];
          int32_t start = fw->diag_c, end = rv->diag_c + (int32_t)L;
          if (rv->diag_c < fw->diag_c) {                  /* dovetail */
            if (!p->allow_dovetail) continue;
            start = rv->diag_c; end = fw->diag_c + (int32_t)L;
          }
          const int32_t fl = end - start;
          if (fl <= 0 || fl > (int32_t)p->max_frag_len) continue;
          joint_t j; j.tid = lc[a].tid; j.li = (int32_t)a; j.ri = (int32_t)b; j.frag_len = fl; j.status = 0;
          jh[npair++] = j;
          const uint32_t sc = lc[a].cov + rcand[b].cov;
          if (sc > best_all) best_all = sc;
        }
      /* post-merge per transcript + consensus over the read; order kept */
      for (uint32_t q = 0; q < npair; ++q) {
        const uint32_t sc = lc[jh[q].li].cov + rcand[jh[q].ri].cov;
        uint32_t best_t = 0;
        for (uint32_t w = 0; w < npair; ++w)
          if (jh[w].tid == jh[q].tid) { const uint32_t s2 = lc[jh[w].li].cov + rcand[jh[w].ri].cov; if (s2 > best_t) best_t = s2; }
        if ((double)sc < p->post_merge_thresh * (double)best_t || (double)sc < p->consensus_frac * (double)best_all) { jh[q].status = 9; }
      }
      for (uint32_t q = 0; q < npair; ++q) if (jh[q].status == 0) jh[nj++] = jh[q];
      if (nj == 0 && p->allow_orphans) {  /* orphans: lefts precede rights (SalmonQuantify.cpp:1407-1420) */
        uint32_t best_c = 0;
        for (uint32_t a = 0; a < nl; ++a) if (okl[a] && lc[a].cov > best_c) best_c = lc[a].cov;
        for (uint32_t b = 0; b < nr; ++b) if (okr[b] && rcand[b].cov > best_c) best_c = rcand[b].cov;
        const double thr = (p->lib_type >= 3 ? 0.0 : p->orphan_thresh) * (double)best_c;
        for (uint32_t a = 0; a < nl; ++a) if (okl[a] && (double)lc[a].cov >= thr) { joint_t j; j.tid = lc[a].tid; j.li = (int32_t)a; j.ri = -1; j.frag_len = 0; j.status = 1; jh[nj++] = j; }
        for (uint32_t b = 0; b < nr; ++b) if (okr[b] && (double)rcand[b].cov >= thr) { joint_t j; j.tid = rcand[b].tid; j.li = -1; j.ri = (int32_t)b; j.frag_len = 0; j.status = 2; jh[nj++] = j; }
      }
    }
    if (nj == 0 || nj > cap) continue;   /* unmapped, or more than maxReadOcc places */
    /* ---- scoring + updateRefMappings (SalmonMappingUtils.hpp:225-281) */
    const int32_t invalidScore = INT_MIN;
    int32_t bestScore = invalidScore, bestDecoyScore = invalidScore;
    uint32_t nperm = 0, nbs = 0;
    for (uint32_t h = 0; h < nj; ++h) {
      int32_t total = 0; int32_t maxPossible = 0; int bad = 0;
      if (jh[h].li >= 0) { int32_t s = dp_score(ix, p, rl, L, lc[jh[h].li].ori, jh[h].tid, lc[jh[h].li].diag_c); local.candidates++; if (s <= NEG_SCORE) bad = 1; total += s; maxPossible += p->ma * (int32_t)L; }
      if (jh[h].ri >= 0) { int32_t s = dp_score(ix, p, rr, L, rcand[jh[h].ri].ori, jh[h].tid, rcand[jh[h].ri].diag_c); local.candidates++; if (s <= NEG_SCORE) bad = 1; total += s; maxPossible += p->ma * (int32_t)L; }
      int32_t hitScore = (!bad && (double)total >= p->min_score_fraction * (double)maxPossible) ? total : invalidScore;
      scores[h] = hitScore;
      {
        /* compatibility with the expected library format (SalmonQuantify.cpp:1467-1517 paired-end, :2141-2147
         * single-end; salmon::utils::compatibleHit, SalmonUtils.cpp:193-298); incompatible mappings are skipped
         * (ignoreIncompat, :1519-1521) */
        const int isOrphan = jh[h].status != 0;
        const int isLeft = jh[h].status != 2;
        const int leftFw = jh[h].li >= 0 && lc[jh[h].li].ori == 0;
        const int rightFw = jh[h].ri >= 0 && rcand[jh[h].ri].ori == 0;
        int isCompat;
        switch (p->lib_type) {
          case 0: isCompat = isOrphan ? 1 : (leftFw != rightFw); break;                         /* IU */
          case 1: isCompat = isOrphan ? ((isLeft && leftFw) || (!isLeft && !rightFw)) : (leftFw && !rightFw); break;   /* ISF: SA */
          case 2: isCompat = isOrphan ? ((isLeft && !leftFw) || (!isLeft && rightFw)) : (!leftFw && rightFw); break;   /* ISR: AS */
          case 3: isCompat = 1; break;                                                          /* U */
          case 4: isCompat = leftFw; break;                                                     /* SF */
          case 5: isCompat = !leftFw; break;                                                    /* SR */
          default: isCompat = 1;
        }
        if (!isCompat) { scores[h] = invalidScore; continue; }
      }
      const int isDecoy = (int32_t)jh[h].tid >= p->first_decoy;
      const double decoyCutoff = (double)(int32_t)(p->decoy_threshold * (double)bestDecoyScore);
      if (isDecoy) { if (hitScore > bestDecoyScore) bestDecoyScore = hitScore; continue; }
      if ((double)hitScore < decoyCutoff || hitScore == invalidScore) continue;
      uint32_t q = 0;
      while (q < nbs && bs_tid[q] != (int32_t)jh[h].tid) ++q;
      if (q == nbs) { bs_tid[nbs] = (int32_t)jh[h].tid; bs_score[nbs] = hitScore; bs_idx[nbs] = (int32_t)h; ++nbs; }
      else if (hitScore > bs_score[q] || (hitScore == bs_score[q] /* and isCompat: always true for IU */)) {
        bs_score[q] = hitScore; scores[bs_idx[q]] = invalidScore; bs_idx[q] = (int32_t)h;
      } else {
        scores[h] = invalidScore;
      }
      if (hitScore > bestScore) bestScore = hitScore;
      perm[nperm].idx = (int32_t)h; perm[nperm].tid = (int32_t)jh[h].tid; ++nperm;
    }
    /* ---- filterAndCollectAlignments (:283-405) */
    if (bestDecoyScore == invalidScore) bestDecoyScore = invalidScore + 1;
    const int32_t decoyThreshold = (int32_t)(p->decoy_threshold * (double)bestDecoyScore);
    const int32_t scoreThreshold = p->hard_filter ? bestScore : decoyThreshold;
    uint32_t nkept = 0;
    for (uint32_t q = 0; q < nperm; ++q)
      if (scores[perm[q].idx] >= scoreThreshold) perm[nkept++] = perm[q];
    qsort(perm, nkept, sizeof(perm_t), cmp_perm);   /* tids are unique after the dedup above */
    uint32_t na = 0;
    const size_t base = (size_t)r * cap;
    for (uint32_t q = 0; q < nkept; ++q) {
      const joint_t* j = &jh[perm[q].idx];
      double v = (double)bestScore - (double)scores[perm[q].idx];
      double estAlnProb = p->hard_filter ? -1.0 : m_exp(-p->score_exp * v);
      if (!p->hard_filter && estAlnProb < p->min_aln_prob) continue;
      const cand_t* first = (j->status == 2) ? &rcand[j->ri] : &lc[j->li];
      aln_tid[base + na] = j->tid;
      aln_score[base + na] = scores[perm[q].idx];
      aln_prob[base + na] = estAlnProb;
      aln_pos[base + na] = first->diag_c;
      aln_mate_pos[base + na] = (j->status == 0) ? rcand[j->ri].diag_c : 0;
      uint8_t fl = (uint8_t)((first->ori == 0) ? 1 : 0);
      if (j->status == 0 && rcand[j->ri].ori == 0) fl |= 2;
      fl |= (uint8_t)(j->status << 2);
      aln_flags[base + na] = fl;
      aln_flen[base + na] = j->frag_len;
      ++na;
    }
    n_aln[r] = na;
    local.kept += na;
    if (na == 0) continue;
    local.mapped++;
    local.label_entries += na;
    /* ---- auxiliary probabilities + label (SalmonQuantify.cpp:599-857), state frozen per batch */
    double auxDenom = LOG_0;
    double aux[256];
    for (uint32_t a = 0; a < na; ++a) {
      const uint32_t tid = aln_tid[base + a];
      const int32_t refLen = (int32_t)(ix->off[tid + 1] - ix->off[tid]);
      const double refLength = refLen > 0 ? (double)refLen : 1.0;
      const uint32_t status = (aln_flags[base + a] >> 2) & 3;
      const int fwd = aln_flags[base + a] & 1, mateFwd = (aln_flags[base + a] >> 1) & 1;
      const double coverage = aln_prob[base + a];
      const double logFragCov = (coverage > 0) ? m_log(coverage) : LOG_1;          /* :602-603 */
      int32_t flen = aln_flen[base + a];
      if (status == 0 && fwd != mateFwd) {                                       /* :629-632 fragLengthPedantic */
        int32_t pos = aln_pos[base + a], mpos = aln_mate_pos[base + a];
        int32_t p1 = fwd ? pos : mpos; p1 = p1 < 0 ? 0 : p1; p1 = p1 > refLen ? refLen : p1;
        int32_t p2 = fwd ? mpos + (int32_t)L : pos + (int32_t)L; p2 = p2 < 0 ? 0 : p2; p2 = p2 > refLen ? refLen : p2;
        flen = (p1 > p2) ? p1 - p2 : p2 - p1;
      }
      double logFragProb = LOG_1;
      if (status != 0) {                                                          /* :642-650 orphan in a PE library */
        int32_t pos = aln_pos[base + a];
        int32_t maxFragLen;
        if (fwd) { int32_t p1 = pos < 0 ? 0 : pos; p1 = p1 > refLen ? refLen : p1; maxFragLen = refLen - p1; }
        else { int32_t p1 = pos + (int32_t)L; p1 = p1 < 0 ? 0 : p1; p1 = p1 > refLen ? refLen : p1; maxFragLen = p1; }
        const double* cm = burnedIn ? fld.cmf_cached : fld.cmf_quirk;              /* DistributionUtils.cpp:145-172 */
        double refLengthCM = tab(cm, fld.max_val, (uint64_t)refLen);
        double maxLenProb = tab(cm, fld.max_val, (uint64_t)maxFragLen);
        logFragProb = (refLengthCM != LOG_0) ? (maxLenProb - refLengthCM) : LOG_EPSILON;
      }
      if (flen > 0 && (burnedIn || useAux)) {                                      /* :658-685 */
        uint64_t fl = (uint64_t)flen;
        if (burnedIn) {
          double lenProb = tab(fld.pmf_cached, fld.max_val, fl);
          double refLengthCM = tab(fld.cmf_cached, fld.max_val, fl);
          int computeMass = ((double)fl < refLength) && (refLengthCM != LOG_0);
          logFragProb = computeMass ? (lenProb - refLengthCM) : LOG_EPSILON;
        } else {
          logFragProb = tab(fld.pmf_live, fld.max_val, fl);
        }
      }
      aux[a] = logFragProb + logFragCov + LOG_1;                                   /* :783 (compatible) */
      auxDenom = logAddDet(auxDenom, aux[a]);
    }
    for (uint32_t a = 0; a < na; ++a) {                                            /* :818-820 */
      weight[base + a] = m_exp(aux[a] - auxDenom);
      label[(size_t)r * 2 * cap + a] = aln_tid[base + a];
    }
    if (p->range_bins > 0) {                                                        /* :845-853 */
      int32_t rangeCount = (int32_t)sqrt((double)na) + (int32_t)p->range_bins;
      for (uint32_t a = 0; a < na; ++a)
        label[(size_t)r * 2 * cap + na + a] = (uint32_t)(int32_t)(weight[base + a] * rangeCount);
    }
    if (on) online_fragment(on, r, L, na, aln_tid + base, aln_pos + base, aln_mate_pos + base, aln_flags + base,
                            aln_flen + base, aux);
  }
  if (ctr) *ctr = local;
  free(lc); free(rcand); free(jh); free(scores); free(perm); free(bs_tid); free(bs_score); free(bs_idx);
  return 0;
}

/* stateless form: the FLD is the prior, the regime is chosen by frag_counter (SalmonQuantify.cpp:496-497) */
int orc_map_reads(const orc_index* ix, const orc_map_params* p, const uint8_t* left,
                  const uint8_t* right, uint32_t n, uint32_t L, uint64_t frag_counter,
                  uint32_t* n_aln, uint32_t* aln_tid, int32_t* aln_score, double* aln_prob,
                  int32_t* aln_pos, int32_t* aln_mate_pos, uint8_t* aln_flags, int32_t* aln_flen,
                  uint32_t* label, double* weight, orc_map_counters* ctr) {
  fld_t fld;
  fld_init(&fld, p->fld_mean, p->fld_sd, p->max_frag_len);
  /* reads are independent here (no online state): chunks of reads in parallel, counters summed (test-harness speed:
   * the at-scale pinning tests map 10^6 pairs) */
  const uint32_t CH = 2048, cap = p->max_read_occ;
  const uint32_t nchunk = (n + CH - 1) / CH;
  int rc = 0;
  orc_map_counters tot;
  memset(&tot, 0, sizeof tot);
#pragma omp parallel for schedule(dynamic, 1)
  for (uint32_t c = 0; c < nchunk; ++c) {
    const size_t o = (size_t)c * CH;
    const uint32_t m = (uint32_t)((o + CH <= n) ? CH : n - o);
    orc_map_counters cc;
    memset(&cc, 0, sizeof cc);
    int r = map_reads_core(ix, p, &fld, frag_counter >= p->num_pre_burnin, frag_counter >= p->num_burnin, NULL, left + o * L,
                           right + o * L, m, L, n_aln + o, aln_tid + o * cap, aln_score + o * cap, aln_prob + o * cap,
                           aln_pos + o * cap, aln_mate_pos + o * cap, aln_flags + o * cap, aln_flen + o * cap,
                           label + o * 2 * cap, weight + o * cap, &cc);
#pragma omp critical
    {
      if (r) rc = r;
      const uint64_t* src = (const uint64_t*)&cc;
      uint64_t* dst = (uint64_t*)&tot;
      for (size_t i = 0; i < sizeof(orc_map_counters) / 8; ++i) dst[i] += src[i];
    }
  }
  if (ctr) *ctr = tot;
  fld_free(&fld);
  return rc;
}

/* ---------------------------------------------------------------- eq-class aggregation */
typedef struct { const uint32_t* lab; uint32_t len; uint32_t frag; } lref_t;
static int cmp_lref(const void* a, const void* b) {
  const lref_t* x = (const lref_t*)a; const lref_t* y = (const lref_t*)b;
  uint32_t m = x->len < y->len ? x->len : y->len;
  for (uint32_t i = 0; i < m; ++i) if (x->lab[i] != y->lab[i]) return x->lab[i] < y->lab[i] ? -1 : 1;
  if (x->len != y->len) return x->len < y->len ? -1 : 1;
  return x->frag < y->frag ? -1 : (x->frag > y->frag);   /* fragment order inside a class */
}

uint64_t orc_eq_aggregate(uint32_t n, uint32_t cap, int binned, const uint32_t* n_aln,
                          const uint32_t* label, const double* weight, uint64_t* out_off,
                          uint32_t* out_ntx, uint32_t* out_label, double* out_weight,
                          uint64_t* out_count) {
  lref_t* refs = (lref_t*)malloc((n ? n : 1) * sizeof(lref_t));
  uint32_t m = 0;
  for (uint32_t r = 0; r < n; ++r)
    if (n_aln[r]) { refs[m].lab = label + (size_t)r * 2 * cap; refs[m].len = n_aln[r] * (binned ? 2 : 1); refs[m].frag = r; ++m; }
  qsort(refs, m, sizeof(lref_t), cmp_lref);
  uint64_t nc = 0, woff = 0;
  uint32_t i = 0;
  while (i < m) {
    uint32_t j = i + 1;
    while (j < m && refs[j].len == refs[i].len && memcmp(refs[j].lab, refs[i].lab, refs[i].len * 4) == 0) ++j;
    uint32_t ntx = refs[i].len / (binned ? 2 : 1);
    out_off[nc] = woff;
    out_ntx[nc] = ntx;
    /* addGroup: count++, weights[i] += w_i in fragment order (EquivalenceClassBuilder.hpp:237-250) */
    for (uint32_t a = 0; a < ntx; ++a) { out_label[woff + a] = refs[i].lab[a]; out_weight[woff + a] = 0.0; }
    for (uint32_t q = i; q < j; ++q)
      for (uint32_t a = 0; a < ntx; ++a) out_weight[woff + a] += weight[(size_t)refs[q].frag * cap + a];
    /* finish(): normalizeAux (:114-123) */
    double s = 0.0;
    for (uint32_t a = 0; a < ntx; ++a) s += out_weight[woff + a];
    double norm = 1.0 / s;
    for (uint32_t a = 0; a < ntx; ++a) out_weight[woff + a] *= norm;
    out_count[nc] = j - i;
    woff += ntx;
    ++nc;
    i = j;
  }
  out_off[nc] = woff;
  free(refs);
  return nc;
}

/* ================================================================ online phase (rows a7, a9)
 * processMiniBatch's state updates (src/quant/SalmonQuantify.cpp:515, 599-623, 749-757, 783-790, 859-1018),
 * ForgettingMassCalculator (include/salmon/internal/quant/ForgettingMassCalculator.hpp:24-92),
 * FragmentLengthDistribution::addVal / pmf / dumpPMF / cacheCMF (src/model/FragmentLengthDistribution.cpp:84-186),
 * ReadExperiment::updateTranscriptLengthsAtomic (include/salmon/internal/quant/ReadExperiment.inl:61-94),
 * correctionFactorsFromMass / computeSmoothedEffectiveLengths (src/util/DistributionUtils.cpp:9-56),
 * normalizeAlphas (src/util/SalmonUtils.cpp:461-529), TranscriptCluster::projectToPolytope
 * (include/salmon/internal/quant/TranscriptCluster.hpp:46-101), ClusterForest (ClusterForest.hpp:29-139).
 *
 * BATCHED SEMANTICS (DESIGN.md): the reference mutates masses and the FLD fragment by fragment from many threads
 * (order-dependent, not reproducible).  Here the state is frozen for the duration of one batch; a batch's
 * contributions are accumulated as integers (multiples of 2^-40 of the batch's largest forgetting mass), hence
 * order-independent and bit-reproducible, and folded into the state at the end of the batch.  Forgetting-mass
 * timesteps advance every `mini_batch` reads as in the reference (miniBatchSize 5000).  The stochastic FLD update
 * (r < exp(logProb), :974-983) draws r from Philox(fragment index, alignment index, 3; seed). */
#define MASS_SCALE 1099511627776.0 /* 2^40 */

struct orc_online {
  const orc_index* ix;
  orc_map_params p;
  uint32_t M, nfld, mini_batch;
  uint64_t seed;
  double *mass, *prior, *log_eff;
  fld_t fld;
  uint64_t min_val;
  uint64_t assigned, frags_seen, timestep;
  int burned_in;
  double* fm; uint64_t n_fm;
  /* per batch */
  uint64_t *mass_acc, *fld_acc;
  uint64_t batch_min, batch_t0, batch_assigned;
  double batch_ref;
};

static double fm_at(orc_online* on, uint64_t t) {   /* ForgettingMassCalculator.hpp:24-40 (forgettingFactor 0.65) */
  const double ff = 0.65;
  while (on->n_fm <= t) {
    uint64_t j = on->n_fm;
    on->fm = (double*)realloc(on->fm, (j + 1) * sizeof(double));
    if (j == 0) on->fm[0] = 0.0;
    else on->fm[j] = on->fm[j - 1] + ff * log((double)j) - log(pow((double)(j + 1), ff) - 1);
    on->n_fm = j + 1;
  }
  return on->fm[t];
}

orc_online* orc_online_create(const orc_index* ix, const orc_map_params* p, uint64_t seed, uint32_t mini_batch) {
  orc_online* on = (orc_online*)calloc(1, sizeof(orc_online));
  on->ix = ix; on->p = *p; on->M = ix->n_txps; on->nfld = p->max_frag_len + 1; on->mini_batch = mini_batch ? mini_batch : 5000;
  on->seed = seed;
  on->mass = (double*)malloc((on->M ? on->M : 1) * sizeof(double));
  on->prior = (double*)malloc((on->M ? on->M : 1) * sizeof(double));
  on->log_eff = (double*)malloc((on->M ? on->M : 1) * sizeof(double));
  for (uint32_t t = 0; t < on->M; ++t) {
    const double len = (double)(ix->off[t + 1] - ix->off[t]);
    on->mass[t] = LOG_0;
    on->prior[t] = m_log(0.005 * len);           /* Transcript(id, name, len, alpha = 0.005): priorMass_ = log(alpha*len) */
    on->log_eff[t] = m_log(len);
  }
  fld_init(&on->fld, p->fld_mean, p->fld_sd, p->max_frag_len);
  on->min_val = p->max_frag_len;
  on->mass_acc = (uint64_t*)calloc(on->M ? on->M : 1, sizeof(uint64_t));
  on->fld_acc = (uint64_t*)calloc(on->nfld, sizeof(uint64_t));
  return on;
}
void orc_online_free(orc_online* on) {
  if (!on) return;
  free(on->mass); free(on->prior); free(on->log_eff); free(on->fm); free(on->mass_acc); free(on->fld_acc);
  fld_free(&on->fld); free(on);
}

static int64_t quant40(double x) { return llrint(x * MASS_SCALE); }

static void online_fragment(orc_online* on, uint32_t r, uint32_t L, uint32_t na, const uint32_t* tid,
                            const int32_t* pos, const int32_t* mate_pos, const uint8_t* flags, const int32_t* flen_raw,
                            const double* aux) {
  const double LOG_EPSILON = log(EPSILON_);
  const orc_index* ix = on->ix;
  const uint64_t t = on->batch_t0 + r / on->mini_batch;
  const double fmv = fm_at(on, t), ref = on->batch_ref;
  double lp[256];
  int32_t fped[256];
  double S = LOG_0;
  for (uint32_t a = 0; a < na; ++a) {
    const uint32_t ti = tid[a];
    const int32_t refLen = (int32_t)(ix->off[ti + 1] - ix->off[ti]);
    const double refLength = refLen > 0 ? (double)refLen : 1.0;
    const uint32_t status = (flags[a] >> 2) & 3;
    const int fwd = flags[a] & 1, mateFwd = (flags[a] >> 1) & 1;
    int32_t flen = flen_raw[a];
    fped[a] = 0;
    if (status == 0 && fwd != mateFwd) {
      int32_t p1 = fwd ? pos[a] : mate_pos[a]; p1 = p1 < 0 ? 0 : p1; p1 = p1 > refLen ? refLen : p1;
      int32_t p2 = fwd ? mate_pos[a] + (int32_t)L : pos[a] + (int32_t)L; p2 = p2 < 0 ? 0 : p2; p2 = p2 > refLen ? refLen : p2;
      flen = (p1 > p2) ? p1 - p2 : p2 - p1;
      fped[a] = flen;
    }
    const double logRefLength = on->burned_in ? on->log_eff[ti] : m_log((double)refLen);      /* :617-623 */
    double startPosProb = -logRefLength;                                                           /* :749-757 */
    if (status == 0) startPosProb = ((double)flen <= refLength) ? -m_log(refLength - (double)flen + 1) : LOG_EPSILON;
    const double transcriptLogCount = logAddDet(on->prior[ti], on->mass[ti]);                       /* mass(initialRound) */
    lp[a] = transcriptLogCount + aux[a] + startPosProb;                                            /* :785 */
    S = logAddDet(S, lp[a]);                                                                        /* :792 */
  }
  const uint64_t g = on->frags_seen + r;
  for (uint32_t a = 0; a < na; ++a) {
    const double nlp = lp[a] - S;                                                                   /* :865 */
    on->mass_acc[tid[a]] += (uint64_t)quant40(m_exp(fmv - ref + nlp));                        /* :871-872 */
    if (!on->burned_in) {                                                                           /* :974-983 */
      uint32_t rnd[4];
      orc_philox4x32((uint32_t)g, (uint32_t)(g >> 32), a, 3u, (uint32_t)on->seed, (uint32_t)(on->seed >> 32), rnd);
      const double u = (double)rnd[0] * (1.0 / 4294967296.0);
      if (u < m_exp(nlp) && fped[a] > 0) {
        /* FragmentLengthDistribution::addVal(len, logForgettingMass), :84-106; kernel = binomial(4, 0.5) */
        static const double kern_lin[5] = {1.0 / 16, 4.0 / 16, 6.0 / 16, 4.0 / 16, 1.0 / 16};
        uint64_t len = (uint64_t)fped[a];
        if (len > on->p.max_frag_len) len = on->p.max_frag_len;
        if (len < on->batch_min) on->batch_min = len;
        int64_t off = (int64_t)len - 2;
        for (int i = 0; i < 5; ++i, ++off)
          if (off > 0 && off < (int64_t)on->nfld)
            on->fld_acc[off] += (uint64_t)quant40(m_exp(fmv - ref + m_log(kern_lin[i])));
      }
    }
  }
  on->batch_assigned++;
}

/* cached effective lengths from the current FLD */
static void online_eff_lengths(orc_online* on) {
  const uint32_t n = on->nfld;
  const uint64_t maxV = n - 1;
  const uint64_t minV = (on->min_val == n - 1) ? 1 : on->min_val;
  double* logPMF = (double*)malloc(n * sizeof(double));
  double sum = LOG_0;
  for (uint64_t i = minV; i <= maxV; ++i) { logPMF[i - minV] = on->fld.hist[i] - on->fld.tot; sum = logAddDet(sum, logPMF[i - minV]); }
  double* pmf = (double*)calloc(maxV + 1, sizeof(double));
  for (uint64_t i = minV; i < maxV; ++i) pmf[i] = 100.0 * m_exp(logPMF[i - minV] - sum);
  const uint64_t maxLen = maxV + 1;
  double* cf = (double*)calloc(maxLen, sizeof(double));
  double vals = 0.0, mult = pmf[0];
  for (uint64_t i = 1; i < maxLen; ++i) {
    vals = pmf[i] * (double)i + vals;
    mult = pmf[i] + mult;
    if (mult > 0) cf[i] = vals / mult;
  }
  for (uint32_t t = 0; t < on->M; ++t) {
    const double origLen = (double)(on->ix->off[t + 1] - on->ix->off[t]);
    const double c = (origLen >= (double)maxLen) ? cf[maxLen - 1] : cf[(uint64_t)origLen];
    double effLen = origLen - c;
    if (effLen < 1.0) effLen = origLen;
    on->log_eff[t] = m_log(effLen);
  }
  free(logPMF); free(pmf); free(cf);
}

int orc_online_batch(orc_online* on, const uint8_t* left, const uint8_t* right, uint32_t n, uint32_t L,
                     uint32_t* n_aln, uint32_t* aln_tid, int32_t* aln_score, double* aln_prob, int32_t* aln_pos,
                     int32_t* aln_mate_pos, uint8_t* aln_flags, int32_t* aln_flen, uint32_t* label, double* weight,
                     orc_map_counters* ctr) {
  const uint32_t nfld = on->nfld;
  const uint64_t nsteps = (n + on->mini_batch - 1) / on->mini_batch;
  on->batch_t0 = on->timestep;
  on->batch_ref = fm_at(on, on->timestep + (nsteps ? nsteps - 1 : 0));
  on->batch_min = on->p.max_frag_len;
  on->batch_assigned = 0;
  const int useAux = on->assigned >= on->p.num_pre_burnin;
  int rc = map_reads_core(on->ix, &on->p, &on->fld, useAux, on->burned_in, on, left, right, n, L, n_aln, aln_tid,
                          aln_score, aln_prob, aln_pos, aln_mate_pos, aln_flags, aln_flen, label, weight, ctr);
  /* fold the batch into the state */
  for (uint32_t t = 0; t < on->M; ++t)
    if (on->mass_acc[t]) {
      on->mass[t] = logAddDet(on->mass[t], on->batch_ref + m_log((double)on->mass_acc[t] * (1.0 / MASS_SCALE)));
      on->mass_acc[t] = 0;
    }
  uint64_t tot_acc = 0;
  for (uint32_t j = 0; j < nfld; ++j)
    if (on->fld_acc[j]) {
      on->fld.hist[j] = logAddDet(on->fld.hist[j], on->batch_ref + m_log((double)on->fld_acc[j] * (1.0 / MASS_SCALE)));
      tot_acc += on->fld_acc[j];
      on->fld_acc[j] = 0;
    }
  if (tot_acc) {
    on->fld.tot = logAddDet(on->fld.tot, on->batch_ref + m_log((double)tot_acc * (1.0 / MASS_SCALE)));
    if (on->batch_min < on->min_val) on->min_val = on->batch_min;
    for (uint32_t j = 0; j < nfld; ++j) on->fld.pmf_live[j] = on->fld.hist[j] - on->fld.tot;
  }
  on->assigned += on->batch_assigned;
  on->frags_seen += n;
  on->timestep += nsteps;
  if (!on->burned_in && on->assigned >= on->p.num_burnin) {            /* SalmonQuantify.cpp:1013-1018 */
    online_eff_lengths(on);
    double tm = LOG_0, cum = LOG_0;                                    /* cacheCMF: getLockedPMF + cmf(pmf) */
    for (uint32_t j = 0; j < nfld; ++j) tm = logAddDet(tm, on->fld.hist[j] - on->fld.tot);
    for (uint32_t j = 0; j < nfld; ++j) {
      on->fld.pmf_cached[j] = (on->fld.hist[j] - on->fld.tot) - tm;
      cum = logAddDet(cum, on->fld.pmf_cached[j]);
      on->fld.cmf_cached[j] = cum;
    }
    on->burned_in = 1;
  }
  return rc;
}

/* scalars[6] = {assigned, frags_seen, timestep, burned_in, min_val, log totMass (as bits of a double)} */
void orc_online_state(const orc_online* on, double* mass_out, double* hist_out, double* log_eff_out, uint64_t* scalars) {
  if (mass_out) memcpy(mass_out, on->mass, on->M * sizeof(double));
  if (hist_out) memcpy(hist_out, on->fld.hist, on->nfld * sizeof(double));
  if (log_eff_out) memcpy(log_eff_out, on->log_eff, on->M * sizeof(double));
  if (scalars) {
    scalars[0] = on->assigned; scalars[1] = on->frags_seen; scalars[2] = on->timestep; scalars[3] = (uint64_t)on->burned_in;
    scalars[4] = on->min_val; scalars[5] = orc_d2u(on->fld.tot);
  }
}

/* normalizeAlphas over the finished classes (transcript parts of the labels): per-transcript unique / total counts,
 * clusters = connected components of the class <-> transcript graph (ClusterForest::mergeClusters per fragment
 * gives the same partition), cluster hit counts, projection.  Members are visited in ascending transcript id. */
static uint32_t uf_find(uint32_t* parent, uint32_t x) { while (parent[x] != x) { parent[x] = parent[parent[x]]; x = parent[x]; } return x; }

int orc_online_finish(orc_online* on, uint64_t n_classes, const uint64_t* off, const uint32_t* tids,
                      const uint64_t* counts, double* projected, double* eff_len, uint64_t* unique, uint64_t* total) {
  const uint32_t M = on->M;
  if (!on->burned_in && on->assigned < on->p.num_burnin) online_eff_lengths(on);   /* SalmonQuantify.cpp:2734-2738 */
  uint32_t* parent = (uint32_t*)malloc((M ? M : 1) * sizeof(uint32_t));
  double* hits = (double*)calloc(M ? M : 1, sizeof(double));
  for (uint32_t t = 0; t < M; ++t) { parent[t] = t; unique[t] = 0; total[t] = 0; projected[t] = 0.0; }
  for (uint64_t c = 0; c < n_classes; ++c) {
    const uint64_t b = off[c], e = off[c + 1];
    if (e == b) continue;
    hits[tids[b]] += (double)counts[c];                      /* updateCluster(first transcript, 1.0, ...) per fragment */
    if (e - b == 1) unique[tids[b]] += counts[c];            /* transcriptUnique, :987-990 */
    for (uint64_t j = b; j < e; ++j) {
      total[tids[j]] += counts[c];                           /* addTotalCount, :795-797 */
      uint32_t ra = uf_find(parent, tids[b]), rb = uf_find(parent, tids[j]);
      if (ra != rb) { if (ra < rb) parent[rb] = ra; else parent[ra] = rb; }
    }
  }
  /* members by cluster, ascending id: counting sort on the root */
  uint32_t* root = (uint32_t*)malloc((M ? M : 1) * sizeof(uint32_t));
  uint32_t* start = (uint32_t*)calloc((size_t)M + 1, sizeof(uint32_t));
  uint32_t* memb = (uint32_t*)malloc((M ? M : 1) * sizeof(uint32_t));
  for (uint32_t t = 0; t < M; ++t) { root[t] = uf_find(parent, t); start[root[t] + 1]++; }
  for (uint32_t t = 0; t < M; ++t) start[t + 1] += start[t];
  uint32_t* fill = (uint32_t*)malloc((M ? M : 1) * sizeof(uint32_t));
  memcpy(fill, start, (M ? M : 1) * sizeof(uint32_t));
  for (uint32_t t = 0; t < M; ++t) memb[fill[root[t]]++] = t;
  uint8_t* bound = (uint8_t*)malloc(M ? M : 1);
  for (uint32_t r = 0; r < M; ++r) {
    const uint32_t b = start[r], e = start[r + 1];
    if (e == b) continue;
    double clusterHits = 0.0, logClusterMass = LOG_0;
    for (uint32_t q = b; q < e; ++q) { clusterHits += hits[memb[q]]; logClusterMass = logAddDet(logClusterMass, on->mass[memb[q]]); }
    const double logClusterCount = m_log(clusterHits);
    int requiresProjection = 0;
    for (uint32_t q = b; q < e; ++q) {
      const uint32_t t = memb[q];
      if (on->mass[t] == LOG_0) projected[t] = 0.0;
      else {
        projected[t] = m_exp((on->mass[t] - logClusterMass) + logClusterCount);
        requiresProjection |= projected[t] > (double)total[t] || projected[t] < (double)unique[t];
      }
    }
    if (e - b > 1 && requiresProjection) {                   /* TranscriptCluster::projectToPolytope */
      const uint32_t cs = e - b;
      memset(bound, 0, cs);
      for (uint32_t round = 0;; ) {
        double unboundCounts = 0.0, boundCounts = 0.0;
        for (uint32_t i = 0; i < cs; ++i) {
          const uint32_t t = memb[b + i];
          if (projected[t] > (double)total[t]) { projected[t] = (double)total[t]; bound[i] = 1; }
          else if (projected[t] < (double)unique[t]) { projected[t] = (double)unique[t]; bound[i] = 1; }
          if (bound[i]) boundCounts += projected[t]; else unboundCounts += projected[t];
        }
        if (fabs(unboundCounts + boundCounts - clusterHits) <= EPSILON_) break;
        if (unboundCounts == 0) { memset(bound, 0, cs); unboundCounts = boundCounts; boundCounts = 0; }
        const double normalizer = (clusterHits - boundCounts) / unboundCounts;
        for (uint32_t i = 0; i < cs; ++i) if (!bound[i]) projected[memb[b + i]] *= normalizer;
        if (++round > 5000) break;
      }
    }
  }
  for (uint32_t t = 0; t < M; ++t) eff_len[t] = m_exp(on->log_eff[t]);   /* CollapsedEMOptimizer.cpp:782-784 */
  free(parent); free(hits); free(root); free(start); free(memb); free(fill); free(bound);
  return 0;
}
