/*
 * tests/oracle_likelihood.c -- TEST INFRASTRUCTURE.  salmon's fragment-likelihood options (--incompatPrior,
 * --noSingleFragProb, --noFragLengthDist, --noEffectiveLengthCorrection; the rule is DESIGN.md section 13) restated on
 * top of the CPU oracle (oracle/map_oracle.c through tests/oracle_rescue.c, both included unchanged for their index,
 * candidates, join, DP, FLD tables and online state), written from the reference's lines, not from the product's
 * map_core.h:
 *   QuantOptionsUtils.cpp:608-616     incompatPrior == 0 or < 1e-100 -> ignoreIncompat, else log(incompatPrior);
 *   SalmonQuantify.cpp:1519-1521      incompatible joint hits are skipped only under ignoreIncompat;
 *   SalmonMappingUtils.hpp:225-281    updateRefMappings: a tie on one transcript goes to the later hit only when it is
 *                                     compatible;
 *   SalmonQuantify.cpp:617-623        logRefLength = log(RefLength) under noEffectiveLengthCorrection or before burn-in;
 *   SalmonQuantify.cpp:640-655        getAmbigFragLengthProb only with modelSingleFragProb and useFragLengthDist, else
 *                                     LOG_EPSILON for an orphan of a paired-end library, LOG_1 for a single-end read;
 *   SalmonQuantify.cpp:657            the fragment-length term of a pair only with useFragLengthDist;
 *   SalmonQuantify.cpp:706-713,783    logAlignCompatProb = isCompat ? LOG_1 : incompatPrior, part of auxProb;
 *   SalmonQuantify.cpp:767-769,812-814  a fragment is compatible when one of its alignments is.
 * The options travel in a struct of their own (orc_lk_opts); orc_map_params is the oracle's, unchanged.
 */
#include "oracle_rescue.c"

typedef struct {
  double incompat_prior;          /* the option's value, a probability */
  int32_t model_single_frag_prob; /* !--noSingleFragProb */
  int32_t use_frag_len_dist;      /* !--noFragLengthDist */
  int32_t no_eff_len_correction;  /* --noEffectiveLengthCorrection */
  int32_t reserved;
} orc_lk_opts;

/* salmon::utils::isCompatible for the inward / unmated formats (SalmonUtils.cpp:138-298): the orientation of the mate(s) */
static int lk_compatible(int lib_type, uint32_t status, int lfw, int rfw) {
  const int orphan = status != 0, isLeft = status != 2;
  switch (lib_type) {
    case 0: return orphan ? 1 : lfw != rfw;
    case 1: return orphan ? ((isLeft && lfw) || (!isLeft && !rfw)) : (lfw && !rfw);
    case 2: return orphan ? ((isLeft && !lfw) || (!isLeft && rfw)) : (!lfw && rfw);
    case 4: return lfw;
    case 5: return !lfw;
    default: return 1;
  }
}

/* processMiniBatch's online update of one fragment (:599-623, 749-792, 859-983) with the chosen logRefLength */
static void lk_online_fragment(orc_online* on, const orc_lk_opts* o, uint32_t r, uint32_t L, uint32_t na, const uint32_t* tid,
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
    const double logRefLength = (o->no_eff_len_correction || !on->burned_in) ? m_log((double)refLen) : on->log_eff[ti];
    double startPosProb = -logRefLength;
    if (status == 0) startPosProb = ((double)flen <= refLength) ? -m_log(refLength - (double)flen + 1) : LOG_EPSILON;
    lp[a] = logAddDet(on->prior[ti], on->mass[ti]) + aux[a] + startPosProb;
    S = logAddDet(S, lp[a]);
  }
  const uint64_t g = on->frags_seen + r;
  for (uint32_t a = 0; a < na; ++a) {
    const double nlp = lp[a] - S;
    on->mass_acc[tid[a]] += (uint64_t)quant40(m_exp(fmv - ref + nlp));
    if (!on->burned_in) {
      uint32_t rnd[4];
      orc_philox4x32((uint32_t)g, (uint32_t)(g >> 32), a, 3u, (uint32_t)on->seed, (uint32_t)(on->seed >> 32), rnd);
      const double u = (double)rnd[0] * (1.0 / 4294967296.0);
      if (u < m_exp(nlp) && fped[a] > 0) {
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

/* one read: updateRefMappings, filterAndCollectAlignments, auxiliary probabilities, label, online update */
static void lk_assign(const orc_index* ix, const orc_map_params* p, const orc_lk_opts* o, const fld_t* fld, int useAux,
                      int burnedIn, orc_online* on, uint32_t r, const uint8_t* rl, const uint8_t* rr, uint32_t L,
                      const cand_t* lc, const cand_t* rc, const joint_t* jh, uint32_t nj, uint32_t* n_aln, uint32_t* tid,
                      int32_t* score, double* prob, int32_t* pos, int32_t* mpos, uint8_t* flags, int32_t* flen,
                      uint32_t* label, double* weight, orc_map_counters* ctr, uint64_t* n_compat) {
  const uint32_t cap = p->max_read_occ;
  const double LOG_EPSILON = log(EPSILON_);
  const int ignoreIncompat = o->incompat_prior < 1e-100 || o->incompat_prior == 0.0;
  const double incompatPrior = ignoreIncompat ? LOG_0 : m_log(o->incompat_prior);
  const size_t NJ = (size_t)(MAXCAND * MAXCAND + 2 * MAXCAND);
  int32_t* sc = (int32_t*)malloc(NJ * sizeof(int32_t));
  int32_t* bs_tid = (int32_t*)malloc(NJ * sizeof(int32_t));
  int32_t* bs_sc = (int32_t*)malloc(NJ * sizeof(int32_t));
  int32_t* bs_idx = (int32_t*)malloc(NJ * sizeof(int32_t));
  uint8_t* compat = (uint8_t*)malloc(NJ);
  perm_t* perm = (perm_t*)malloc(NJ * sizeof(perm_t));
  int32_t best = INT_MIN, bestDecoy = INT_MIN;
  uint32_t nperm = 0, nbs = 0;
  n_aln[r] = 0;
  for (uint32_t h = 0; h < nj; ++h) {
    int32_t tot = 0, maxPossible = 0;
    int bad = 0;
    if (jh[h].li >= 0) { const int32_t s = orc_dp_score(ix, p, rl, L, lc[jh[h].li].ori, jh[h].tid, lc[jh[h].li].diag_c); ctr->candidates++; if (s <= NEG_SCORE) bad = 1; tot += s; maxPossible += p->ma * (int32_t)L; }
    if (jh[h].ri >= 0) { const int32_t s = orc_dp_score(ix, p, rr, L, rc[jh[h].ri].ori, jh[h].tid, rc[jh[h].ri].diag_c); ctr->candidates++; if (s <= NEG_SCORE) bad = 1; tot += s; maxPossible += p->ma * (int32_t)L; }
    const int32_t hs = (!bad && (double)tot >= p->min_score_fraction * (double)maxPossible) ? tot : INT_MIN;
    sc[h] = hs;
    const int isCompat = lk_compatible(p->lib_type, jh[h].status, jh[h].li >= 0 && lc[jh[h].li].ori == 0,
                                       jh[h].ri >= 0 && rc[jh[h].ri].ori == 0);
    compat[h] = (uint8_t)isCompat;
    if (!isCompat && ignoreIncompat) { sc[h] = INT_MIN; continue; }   /* the hit never reaches updateRefMappings */
    const double cutoff = (double)(int32_t)(p->decoy_threshold * (double)bestDecoy);
    if ((int32_t)jh[h].tid >= p->first_decoy) { if (hs > bestDecoy) bestDecoy = hs; continue; }
    if ((double)hs < cutoff || hs == INT_MIN) continue;
    uint32_t q = 0;
    while (q < nbs && bs_tid[q] != (int32_t)jh[h].tid) ++q;
    if (q == nbs) { bs_tid[nbs] = (int32_t)jh[h].tid; bs_sc[nbs] = hs; bs_idx[nbs] = (int32_t)h; ++nbs; }
    else if (hs > bs_sc[q] || (hs == bs_sc[q] && isCompat)) { bs_sc[q] = hs; sc[bs_idx[q]] = INT_MIN; bs_idx[q] = (int32_t)h; }
    else sc[h] = INT_MIN;
    if (hs > best) best = hs;
    perm[nperm].idx = (int32_t)h; perm[nperm].tid = (int32_t)jh[h].tid; ++nperm;
  }
  if (bestDecoy == INT_MIN) bestDecoy = INT_MIN + 1;
  const int32_t thr = p->hard_filter ? best : (int32_t)(p->decoy_threshold * (double)bestDecoy);
  uint32_t nk = 0;
  for (uint32_t q = 0; q < nperm; ++q) if (sc[perm[q].idx] >= thr) perm[nk++] = perm[q];
  qsort(perm, nk, sizeof(perm_t), cmp_perm);
  const size_t b = (size_t)r * cap;
  uint8_t kept_compat[256];
  uint32_t na = 0;
  for (uint32_t q = 0; q < nk; ++q) {
    const joint_t* j = &jh[perm[q].idx];
    const double est = p->hard_filter ? -1.0 : m_exp(-p->score_exp * ((double)best - (double)sc[perm[q].idx]));
    if (!p->hard_filter && est < p->min_aln_prob) continue;
    const cand_t* first = j->status == 2 ? &rc[j->ri] : &lc[j->li];
    tid[b + na] = j->tid; score[b + na] = sc[perm[q].idx]; prob[b + na] = est;
    pos[b + na] = first->diag_c; mpos[b + na] = j->status == 0 ? rc[j->ri].diag_c : 0;
    uint8_t fl = (uint8_t)(first->ori == 0 ? 1 : 0);
    if (j->status == 0 && rc[j->ri].ori == 0) fl |= 2;
    flags[b + na] = (uint8_t)(fl | (j->status << 2));
    flen[b + na] = j->frag_len;
    kept_compat[na] = compat[perm[q].idx];
    ++na;
  }
  n_aln[r] = na;
  ctr->kept += na;
  free(sc); free(bs_tid); free(bs_sc); free(bs_idx); free(compat); free(perm);
  if (!na) return;
  ctr->mapped++;
  ctr->label_entries += na;
  const int singleEndLib = p->lib_type >= 3;
  int hasCompatibleMapping = 0;
  double aux[256], den = LOG_0;
  for (uint32_t a = 0; a < na; ++a) {
    const uint32_t t = tid[b + a];
    const int32_t refLen = (int32_t)(ix->off[t + 1] - ix->off[t]);
    const double refLength = refLen > 0 ? (double)refLen : 1.0;
    const uint32_t status = (flags[b + a] >> 2) & 3;
    const int fwd = flags[b + a] & 1, mfwd = (flags[b + a] >> 1) & 1;
    const int unexpectedOrphan = !singleEndLib && status != 0;   /* isUnexpectedOrphan */
    int32_t fl = flen[b + a];
    if (status == 0 && fwd != mfwd) {
      int32_t p1 = fwd ? pos[b + a] : mpos[b + a]; p1 = p1 < 0 ? 0 : (p1 > refLen ? refLen : p1);
      int32_t p2 = fwd ? mpos[b + a] + (int32_t)L : pos[b + a] + (int32_t)L; p2 = p2 < 0 ? 0 : (p2 > refLen ? refLen : p2);
      fl = p1 > p2 ? p1 - p2 : p2 - p1;
    }
    double lfp = LOG_1;
    if (o->model_single_frag_prob && o->use_frag_len_dist && (singleEndLib || unexpectedOrphan)) {
      int32_t maxFragLen;   /* getAmbigFragLengthProb */
      if (fwd) { int32_t p1 = pos[b + a] < 0 ? 0 : pos[b + a]; p1 = p1 > refLen ? refLen : p1; maxFragLen = refLen - p1; }
      else { int32_t p1 = pos[b + a] + (int32_t)L; p1 = p1 < 0 ? 0 : p1; p1 = p1 > refLen ? refLen : p1; maxFragLen = p1; }
      const double* cm = burnedIn ? fld->cmf_cached : fld->cmf_quirk;
      const double rcm = tab(cm, fld->max_val, (uint64_t)refLen), mlp = tab(cm, fld->max_val, (uint64_t)maxFragLen);
      lfp = rcm != LOG_0 ? mlp - rcm : LOG_EPSILON;
    } else if (unexpectedOrphan) {
      lfp = LOG_EPSILON;
    }
    if (fl > 0 && o->use_frag_len_dist && (burnedIn || useAux)) {
      if (burnedIn) {
        const double cm = tab(fld->cmf_cached, fld->max_val, (uint64_t)fl);
        lfp = ((double)fl < refLength && cm != LOG_0) ? tab(fld->pmf_cached, fld->max_val, (uint64_t)fl) - cm : LOG_EPSILON;
      } else {
        lfp = tab(fld->pmf_live, fld->max_val, (uint64_t)fl);
      }
    }
    const double logAlignCompatProb = kept_compat[a] ? LOG_1 : incompatPrior;
    if (logAlignCompatProb == LOG_1) hasCompatibleMapping = 1;
    aux[a] = lfp + (prob[b + a] > 0 ? m_log(prob[b + a]) : LOG_1) + logAlignCompatProb;
    den = logAddDet(den, aux[a]);
  }
  if (hasCompatibleMapping) ++*n_compat;
  for (uint32_t a = 0; a < na; ++a) { weight[b + a] = m_exp(aux[a] - den); label[(size_t)r * 2 * cap + a] = tid[b + a]; }
  if (p->range_bins > 0) {
    const int32_t rcnt = (int32_t)sqrt((double)na) + (int32_t)p->range_bins;
    for (uint32_t a = 0; a < na; ++a) label[(size_t)r * 2 * cap + na + a] = (uint32_t)(int32_t)(weight[b + a] * rcnt);
  }
  if (on) lk_online_fragment(on, o, r, L, na, tid + b, pos + b, mpos + b, flags + b, flen + b, aux);
}

/* a batch: stateless (on == NULL; regime from frag_counter, FLD = prior) or through the online state (the batch set-up
 * and fold of orc_online_batch, with the burn-in's effective lengths) */
static int lk_batch(orc_online* on, const orc_index* ix, const orc_map_params* p, const orc_lk_opts* o, const uint8_t* left,
                    const uint8_t* right, uint32_t n, uint32_t L, uint64_t frag_counter, uint32_t* n_aln, uint32_t* tid,
                    int32_t* score, double* prob, int32_t* pos, int32_t* mpos, uint8_t* flags, int32_t* flen, uint32_t* label,
                    double* weight, orc_map_counters* ctr, uint64_t* n_compat) {
  const uint32_t cap = p->max_read_occ;
  fld_t prior;
  const fld_t* fld = &prior;
  int useAux, burnedIn;
  if (on) {
    const uint64_t nsteps = (n + on->mini_batch - 1) / on->mini_batch;
    on->batch_t0 = on->timestep;
    on->batch_ref = fm_at(on, on->timestep + (nsteps ? nsteps - 1 : 0));
    on->batch_min = on->p.max_frag_len;
    on->batch_assigned = 0;
    useAux = on->assigned >= p->num_pre_burnin; burnedIn = on->burned_in; fld = &on->fld;
  } else {
    fld_init(&prior, p->fld_mean, p->fld_sd, p->max_frag_len);
    useAux = frag_counter >= p->num_pre_burnin; burnedIn = frag_counter >= p->num_burnin;
  }
  orc_map_counters tot;
  memset(&tot, 0, sizeof tot);
  *n_compat = 0;
  cand_t lc[MAXCAND], rc[MAXCAND];
  joint_t* jh = (joint_t*)malloc((size_t)(MAXCAND * MAXCAND + 2 * MAXCAND) * sizeof(joint_t));
  for (uint32_t r = 0; r < n; ++r) {
    const uint8_t* rl = left + (size_t)r * L;
    const uint8_t* rr = right + (size_t)r * L;
    n_aln[r] = 0;
    const uint32_t nl = mate_candidates(ix, p, rl, L, lc, &tot), nr = mate_candidates(ix, p, rr, L, rc, &tot);
    const uint32_t nj = rs_joint_hits(p, lc, nl, rc, nr, L, jh);
    if (nj == 0 || nj > cap) continue;
    lk_assign(ix, p, o, fld, useAux, burnedIn, on, r, rl, rr, L, lc, rc, jh, nj, n_aln, tid, score, prob, pos, mpos, flags,
              flen, label, weight, &tot, n_compat);
  }
  free(jh);
  if (ctr) *ctr = tot;
  if (!on) { fld_free(&prior); return 0; }
  const uint32_t nfld = on->nfld;
  const uint64_t nsteps = (n + on->mini_batch - 1) / on->mini_batch;
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
  if (!on->burned_in && on->assigned >= on->p.num_burnin) {
    online_eff_lengths(on);
    double tm = LOG_0, cum = LOG_0;
    for (uint32_t j = 0; j < nfld; ++j) tm = logAddDet(tm, on->fld.hist[j] - on->fld.tot);
    for (uint32_t j = 0; j < nfld; ++j) {
      on->fld.pmf_cached[j] = (on->fld.hist[j] - on->fld.tot) - tm;
      cum = logAddDet(cum, on->fld.pmf_cached[j]);
      on->fld.cmf_cached[j] = cum;
    }
    on->burned_in = 1;
  }
  return 0;
}

int orc_lk_map_reads(const orc_index* ix, const orc_map_params* p, const orc_lk_opts* o, const uint8_t* left,
                     const uint8_t* right, uint32_t n, uint32_t L, uint64_t frag_counter, uint32_t* n_aln, uint32_t* tid,
                     int32_t* score, double* prob, int32_t* pos, int32_t* mpos, uint8_t* flags, int32_t* flen,
                     uint32_t* label, double* weight, orc_map_counters* ctr, uint64_t* n_compat) {
  return lk_batch(NULL, ix, p, o, left, right, n, L, frag_counter, n_aln, tid, score, prob, pos, mpos, flags, flen, label,
                  weight, ctr, n_compat);
}
int orc_lk_online_batch(orc_online* on, const orc_lk_opts* o, const uint8_t* left, const uint8_t* right, uint32_t n,
                        uint32_t L, uint32_t* n_aln, uint32_t* tid, int32_t* score, double* prob, int32_t* pos,
                        int32_t* mpos, uint8_t* flags, int32_t* flen, uint32_t* label, double* weight,
                        orc_map_counters* ctr, uint64_t* n_compat) {
  return lk_batch(on, on->ix, &on->p, o, left, right, n, L, 0, n_aln, tid, score, prob, pos, mpos, flags, flen, label,
                  weight, ctr, n_compat);
}
