/*
 * tests/oracle_softclip.c -- TEST INFRASTRUCTURE.  The scoring modes of the banded DP (--softclipOverhangs,
 * --softclip; the rule is DESIGN.md section 12) restated on top of the CPU oracle (oracle/map_oracle.c and the rescue
 * restatement tests/oracle_rescue.c, both included unchanged for their index, candidates, join, search, assignment
 * arithmetic and online state), written from the option texts, not from the product's map_core.h:
 *   mode 0  end-to-end: the oracle's own recurrence;
 *   mode 1  overhangs, in two forms that must agree:
 *             form 0  a path may also start at any row in the cell of reference column 0 and end at any row in the cell
 *                     of column tlen-1;
 *             form 1  cells outside the transcript are live, score 0 for any base and take part in no gap; a path must
 *                     hold at least one base inside the transcript;
 *   mode 2  soft-clip: every live cell may start a path (diagonal predecessor floored at 0); the score is the best live
 *           cell of any row.
 * The per-read path (join, optional orphan rescue, updateRefMappings, filterAndCollectAlignments, auxiliary
 * probabilities, labels, online update) is the oracle's, with the DP of the chosen mode.
 */
#include "oracle_rescue.c"

int32_t orc_sc_dp_score(const orc_index* ix, const orc_map_params* p, const uint8_t* read, uint32_t L, uint32_t ori,
                        uint32_t tid, int32_t diag_c, int mode, int form) {
  const int32_t B = (int32_t)p->band, W = 2 * B + 1;
  const int64_t tlen = (int64_t)(ix->off[tid + 1] - ix->off[tid]);
  const uint8_t* ref = ix->codes + ix->off[tid];
  const int zero_outside = mode == 1 && form == 1;
  int32_t Hp[128], Ep[128], Hc[128], Ec[128];
  uint8_t Ap[128], Ac[128];   /* form 1: the cell's path holds a base inside the transcript */
  for (int32_t j = 0; j < W; ++j) { Hp[j] = 0; Ep[j] = NEG_SCORE; Ap[j] = 0; }
  int32_t best = NEG_SCORE;
  for (uint32_t i = 0; i < L; ++i) {
    const uint8_t rb = ori ? (uint8_t)(read[L - 1 - i] > 3 ? 4 : 3 - read[L - 1 - i]) : read[i];
    int32_t Fprev = NEG_SCORE, Hleft = NEG_SCORE;
    for (int32_t j = 0; j < W; ++j) {
      const int64_t r = (int64_t)diag_c + (int64_t)i + (j - B);
      const int inside = r >= 0 && r < tlen;
      int32_t h = NEG_SCORE, e = NEG_SCORE, f = NEG_SCORE;
      uint8_t a = 0;
      if (inside) {
        const int32_t s = (rb < 4 && rb == ref[r]) ? p->ma : p->mp;
        int32_t diag = Hp[j];
        if (mode == 2 && diag < 0) diag = 0;                        /* any live cell starts a path */
        if (mode == 1 && form == 0 && r == 0 && diag < 0) diag = 0;  /* start at column 0 */
        const int32_t m = diag + s;
        if (j + 1 < W) { const int32_t x = Hp[j + 1] - p->go - p->ge, y = Ep[j + 1] - p->ge; e = x > y ? x : y; }
        if (j > 0) { const int32_t x = Hleft - p->go - p->ge, y = Fprev - p->ge; f = x > y ? x : y; }
        h = m;
        if (e > h) h = e;
        if (f > h) h = f;
        if (h < NEG_SCORE) h = NEG_SCORE;
        if (e < NEG_SCORE) e = NEG_SCORE;
        if (f < NEG_SCORE) f = NEG_SCORE;
        a = h > NEG_SCORE;
        if (mode == 2 && h > best) best = h;                                       /* end anywhere */
        if (mode == 1 && form == 0 && r == tlen - 1 && h > best) best = h;         /* end at column tlen-1 */
      } else if (zero_outside) {
        if (r < 0) { h = 0; a = 0; }                 /* before the transcript: nothing aligned yet */
        else { h = Hp[j]; a = Ap[j]; }               /* after it: the diagonal predecessor, base scores 0 */
      }
      Hc[j] = h; Ec[j] = e; Ac[j] = a;
      Hleft = inside ? h : NEG_SCORE;                /* no gap opens from a cell outside the transcript */
      Fprev = f;
    }
    memcpy(Hp, Hc, W * sizeof(int32_t));
    memcpy(Ep, Ec, W * sizeof(int32_t));
    memcpy(Ap, Ac, (size_t)W);
  }
  for (int32_t j = 0; j < W; ++j)
    if ((!zero_outside || Ap[j]) && Hp[j] > best) best = Hp[j];
  return best;
}

/* the edit limit of the mate search: a base left unaligned (modes 1, 2) costs ma against a perfect score */
int32_t orc_sc_edit_limit(const orc_map_params* p, int mode, uint32_t L) {
  int32_t per = (p->ma - p->mp) < p->ge ? (p->ma - p->mp) : p->ge;
  if (mode != 0 && p->ma < per) per = p->ma;
  if (per <= 0) return (int32_t)L;
  const double k = (1.0 - p->min_score_fraction) * p->ma * (double)L / per;
  return k < 0 ? 0 : (k >= L ? (int32_t)L : (int32_t)k);
}

typedef struct { const orc_index* ix; const orc_map_params* p; int mode; } sc_ctx;

static int32_t sc_dp(const sc_ctx* c, const uint8_t* read, uint32_t L, const cand_t* cd) {
  return orc_sc_dp_score(c->ix, c->p, read, L, cd->ori, cd->tid, cd->diag_c, c->mode, 0);
}

/* rs_rescue_read with the mode's DP and edit limit */
static uint32_t sc_rescue_read(const sc_ctx* c, const uint8_t* rl, const uint8_t* rr, uint32_t L, cand_t* lc, uint32_t* nl,
                               cand_t* rc, uint32_t* nr, const joint_t* orph, uint32_t nj, joint_t* jh, uint64_t* ctr3) {
  const orc_index* ix = c->ix;
  const orc_map_params* p = c->p;
  const int32_t K = orc_sc_edit_limit(p, c->mode, L);
  uint8_t* pat = (uint8_t*)malloc(L);
  uint32_t np = 0;
  for (uint32_t h = 0; h < nj; ++h) {
    const int left = orph[h].status == 1;
    const cand_t anc = left ? lc[orph[h].li] : rc[orph[h].ri];
    const uint8_t* own = left ? rl : rr;
    const uint8_t* other = left ? rr : rl;
    if (!rs_passes(p, sc_dp(c, own, L, &anc), L)) continue;
    const int afw = anc.ori == 0;
    if (!rs_pair_compatible(p->lib_type, left ? afw : !afw, left ? !afw : afw)) continue;
    ctr3[1]++;
    const int64_t tlen = (int64_t)(ix->off[anc.tid + 1] - ix->off[anc.tid]);
    int64_t lo = afw ? anc.diag_c : (int64_t)anc.diag_c + L - p->max_frag_len;
    int64_t hi = afw ? (int64_t)anc.diag_c + p->max_frag_len : (int64_t)anc.diag_c + L;
    if (lo < 0) lo = 0;
    if (hi > tlen) hi = tlen;
    if (hi <= lo) continue;
    for (uint32_t i = 0; i < L; ++i) pat[i] = afw ? (other[L - 1 - i] > 3 ? 4 : 3 - other[L - 1 - i]) : other[i];
    int32_t d, e;
    orc_sellers_infix(pat, L, ix->codes + ix->off[anc.tid] + lo, (uint32_t)(hi - lo), K, &d, &e);
    if (d < 0) continue;
    cand_t res;
    memset(&res, 0, sizeof res);
    res.tid = anc.tid; res.ori = afw ? 1 : 0; res.diag_c = (int32_t)(lo + e) - (int32_t)L + 1;
    if (!rs_passes(p, sc_dp(c, other, L, &res), L)) continue;
    const cand_t* fw = afw ? &anc : &res;
    const cand_t* rv = afw ? &res : &anc;
    int32_t s = fw->diag_c, en = rv->diag_c + (int32_t)L;
    if (rv->diag_c < fw->diag_c) {
      if (!p->allow_dovetail) continue;
      s = rv->diag_c; en = fw->diag_c + (int32_t)L;
    }
    if (en - s <= 0 || en - s > (int32_t)p->max_frag_len) continue;
    const cand_t* L_ = left ? &anc : &res;
    const cand_t* R_ = left ? &res : &anc;
    int dup = 0;
    for (uint32_t q = 0; q < np; ++q)
      if (lc[jh[q].li].tid == L_->tid && lc[jh[q].li].ori == L_->ori && lc[jh[q].li].diag_c == L_->diag_c &&
          rc[jh[q].ri].ori == R_->ori && rc[jh[q].ri].diag_c == R_->diag_c) dup = 1;
    if (dup) continue;
    uint32_t* n = left ? nr : nl;
    if (*n >= MAXCAND) { ctr3[2]++; continue; }
    joint_t j = {anc.tid, 0, 0, en - s, 0};
    if (left) { rc[*n] = res; j.li = orph[h].li; j.ri = (int32_t)*n; }
    else { lc[*n] = res; j.li = (int32_t)*n; j.ri = orph[h].ri; }
    ++*n;
    jh[np++] = j;
  }
  free(pat);
  return np;
}

/* updateRefMappings + filterAndCollectAlignments + auxiliary probabilities + label of one read (map_reads_core's
 * statement, SalmonMappingUtils.hpp:225-405, SalmonQuantify.cpp:599-857) with the mode's DP */
static void sc_assign(const sc_ctx* c, const fld_t* fld, int useAux, int burnedIn, orc_online* on, uint32_t r,
                      const uint8_t* rl, const uint8_t* rr, uint32_t L, const cand_t* lc, const cand_t* rc, const joint_t* jh,
                      uint32_t nj, uint32_t* n_aln, uint32_t* tid, int32_t* score, double* prob, int32_t* pos, int32_t* mpos,
                      uint8_t* flags, int32_t* flen, uint32_t* label, double* weight, orc_map_counters* ctr) {
  const orc_index* ix = c->ix;
  const orc_map_params* p = c->p;
  const uint32_t cap = p->max_read_occ;
  const double LOG_EPSILON = log(EPSILON_);
  const size_t NJ = (size_t)(MAXCAND * MAXCAND + 2 * MAXCAND);
  int32_t* sc = (int32_t*)malloc(NJ * sizeof(int32_t));
  int32_t* bs_tid = (int32_t*)malloc(NJ * sizeof(int32_t));
  int32_t* bs_sc = (int32_t*)malloc(NJ * sizeof(int32_t));
  int32_t* bs_idx = (int32_t*)malloc(NJ * sizeof(int32_t));
  perm_t* perm = (perm_t*)malloc(NJ * sizeof(perm_t));
  int32_t best = INT_MIN, bestDecoy = INT_MIN;
  uint32_t nperm = 0, nbs = 0;
  n_aln[r] = 0;
  for (uint32_t h = 0; h < nj; ++h) {
    int32_t tot = 0, maxPossible = 0;
    int bad = 0;
    if (jh[h].li >= 0) { const int32_t s = sc_dp(c, rl, L, &lc[jh[h].li]); ctr->candidates++; if (s <= NEG_SCORE) bad = 1; tot += s; maxPossible += p->ma * (int32_t)L; }
    if (jh[h].ri >= 0) { const int32_t s = sc_dp(c, rr, L, &rc[jh[h].ri]); ctr->candidates++; if (s <= NEG_SCORE) bad = 1; tot += s; maxPossible += p->ma * (int32_t)L; }
    const int32_t hs = (!bad && (double)tot >= p->min_score_fraction * (double)maxPossible) ? tot : INT_MIN;
    sc[h] = hs;
    {   /* compatibility with the expected library format, as map_reads_core states it */
      const int orphan = jh[h].status != 0, isLeft = jh[h].status != 2;
      const int lfw = jh[h].li >= 0 && lc[jh[h].li].ori == 0, rfw = jh[h].ri >= 0 && rc[jh[h].ri].ori == 0;
      int ok;
      switch (p->lib_type) {
        case 0: ok = orphan ? 1 : lfw != rfw; break;
        case 1: ok = orphan ? ((isLeft && lfw) || (!isLeft && !rfw)) : (lfw && !rfw); break;
        case 2: ok = orphan ? ((isLeft && !lfw) || (!isLeft && rfw)) : (!lfw && rfw); break;
        case 4: ok = lfw; break;
        case 5: ok = !lfw; break;
        default: ok = 1;
      }
      if (!ok) { sc[h] = INT_MIN; continue; }
    }
    const double cutoff = (double)(int32_t)(p->decoy_threshold * (double)bestDecoy);
    if ((int32_t)jh[h].tid >= p->first_decoy) { if (hs > bestDecoy) bestDecoy = hs; continue; }
    if ((double)hs < cutoff || hs == INT_MIN) continue;
    uint32_t q = 0;
    while (q < nbs && bs_tid[q] != (int32_t)jh[h].tid) ++q;
    if (q == nbs) { bs_tid[nbs] = (int32_t)jh[h].tid; bs_sc[nbs] = hs; bs_idx[nbs] = (int32_t)h; ++nbs; }
    else if (hs >= bs_sc[q]) { bs_sc[q] = hs; sc[bs_idx[q]] = INT_MIN; bs_idx[q] = (int32_t)h; }
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
    ++na;
  }
  n_aln[r] = na;
  ctr->kept += na;
  free(sc); free(bs_tid); free(bs_sc); free(bs_idx); free(perm);
  if (!na) return;
  ctr->mapped++;
  ctr->label_entries += na;
  double aux[256], den = LOG_0;
  for (uint32_t a = 0; a < na; ++a) {
    const uint32_t t = tid[b + a];
    const int32_t refLen = (int32_t)(ix->off[t + 1] - ix->off[t]);
    const double refLength = refLen > 0 ? (double)refLen : 1.0;
    const uint32_t status = (flags[b + a] >> 2) & 3;
    const int fwd = flags[b + a] & 1, mfwd = (flags[b + a] >> 1) & 1;
    int32_t fl = flen[b + a];
    if (status == 0 && fwd != mfwd) {   /* fragLengthPedantic */
      int32_t p1 = fwd ? pos[b + a] : mpos[b + a]; p1 = p1 < 0 ? 0 : (p1 > refLen ? refLen : p1);
      int32_t p2 = fwd ? mpos[b + a] + (int32_t)L : pos[b + a] + (int32_t)L; p2 = p2 < 0 ? 0 : (p2 > refLen ? refLen : p2);
      fl = p1 > p2 ? p1 - p2 : p2 - p1;
    }
    double lfp = LOG_1;
    if (status != 0) {   /* orphan in a paired-end library */
      int32_t maxFragLen;
      if (fwd) { int32_t p1 = pos[b + a] < 0 ? 0 : pos[b + a]; p1 = p1 > refLen ? refLen : p1; maxFragLen = refLen - p1; }
      else { int32_t p1 = pos[b + a] + (int32_t)L; p1 = p1 < 0 ? 0 : p1; p1 = p1 > refLen ? refLen : p1; maxFragLen = p1; }
      const double* cm = burnedIn ? fld->cmf_cached : fld->cmf_quirk;
      const double rcm = tab(cm, fld->max_val, (uint64_t)refLen), mlp = tab(cm, fld->max_val, (uint64_t)maxFragLen);
      lfp = rcm != LOG_0 ? mlp - rcm : LOG_EPSILON;
    }
    if (fl > 0 && (burnedIn || useAux)) {
      if (burnedIn) {
        const double cm = tab(fld->cmf_cached, fld->max_val, (uint64_t)fl);
        lfp = ((double)fl < refLength && cm != LOG_0) ? tab(fld->pmf_cached, fld->max_val, (uint64_t)fl) - cm : LOG_EPSILON;
      } else {
        lfp = tab(fld->pmf_live, fld->max_val, (uint64_t)fl);
      }
    }
    aux[a] = lfp + (prob[b + a] > 0 ? m_log(prob[b + a]) : LOG_1) + LOG_1;
    den = logAddDet(den, aux[a]);
  }
  for (uint32_t a = 0; a < na; ++a) { weight[b + a] = m_exp(aux[a] - den); label[(size_t)r * 2 * cap + a] = tid[b + a]; }
  if (p->range_bins > 0) {
    const int32_t rcnt = (int32_t)sqrt((double)na) + (int32_t)p->range_bins;
    for (uint32_t a = 0; a < na; ++a) label[(size_t)r * 2 * cap + na + a] = (uint32_t)(int32_t)(weight[b + a] * rcnt);
  }
  if (on) online_fragment(on, r, L, na, tid + b, pos + b, mpos + b, flags + b, flen + b, aux);
}

/* a batch in the given mode, with or without rescue: stateless (on == NULL; regime from frag_counter, FLD = prior) or
 * through the online state (the batch set-up and fold of orc_online_batch).  ctr3: fragments rescued, searches, anchors
 * without room. */
static int sc_batch(orc_online* on, const orc_index* ix, const orc_map_params* p, int mode, int rescue, const uint8_t* left,
                    const uint8_t* right, uint32_t n, uint32_t L, uint64_t frag_counter, uint32_t* n_aln, uint32_t* tid,
                    int32_t* score, double* prob, int32_t* pos, int32_t* mpos, uint8_t* flags, int32_t* flen, uint32_t* label,
                    double* weight, orc_map_counters* ctr, uint64_t* ctr3) {
  const uint32_t cap = p->max_read_occ;
  const sc_ctx c = {ix, p, mode};
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
  ctr3[0] = ctr3[1] = ctr3[2] = 0;
  cand_t lc[MAXCAND], rc[MAXCAND];
  joint_t* jh = (joint_t*)malloc((size_t)(MAXCAND * MAXCAND + 2 * MAXCAND) * sizeof(joint_t));
  joint_t rj[2 * MAXCAND];
  for (uint32_t r = 0; r < n; ++r) {
    const uint8_t* rl = left + (size_t)r * L;
    const uint8_t* rr = right + (size_t)r * L;
    n_aln[r] = 0;
    uint32_t nl = mate_candidates(ix, p, rl, L, lc, &tot), nr = mate_candidates(ix, p, rr, L, rc, &tot);
    const uint32_t nj = rs_joint_hits(p, lc, nl, rc, nr, L, jh);
    if (nj == 0 || nj > cap) continue;
    int orphans_only = rescue && p->lib_type < 3;
    for (uint32_t h = 0; h < nj && orphans_only; ++h) if (jh[h].status == 0) orphans_only = 0;
    const uint32_t np = orphans_only ? sc_rescue_read(&c, rl, rr, L, lc, &nl, rc, &nr, jh, nj, rj, ctr3) : 0;
    if (np) ctr3[0]++;
    sc_assign(&c, fld, useAux, burnedIn, on, r, rl, rr, L, lc, rc, np ? rj : jh, np ? np : nj, n_aln, tid, score, prob,
              pos, mpos, flags, flen, label, weight, &tot);
  }
  free(jh);
  if (ctr) *ctr = tot;
  if (!on) { fld_free(&prior); return 0; }
  /* fold the batch into the state (orc_online_batch) */
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

int orc_sc_map_reads(const orc_index* ix, const orc_map_params* p, int mode, int rescue, const uint8_t* left,
                     const uint8_t* right, uint32_t n, uint32_t L, uint64_t frag_counter, uint32_t* n_aln, uint32_t* tid,
                     int32_t* score, double* prob, int32_t* pos, int32_t* mpos, uint8_t* flags, int32_t* flen,
                     uint32_t* label, double* weight, orc_map_counters* ctr, uint64_t* ctr3) {
  return sc_batch(NULL, ix, p, mode, rescue, left, right, n, L, frag_counter, n_aln, tid, score, prob, pos, mpos, flags, flen,
                  label, weight, ctr, ctr3);
}
int orc_sc_online_batch(orc_online* on, int mode, int rescue, const uint8_t* left, const uint8_t* right, uint32_t n,
                        uint32_t L, uint32_t* n_aln, uint32_t* tid, int32_t* score, double* prob, int32_t* pos,
                        int32_t* mpos, uint8_t* flags, int32_t* flen, uint32_t* label, double* weight,
                        orc_map_counters* ctr, uint64_t* ctr3) {
  return sc_batch(on, on->ix, &on->p, mode, rescue, left, right, n, L, 0, n_aln, tid, score, prob, pos, mpos, flags, flen,
                  label, weight, ctr, ctr3);
}
