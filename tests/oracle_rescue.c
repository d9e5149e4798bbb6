/*
 * tests/oracle_rescue.c -- TEST INFRASTRUCTURE.  Orphan rescue (--recoverOrphans; the rule is DESIGN.md section 11)
 * restated on top of the CPU oracle (oracle/map_oracle.c, included unchanged for its index, candidates, DP, assignment
 * and online state), written from salmon's call site (src/quant/SalmonQuantify.cpp:1342-1364), not from the product's
 * map_core.h:
 *   - rescue only when the join produced no pair and the read has no more than maxReadOcc joint hits;
 *   - each orphan whose own score passes and whose pair would fit the library type is an anchor; its transcript is
 *     searched within the maximum fragment length for the other mate with a plain O(W*L) Sellers DP (infix edit
 *     distance, limit K) -- no bit-parallel code shared with the product;
 *   - the place found is scored by the oracle's DP, must pass and form a concordant pair; identical pairs count once;
 *     the mate's candidate list holds at most MAXCAND entries;
 *   - "if we recovered a mate, then we have no orphans" (:1362): the read's mappings are the rescued pairs.
 * Reads without a rescue go through the oracle's own map_reads_core, one read at a time.
 */
#include "../oracle/map_oracle.c"

/* smallest infix edit distance of pat in text and the leftmost end at that distance; -1 / -1 above K.  Code 4 (N) in
 * either sequence matches nothing. */
void orc_sellers_infix(const uint8_t* pat, uint32_t m, const uint8_t* text, uint32_t n, int32_t K, int32_t* dist, int32_t* end) {
  int32_t* col = (int32_t*)malloc((m + 1) * sizeof(int32_t));
  for (uint32_t i = 0; i <= m; ++i) col[i] = (int32_t)i;
  int32_t best = K + 1, bend = -1;
  for (uint32_t j = 0; j < n; ++j) {
    int32_t diag = col[0];   /* D[0][j-1] */
    col[0] = 0;              /* free start */
    for (uint32_t i = 1; i <= m; ++i) {
      const int32_t up = col[i];
      const int match = pat[i - 1] < 4 && pat[i - 1] == text[j];
      int32_t v = diag + (match ? 0 : 1);
      if (up + 1 < v) v = up + 1;
      if (col[i - 1] + 1 < v) v = col[i - 1] + 1;
      diag = up;
      col[i] = v;
    }
    if (col[m] < best) { best = col[m]; bend = (int32_t)j; }
  }
  free(col);
  *dist = bend >= 0 ? best : -1;
  *end = bend;
}

/* the oracle's join, as oracle_sam.c states it (pairs, else orphans) */
static uint32_t rs_joint_hits(const orc_map_params* p, const cand_t* lc, uint32_t nl, const cand_t* rc, uint32_t nr,
                              uint32_t L, joint_t* out) {
  uint8_t okl[MAXCAND], okr[MAXCAND];
  for (uint32_t a = 0; a < nl; ++a) {
    uint32_t best = 0;
    for (uint32_t q = 0; q < nl; ++q) if (lc[q].tid == lc[a].tid && lc[q].cov > best) best = lc[q].cov;
    okl[a] = (double)lc[a].cov >= p->pre_merge_thresh * (double)best;
  }
  for (uint32_t b = 0; b < nr; ++b) {
    uint32_t best = 0;
    for (uint32_t q = 0; q < nr; ++q) if (rc[q].tid == rc[b].tid && rc[q].cov > best) best = rc[q].cov;
    okr[b] = (double)rc[b].cov >= p->pre_merge_thresh * (double)best;
  }
  uint32_t np = 0, best_all = 0, nj = 0;
  for (uint32_t a = 0; a < nl; ++a)
    for (uint32_t b = 0; b < nr; ++b) {
      if (!okl[a] || !okr[b] || lc[a].tid != rc[b].tid || lc[a].ori == rc[b].ori) continue;
      const cand_t* fw = lc[a].ori == 0 ? &lc[a] : &rc[b];
      const cand_t* rv = lc[a].ori == 0 ? &rc[b] : &lc[a];
      int32_t s = fw->diag_c, e = rv->diag_c + (int32_t)L;
      if (rv->diag_c < fw->diag_c) {
        if (!p->allow_dovetail) continue;
        s = rv->diag_c; e = fw->diag_c + (int32_t)L;
      }
      if (e - s <= 0 || e - s > (int32_t)p->max_frag_len) continue;
      joint_t j = {lc[a].tid, (int32_t)a, (int32_t)b, e - s, 0};
      out[np++] = j;
      if (lc[a].cov + rc[b].cov > best_all) best_all = lc[a].cov + rc[b].cov;
    }
  for (uint32_t q = 0; q < np; ++q) {
    const uint32_t sc = lc[out[q].li].cov + rc[out[q].ri].cov;
    uint32_t best_t = 0;
    for (uint32_t w = 0; w < np; ++w)
      if (out[w].tid == out[q].tid && lc[out[w].li].cov + rc[out[w].ri].cov > best_t) best_t = lc[out[w].li].cov + rc[out[w].ri].cov;
    if (!((double)sc < p->post_merge_thresh * (double)best_t || (double)sc < p->consensus_frac * (double)best_all)) out[nj++] = out[q];
  }
  if (nj == 0 && p->allow_orphans) {
    uint32_t best_c = 0;
    for (uint32_t a = 0; a < nl; ++a) if (okl[a] && lc[a].cov > best_c) best_c = lc[a].cov;
    for (uint32_t b = 0; b < nr; ++b) if (okr[b] && rc[b].cov > best_c) best_c = rc[b].cov;
    const double thr = (p->lib_type >= 3 ? 0.0 : p->orphan_thresh) * (double)best_c;
    for (uint32_t a = 0; a < nl; ++a) if (okl[a] && (double)lc[a].cov >= thr) { joint_t j = {lc[a].tid, (int32_t)a, -1, 0, 1}; out[nj++] = j; }
    for (uint32_t b = 0; b < nr; ++b) if (okr[b] && (double)rc[b].cov >= thr) { joint_t j = {rc[b].tid, -1, (int32_t)b, 0, 2}; out[nj++] = j; }
  }
  return nj;
}

static int rs_pair_compatible(int lib_type, int lfw, int rfw) {   /* SalmonUtils.cpp:193-298, paired mappings */
  switch (lib_type) {
    case 0: return lfw != rfw;
    case 1: return lfw && !rfw;
    case 2: return !lfw && rfw;
    default: return 1;
  }
}
static int rs_passes(const orc_map_params* p, int32_t s, uint32_t L) {
  return s > NEG_SCORE && (double)s >= p->min_score_fraction * (double)(p->ma * (int32_t)L);
}

/* the read's rescued pairs (status 0) into jh, the rescued candidates appended to lc / rc; returns their number */
static uint32_t rs_rescue_read(const orc_index* ix, const orc_map_params* p, const uint8_t* rl, const uint8_t* rr,
                               uint32_t L, cand_t* lc, uint32_t* nl, cand_t* rc, uint32_t* nr, const joint_t* orph,
                               uint32_t nj, joint_t* jh, uint64_t* ctr3) {
  const int32_t per = (p->ma - p->mp) < p->ge ? (p->ma - p->mp) : p->ge;
  int32_t K = (int32_t)L;
  if (per > 0) { const double k = (1.0 - p->min_score_fraction) * p->ma * (double)L / per; K = k < 0 ? 0 : (k >= L ? (int32_t)L : (int32_t)k); }
  uint8_t* pat = (uint8_t*)malloc(L);
  uint32_t np = 0;
  for (uint32_t h = 0; h < nj; ++h) {
    const int left = orph[h].status == 1;
    const cand_t anc = left ? lc[orph[h].li] : rc[orph[h].ri];
    const uint8_t* own = left ? rl : rr;
    const uint8_t* other = left ? rr : rl;
    if (!rs_passes(p, dp_score(ix, p, own, L, anc.ori, anc.tid, anc.diag_c), L)) continue;
    const int afw = anc.ori == 0;
    if (!rs_pair_compatible(p->lib_type, left ? afw : !afw, left ? !afw : afw)) continue;
    ctr3[1]++;
    /* window: within one maximum fragment length downstream (anchor forward) or upstream (anchor reverse) */
    const int64_t tlen = (int64_t)(ix->off[anc.tid + 1] - ix->off[anc.tid]);
    int64_t lo = afw ? anc.diag_c : (int64_t)anc.diag_c + L - p->max_frag_len;
    int64_t hi = afw ? (int64_t)anc.diag_c + p->max_frag_len : (int64_t)anc.diag_c + L;
    if (lo < 0) lo = 0;
    if (hi > tlen) hi = tlen;
    if (hi <= lo) continue;
    for (uint32_t i = 0; i < L; ++i)   /* forward anchor: the mate lies on the other strand */
      pat[i] = afw ? (other[L - 1 - i] > 3 ? 4 : 3 - other[L - 1 - i]) : other[i];
    int32_t d, e;
    orc_sellers_infix(pat, L, ix->codes + ix->off[anc.tid] + lo, (uint32_t)(hi - lo), K, &d, &e);
    if (d < 0) continue;
    cand_t res;
    memset(&res, 0, sizeof res);
    res.tid = anc.tid; res.ori = afw ? 1 : 0; res.diag_c = (int32_t)(lo + e) - (int32_t)L + 1;
    if (!rs_passes(p, dp_score(ix, p, other, L, res.ori, res.tid, res.diag_c), L)) continue;
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

/* updateRefMappings + filterAndCollectAlignments + auxiliary probabilities + label for a read whose joint hits are the
 * rescued pairs (SalmonMappingUtils.hpp:225-405, SalmonQuantify.cpp:599-857), state frozen per batch */
static void rs_assign(const orc_index* ix, const orc_map_params* p, const fld_t* fld, int useAux, int burnedIn,
                      orc_online* on, uint32_t r, const uint8_t* rl, const uint8_t* rr, uint32_t L, const cand_t* lc,
                      const cand_t* rc, const joint_t* jh, uint32_t nj, uint32_t* n_aln, uint32_t* tid, int32_t* score,
                      double* prob, int32_t* pos, int32_t* mpos, uint8_t* flags, int32_t* flen, uint32_t* label,
                      double* weight, orc_map_counters* ctr) {
  const uint32_t cap = p->max_read_occ;
  const double LOG_EPSILON = log(EPSILON_);
  int32_t sc[2 * MAXCAND], bs_tid[2 * MAXCAND], bs_sc[2 * MAXCAND], bs_idx[2 * MAXCAND];
  perm_t perm[2 * MAXCAND];
  int32_t best = INT_MIN, bestDecoy = INT_MIN;
  uint32_t nperm = 0, nbs = 0;
  for (uint32_t h = 0; h < nj; ++h) {
    const int32_t s1 = dp_score(ix, p, rl, L, lc[jh[h].li].ori, jh[h].tid, lc[jh[h].li].diag_c);
    const int32_t s2 = dp_score(ix, p, rr, L, rc[jh[h].ri].ori, jh[h].tid, rc[jh[h].ri].diag_c);
    const int bad = s1 <= NEG_SCORE || s2 <= NEG_SCORE;
    const int32_t hs = (!bad && (double)(s1 + s2) >= p->min_score_fraction * (double)(2 * p->ma * (int32_t)L)) ? s1 + s2 : INT_MIN;
    sc[h] = hs;
    if (!rs_pair_compatible(p->lib_type, lc[jh[h].li].ori == 0, rc[jh[h].ri].ori == 0)) { sc[h] = INT_MIN; continue; }
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
    tid[b + na] = j->tid; score[b + na] = sc[perm[q].idx]; prob[b + na] = est;
    pos[b + na] = lc[j->li].diag_c; mpos[b + na] = rc[j->ri].diag_c;
    flags[b + na] = (uint8_t)((lc[j->li].ori == 0 ? 1 : 0) | (rc[j->ri].ori == 0 ? 2 : 0));
    flen[b + na] = j->frag_len;
    ++na;
  }
  n_aln[r] = na;
  ctr->kept += na;
  if (!na) return;
  ctr->mapped++;
  ctr->label_entries += na;
  double aux[2 * MAXCAND], den = LOG_0;
  for (uint32_t a = 0; a < na; ++a) {
    const uint32_t t = tid[b + a];
    const int32_t refLen = (int32_t)(ix->off[t + 1] - ix->off[t]);
    const int fwd = flags[b + a] & 1, mfwd = (flags[b + a] >> 1) & 1;
    int32_t fl = flen[b + a];
    if (fwd != mfwd) {   /* fragLengthPedantic */
      int32_t p1 = fwd ? pos[b + a] : mpos[b + a]; p1 = p1 < 0 ? 0 : (p1 > refLen ? refLen : p1);
      int32_t p2 = fwd ? mpos[b + a] + (int32_t)L : pos[b + a] + (int32_t)L; p2 = p2 < 0 ? 0 : (p2 > refLen ? refLen : p2);
      fl = p1 > p2 ? p1 - p2 : p2 - p1;
    }
    double lfp = LOG_1;
    if (fl > 0 && (burnedIn || useAux)) {
      if (burnedIn) {
        const double cm = tab(fld->cmf_cached, fld->max_val, (uint64_t)fl);
        lfp = ((double)fl < (refLen > 0 ? (double)refLen : 1.0) && cm != LOG_0) ? tab(fld->pmf_cached, fld->max_val, (uint64_t)fl) - cm : LOG_EPSILON;
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

/* a batch with rescue: stateless (on == NULL; regime from frag_counter, FLD = prior) or through the online state
 * (the batch set-up and fold of orc_online_batch).  ctr3: fragments rescued, searches, anchors without room. */
static int rs_batch(orc_online* on, const orc_index* ix, const orc_map_params* p, const uint8_t* left, const uint8_t* right,
                    uint32_t n, uint32_t L, uint64_t frag_counter, uint32_t* n_aln, uint32_t* tid, int32_t* score,
                    double* prob, int32_t* pos, int32_t* mpos, uint8_t* flags, int32_t* flen, uint32_t* label,
                    double* weight, orc_map_counters* ctr, uint64_t* ctr3) {
  const uint32_t cap = p->max_read_occ;
  fld_t prior;
  const fld_t* fld = &prior;
  int useAux, burnedIn;
  uint64_t t0 = 0, fs0 = 0;
  if (on) {
    const uint64_t nsteps = (n + on->mini_batch - 1) / on->mini_batch;
    on->batch_t0 = on->timestep;
    on->batch_ref = fm_at(on, on->timestep + (nsteps ? nsteps - 1 : 0));
    on->batch_min = on->p.max_frag_len;
    on->batch_assigned = 0;
    useAux = on->assigned >= p->num_pre_burnin; burnedIn = on->burned_in; fld = &on->fld;
    t0 = on->batch_t0; fs0 = on->frags_seen;
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
    orc_map_counters cc;
    memset(&cc, 0, sizeof cc);
    uint32_t nl = mate_candidates(ix, p, rl, L, lc, &cc), nr = mate_candidates(ix, p, rr, L, rc, &cc);
    const uint32_t nj = rs_joint_hits(p, lc, nl, rc, nr, L, jh);
    int orphans_only = nj > 0 && nj <= cap && p->lib_type < 3;
    for (uint32_t h = 0; h < nj && orphans_only; ++h) if (jh[h].status == 0) orphans_only = 0;
    uint32_t np = 0;
    if (orphans_only) np = rs_rescue_read(ix, p, rl, rr, L, lc, &nl, rc, &nr, jh, nj, rj, ctr3);
    if (np) {
      ctr3[0]++;
      tot.lookups += cc.lookups; tot.postings += cc.postings; tot.seeds += cc.seeds;
      n_aln[r] = 0;
      rs_assign(ix, p, fld, useAux, burnedIn, on, r, rl, rr, L, lc, rc, rj, np, n_aln, tid, score, prob, pos, mpos, flags,
                flen, label, weight, &tot);
      continue;
    }
    /* no rescue: the oracle's own path for this one read (its online update keyed to the read's place in the batch) */
    const size_t b = (size_t)r * cap;
    if (on) { on->batch_t0 = t0 + r / on->mini_batch; on->frags_seen = fs0 + r; }
    map_reads_core(ix, p, fld, useAux, burnedIn, on, rl, rr, 1, L, n_aln + r, tid + b, score + b, prob + b, pos + b,
                   mpos + b, flags + b, flen + b, label + (size_t)r * 2 * cap, weight + b, &cc);
    if (on) { on->batch_t0 = t0; on->frags_seen = fs0; }
    const uint64_t* src = (const uint64_t*)&cc;
    uint64_t* dst = (uint64_t*)&tot;
    for (size_t i = 0; i < sizeof(orc_map_counters) / 8; ++i) dst[i] += src[i];
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

int orc_rescue_map_reads(const orc_index* ix, const orc_map_params* p, const uint8_t* left, const uint8_t* right, uint32_t n,
                         uint32_t L, uint64_t frag_counter, uint32_t* n_aln, uint32_t* tid, int32_t* score, double* prob,
                         int32_t* pos, int32_t* mpos, uint8_t* flags, int32_t* flen, uint32_t* label, double* weight,
                         orc_map_counters* ctr, uint64_t* ctr3) {
  return rs_batch(NULL, ix, p, left, right, n, L, frag_counter, n_aln, tid, score, prob, pos, mpos, flags, flen, label,
                  weight, ctr, ctr3);
}
int orc_rescue_online_batch(orc_online* on, const uint8_t* left, const uint8_t* right, uint32_t n, uint32_t L,
                            uint32_t* n_aln, uint32_t* tid, int32_t* score, double* prob, int32_t* pos, int32_t* mpos,
                            uint8_t* flags, int32_t* flen, uint32_t* label, double* weight, orc_map_counters* ctr,
                            uint64_t* ctr3) {
  return rs_batch(on, on->ix, &on->p, left, right, n, L, 0, n_aln, tid, score, prob, pos, mpos, flags, flen, label, weight,
                  ctr, ctr3);
}
