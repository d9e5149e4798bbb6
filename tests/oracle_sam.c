/*
 * tests/oracle_sam.c -- TEST INFRASTRUCTURE.  The SAM side output of the mapping step, restated on top of the CPU
 * oracle (oracle/map_oracle.c, included unchanged for its index, candidates and DP) and written from salmon's code, not
 * from the product's map_core.h:
 *   - per-mate scores: the oracle's DP score of each mate of each kept alignment (salmon's score / mateScore);
 *   - decoy-only fragments: MappingScoreInfo::update_decoy_mappings collects the joint hits whose score equals the best
 *     decoy score, in joint-hit order (SalmonMappingUtils.hpp:124-139); haveOnlyDecoyMappings (:115-122) decides
 *     whether they are written; filterAndCollectAlignmentsDecoy (:407-470) turns them into alignments.
 * The kept alignments themselves come from orc_map_reads, which the caller runs first.
 */
#include "../oracle/map_oracle.c"

/* the joint hits of one read as the oracle's join forms them (MAPSPEC step 4): pairs, else orphans */
static uint32_t sam_joint_hits(const orc_map_params* p, const cand_t* lc, uint32_t nl, const cand_t* rc, uint32_t nr,
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

static int sam_compatible(int lib_type, uint32_t status, int lfw, int rfw) {   /* SalmonUtils.cpp:193-298 */
  const int orphan = status != 0, left = status != 2;
  switch (lib_type) {
    case 0: return orphan ? 1 : lfw != rfw;
    case 1: return orphan ? ((left && lfw) || (!left && !rfw)) : (lfw && !rfw);
    case 2: return orphan ? ((left && !lfw) || (!left && rfw)) : (!lfw && rfw);
    case 4: return lfw;
    case 5: return !lfw;
    default: return 1;
  }
}

/* n_aln / tid / pos / mate_pos / flags / flen: orc_map_reads' output for the same reads (cap entries per read).
 * Out: n_out, decoy, score1 / score2 per written alignment; for decoy-only reads the decoy alignments are written into
 * tid / pos / mate_pos / flags / flen. */
int orc_sam_side(const orc_index* ix, const orc_map_params* p, const uint8_t* left, const uint8_t* right, uint32_t n,
                 uint32_t L, const uint32_t* n_aln, uint32_t* tid, int32_t* pos, int32_t* mate_pos, uint8_t* flags,
                 int32_t* flen, uint32_t* n_out, uint8_t* decoy, int32_t* score1, int32_t* score2) {
  const uint32_t cap = p->max_read_occ;
  orc_map_counters ctr;
  memset(&ctr, 0, sizeof ctr);
  cand_t* lc = (cand_t*)malloc(MAXCAND * sizeof(cand_t));
  cand_t* rc = (cand_t*)malloc(MAXCAND * sizeof(cand_t));
  joint_t* jh = (joint_t*)malloc((size_t)(MAXCAND * MAXCAND + 2 * MAXCAND) * sizeof(joint_t));
  int32_t* s1 = (int32_t*)malloc((size_t)(MAXCAND * MAXCAND + 2 * MAXCAND) * sizeof(int32_t));
  int32_t* s2 = (int32_t*)malloc((size_t)(MAXCAND * MAXCAND + 2 * MAXCAND) * sizeof(int32_t));
  for (uint32_t r = 0; r < n; ++r) {
    const uint8_t* rl = left + (size_t)r * L;
    const uint8_t* rr = right + (size_t)r * L;
    const size_t b = (size_t)r * cap;
    n_out[r] = n_aln[r];
    decoy[r] = 0;
    if (n_aln[r] > 0) {   /* each mate's own score at the place the alignment puts it */
      for (uint32_t a = 0; a < n_aln[r]; ++a) {
        const uint32_t st = (flags[b + a] >> 2) & 3, fw1 = flags[b + a] & 1, fw2 = (flags[b + a] >> 1) & 1;
        score1[b + a] = score2[b + a] = 0;
        if (st == 0 || st == 1) score1[b + a] = dp_score(ix, p, rl, L, fw1 ? 0 : 1, tid[b + a], pos[b + a]);
        if (st == 0) score2[b + a] = dp_score(ix, p, rr, L, fw2 ? 0 : 1, tid[b + a], mate_pos[b + a]);
        if (st == 2) score2[b + a] = dp_score(ix, p, rr, L, fw1 ? 0 : 1, tid[b + a], pos[b + a]);
      }
      continue;
    }
    const uint32_t nl = mate_candidates(ix, p, rl, L, lc, &ctr), nr = mate_candidates(ix, p, rr, L, rc, &ctr);
    const uint32_t nj = sam_joint_hits(p, lc, nl, rc, nr, L, jh);
    if (nj == 0 || nj > cap) continue;
    /* updateRefMappings' score bookkeeping (SalmonMappingUtils.hpp:225-281) with the decoy hits collected */
    int32_t best = INT_MIN, best_decoy = INT_MIN;
    uint32_t hits[MAXCAND * MAXCAND + 2 * MAXCAND], nh = 0;
    for (uint32_t h = 0; h < nj; ++h) {
      int32_t tot = 0, maxp = 0;
      int bad = 0;
      s1[h] = s2[h] = 0;
      if (jh[h].li >= 0) { s1[h] = dp_score(ix, p, rl, L, lc[jh[h].li].ori, jh[h].tid, lc[jh[h].li].diag_c); bad |= s1[h] <= NEG_SCORE; tot += s1[h]; maxp += p->ma * (int32_t)L; }
      if (jh[h].ri >= 0) { s2[h] = dp_score(ix, p, rr, L, rc[jh[h].ri].ori, jh[h].tid, rc[jh[h].ri].diag_c); bad |= s2[h] <= NEG_SCORE; tot += s2[h]; maxp += p->ma * (int32_t)L; }
      const int32_t score = (!bad && (double)tot >= p->min_score_fraction * (double)maxp) ? tot : INT_MIN;
      if (!sam_compatible(p->lib_type, jh[h].status, jh[h].li >= 0 && lc[jh[h].li].ori == 0, jh[h].ri >= 0 && rc[jh[h].ri].ori == 0))
        continue;
      if ((int32_t)jh[h].tid >= p->first_decoy) {            /* update_decoy_mappings */
        if (score > best_decoy) { best_decoy = score; nh = 0; hits[nh++] = h; }
        else if (score == best_decoy) hits[nh++] = h;
        continue;
      }
      const double cutoff = (double)(int32_t)(p->decoy_threshold * (double)best_decoy);
      if (score != INT_MIN && (double)score >= cutoff && score > best) best = score;
    }
    /* haveOnlyDecoyMappings */
    if (!(best < (int32_t)(p->decoy_threshold * (double)best_decoy) && best_decoy > INT_MIN)) continue;
    for (uint32_t k = 0; k < nh && k < cap; ++k) {
      const joint_t* j = &jh[hits[k]];
      const cand_t* first = j->status == 2 ? &rc[j->ri] : &lc[j->li];
      tid[b + k] = j->tid;
      pos[b + k] = first->diag_c;
      mate_pos[b + k] = j->status == 0 ? rc[j->ri].diag_c : 0;
      flags[b + k] = (uint8_t)((first->ori == 0 ? 1 : 0) | (j->status == 0 && rc[j->ri].ori == 0 ? 2 : 0) | (j->status << 2));
      flen[b + k] = j->frag_len;
      score1[b + k] = s1[hits[k]];
      score2[b + k] = s2[hits[k]];
    }
    n_out[r] = nh < cap ? nh : cap;
    decoy[r] = nh ? 1 : 0;
  }
  free(lc); free(rc); free(jh); free(s1); free(s2);
  return 0;
}
