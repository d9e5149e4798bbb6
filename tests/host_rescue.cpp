// tests/host_rescue.cpp -- TEST INFRASTRUCTURE.  The product's orphan rescue (salmon_b200/csrc/map_core.h: anchors,
// window, bit-vector search, commit, assign_read with the rescued pairs) compiled for the HOST, so that it can be
// checked against edlib's goldens and the independent restatement (tests/oracle_rescue.c) without a GPU.
#include <stdint.h>
#include <string.h>
#include <vector>

#include "../salmon_b200/csrc/map_core.h"

using namespace sbmap;

// the serial bit-vector search on one (pattern, text) case
extern "C" void hrs_myers(const uint8_t* pat, uint32_t m, const uint8_t* text, uint32_t n, int32_t K, int32_t* dist,
                          int32_t* end) {
  myers_infix_any([&](uint32_t i) { return pat[i]; }, m, n, [&](uint32_t j) { return text[j]; }, K, *dist, *end);
}

extern "C" int32_t hrs_edit_limit(const Params* p, uint32_t L) { return rescue_edit_limit(*p, L); }

// hmc_map_reads (tests/host_map_core.cpp) with the rescue step between the DP scores and the assignment.
// rescue3: fragments rescued, searches, anchors without room.
extern "C" int hrs_map_reads(uint32_t n_txps, uint32_t k, const uint64_t* tx_off, const uint8_t* codes,
                             const void* table, uint64_t table_capacity, const void* postings, const Params* p,
                             const double* fld4, const uint8_t* left, const uint8_t* right, uint32_t n, uint32_t L,
                             uint64_t frag_counter, uint32_t* n_aln, uint32_t* tid, int32_t* score, double* prob,
                             int32_t* pos, int32_t* mate_pos, uint8_t* flags, int32_t* flen, uint32_t* label,
                             double* weight, unsigned long long* rescue3) {
  IndexView ix;
  ix.n_txps = n_txps; ix.k = k; ix.mask = table_capacity - 1; ix.tx_off = tx_off; ix.codes = codes;
  ix.table = (const TableEntry*)table; ix.post = (const Posting*)postings;
  ix.packed = nullptr; ix.tx_has_n = nullptr;
  const uint32_t nf = p->max_frag_len + 1;
  FldView fld;
  fld.max_val = p->max_frag_len; fld.pmf_live = fld4; fld.pmf_cached = fld4 + nf; fld.cmf_cached = fld4 + 2 * nf;
  fld.cmf_quirk = fld4 + 3 * nf;
  const uint32_t cap = p->max_read_occ;
  std::vector<uint64_t> keys(MAXSEEDS);
  std::vector<Cand> lc(MAXCAND), rc(MAXCAND);
  std::vector<int32_t> sl(MAXCAND), sr(MAXCAND), sc(cap), pi(cap), pt(cap), b1(cap), b2(cap), b3(cap);
  std::vector<Joint> jh(cap), pre(2 * MAXCAND);
  uint8_t side[2 * MAXCAND], ci[2 * MAXCAND];
  int32_t rdiag[2 * MAXCAND], rscore[2 * MAXCAND];
  Counters ctr;
  memset(&ctr, 0, sizeof(ctr));
  rescue3[0] = rescue3[1] = rescue3[2] = 0;
  const bool useAux = frag_counter >= p->num_pre_burnin, burnedIn = frag_counter >= p->num_burnin;
  for (uint32_t r = 0; r < n; ++r) {
    const uint8_t* rl = left + (size_t)r * L;
    const uint8_t* rr = right + (size_t)r * L;
    uint32_t nl = mate_candidates(ix, *p, rl, L, keys.data(), 1, lc.data(), ctr);
    uint32_t nr = mate_candidates(ix, *p, rr, L, keys.data(), 1, rc.data(), ctr);
    unsigned long long used_l = 0, used_r = 0;
    const uint32_t nj = for_each_joint(*p, lc.data(), nl, rc.data(), nr, L, [&](const Joint& j, uint32_t) {
      if (j.li >= 0) used_l |= 1ull << j.li;
      if (j.ri >= 0) used_r |= 1ull << j.ri;
    });
    ReadOut o;
    o.n_aln = n_aln + r; o.tid = tid + (size_t)r * cap; o.score = score + (size_t)r * cap; o.prob = prob + (size_t)r * cap;
    o.pos = pos + (size_t)r * cap; o.mate_pos = mate_pos + (size_t)r * cap; o.flags = flags + (size_t)r * cap;
    o.flen = flen + (size_t)r * cap; o.label = label + (size_t)r * 2 * cap; o.weight = weight + (size_t)r * cap;
    *o.n_aln = 0;
    if (nj == 0 || nj > cap) continue;
    for (uint32_t a = 0; a < nl; ++a)
      if (used_l >> a & 1) sl[a] = dp_score_serial(ix, *p, rl, L, lc[a].ori_cov >> 31, lc[a].tid, lc[a].diag_c);
    for (uint32_t a = 0; a < nr; ++a)
      if (used_r >> a & 1) sr[a] = dp_score_serial(ix, *p, rr, L, rc[a].ori_cov >> 31, rc[a].tid, rc[a].diag_c);
    uint32_t np = 0;
    if (p->recover_orphans && p->lib_type < 3) {
      const uint32_t na = rescue_anchors(*p, lc.data(), nl, rc.data(), nr, sl.data(), sr.data(), L, side, ci);
      rescue3[1] += na;
      for (uint32_t a = 0; a < na; ++a) {
        const Cand& anc = side[a] == 0 ? lc[ci[a]] : rc[ci[a]];
        const uint8_t* mate = side[a] == 0 ? rr : rl;
        rscore[a] = INVALID_SCORE;
        if (rescue_search_serial(ix, *p, anc, mate, L, rdiag[a])) {
          const Cand res = rescue_cand(anc, rdiag[a]);
          rscore[a] = dp_score_serial(ix, *p, mate, L, res.ori_cov >> 31, res.tid, res.diag_c);
        }
      }
      uint32_t no_room = 0;
      np = rescue_commit(*p, L, lc.data(), nl, rc.data(), nr, sl.data(), sr.data(), na, side, ci, rdiag, rscore,
                         pre.data(), no_room);
      rescue3[0] += np ? 1 : 0;
      rescue3[2] += no_room;
    }
    assign_read(ix, *p, fld, useAux, burnedIn, lc.data(), nl, rc.data(), nr, sl.data(), sr.data(), L, sc.data(),
                pi.data(), pt.data(), b1.data(), b2.data(), b3.data(), jh.data(), o, ctr, nullptr, 0, nullptr, nullptr,
                np ? pre.data() : nullptr, np);
  }
  return 0;
}
