// tests/host_map_core.cpp -- TEST INFRASTRUCTURE.  Compiles the product's per-read Stage A logic
// (salmon_b200/csrc/map_core.h, the code the CUDA kernels run) for the HOST so that it can be
// checked against the independent oracle (oracle/map_oracle.c) without a GPU.  Not part of the
// product library; the product has no CPU path.
#include <stdint.h>
#include <string.h>
#include <vector>

#include "../salmon_b200/csrc/map_core.h"

using namespace sbmap;

extern "C" int hmc_map_reads(uint32_t n_txps, uint32_t k, const uint64_t* tx_off, const uint8_t* codes,
                             const void* table, uint64_t table_capacity, const void* postings,
                             const Params* p, const double* fld4 /* 4*(max_frag_len+1) */,
                             const uint8_t* left, const uint8_t* right, uint32_t n, uint32_t L,
                             uint64_t frag_counter, uint32_t* n_aln, uint32_t* tid, int32_t* score, double* prob,
                             int32_t* pos, int32_t* mate_pos, uint8_t* flags, int32_t* flen, uint32_t* label,
                             double* weight, unsigned long long* counters7) {
  IndexView ix;
  ix.n_txps = n_txps; ix.k = k; ix.mask = table_capacity - 1; ix.tx_off = tx_off; ix.codes = codes;
  ix.table = (const TableEntry*)table; ix.post = (const Posting*)postings;
  ix.packed = nullptr; ix.tx_has_n = nullptr;   // the serial forms read the byte codes
  const uint32_t nf = p->max_frag_len + 1;
  FldView fld;
  fld.max_val = p->max_frag_len; fld.pmf_live = fld4; fld.pmf_cached = fld4 + nf; fld.cmf_cached = fld4 + 2 * nf;
  fld.cmf_quirk = fld4 + 3 * nf;
  const uint32_t cap = p->max_read_occ;
  std::vector<uint64_t> keys(MAXSEEDS);
  std::vector<Cand> lc(MAXCAND), rc(MAXCAND);
  std::vector<int32_t> sl(MAXCAND), sr(MAXCAND), sc(cap), pi(cap), pt(cap), b1(cap), b2(cap), b3(cap);
  std::vector<Joint> jh(cap);
  Counters ctr;
  memset(&ctr, 0, sizeof(ctr));
  const bool useAux = frag_counter >= p->num_pre_burnin, burnedIn = frag_counter >= p->num_burnin;
  for (uint32_t r = 0; r < n; ++r) {
    const uint8_t* rl = left + (size_t)r * L;
    const uint8_t* rr = right + (size_t)r * L;
    const uint32_t nl = mate_candidates(ix, *p, rl, L, keys.data(), 1, lc.data(), ctr);
    const uint32_t nr = mate_candidates(ix, *p, rr, L, keys.data(), 1, rc.data(), ctr);
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
      if (used_l >> a & 1) { sl[a] = dp_score_serial(ix, *p, rl, L, lc[a].ori_cov >> 31, lc[a].tid, lc[a].diag_c); ctr.candidates++; }
    for (uint32_t a = 0; a < nr; ++a)
      if (used_r >> a & 1) { sr[a] = dp_score_serial(ix, *p, rr, L, rc[a].ori_cov >> 31, rc[a].tid, rc[a].diag_c); ctr.candidates++; }
    assign_read(ix, *p, fld, useAux, burnedIn, lc.data(), nl, rc.data(), nr, sl.data(), sr.data(), L, sc.data(),
                pi.data(), pt.data(), b1.data(), b2.data(), b3.data(), jh.data(), o, ctr);
  }
  counters7[0] = ctr.lookups; counters7[1] = ctr.postings; counters7[2] = ctr.seeds; counters7[3] = ctr.candidates;
  counters7[4] = ctr.kept; counters7[5] = ctr.label_entries; counters7[6] = ctr.mapped;
  return 0;
}

// CPU port for bench.py's cpu_baseline / reference arm: the same per-read logic over all host threads (OpenMP,
// reads are independent), outputs discarded except the per-read alignment count and the counters.  The online
// state is not advanced (stateless regime from frag_counter), which is what the reference's mapping threads cost.
#include <omp.h>
extern "C" int hmc_map_throughput(uint32_t n_txps, uint32_t k, const uint64_t* tx_off, const uint8_t* codes,
                                  const void* table, uint64_t table_capacity, const void* postings, const Params* p,
                                  const double* fld4, const uint8_t* left, const uint8_t* right, uint32_t n, uint32_t L,
                                  uint64_t frag_counter, int n_threads, uint32_t* n_aln, unsigned long long* counters7) {
  IndexView ix;
  ix.n_txps = n_txps; ix.k = k; ix.mask = table_capacity - 1; ix.tx_off = tx_off; ix.codes = codes;
  ix.table = (const TableEntry*)table; ix.post = (const Posting*)postings;
  ix.packed = nullptr; ix.tx_has_n = nullptr;
  const uint32_t nf = p->max_frag_len + 1;
  FldView fld;
  fld.max_val = p->max_frag_len; fld.pmf_live = fld4; fld.pmf_cached = fld4 + nf; fld.cmf_cached = fld4 + 2 * nf;
  fld.cmf_quirk = fld4 + 3 * nf;
  const uint32_t cap = p->max_read_occ;
  const bool useAux = frag_counter >= p->num_pre_burnin, burnedIn = frag_counter >= p->num_burnin;
  unsigned long long tot[7] = {0, 0, 0, 0, 0, 0, 0};
  if (n_threads > 0) omp_set_num_threads(n_threads);
#pragma omp parallel
  {
    std::vector<uint64_t> keys(MAXSEEDS);
    std::vector<Cand> lc(MAXCAND), rc(MAXCAND);
    std::vector<int32_t> sl(MAXCAND), sr(MAXCAND), sc(cap), pi(cap), pt(cap), b1(cap), b2(cap), b3(cap);
    std::vector<Joint> jh(cap);
    std::vector<uint32_t> o_tid(cap), o_label(2 * cap);
    std::vector<int32_t> o_score(cap), o_pos(cap), o_mpos(cap), o_flen(cap);
    std::vector<double> o_prob(cap), o_weight(cap);
    std::vector<uint8_t> o_flags(cap);
    Counters ctr;
    memset(&ctr, 0, sizeof(ctr));
#pragma omp for schedule(dynamic, 256)
    for (int64_t r = 0; r < (int64_t)n; ++r) {
      const uint8_t* rl = left + (size_t)r * L;
      const uint8_t* rr = right + (size_t)r * L;
      const uint32_t nl = mate_candidates(ix, *p, rl, L, keys.data(), 1, lc.data(), ctr);
      const uint32_t nr = mate_candidates(ix, *p, rr, L, keys.data(), 1, rc.data(), ctr);
      unsigned long long used_l = 0, used_r = 0;
      const uint32_t nj = for_each_joint(*p, lc.data(), nl, rc.data(), nr, L, [&](const Joint& j, uint32_t) {
        if (j.li >= 0) used_l |= 1ull << j.li;
        if (j.ri >= 0) used_r |= 1ull << j.ri;
      });
      uint32_t na = 0;
      ReadOut o;
      o.n_aln = &na; o.tid = o_tid.data(); o.score = o_score.data(); o.prob = o_prob.data(); o.pos = o_pos.data();
      o.mate_pos = o_mpos.data(); o.flags = o_flags.data(); o.flen = o_flen.data(); o.label = o_label.data();
      o.weight = o_weight.data();
      if (nj != 0 && nj <= cap) {
        for (uint32_t a = 0; a < nl; ++a)
          if (used_l >> a & 1) { sl[a] = dp_score_serial(ix, *p, rl, L, lc[a].ori_cov >> 31, lc[a].tid, lc[a].diag_c); ctr.candidates++; }
        for (uint32_t a = 0; a < nr; ++a)
          if (used_r >> a & 1) { sr[a] = dp_score_serial(ix, *p, rr, L, rc[a].ori_cov >> 31, rc[a].tid, rc[a].diag_c); ctr.candidates++; }
        assign_read(ix, *p, fld, useAux, burnedIn, lc.data(), nl, rc.data(), nr, sl.data(), sr.data(), L, sc.data(),
                    pi.data(), pt.data(), b1.data(), b2.data(), b3.data(), jh.data(), o, ctr);
      }
      if (n_aln) n_aln[r] = na;
    }
#pragma omp critical
    {
      tot[0] += ctr.lookups; tot[1] += ctr.postings; tot[2] += ctr.seeds; tot[3] += ctr.candidates;
      tot[4] += ctr.kept; tot[5] += ctr.label_entries; tot[6] += ctr.mapped;
    }
  }
  for (int i = 0; i < 7; ++i) counters7[i] = tot[i];
  return 0;
}

// the product's serial seed / chain form on one mate (tests/test_seed_paths_cpu.py): candidates in (tid, ori, diag_c)
// order, counters3 = {lookups, postings, seeds} of this mate
extern "C" uint32_t hmc_mate_candidates(uint32_t n_txps, uint32_t k, const uint64_t* tx_off, const uint8_t* codes,
                                        const void* table, uint64_t table_capacity, const void* postings, const Params* p,
                                        const uint8_t* read, uint32_t L, Cand* out /* [MAXCAND] */,
                                        unsigned long long* counters3) {
  IndexView ix;
  ix.n_txps = n_txps; ix.k = k; ix.mask = table_capacity - 1; ix.tx_off = tx_off; ix.codes = codes;
  ix.table = (const TableEntry*)table; ix.post = (const Posting*)postings;
  ix.packed = nullptr; ix.tx_has_n = nullptr;
  std::vector<uint64_t> keys(MAXSEEDS);
  Counters ctr;
  memset(&ctr, 0, sizeof(ctr));
  const uint32_t n = mate_candidates(ix, *p, read, L, keys.data(), 1, out, ctr);
  counters3[0] = ctr.lookups; counters3[1] = ctr.postings; counters3[2] = ctr.seeds;
  return n;
}

// the product's serial DP form on one reference (tests/test_dp_vs_edlib.py)
extern "C" int32_t hmc_dp_score(const uint64_t* tx_off, const uint8_t* codes, const Params* p, const uint8_t* read, uint32_t L,
                                uint32_t ori, uint32_t tid, int32_t diag_c) {
  IndexView ix;
  memset(&ix, 0, sizeof ix);
  ix.n_txps = tid + 1; ix.tx_off = tx_off; ix.codes = codes;
  return dp_score_serial(ix, *p, read, L, ori, tid, diag_c);
}
