// map_core.h -- Stage A per-read logic of the product (sm_90a device code; also compiles for
// the host so that tests can run the SAME code against the independent oracle without a GPU).
//
// MAPSPEC (DESIGN.md "Stage A"): seeds sampled every `stride` bases -> hash lookup of the
// canonical k-mer -> postings (transcript, offset) -> seeds keyed (tid, ori, diag, qpos) ->
// sorted -> chains by single linkage on the diagonal -> candidates filtered by coverage ->
// inward pairing (IU) or orphans -> banded affine glocal DP score per mate -> salmon's own
// updateRefMappings / filterAndCollectAlignments / auxiliary-probability / label arithmetic
// (include/salmon/internal/quant/SalmonMappingUtils.hpp:225-405, src/quant/SalmonQuantify.cpp:599-857).
// The mapping core replaces pufferfish's MemCollector / MemChainer / joinReadsAndFilter /
// PuffAligner (call sites src/quant/SalmonQuantify.cpp:1266-1288,1339-1341,1523), whose source
// is not in the reference tree.
#pragma once
#include <stdint.h>

#include "../../include/sb_detmath.h"

#ifndef __CUDACC__
#include <math.h>
#endif

namespace sbmap {

constexpr int MAXSEEDS = 2048;
constexpr int MAXCAND = 64;
constexpr int32_t NEG_SCORE = -(1 << 28);
constexpr int32_t INVALID_SCORE = (-2147483647 - 1);
constexpr uint64_t EMPTY_KEY = ~0ull;

struct Params {
  uint32_t k, stride, max_occs_per_hit, max_read_occ, max_frag_len, band, chain_gap, range_bins;
  int32_t ma, mp, go, ge, hard_filter, first_decoy;
  double consensus_frac, min_score_fraction, score_exp, min_aln_prob, decoy_threshold;
  double fld_mean, fld_sd;
  uint64_t num_pre_burnin, num_burnin;
  uint64_t seed;
  uint32_t mini_batch, reserved;
  double pre_merge_thresh, post_merge_thresh, orphan_thresh;   // join policy (see sb_map_params)
  int32_t allow_dovetail, allow_orphans;
  int32_t lib_type, reserved3;      // expected library format (SB_LIB_*)
};

struct TableEntry {
  uint64_t key;   // canonical k-mer, EMPTY_KEY if free
  uint32_t off;   // first posting
  uint32_t cnt;   // number of postings
};
struct Posting {
  uint32_t tid;
  uint32_t tpos_rc;   // bits 0..30: offset in the transcript; bit 31: the reference k-mer there is the
                      // reverse complement of the canonical k-mer (orientation without touching the sequence)
};
constexpr uint32_t PACK_GUARD_BASES = 512;   // guard bases in front of / behind the 2-bit packed reference

struct IndexView {
  uint32_t n_txps, k;
  uint64_t mask;             // table capacity - 1 (power of two)
  const uint64_t* tx_off;    // [n_txps+1] base offsets into codes
  const uint8_t* codes;      // one base per byte: 0..3, 4 = N
  const TableEntry* table;
  const Posting* post;       // ascending (tid, tpos) per k-mer
  const uint64_t* packed;    // 2-bit codes, base g at bits 2*((g+GUARD)&31) of word (g+GUARD)>>5 (N stored as 0)
  const uint8_t* tx_has_n;   // [n_txps] transcript contains a non-ACGT base (packed form unusable)
};

// FLD tables (log space), built on the host from the prior (FragmentLengthDistribution.cpp:22-78)
struct FldView {
  uint32_t max_val;
  const double* pmf_live;    // hist - totMass                      (:122-132)
  const double* pmf_cached;  // renormalised copy used after burn-in (:163-175)
  const double* cmf_cached;  // (:190-201)
  const double* cmf_quirk;   // LogCMFCache before burn-in (DistributionUtils.cpp:103-116)
};

struct Cand {
  uint32_t tid;
  int32_t diag_c;
  uint32_t ori_cov;  // bit 31 = orientation (1 = read maps reverse-complemented), low bits = coverage
};

struct Counters {
  unsigned long long lookups, postings, seeds, candidates, kept, label_entries, mapped;
  unsigned long long lib_mask_sum[4];   // fragments that showed ISF / ISR / SF / SR among their kept mappings
};

SB_HD uint64_t mix64(uint64_t x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
  return x;
}

SB_HD bool index_lookup(const IndexView& ix, uint64_t canon, uint32_t& off, uint32_t& cnt) {
  uint64_t h = mix64(canon) & ix.mask;
  for (;;) {
    const TableEntry e = ix.table[h];
    if (e.key == canon) { off = e.off; cnt = e.cnt; return true; }
    if (e.key == EMPTY_KEY) return false;
    h = (h + 1) & ix.mask;
  }
}

// seed key: tid(32) | ori(1) | diag + 2^21 (22) | qpos (9)
SB_HD uint64_t seed_key(uint32_t tid, uint32_t ori, int32_t diag, int32_t qpos) {
  return ((uint64_t)tid << 32) | ((uint64_t)ori << 31) | ((uint64_t)(uint32_t)(diag + (1 << 21)) << 9) |
         (uint64_t)(uint32_t)qpos;
}
SB_HD uint32_t key_tid(uint64_t k) { return (uint32_t)(k >> 32); }
SB_HD uint32_t key_ori(uint64_t k) { return (uint32_t)(k >> 31) & 1u; }
SB_HD int32_t key_diag(uint64_t k) { return (int32_t)((k >> 9) & 0x3fffffu) - (1 << 21); }
SB_HD int32_t key_qpos(uint64_t k) { return (int32_t)(k & 0x1ffu); }

// in-place heapsort of n u64 keys stored with a stride (interleaved per-thread scratch)
SB_HD void heapsort_u64(uint64_t* a, size_t stride, uint32_t n) {
  if (n < 2) return;
  for (uint32_t start = n / 2; start-- > 0;) {
    uint32_t root = start;
    const uint64_t v = a[(size_t)root * stride];
    for (;;) {
      uint32_t child = 2 * root + 1;
      if (child >= n) break;
      if (child + 1 < n && a[(size_t)child * stride] < a[(size_t)(child + 1) * stride]) ++child;
      if (v >= a[(size_t)child * stride]) break;
      a[(size_t)root * stride] = a[(size_t)child * stride];
      root = child;
    }
    a[(size_t)root * stride] = v;
  }
  for (uint32_t end = n - 1; end > 0; --end) {
    const uint64_t v = a[(size_t)end * stride];
    a[(size_t)end * stride] = a[0];
    uint32_t root = 0;
    for (;;) {
      uint32_t child = 2 * root + 1;
      if (child >= end) break;
      if (child + 1 < end && a[(size_t)child * stride] < a[(size_t)(child + 1) * stride]) ++child;
      if (v >= a[(size_t)child * stride]) break;
      a[(size_t)root * stride] = a[(size_t)child * stride];
      root = child;
    }
    a[(size_t)root * stride] = v;
  }
}

// Seeds + chains of one mate.  read: L byte codes.  keys: scratch for MAXSEEDS keys (strided).
// Returns the number of candidates written to out[] in (tid, ori, diag_c) order.
SB_HD uint32_t mate_candidates(const IndexView& ix, const Params& p, const uint8_t* read, uint32_t L,
                               uint64_t* keys, size_t kstride, Cand* out, Counters& ctr) {
  const uint32_t K = p.k;
  if (L < K) return 0;
  uint32_t ns = 0;
  for (uint32_t i = 0;; i += p.stride) {
    uint32_t pos_i = i;
    bool last = false;
    if (i > L - K) {
      if ((L - K) % p.stride == 0) break;
      pos_i = L - K;
      last = true;
    }
    uint64_t fw = 0, rc = 0;
    bool bad = false;
    for (uint32_t j = 0; j < K; ++j) {
      const uint8_t c = read[pos_i + j];
      if (c > 3) { bad = true; break; }
      fw = (fw << 2) | c;
      rc |= (uint64_t)(3 - c) << (2 * j);
    }
    if (!bad) {
      const uint64_t canon = fw < rc ? fw : rc;
      ctr.lookups++;
      uint32_t off, cnt;
      if (index_lookup(ix, canon, off, cnt) && cnt <= p.max_occs_per_hit) {
        const uint32_t read_rc = (fw < rc) ? 0u : 1u;   // the read k-mer is the reverse complement of the canonical one
        for (uint32_t q = 0; q < cnt && ns < (uint32_t)MAXSEEDS; ++q) {
          ctr.postings++;
          const Posting po = ix.post[off + q];
          const uint32_t tpos = po.tpos_rc & 0x7fffffffu;
          const uint32_t ori = read_rc ^ (po.tpos_rc >> 31);
          const int32_t qpos = ori ? (int32_t)(L - K - pos_i) : (int32_t)pos_i;
          keys[(size_t)ns * kstride] = seed_key(po.tid, ori, (int32_t)tpos - qpos, qpos);
          ++ns;
        }
      }
    }
    if (last) break;
  }
  ctr.seeds += ns;
  heapsort_u64(keys, kstride, ns);
  // chains -> candidates; coverage = bases of the read covered by the chain's seeds
  uint32_t nc = 0, best = 0;
  uint32_t i = 0;
  // pass 1: best coverage (candidates are re-derived in pass 2 to avoid storing all of them)
  for (int pass = 0; pass < 2; ++pass) {
    i = 0;
    nc = 0;
    uint32_t n_over = 0;
    while (i < ns) {
      const uint64_t k0 = keys[(size_t)i * kstride];
      uint64_t cover[4] = {0, 0, 0, 0};
      int32_t dmin = key_diag(k0), dmax = dmin, prev = dmin;
      uint32_t j = i;
      while (j < ns) {
        const uint64_t kj = keys[(size_t)j * kstride];
        if (key_tid(kj) != key_tid(k0) || key_ori(kj) != key_ori(k0)) break;
        const int32_t dj = key_diag(kj);
        if (j > i && dj - prev > (int32_t)p.chain_gap) break;
        prev = dj;
        dmax = dj;
        const int32_t q0 = key_qpos(kj);
        for (uint32_t b = 0; b < K; ++b) {
          const int32_t q = q0 + (int32_t)b;
          if (q >= 0 && q < 256) cover[q >> 6] |= 1ull << (q & 63);
        }
        ++j;
      }
      uint32_t cov = 0;
      for (int w = 0; w < 4; ++w) {
#if defined(__CUDA_ARCH__)
        cov += (uint32_t)__popcll(cover[w]);
#else
        cov += (uint32_t)__builtin_popcountll(cover[w]);
#endif
      }
      if (pass == 0) {
        if (cov > best) best = cov;
      } else if ((double)cov >= p.consensus_frac * (double)best) {
        if (nc < (uint32_t)MAXCAND) {
          out[nc].tid = key_tid(k0);
          out[nc].diag_c = dmin + (dmax - dmin) / 2;
          out[nc].ori_cov = (key_ori(k0) << 31) | cov;
          ++nc;
        } else {
          ++n_over;
        }
      }
      i = j;
    }
    if (pass == 1 && n_over) {
      // more than MAXCAND survivors: keep the MAXCAND best by (coverage desc, tid, ori, diag_c).
      // Rare; done by re-walking the chains and replacing the current worst entry.
      // (worst = smallest coverage, ties: largest (tid, ori, diag_c))
      i = 0;
      uint32_t seen = 0;
      while (i < ns) {
        const uint64_t k0 = keys[(size_t)i * kstride];
        uint64_t cover[4] = {0, 0, 0, 0};
        int32_t dmin = key_diag(k0), dmax = dmin, prev = dmin;
        uint32_t j = i;
        while (j < ns) {
          const uint64_t kj = keys[(size_t)j * kstride];
          if (key_tid(kj) != key_tid(k0) || key_ori(kj) != key_ori(k0)) break;
          const int32_t dj = key_diag(kj);
          if (j > i && dj - prev > (int32_t)p.chain_gap) break;
          prev = dj; dmax = dj;
          const int32_t q0 = key_qpos(kj);
          for (uint32_t b = 0; b < K; ++b) {
            const int32_t q = q0 + (int32_t)b;
            if (q >= 0 && q < 256) cover[q >> 6] |= 1ull << (q & 63);
          }
          ++j;
        }
        uint32_t cov = 0;
        for (int w = 0; w < 4; ++w) {
#if defined(__CUDA_ARCH__)
          cov += (uint32_t)__popcll(cover[w]);
#else
          cov += (uint32_t)__builtin_popcountll(cover[w]);
#endif
        }
        if ((double)cov >= p.consensus_frac * (double)best) {
          if (seen >= (uint32_t)MAXCAND) {
            // candidate beyond the first MAXCAND: replace the worst kept one if this is better
            uint32_t wi = 0;
            for (uint32_t c = 1; c < (uint32_t)MAXCAND; ++c) {
              const uint32_t cw = out[wi].ori_cov & 0x7fffffffu, cc = out[c].ori_cov & 0x7fffffffu;
              const bool worse = cc < cw || (cc == cw && (out[c].tid > out[wi].tid ||
                                 (out[c].tid == out[wi].tid && ((out[c].ori_cov >> 31) > (out[wi].ori_cov >> 31) ||
                                 ((out[c].ori_cov >> 31) == (out[wi].ori_cov >> 31) && out[c].diag_c > out[wi].diag_c)))));
              if (worse) wi = c;
            }
            const uint32_t cw = out[wi].ori_cov & 0x7fffffffu;
            const int32_t dc = dmin + (dmax - dmin) / 2;
            const bool better = cov > cw || (cov == cw && (key_tid(k0) < out[wi].tid ||
                                (key_tid(k0) == out[wi].tid && (key_ori(k0) < (out[wi].ori_cov >> 31) ||
                                (key_ori(k0) == (out[wi].ori_cov >> 31) && dc < out[wi].diag_c)))));
            if (better) {
              out[wi].tid = key_tid(k0);
              out[wi].diag_c = dc;
              out[wi].ori_cov = (key_ori(k0) << 31) | cov;
            }
          }
          ++seen;
        }
        i = j;
      }
      // restore (tid, ori, diag_c) order (insertion sort, MAXCAND entries)
      for (uint32_t a = 1; a < (uint32_t)MAXCAND; ++a) {
        const Cand v = out[a];
        uint32_t b = a;
        while (b > 0) {
          const Cand& u = out[b - 1];
          const bool gt = u.tid > v.tid || (u.tid == v.tid && ((u.ori_cov >> 31) > (v.ori_cov >> 31) ||
                          ((u.ori_cov >> 31) == (v.ori_cov >> 31) && u.diag_c > v.diag_c)));
          if (!gt) break;
          out[b] = out[b - 1];
          --b;
        }
        out[b] = v;
      }
    }
  }
  return nc;
}

// ---- joint hits (library type IU).  Enumerated in the oracle's order: left-major.
struct Joint {
  uint32_t tid;
  int32_t li, ri;       // candidate indices, -1 if absent
  int32_t frag_len;
  uint32_t status;      // 0 paired, 1 left orphan, 2 right orphan
};

// Join policy (MAPSPEC step 4; the knobs salmon sets on pufferfish's MappingConstraintPolicy,
// SalmonMappingUtils.hpp:208-220, semantics from the option texts ProgramOptionsGenerator.cpp:111-137,198-201):
//   (1) pre-merge: per mate and transcript, a chain with coverage < pre_merge_thresh x (best coverage of that mate on
//       that transcript) takes no part;
//   (2) a pair = one chain of each mate on the same transcript, opposite orientations, the forward mate not behind the
//       reverse mate (unless allow_dovetail), 0 < fragment length <= max_frag_len; its score = sum of the coverages;
//   (3) post-merge: per transcript, pairs with score < post_merge_thresh x (best pair score on it) are dropped;
//   (4) consensus: pairs with score < consensus_frac x (best pair score of the read) are dropped;
//   (5) no pair at all -> orphans, if allow_orphans: chains with coverage >= orphan_thresh x (best chain coverage of
//       the read), lefts before rights (SalmonQuantify.cpp:1407-1420).
// Candidate lists are sorted by (transcript, orientation, diagonal), so the chains of a transcript are one run in each.
SB_HD uint32_t sbm_maxu(uint32_t a, uint32_t b) { return a > b ? a : b; }
// Is a joint hit compatible with the expected library format?  (SalmonQuantify.cpp:1467-1517 for paired-end libraries,
// :2141-2147 single-end; = salmon::utils::isCompatible, src/util/SalmonUtils.cpp:138-298.)  status: 0 pair, 1 left
// orphan, 2 right orphan; first_fw: the (left, or for a right orphan the right) mate maps forward.
SB_HD bool lib_compatible(int32_t lib_type, uint32_t status, bool left_fw, bool right_fw) {
  switch (lib_type) {
    case 0: return status != 0 || left_fw != right_fw;                    // IU: orphans always, pairs on opposite strands
    case 1: return status == 0 ? (left_fw && !right_fw) : (status == 1 ? left_fw : !right_fw);   // ISF (strandedness SA)
    case 2: return status == 0 ? (!left_fw && right_fw) : (status == 1 ? !left_fw : right_fw);   // ISR (AS)
    case 3: return true;                                                  // U
    case 4: return left_fw;                                               // SF
    case 5: return !left_fw;                                              // SR
    default: return true;
  }
}
SB_HD bool pair_geometry(const Params& p, const Cand& l, const Cand& r, uint32_t L, int32_t& fl) {
  if (l.tid != r.tid || (l.ori_cov >> 31) == (r.ori_cov >> 31)) return false;
  const Cand& fw = ((l.ori_cov >> 31) == 0) ? l : r;      // the mate that maps forward
  const Cand& rv = ((l.ori_cov >> 31) == 0) ? r : l;
  int32_t start = fw.diag_c, end = rv.diag_c + (int32_t)L;
  if (rv.diag_c < fw.diag_c) {                              // the reverse mate starts before the forward mate: dovetail
    if (!p.allow_dovetail) return false;
    start = rv.diag_c; end = fw.diag_c + (int32_t)L;
  }
  fl = end - start;
  return fl > 0 && fl <= (int32_t)p.max_frag_len;
}
SB_HD uint32_t cand_cov(const Cand& c) { return c.ori_cov & 0x7fffffffu; }
// chain c of `list` passes the pre-merge filter (1)
SB_HD bool pre_merge_keep(const Params& p, const Cand* list, uint32_t n, uint32_t c) {
  uint32_t best = 0;
  for (uint32_t q = c; q < n && list[q].tid == list[c].tid; ++q) best = sbm_maxu(best, cand_cov(list[q]));
  for (uint32_t q = c; q-- > 0 && list[q].tid == list[c].tid;) best = sbm_maxu(best, cand_cov(list[q]));
  return (double)cand_cov(list[c]) >= p.pre_merge_thresh * (double)best;
}

// visits joint hits in order; F(const Joint&, index) ; returns the number of joint hits
template <class F>
SB_HD uint32_t for_each_joint(const Params& p, const Cand* lc, uint32_t nl, const Cand* rc, uint32_t nr,
                              uint32_t L, F&& f) {
  // pre-merge masks
  unsigned long long keep_l = 0, keep_r = 0;
  for (uint32_t a = 0; a < nl; ++a) if (pre_merge_keep(p, lc, nl, a)) keep_l |= 1ull << a;
  for (uint32_t b = 0; b < nr; ++b) if (pre_merge_keep(p, rc, nr, b)) keep_r |= 1ull << b;
  // best pair score of the read (4)
  uint32_t best_all = 0;
  for (uint32_t a = 0; a < nl; ++a) {
    if (!(keep_l >> a & 1)) continue;
    for (uint32_t b = 0; b < nr; ++b) {
      int32_t fl;
      if ((keep_r >> b & 1) && pair_geometry(p, lc[a], rc[b], L, fl)) best_all = sbm_maxu(best_all, cand_cov(lc[a]) + cand_cov(rc[b]));
    }
  }
  uint32_t nj = 0;
  if (best_all > 0) {
    uint32_t a0 = 0;
    while (a0 < nl) {                       // runs of one transcript in the left list
      uint32_t a1 = a0;
      while (a1 < nl && lc[a1].tid == lc[a0].tid) ++a1;
      uint32_t best_t = 0;                  // best pair score on this transcript (3)
      for (uint32_t a = a0; a < a1; ++a) {
        if (!(keep_l >> a & 1)) continue;
        for (uint32_t b = 0; b < nr; ++b) {
          int32_t fl;
          if ((keep_r >> b & 1) && pair_geometry(p, lc[a], rc[b], L, fl)) best_t = sbm_maxu(best_t, cand_cov(lc[a]) + cand_cov(rc[b]));
        }
      }
      if (best_t > 0)
        for (uint32_t a = a0; a < a1; ++a) {
          if (!(keep_l >> a & 1)) continue;
          for (uint32_t b = 0; b < nr; ++b) {
            int32_t fl;
            if (!(keep_r >> b & 1) || !pair_geometry(p, lc[a], rc[b], L, fl)) continue;
            const double sc = (double)(cand_cov(lc[a]) + cand_cov(rc[b]));
            if (sc < p.post_merge_thresh * (double)best_t || sc < p.consensus_frac * (double)best_all) continue;
            Joint j;
            j.tid = lc[a].tid; j.li = (int32_t)a; j.ri = (int32_t)b; j.frag_len = fl; j.status = 0;
            f(j, nj);
            ++nj;
          }
        }
      a0 = a1;
    }
  }
  if (nj == 0 && p.allow_orphans) {
    uint32_t best_c = 0;
    for (uint32_t a = 0; a < nl; ++a) if (keep_l >> a & 1) best_c = sbm_maxu(best_c, cand_cov(lc[a]));
    for (uint32_t b = 0; b < nr; ++b) if (keep_r >> b & 1) best_c = sbm_maxu(best_c, cand_cov(rc[b]));
    const double thr = (p.lib_type >= 3 ? 0.0 : p.orphan_thresh) * (double)best_c;   // single-end: consensus filter only (joinReadsAndFilterSingle)
    for (uint32_t a = 0; a < nl; ++a) {
      if (!(keep_l >> a & 1) || (double)cand_cov(lc[a]) < thr) continue;
      Joint j; j.tid = lc[a].tid; j.li = (int32_t)a; j.ri = -1; j.frag_len = 0; j.status = 1;
      f(j, nj); ++nj;
    }
    for (uint32_t b = 0; b < nr; ++b) {
      if (!(keep_r >> b & 1) || (double)cand_cov(rc[b]) < thr) continue;
      Joint j; j.tid = rc[b].tid; j.li = -1; j.ri = (int32_t)b; j.frag_len = 0; j.status = 2;
      f(j, nj); ++nj;
    }
  }
  return nj;
}

// ---- banded affine glocal DP, serial form (host tests; device fallback).  The warp form in
// map.cu computes the same recurrences with lanes = band cells.
SB_HD int32_t dp_score_serial(const IndexView& ix, const Params& p, const uint8_t* read, uint32_t L,
                              uint32_t ori, uint32_t tid, int32_t diag_c) {
  const int32_t B = (int32_t)p.band, W = 2 * B + 1;
  const int64_t tlen = (int64_t)(ix.tx_off[tid + 1] - ix.tx_off[tid]);
  const uint8_t* ref = ix.codes + ix.tx_off[tid];
  int32_t H[64], E[64];
  for (int32_t j = 0; j < W; ++j) { H[j] = 0; E[j] = NEG_SCORE; }
  for (uint32_t i = 0; i < L; ++i) {
    const uint8_t c = ori ? read[L - 1 - i] : read[i];
    const uint8_t rb = ori ? (uint8_t)(c > 3 ? 4 : 3 - c) : c;
    int32_t Fprev = NEG_SCORE, Hleft = NEG_SCORE;
    int32_t Hn_next_diag;  // H[j+1] of the previous row must be read before H[j+1] is overwritten
    for (int32_t j = 0; j < W; ++j) {
      const int64_t r = (int64_t)diag_c + (int64_t)i + (j - B);
      const int32_t Hup = (j + 1 < W) ? H[j + 1] : NEG_SCORE;   // previous row, lane j+1 (not yet overwritten)
      const int32_t Eup = (j + 1 < W) ? E[j + 1] : NEG_SCORE;
      int32_t h = NEG_SCORE, e = NEG_SCORE, f = NEG_SCORE;
      if (r >= 0 && r < tlen) {
        const int32_t s = (rb < 4 && rb == ref[r]) ? p.ma : p.mp;
        const int32_t m = H[j] + s;
        if (j + 1 < W) { const int32_t a = Hup - p.go - p.ge, b = Eup - p.ge; e = a > b ? a : b; }
        if (j > 0) { const int32_t a = Hleft - p.go - p.ge, b = Fprev - p.ge; f = a > b ? a : b; }
        h = m;
        if (e > h) h = e;
        if (f > h) h = f;
        if (h < NEG_SCORE) h = NEG_SCORE;
        if (e < NEG_SCORE) e = NEG_SCORE;
        if (f < NEG_SCORE) f = NEG_SCORE;
      }
      (void)Hn_next_diag;
      H[j] = h; E[j] = e;     // lane j of the previous row is no longer needed (lane j-1 used H[j] already)
      Hleft = h; Fprev = f;
    }
  }
  int32_t best = NEG_SCORE;
  for (int32_t j = 0; j < W; ++j) if (H[j] > best) best = H[j];
  return best;
}

// ---- salmon-owned arithmetic on the log scale (deterministic exp/log, sb_detmath.h)
SB_HD double log0() { return sbm_u2d(0x7ff0000000000000ull); }   // LOG_0 = HUGE_VAL (SalmonMath.hpp:40)
SB_HD double dabs(double x) { return x < 0 ? -x : x; }
SB_HD double log_add(double x, double y) {                       // SalmonMath.hpp:54-66
  if (dabs(x) == log0()) return y;
  if (dabs(y) == log0()) return x;
  if (y > x) { const double t = x; x = y; y = t; }
  return x + sbm_det_log(1 + sbm_det_exp(y - x));
}
SB_HD double tabv(const double* t, uint32_t max_val, uint64_t len) { return t[len > max_val ? max_val : len]; }

// ---- online phase (processMiniBatch's state updates, src/quant/SalmonQuantify.cpp:599-623, 749-757, 783-792,
// 859-983) with BATCHED SEMANTICS: the state (masses, FLD) is frozen while a batch is processed; the batch's
// contributions are accumulated as integers -- multiples of 2^-40 of the batch's largest forgetting mass -- so
// the sums do not depend on the order in which threads add them, and folded into the state afterwards.
struct OnlineView {
  const double* mass;        // [M] log mass (+inf = none), Transcript::mass_
  const double* prior;       // [M] log(0.005 * length), Transcript::priorMass_
  const double* log_eff;     // [M] cached log effective length (used once burned in)
  unsigned long long* mass_acc;   // [M]
  unsigned long long* fld_acc;    // [max_frag_len + 1]
  unsigned int* batch_min;        // smallest fragment length added to the FLD in this batch
  const double* fm_rel;      // [timesteps of the batch] log forgetting mass minus the batch's largest
  const unsigned long long* tap_q;   // [timesteps * 5] FLD kernel taps (binomial(4, 1/2)) x forgetting mass, quantised
  uint32_t mini_batch, max_frag_len;
  uint64_t frag_base;        // global index of the batch's first fragment (RNG stream)
  uint64_t seed;
};
constexpr double MASS_SCALE = 1099511627776.0;   // 2^40

// Philox-4x32-10 (Salmon, Moraes, Dror, Shaw, SC'11): r < exp(logProb) of the stochastic FLD update (:974-983)
SB_HD uint32_t philox_first(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
  for (int i = 0; i < 10; ++i) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n1 = (uint32_t)p1, n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1, n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return c0;
}
SB_HD void acc_add(unsigned long long* p, unsigned long long v) {
#if defined(__CUDA_ARCH__)
  atomicAdd(p, v);
#else
  *p += v;
#endif
}
SB_HD void acc_min(unsigned int* p, unsigned int v) {
#if defined(__CUDA_ARCH__)
  atomicMin(p, v);
#else
  if (v < *p) *p = v;
#endif
}
SB_HD long long quant40(double x) {
#if defined(__CUDA_ARCH__)
  return __double2ll_rn(SB_MUL(x, MASS_SCALE));
#else
  return llrint(x * MASS_SCALE);
#endif
}
// QuasiAlignment::fragLengthPedantic for an inward pair: span of the outer ends clamped to the transcript
SB_HD int32_t pedantic_flen(int fwd, int32_t pos, int32_t mpos, int32_t L, int32_t refLen) {
  int32_t p1 = fwd ? pos : mpos; p1 = p1 < 0 ? 0 : p1; p1 = p1 > refLen ? refLen : p1;
  int32_t p2 = fwd ? mpos + L : pos + L; p2 = p2 < 0 ? 0 : p2; p2 = p2 > refLen ? refLen : p2;
  return (p1 > p2) ? p1 - p2 : p2 - p1;
}

// Per-read output of the assignment step.  cap = max_read_occ entries per read.
struct ReadOut {
  uint32_t* n_aln;       // [1]
  uint32_t* tid;         // [cap]
  int32_t* score;        // [cap]
  double* prob;          // [cap]
  int32_t* pos;          // [cap]
  int32_t* mate_pos;     // [cap]
  uint8_t* flags;        // [cap]  bit0 fwd, bit1 mate fwd, bits 2-3 mate status
  int32_t* flen;         // [cap]
  uint32_t* label;       // [2*cap] transcripts then range bins
  double* weight;        // [cap]
};

// updateRefMappings + filterAndCollectAlignments + auxiliary probabilities + label, for one read.
// score_l / score_r: DP score per left / right candidate.  perm_* scratch: >= nj entries each.
SB_HD void assign_read(const IndexView& ix, const Params& p, const FldView& fld, bool useAux, bool burnedIn,
                       const Cand* lc, uint32_t nl, const Cand* rcd, uint32_t nr, const int32_t* score_l,
                       const int32_t* score_r, uint32_t L, int32_t* sc, int32_t* perm_idx, int32_t* perm_tid,
                       int32_t* bs_tid, int32_t* bs_score, int32_t* bs_idx, Joint* jh, const ReadOut& o,
                       Counters& ctr, const OnlineView* on = nullptr, uint32_t read_in_batch = 0,
                       double* lpbuf = nullptr /* >= cap doubles */) {
  const double LOG_EPSILON = -24.006680182952184;   // log(0.375e-10), SalmonMath.hpp:44-45 (libm and sbm_det_log agree)
  const uint32_t cap = p.max_read_occ;
  *o.n_aln = 0;
  uint32_t nj = 0;
  const uint32_t total = for_each_joint(p, lc, nl, rcd, nr, L, [&](const Joint& j, uint32_t k) {
    if (k < cap) jh[k] = j;
  });
  nj = total;
  if (nj == 0 || nj > cap) return;
  // ---- SalmonMappingUtils.hpp:225-281
  int32_t bestScore = INVALID_SCORE, bestDecoyScore = INVALID_SCORE;
  uint32_t nperm = 0, nbs = 0;
  for (uint32_t h = 0; h < nj; ++h) {
    int32_t tot = 0, maxPossible = 0;
    bool bad = false;
    if (jh[h].li >= 0) { const int32_t s = score_l[jh[h].li]; if (s <= NEG_SCORE) bad = true; tot += s; maxPossible += p.ma * (int32_t)L; }
    if (jh[h].ri >= 0) { const int32_t s = score_r[jh[h].ri]; if (s <= NEG_SCORE) bad = true; tot += s; maxPossible += p.ma * (int32_t)L; }
    const int32_t hitScore = (!bad && (double)tot >= p.min_score_fraction * (double)maxPossible) ? tot : INVALID_SCORE;
    sc[h] = hitScore;
    {   // mappings incompatible with the library format are ignored (ignoreIncompat, SalmonQuantify.cpp:1519-1521)
      const bool lfw = jh[h].li >= 0 && (lc[jh[h].li].ori_cov >> 31) == 0;
      const bool rfw = jh[h].ri >= 0 && (rcd[jh[h].ri].ori_cov >> 31) == 0;
      if (!lib_compatible(p.lib_type, jh[h].status, lfw, rfw)) { sc[h] = INVALID_SCORE; continue; }
    }
    const bool isDecoy = (int32_t)jh[h].tid >= p.first_decoy;
    const double decoyCutoff = (double)(int32_t)(p.decoy_threshold * (double)bestDecoyScore);
    if (isDecoy) { if (hitScore > bestDecoyScore) bestDecoyScore = hitScore; continue; }
    if ((double)hitScore < decoyCutoff || hitScore == INVALID_SCORE) continue;
    uint32_t q = 0;
    while (q < nbs && bs_tid[q] != (int32_t)jh[h].tid) ++q;
    if (q == nbs) { bs_tid[nbs] = (int32_t)jh[h].tid; bs_score[nbs] = hitScore; bs_idx[nbs] = (int32_t)h; ++nbs; }
    else if (hitScore >= bs_score[q]) { bs_score[q] = hitScore; sc[bs_idx[q]] = INVALID_SCORE; bs_idx[q] = (int32_t)h; }  // isCompat is always true for IU
    else { sc[h] = INVALID_SCORE; }
    if (hitScore > bestScore) bestScore = hitScore;
    perm_idx[nperm] = (int32_t)h; perm_tid[nperm] = (int32_t)jh[h].tid; ++nperm;
  }
  // ---- :283-405
  if (bestDecoyScore == INVALID_SCORE) bestDecoyScore = INVALID_SCORE + 1;
  const int32_t decoyThreshold = (int32_t)(p.decoy_threshold * (double)bestDecoyScore);
  const int32_t scoreThreshold = p.hard_filter ? bestScore : decoyThreshold;
  uint32_t nk = 0;
  for (uint32_t q = 0; q < nperm; ++q)
    if (sc[perm_idx[q]] >= scoreThreshold) { perm_idx[nk] = perm_idx[q]; perm_tid[nk] = perm_tid[q]; ++nk; }
  for (uint32_t a = 1; a < nk; ++a) {   // sort by transcript id (unique after the dedup above)
    const int32_t vi = perm_idx[a], vt = perm_tid[a];
    uint32_t b = a;
    while (b > 0 && perm_tid[b - 1] > vt) { perm_idx[b] = perm_idx[b - 1]; perm_tid[b] = perm_tid[b - 1]; --b; }
    perm_idx[b] = vi; perm_tid[b] = vt;
  }
  uint32_t na = 0;
  for (uint32_t q = 0; q < nk; ++q) {
    const Joint& j = jh[perm_idx[q]];
    const double v = (double)bestScore - (double)sc[perm_idx[q]];
    const double estAlnProb = p.hard_filter ? -1.0 : sbm_det_exp(-p.score_exp * v);
    if (!p.hard_filter && estAlnProb < p.min_aln_prob) continue;
    const Cand& first = (j.status == 2) ? rcd[j.ri] : lc[j.li];
    o.tid[na] = j.tid;
    o.score[na] = sc[perm_idx[q]];
    o.prob[na] = estAlnProb;
    o.pos[na] = first.diag_c;
    o.mate_pos[na] = (j.status == 0) ? rcd[j.ri].diag_c : 0;
    uint8_t fl = (uint8_t)(((first.ori_cov >> 31) == 0) ? 1 : 0);
    if (j.status == 0 && (rcd[j.ri].ori_cov >> 31) == 0) fl |= 2;
    fl |= (uint8_t)(j.status << 2);
    o.flags[na] = fl;
    o.flen[na] = j.frag_len;
    ++na;
  }
  *o.n_aln = na;
  ctr.kept += na;
  if (na == 0) return;
  ctr.mapped++;
  {   // observed formats of this fragment (libTypeCountsPerFrag, SalmonQuantify.cpp:765,1000-1002): bit 0 ISF, 1 ISR, 2 SF, 3 SR
    uint32_t m = 0;
    for (uint32_t a = 0; a < na; ++a) {
      const uint32_t st = (o.flags[a] >> 2) & 3;
      const bool fw = (o.flags[a] & 1) != 0;
      m |= st == 0 ? (fw ? 1u : 2u) : (fw ? 4u : 8u);
    }
    ctr.lib_mask_sum[0] += m & 1u; ctr.lib_mask_sum[1] += (m >> 1) & 1u; ctr.lib_mask_sum[2] += (m >> 2) & 1u; ctr.lib_mask_sum[3] += (m >> 3) & 1u;
  }
  ctr.label_entries += na;
  // ---- SalmonQuantify.cpp:599-857 (state frozen per batch); aux kept in o.weight until normalised
  double auxDenom = log0(), sumLp = log0();
  for (uint32_t a = 0; a < na; ++a) {
    const uint32_t tid = o.tid[a];
    const int32_t refLen = (int32_t)(ix.tx_off[tid + 1] - ix.tx_off[tid]);
    const double refLength = refLen > 0 ? (double)refLen : 1.0;
    const uint32_t status = (o.flags[a] >> 2) & 3;
    const int fwd = o.flags[a] & 1, mateFwd = (o.flags[a] >> 1) & 1;
    const double coverage = o.prob[a];
    const double logFragCov = (coverage > 0) ? sbm_det_log(coverage) : 0.0;
    int32_t flen = o.flen[a];
    if (status == 0 && fwd != mateFwd) {
      const int32_t pos = o.pos[a], mpos = o.mate_pos[a];
      int32_t p1 = fwd ? pos : mpos; p1 = p1 < 0 ? 0 : p1; p1 = p1 > refLen ? refLen : p1;
      int32_t p2 = fwd ? mpos + (int32_t)L : pos + (int32_t)L; p2 = p2 < 0 ? 0 : p2; p2 = p2 > refLen ? refLen : p2;
      flen = (p1 > p2) ? p1 - p2 : p2 - p1;
    }
    double logFragProb = 0.0;
    if (status != 0) {
      const int32_t pos = o.pos[a];
      int32_t maxFragLen;
      if (fwd) { int32_t p1 = pos < 0 ? 0 : pos; p1 = p1 > refLen ? refLen : p1; maxFragLen = refLen - p1; }
      else { int32_t p1 = pos + (int32_t)L; p1 = p1 < 0 ? 0 : p1; p1 = p1 > refLen ? refLen : p1; maxFragLen = p1; }
      const double* cm = burnedIn ? fld.cmf_cached : fld.cmf_quirk;
      const double refLengthCM = tabv(cm, fld.max_val, (uint64_t)refLen);
      const double maxLenProb = tabv(cm, fld.max_val, (uint64_t)maxFragLen);
      logFragProb = (refLengthCM != log0()) ? (maxLenProb - refLengthCM) : LOG_EPSILON;
    }
    if (flen > 0 && (burnedIn || useAux)) {
      const uint64_t fl = (uint64_t)flen;
      if (burnedIn) {
        const double lenProb = tabv(fld.pmf_cached, fld.max_val, fl);
        const double refLengthCM = tabv(fld.cmf_cached, fld.max_val, fl);
        const bool computeMass = ((double)fl < refLength) && (refLengthCM != log0());
        logFragProb = computeMass ? (lenProb - refLengthCM) : LOG_EPSILON;
      } else {
        logFragProb = tabv(fld.pmf_live, fld.max_val, fl);
      }
    }
    const double aux = logFragProb + logFragCov + 0.0;
    o.weight[a] = aux;
    auxDenom = log_add(auxDenom, aux);
    if (on) {   // aln.logProb = transcriptLogCount + auxProb + startPosProb  (:607-623, 749-757, 785)
      const double logRefLength = burnedIn ? on->log_eff[tid] : sbm_det_log((double)refLen);
      double startPosProb = -logRefLength;
      if (status == 0) startPosProb = ((double)flen <= refLength) ? -sbm_det_log(refLength - (double)flen + 1) : LOG_EPSILON;
      lpbuf[a] = log_add(on->prior[tid], on->mass[tid]) + aux + startPosProb;
      sumLp = log_add(sumLp, lpbuf[a]);
    }
  }
  for (uint32_t a = 0; a < na; ++a) {
    o.weight[a] = sbm_det_exp(o.weight[a] - auxDenom);
    o.label[a] = o.tid[a];
  }
  if (p.range_bins > 0) {
    const int32_t rangeCount = (int32_t)sqrt((double)na) + (int32_t)p.range_bins;
    for (uint32_t a = 0; a < na; ++a) o.label[na + a] = (uint32_t)(int32_t)(o.weight[a] * rangeCount);
  }
  if (on) {   // :859-983: normalise, add mass (x forgetting mass), stochastic FLD update
    const uint32_t step = read_in_batch / on->mini_batch;
    const double fm = on->fm_rel[step];
    const uint64_t g = on->frag_base + read_in_batch;
    for (uint32_t a = 0; a < na; ++a) {
      const double nlp = lpbuf[a] - sumLp;
      acc_add(on->mass_acc + o.tid[a], (unsigned long long)quant40(sbm_det_exp(fm + nlp)));
      if (!burnedIn) {
        const uint32_t status = (o.flags[a] >> 2) & 3;
        const int fwd = o.flags[a] & 1, mateFwd = (o.flags[a] >> 1) & 1;
        if (status != 0 || fwd == mateFwd) continue;          // fragLengthPedantic is 0 for anything but an inward pair
        const uint32_t x = philox_first((uint32_t)g, (uint32_t)(g >> 32), a, 3u, (uint32_t)on->seed, (uint32_t)(on->seed >> 32));
        const double u = (double)x * (1.0 / 4294967296.0);
        if (!(u < sbm_det_exp(nlp))) continue;
        const uint32_t tid = o.tid[a];
        const int32_t refLen = (int32_t)(ix.tx_off[tid + 1] - ix.tx_off[tid]);
        const int32_t fped = pedantic_flen(fwd, o.pos[a], o.mate_pos[a], (int32_t)L, refLen);
        if (fped <= 0) continue;
        uint32_t len = (uint32_t)fped;                         // FragmentLengthDistribution::addVal (:84-106)
        if (len > on->max_frag_len) len = on->max_frag_len;
        acc_min(on->batch_min, len);
        int64_t off = (int64_t)len - 2;
        for (int i = 0; i < 5; ++i, ++off)
          if (off > 0 && off <= (int64_t)on->max_frag_len) acc_add(on->fld_acc + off, on->tap_q[step * 5 + i]);
      }
    }
  }
}

}  // namespace sbmap
