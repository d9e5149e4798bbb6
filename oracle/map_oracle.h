/*
 * oracle/map_oracle.h -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU statement of Stage A (SURVEY.md section 8 rows a1-a8): per-read mapping, scoring,
 * alignment filtering, auxiliary probabilities, equivalence-class labels and aggregation.
 *
 * PARITY UNPINNED for the mapping core: rows a2-a4 live in COMBINE-lab/pufferfish @ ace68c1c
 * (MemCollector / MemChainer / joinReadsAndFilter / PuffAligner / ksw2pp), which is NOT in
 * the salmon source tree and has no tests or golden vectors in the salmon tree (SURVEY.md 8c).  The
 * seed -> chain -> join -> banded-affine-DP algorithm below is this project's own, documented
 * in DESIGN.md ("Stage A, MAPSPEC"); it follows the call sites and option semantics salmon
 * shows (initMapperSettings, include/salmon/internal/quant/SalmonMappingUtils.hpp:153-223;
 * src/cli/ProgramOptionsGenerator.cpp:85-289) but cannot be checked against pufferfish.
 *
 * The salmon-OWNED arithmetic is restated from the tree and cites file:line:
 *   updateRefMappings            SalmonMappingUtils.hpp:225-281
 *   filterAndCollectAlignments   SalmonMappingUtils.hpp:283-405
 *   processMiniBatch (aux probs, labels, range factorisation)  src/quant/SalmonQuantify.cpp:599-857
 *   FragmentLengthDistribution   src/model/FragmentLengthDistribution.cpp:22-175
 *   LogCMFCache                  src/util/DistributionUtils.cpp:100-172
 *   logAdd                       include/salmon/internal/util/SalmonMath.hpp:54-66
 *   EquivalenceClassBuilder      include/salmon/internal/quant/EquivalenceClassBuilder.hpp:165-181,237-250
 */
#ifndef SB_MAP_ORACLE_H
#define SB_MAP_ORACLE_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct orc_map_params {
  uint32_t k;                 /* 31 */
  uint32_t stride;            /* seed sampling stride along the read */
  uint32_t max_occs_per_hit;  /* maxOccsPerHit 1000 */
  uint32_t max_read_occ;      /* maxReadOcc 200 */
  uint32_t max_frag_len;      /* fragLenDistMax 1000 */
  uint32_t band;              /* bandwidth 15 */
  uint32_t chain_gap;         /* max diagonal gap inside one chain (8) */
  uint32_t range_bins;        /* rangeFactorizationBins 4 */
  int32_t ma, mp, go, ge;     /* 2, -4, 6, 2 */
  int32_t hard_filter;        /* hardFilter */
  int32_t first_decoy;        /* firstDecoyIndex (>= n_txps: no decoys) */
  double consensus_frac;      /* 1 - consensusSlack = 0.65 */
  double min_score_fraction;  /* 0.65 */
  double score_exp;           /* 1.0 */
  double min_aln_prob;        /* 1e-5 */
  double decoy_threshold;     /* 1.0 */
  double fld_mean, fld_sd;    /* 250, 25 */
  uint64_t num_pre_burnin;    /* 5000 */
  uint64_t num_burnin;        /* 5000000 */
  /* join policy as salmon configures pufferfish's MappingConstraintPolicy (SalmonMappingUtils.hpp:208-220; option
   * texts ProgramOptionsGenerator.cpp:111-137,198-201; defaults SalmonDefaults.hpp:28-30,46) */
  double pre_merge_thresh;    /* 0.75 */
  double post_merge_thresh;   /* 0.9 */
  double orphan_thresh;       /* 0.95 */
  int32_t allow_dovetail;     /* 0 */
  int32_t allow_orphans;      /* 1 */
  int32_t lib_type;           /* expected library format: 0 IU, 1 ISF, 2 ISR (paired-end, inward); 3 U, 4 SF, 5 SR (single-end) */
  int32_t reserved3;
} orc_map_params;

/* per-dataset counters for the roofline accounting of SURVEY.md section 8d */
typedef struct orc_map_counters {
  uint64_t lookups;      /* L: k-mer lookups issued */
  uint64_t postings;     /* P: postings read */
  uint64_t seeds;        /* seeds kept */
  uint64_t candidates;   /* A: mate alignments scored (DP invocations) */
  uint64_t kept;         /* K: alignments kept after filtering */
  uint64_t label_entries;/* sum of label sizes (transcript part) */
  uint64_t mapped;       /* fragments with >= 1 kept alignment */
} orc_map_counters;

typedef struct orc_index orc_index;

/* codes: one base per byte, 0..3 = A,C,G,T, 4 = N; seq_off[n+1] base offsets */
orc_index* orc_index_build(uint32_t n_txps, const uint64_t* seq_off, const uint8_t* codes, uint32_t k);
void orc_index_free(orc_index*);
uint64_t orc_index_n_kmers(const orc_index*);

/* Map n fixed-length pairs.  cap = max_read_occ.  Outputs per read r (arrays sized n*cap
 * unless noted): kept alignments in transcript order.  frag_counter = number of fragments
 * assigned before this batch (selects the pre-burn-in / burn-in regime for the whole batch). */
int orc_map_reads(const orc_index* idx, const orc_map_params* p, const uint8_t* left,
                  const uint8_t* right, uint32_t n, uint32_t read_len, uint64_t frag_counter,
                  uint32_t* n_aln /*[n]*/, uint32_t* aln_tid, int32_t* aln_score, double* aln_prob,
                  int32_t* aln_pos, int32_t* aln_mate_pos, uint8_t* aln_flags, int32_t* aln_flen,
                  uint32_t* label /*[n*2*cap]: tids then range bins*/, double* weight /*[n*cap]*/,
                  orc_map_counters* ctr);

/* EquivalenceClassBuilder: addGroup per fragment in order, finish() (normalise weights).
 * Classes are emitted sorted by label (lexicographic) -- a canonical order for comparison.
 * Returns the number of classes; out arrays must hold n entries (classes) / sum of n_aln
 * (labels, weights).  out_label_len[c] = full label length (2x transcripts when binned). */
uint64_t orc_eq_aggregate(uint32_t n, uint32_t cap, int binned, const uint32_t* n_aln,
                          const uint32_t* label, const double* weight, uint64_t* out_off,
                          uint32_t* out_ntx, uint32_t* out_label, double* out_weight,
                          uint64_t* out_count);

/* FLD tables (log pmf, log cmf over 0..max_val) as the prior N(mean, sd) gives them. */
void orc_fld_tables(double mean, double sd, uint32_t max_val, double* log_pmf, double* log_cmf);

/* ---- online phase with batched semantics (see map_oracle.c): masses, FLD, burn-in, normalizeAlphas ---- */
typedef struct orc_online orc_online;
orc_online* orc_online_create(const orc_index* idx, const orc_map_params* p, uint64_t seed, uint32_t mini_batch);
void orc_online_free(orc_online*);
/* like orc_map_reads, from the state's FLD / regime; then folds the batch into the state */
int orc_online_batch(orc_online* on, const uint8_t* left, const uint8_t* right, uint32_t n, uint32_t read_len,
                     uint32_t* n_aln, uint32_t* aln_tid, int32_t* aln_score, double* aln_prob, int32_t* aln_pos,
                     int32_t* aln_mate_pos, uint8_t* aln_flags, int32_t* aln_flen, uint32_t* label, double* weight,
                     orc_map_counters* ctr);
/* mass_out[M] (log, +inf = none), hist_out[max_frag_len+1] (log), log_eff_out[M],
 * scalars[6] = {assigned, frags_seen, timestep, burned_in, min_val, bits of log totMass} */
void orc_online_state(const orc_online* on, double* mass_out, double* hist_out, double* log_eff_out, uint64_t* scalars);
/* normalizeAlphas over the finished classes (transcript part of the labels) */
int orc_online_finish(orc_online* on, uint64_t n_classes, const uint64_t* off, const uint32_t* tids,
                      const uint64_t* counts, double* projected, double* eff_len, uint64_t* unique, uint64_t* total);

/* exp / log of the per-alignment arithmetic: 0 = the platform libm (default: what the reference calls), 1 = the
 * fdlibm restatement of orc_math.h (bit-exact regression mode, the algorithm of the product's device code) */
void orc_set_math_mode(int mode);
int orc_get_math_mode(void);
void orc_math_probe(int mode, uint64_t nx, const double* x, double* ex, uint64_t ny, const double* y, double* ly);

/* test hook: banded affine glocal DP score of one read on reference `tid` around diagonal `diag_c` (read base i faces
 * reference position diag_c + i); ori 1 = the read's reverse complement */
int32_t orc_dp_score(const orc_index* ix, const orc_map_params* p, const uint8_t* read, uint32_t L, uint32_t ori,
                     uint32_t tid, int32_t diag_c);

/* test hook: the candidates of one mate (at most 64, in (tid, ori, diag_c) order) and what its seeds look like.  The
 * fields tell which path of the product's seed kernel the mate takes (tests/test_seed_paths_cpu.py). */
typedef struct orc_cand { uint32_t tid, ori; int32_t diag_c; uint32_t cov; } orc_cand;
typedef struct orc_mate_info {
  uint32_t lookups;            /* valid k-mer lookups (no N) */
  uint32_t postings_all;       /* postings of the accepted lookups, before the 2048-seed cut */
  uint32_t seeds;              /* seeds kept (after the cut) */
  uint32_t cut_round;          /* 0: no cut; else the round of 32 seed positions whose lookup the cut fell in (1, 2) */
  uint32_t distinct;           /* distinct (tid, ori, diag) keys among the kept seeds */
  uint32_t chains;
  uint32_t survivors;          /* chains at or above the consensus threshold, before the top-64 cut */
  uint32_t straddle_seeds;     /* chains whose seeds cross a 32-key boundary of the sorted seed array */
  uint32_t straddle_distinct;  /* the same over the sorted array of distinct keys */
} orc_mate_info;
uint32_t orc_mate_candidates(const orc_index* ix, const orc_map_params* p, const uint8_t* read, uint32_t L,
                             orc_cand* out /*[64]*/, orc_mate_info* info);

#ifdef __cplusplus
}
#endif
#endif
