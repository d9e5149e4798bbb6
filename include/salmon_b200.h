/*
 * salmon_b200.h -- C ABI of libsalmon_b200.so (H100 / sm_90a).
 *
 * Drop-in boundary for Salmon's quantification hot path (SURVEY.md section 8b).
 * The reference has no FFI layer; the seams are ordinary C++ calls.  Each entry
 * point below names the reference call it replaces (file:line relative to
 * COMBINE-lab/salmon v1.11.4).  Plain pointers and sizes only; all pointers are
 * HOST pointers unless a name ends in _dev.  Return 0 on success, negative on
 * error (message via sb_last_error()); sb_em_optimize returns 1 where the
 * reference returns `false` ("Total alpha weight was too small").
 *
 * There is no CPU fallback: every compute entry point fails with
 * SB_ERR_NO_DEVICE if no CUDA device is usable.
 */
#ifndef SALMON_B200_H
#define SALMON_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SB_OK 0
#define SB_ERR_INVALID (-1)
#define SB_ERR_NO_DEVICE (-2)
#define SB_ERR_CUDA (-3)
#define SB_ERR_NOMEM (-4)
#define SB_ERR_NCCL (-5)
#define SB_ERR_STATE (-6)

/* ---- library ---------------------------------------------------------- */
int sb_version(void);                 /* 10000*major + 100*minor + patch */
const char* sb_last_error(void);      /* thread-local, never NULL */
int sb_device_count(void);            /* number of usable CUDA devices (0 if none) */

/* ---- equivalence classes ---------------------------------------------- */
/* Host view of EquivalenceClassBuilder<TGValue>::eqVec() after finish()
 * (include/salmon/internal/quant/EquivalenceClassBuilder.hpp:165-181,210-223):
 * class c has transcripts tids[off[c]..off[c+1]) (sorted ascending, as
 * TranscriptGroup keeps them), TGValue::weights in `weights` (normalised to sum
 * 1 per class by finish()), TGValue::count in `counts`. */
typedef struct sb_eq_csr {
  uint64_t n_classes;
  uint32_t n_txps;
  const uint64_t* off;     /* [n_classes+1] */
  const uint32_t* tids;    /* [off[n_classes]] */
  const double* weights;   /* [off[n_classes]] */
  const uint64_t* counts;  /* [n_classes] */
} sb_eq_csr;

/* ---- EM / VBEM optimiser ---------------------------------------------- */
/* The SalmonOpts fields CollapsedEMOptimizer::optimize reads
 * (src/inference/CollapsedEMOptimizer.cpp:743-773,785,791,805,817,862). */
typedef struct sb_em_params {
  int32_t use_vbem;             /* sopt.useVBOpt (default 1) */
  int32_t per_txp_prior;        /* sopt.perTranscriptPrior (default 1) */
  int32_t init_uniform;         /* sopt.initUniform */
  int32_t eq_class_mode;        /* sopt.eqClassMode */
  int32_t no_rich_eq;           /* sopt.noRichEqClasses */
  int32_t no_length_correction; /* sopt.noLengthCorrection */
  int32_t alt_init;             /* sopt.meta || sopt.alternativeInitMode */
  int32_t bootstrap_reproject;  /* sopt.bootstrapReproject: sb_bootstrap ends each replicate with one update against the
                                   original class counts (CollapsedEMOptimizer.cpp:495-505); 0 = off */
  double vb_prior;              /* sopt.vbPrior (1e-2) */
  double tol;                   /* relDiffTolerance (0.01) */
  double num_required_frags;    /* sopt.numRequiredFragments (5e7) */
  uint32_t min_iter;            /* 100 (:890); 50 for bootstraps (:411) */
  uint32_t max_iter;            /* 10000 (pipeline/MappingPipelineStages.cpp:49) */
} sb_em_params;

typedef struct sb_em_stats {
  uint32_t iters;
  uint32_t converged;
  double max_rel_diff;     /* of the last iteration */
  double alpha_sum;        /* after truncation (:1004-1014) */
  uint64_t n_degenerate;   /* markDegenerateClasses (:330-394) */
  uint64_t n_multi_classes;/* valid classes with >1 transcript kept on device */
  uint64_t nnz_multi;      /* their label entries */
  uint32_t n_active_txps;  /* transcripts in >=1 such class */
  uint32_t gpu_launches;   /* kernels this library launched in the last call */
  float prepare_ms;        /* device time of sb_em_prepare (CUDA events) */
  float run_ms;            /* device time of the iteration loop (CUDA events) */
  float loop_kernel_ms;    /* device time of the persistent iteration kernel(s) only */
  uint32_t loop_kernel_launches;
} sb_em_stats;

void sb_em_default_params(sb_em_params* p);

typedef struct sb_em_ctx sb_em_ctx;

/* One context per GPU (one process per GPU in multi-GPU runs). */
sb_em_ctx* sb_em_create(int device);
void sb_em_destroy(sb_em_ctx* ctx);

/* Replaces `bool CollapsedEMOptimizer::optimize(ExpT&, SalmonOpts&, double tol,
 * uint32_t maxIter)` (include/salmon/internal/inference/CollapsedEMOptimizer.hpp:22-28;
 * src/inference/CollapsedEMOptimizer.cpp:732-1035).  Inputs per transcript are
 * what optimize reads from Transcript: projectedCounts (:780), the effective
 * length it would compute at :782-784, uniqueCount() (:790).  alpha_out[M]
 * receives what :1031 stores with setSharedCount().  Host buffers in and out;
 * this call = upload + prepare + run + download. */
int sb_em_optimize(sb_em_ctx* ctx, const sb_eq_csr* eq, const sb_em_params* p,
                   const double* projected_counts, const double* eff_len,
                   const uint64_t* unique_counts, double* alpha_out,
                   sb_em_stats* stats);

/* The same call split into its stages, so that a caller (or bench.py) can keep
 * the classes resident in HBM and time the stages separately. */
int sb_em_upload(sb_em_ctx* ctx, const sb_eq_csr* eq,
                 const double* projected_counts, const double* eff_len,
                 const uint64_t* unique_counts);
/* sb_em_prepare refuses (SB_ERR_INVALID) a negative or non-finite vb_prior. */
int sb_em_prepare(sb_em_ctx* ctx, const sb_em_params* p, sb_em_stats* stats);
int sb_em_run(sb_em_ctx* ctx, sb_em_stats* stats);   /* re-runnable: restarts from the prepared state */
int sb_em_download(sb_em_ctx* ctx, double* alpha_out, sb_em_stats* stats);

/* Debug/parity taps (tests): combinedWeights (:862-870) and validity flags. */
int sb_em_get_combined(sb_em_ctx* ctx, double* combined_out, uint8_t* valid_out);

/* The combined weights `--skipQuant --dumpEqWeights` writes (MappingPipelineStages.cpp:112-162): per class,
 * count * w / max(eff_len, 1) normalised to sum 1 (w = 1 with no_rich_eq), computed on the device with the arithmetic
 * of sb_em_prepare's combinedWeights.  eff_len = sb_map_result.eff_len (the transcript lengths under
 * --noEffectiveLengthCorrection).  combined_out[eq->off[n_classes]].  Uploads the table into ctx (a later
 * sb_em_prepare needs its own sb_em_upload). */
int sb_eq_combined_weights(sb_em_ctx* ctx, const sb_eq_csr* eq, const double* eff_len, int no_rich_eq,
                           double* combined_out);

/* ---- bootstraps and Gibbs samples ----------------------------------------
 * Both run on the context sb_em_optimize (or upload+prepare+run) left behind: the class table,
 * combinedWeights, validity flags and effective lengths stay resident in HBM.  Each sample
 * is handed to the callback on the calling thread (the reference serialises its
 * writeBootstrap callback with a mutex, src/output/GZipWriter.cpp:766-771); a non-zero
 * return stops sampling.  Draws are a pure function of `seed` (Philox-4x32-10; stream
 * layout in oracle/em_oracle.h), unlike the reference's random_device seeding. */
typedef int (*sb_sample_cb)(const double* alpha, uint32_t n_txps, void* user);

/* Replaces CollapsedEMOptimizer::gatherBootstraps (CollapsedEMOptimizer.hpp:30-34;
 * src/inference/CollapsedEMOptimizer.cpp:554-690, doBootstrap :398-552).  p carries
 * min_iter = 50 (:411), tol, max_iter and the VBEM switch; num_mapped_frags is
 * readExp.numMappedFragments() (:572-573, used by the degenerate marking :608-621).
 * Returns 1 where doBootstrap returns false (:521-525).  With p->bootstrap_reproject each replicate's converged
 * alpha takes one more EM / VBEM update against the original counts of the classes the replicates resample, before
 * the truncation (:495-505); that update drops a class whose denominator is at most DBL_MIN times the largest count of a
 * multi-transcript class, so that count / denominator stays finite. */
int sb_bootstrap(sb_em_ctx* ctx, const sb_em_params* p, double num_mapped_frags,
                 uint32_t n_bootstraps, uint64_t seed, sb_sample_cb cb, void* user);
/* Parity tap: per input class, the count drawn by the last replicate.  Single-transcript classes
 * on the same transcript share one count: each of them reports what all of them drew together. */
int sb_bootstrap_last_counts(sb_em_ctx* ctx, uint64_t* counts_out);

/* Replaces CollapsedGibbsSampler::sample (CollapsedGibbsSampler.hpp:18-21;
 * src/inference/CollapsedGibbsSampler.cpp:317-508, round :92-278).  alphas_init =
 * Transcript::projectedCounts as writeAbundances leaves it (= sharedCount, GZipWriter.cpp:711-715);
 * use_vbem / per_txp_prior / vb_prior select the prior (:357-371); thinning = sopt.thinningFactor
 * (16); no_gamma_draw = sopt.noGammaDraw. */
int sb_gibbs(sb_em_ctx* ctx, const double* alphas_init, int use_vbem, int per_txp_prior,
             double vb_prior, uint32_t n_samples, uint32_t thinning, int no_gamma_draw,
             double num_mapped_frags, uint64_t seed, sb_sample_cb cb, void* user);
/* Parity tap: the per-transcript state the last Gibbs round left, M doubles each.  mu_out: the
 * gamma draws (count+prior ~ Gamma, scale 1/(0.1+effLen)) or, with no_gamma_draw, the means
 * (count+prior)/effLen; 0 for inactive transcripts.  cnt_out: the counts that round's singletons
 * and category draws produced.  SB_ERR_STATE if no sb_gibbs has run on the current table. */
int sb_gibbs_last_state(sb_em_ctx* ctx, double* mu_out, double* cnt_out);

/* ---- output seam (host code): the reference's file formats ---------------------------------
 * TPM as GZipWriter::writeAbundances computes it (src/output/GZipWriter.cpp:719-736). */
int sb_tpm(uint32_t n_txps, const double* alpha, const double* eff_len, double num_mapped_frags, double* tpm_out);
/* quant.sf (GZipWriter.cpp:684-739): Name, Length (CompleteLength), EffectiveLength %.{sig}f, TPM %f, NumReads %.{sig}f */
int sb_write_quant_sf(const char* path, uint32_t n_txps, const char* const* names, const uint32_t* complete_len,
                      const double* eff_len, const double* alpha, double num_mapped_frags, int sig_digits);
/* aux_info/eq_classes.txt[.gz] (GZipWriter.cpp:64-168; gzip when the path ends in .gz).  weights != NULL is the
 * --dumpEqWeights layout the --eqclasses reader expects (src/util/SalmonUtils.cpp:1026-1122); weights == NULL
 * collapses range-factorised classes by transcript set like the reference (:86-113). */
int sb_write_eq_classes(const char* path, uint32_t n_txps, const char* const* names, uint64_t n_classes,
                        const uint64_t* off, const uint32_t* tids, const double* weights, const uint64_t* counts);

/* ---- input seam (SURVEY.md 8f-1, host code): what sits immediately before B1 / B3 in the reference ---------------
 * sb_reads_*: FASTQ / FASTA read files (plain or gzip) -> batches of base codes.  Replaces FQFeeder's
 * fastx_parser<ReadPair> / <ReadSeq> as salmon drives it (src/quant/SalmonQuantify.cpp:2357-2373 construction,
 * :2419-2430 start, :1118-1141 the ReadGroup loop).  One splitter thread per mate stream cuts record-aligned
 * blocks, sb_reads_next translates a batch with n_threads OpenMP threads straight into the caller's buffers
 * (0..3 = A,C,G,T, 4 = anything else; one byte per base, `stride` bytes per read, the tail padded with 4).
 * files2 == NULL: single-end.  4-line FASTQ and 2-line FASTA records; mates are paired by record index. */
typedef struct sb_reads sb_reads;
sb_reads* sb_reads_open(const char* const* files1, const char* const* files2, uint32_t n_files, uint32_t n_threads);
/* Returns the number of reads (pairs) delivered, 0 at the end of the input, < 0 on error (malformed record, mate
 * files of different length, a read longer than `stride`). */
int64_t sb_reads_next(sb_reads* r, uint32_t max_pairs, uint32_t stride, uint8_t* left, uint8_t* right,
                      uint32_t* len_left, uint32_t* len_right);
/* Lengths of the next records without delivering them: returns how many reads (pairs) the next sb_reads_next call can
 * deliver, up to max_pairs (fewer only at the end of the input); *uniform_len = their common length when every read of
 * both mates has the same one, else 0 (a caller that groups reads by length then takes the usual case straight into its
 * [n, L] buffer with stride = L).  sb_reads_skip drops the next n reads unread (another shard's batch). */
int64_t sb_reads_peek(sb_reads* r, uint32_t max_pairs, uint32_t* uniform_len);
int64_t sb_reads_skip(sb_reads* r, uint32_t n);
int sb_reads_paired(const sb_reads* r);   /* 1: two mate streams, 0: single-end */
void sb_reads_close(sb_reads* r);

/* The --eqclasses input (src/util/SalmonUtils.cpp:1024-1122 readEquivCounts): N, C, N names, C lines
 * `k t_1..t_k [w_1..w_k] count`, then optional `name effective_length` lines (missing -> 100.0, :1109-1116). */
typedef struct sb_eq_file {
  uint32_t n_txps, has_weights;
  uint64_t n_classes;
  const char* const* names;   /* [n_txps] */
  const uint64_t* off;        /* [n_classes+1] */
  const uint32_t* tids;
  const double* weights;      /* NULL when the file has none (--dumpEq without --dumpEqWeights) */
  const uint64_t* counts;
  const double* eff_len;      /* [n_txps] */
  uint32_t n_missing_eff_len, reserved;
} sb_eq_file;
int sb_eq_file_read(const char* path, sb_eq_file** out);
void sb_eq_file_free(sb_eq_file* f);

/* aux_info/bootstrap/bootstraps.gz (src/output/GZipWriter.cpp:765-789 writeBootstrap): every sample is n raw doubles
 * appended to one gzip member (level 6, deflated in 128 KiB slices by a thread team the way pigz does it); write() may
 * be called from several threads (the sb_bootstrap / sb_gibbs callback).  close() returns the number of samples written,
 * or a negative code when the file could not be completed (full disk). */
typedef struct sb_bootstrap_writer sb_bootstrap_writer;
sb_bootstrap_writer* sb_bootstrap_writer_open(const char* path);
int sb_bootstrap_writer_write(sb_bootstrap_writer* w, const double* sample, uint32_t n);
int64_t sb_bootstrap_writer_close(sb_bootstrap_writer* w);

/* Transcript FASTA (plain / gzip, multi-line) -> the arrays sb_index_build takes, with the `salmon index` options of
 * src/index/BuildSalmonIndex.cpp:72-124: --gencode (name ends at the first '|'), --decoys (names listed in a file;
 * decoys must come last, first_decoy feeds sb_map_params.first_decoy), --no-clip (poly-A clipping off: by default a
 * run of more than 10 trailing A is removed), --keepDuplicates (by default sequence-identical transcripts are
 * dropped, the first one is kept).  Non-ACGT bases become code 4 (no k-mers; the reference's pufferfish replaces
 * them with random bases -- documented deviation).  complete_len = length before clipping (quant.sf "Length"). */
typedef struct sb_txome {
  uint32_t n_txps, first_decoy;      /* first_decoy == n_txps: no decoys */
  const char* const* names;
  const uint64_t* seq_off;           /* [n_txps+1] */
  const uint8_t* codes;
  const uint32_t* complete_len;
  uint32_t n_duplicates_removed, n_clipped, n_short, reserved;
} sb_txome;
int sb_txome_read_fasta(const char* path, uint32_t k, int gencode, const char* decoys_path, int no_clip,
                        int keep_duplicates, sb_txome** out);
void sb_txome_free(sb_txome* t);

/* ---- Stage A: index, per-read mapping, equivalence-class builder ------------------
 * Seam B1: the body of processReads<IndexT> (src/quant/SalmonQuantify.cpp:1026-1874: per read
 * MemCollector / findChains / joinReadsAndFilter / PuffAligner::calculateAlignments /
 * updateRefMappings / filterAndCollectAlignments, then processMiniBatch :426-1023) and seam B2:
 * EquivalenceClassBuilder<TGValue>::addGroup / finish / eqVec
 * (include/salmon/internal/quant/EquivalenceClassBuilder.hpp:165-181,210-223,237-250).
 * The mapping core (pufferfish) is not in the reference tree; the algorithm here is this
 * project's own (DESIGN.md "MAPSPEC").  Reads are passed as one base per byte
 * (0..3 = A,C,G,T; 4 = N), n_pairs x read_len, fixed length per batch. */
typedef struct sb_index sb_index;
/* Replaces SalmonIndex::build -> pufferfishIndex() for the purposes of this path
 * (include/salmon/internal/index/SalmonIndex.hpp:106-118): canonical k-mer hash table ->
 * postings (transcript, offset); own in-memory format.  seq_off[n_txps+1]: base offsets. */
sb_index* sb_index_build(uint32_t n_txps, const uint64_t* seq_off, const uint8_t* codes, uint32_t k);
void sb_index_free(sb_index* ix);
/* Reference metadata carried by the index (what `salmon quant` prints in quant.sf): names, lengths before poly-A
 * clipping, index of the first decoy (== n_txps: none).  Optional; get returns NULL arrays when never set. */
int sb_index_set_meta(sb_index* ix, const char* const* names, const uint32_t* complete_len, uint32_t first_decoy);
int sb_index_get_meta(const sb_index* ix, uint32_t* n_txps, uint32_t* k, uint32_t* first_decoy,
                      const char* const** names, const uint32_t** complete_len);
/* On-disk form (own binary format, one file; `salmon index -i dir` analog).  NOT the pufferfish / SSHash layout
 * (that source is absent from the reference tree; SURVEY.md 8f-2). */
int sb_index_save(const sb_index* ix, const char* path);
sb_index* sb_index_load(const char* path);

/* Creates the CUDA context of `device` (this takes seconds on a large GPU).  Optional: a front end calls it from a
 * thread of its own while it loads the index from disk, so that the two overlap (sb_salmon does). */
int sb_device_init(int device);
/* out4 = {distinct k-mers, postings, table capacity, bytes} */
int sb_index_info(const sb_index* ix, uint64_t* out4);
/* Raw views of the index arrays (for serialisation): table = {u64 key, u32 first posting, u32 count}
 * x capacity (open addressing, linear probing, key ~0 = free); postings = {u32 transcript, u32 offset}. */
int sb_index_host_arrays(const sb_index* ix, const uint64_t** tx_off, const uint8_t** codes,
                         const void** table, uint64_t* table_capacity, const void** postings,
                         uint64_t* n_postings);

/* SalmonOpts fields of the mapping / assignment path (defaults: SalmonDefaults.hpp:10-99;
 * initMapperSettings, SalmonMappingUtils.hpp:153-223). */
typedef struct sb_map_params {
  uint32_t k;                 /* 31 */
  uint32_t stride;            /* seed sampling stride (MAPSPEC) */
  uint32_t max_occs_per_hit;  /* maxOccsPerHit 1000 */
  uint32_t max_read_occ;      /* maxReadOcc 200; at most 1000 (device memory grows with it: DESIGN.md section 14) */
  uint32_t max_frag_len;      /* fragLenDistMax 1000 */
  uint32_t band;              /* bandwidth 15 */
  uint32_t chain_gap;         /* MAPSPEC: diagonal gap inside a chain */
  uint32_t range_bins;        /* rangeFactorizationBins 4 */
  int32_t ma, mp, go, ge;     /* 2 -4 6 2 */
  int32_t hard_filter;        /* hardFilter */
  int32_t first_decoy;        /* firstDecoyIndex */
  double consensus_frac;      /* 1 - consensusSlack */
  double min_score_fraction;  /* 0.65 */
  double score_exp;           /* 1.0 */
  double min_aln_prob;        /* 1e-5 */
  double decoy_threshold;     /* 1.0 */
  double fld_mean, fld_sd;    /* 250, 25 */
  uint64_t num_pre_burnin;    /* numPreBurninFrags 5000 */
  uint64_t num_burnin;        /* numBurninFrags 5000000 */
  uint64_t seed;              /* stream of the stochastic FLD update (the reference seeds from random_device) */
  uint32_t mini_batch;        /* reads per forgetting-mass timestep (miniBatchSize 5000) */
  uint32_t reserved2;
  /* join policy (pufferfish::util::MappingConstraintPolicy as salmon configures it, SalmonMappingUtils.hpp:208-220;
   * option texts src/cli/ProgramOptionsGenerator.cpp:111-137,198-201): */
  double pre_merge_thresh;    /* preMergeChainSubThresh 0.75: per mate and transcript, chains below this fraction of the best are dropped */
  double post_merge_thresh;   /* postMergeChainSubThresh 0.9: per transcript, chain pairs below this fraction of the best pair are dropped */
  double orphan_thresh;       /* orphanChainSubThresh 0.95: without a concordant pair, orphans below this fraction of the best chain are dropped */
  int32_t allow_dovetail;     /* allowDovetail (false): dovetailing mates count as concordant */
  int32_t allow_orphans;      /* !discardOrphansQuasi (true): orphan mappings when no pair exists */
  /* expected library format (LibraryFormat, -l): SB_LIB_IU / ISF / ISR (paired-end, inward) or SB_LIB_U / SF / SR
   * (single-end: sb_map_batch with right == NULL).  Mappings that are not compatible with it are ignored
   * (incompatPrior = 0 -> ignoreIncompat, SalmonQuantify.cpp:1467-1521,2141-2150; rules src/util/SalmonUtils.cpp:138-298) */
  int32_t lib_type;
  /* --recoverOrphans (0 = off; paired-end, warp kernels only): for a read whose joint hits are orphans only, search each
   * anchor's transcript within max_frag_len for the missing mate (infix edit distance) and turn the orphans into the
   * pairs found (rule: DESIGN.md section 11).  Single-end libraries ignore it. */
  int32_t recover_orphans;
  /* scoring mode of the banded DP (rule: DESIGN.md section 12): 0 = end-to-end (default), 1 = --softclipOverhangs
   * (read bases hanging over either transcript end are left unaligned and add nothing to the score), 2 = --softclip
   * (any stretch of the read may be left unaligned at either end: the score is the best local alignment inside the
   * band; includes 1).  The acceptance threshold stays minScoreFraction * ma * read length.  Other values are refused;
   * variant 0 of the mapping kernels supports 0 only. */
  int32_t softclip;
  /* fragment likelihood of each kept mapping (rule: DESIGN.md section 13); all zero = salmon's defaults.
   * no_single_frag_prob (--noSingleFragProb): an orphan of a paired-end library gets log P = LOG_EPSILON and a single-end
   * read LOG_1 instead of the ambiguous-length probability.  no_frag_len_dist (--noFragLengthDist): no fragment-length
   * term at all (orphans and single-end reads as under no_single_frag_prob); needs no_eff_len_correction.
   * no_eff_len_correction (--noEffectiveLengthCorrection): transcript lengths replace effective lengths in the online
   * phase after burn-in and in sb_map_result.eff_len (what the optimiser, the samplers and quant.sf take). */
  int32_t no_single_frag_prob;
  int32_t no_frag_len_dist;
  int32_t no_eff_len_correction;
  /* --incompatPrior as a probability: 0 (or below 1e-100) = mappings incompatible with lib_type are ignored (the
   * default); otherwise they stay in and carry log(incompat_prior) in their auxiliary probability.  In [0, 1]. */
  double incompat_prior;
} sb_map_params;
/* Only sb_quant_files takes these two: the library type is detected from the first 50 000 fragments that show a
 * strand, as LibraryTypeDetector does (include/salmon/internal/model/LibraryTypeDetector.hpp:34-140): until then every
 * mapping counts as compatible, afterwards the detected type applies (checked after every batch). */
#define SB_LIB_AUTO_PAIRED 6
#define SB_LIB_AUTO_SINGLE 7
#define SB_LIB_IU 0
#define SB_LIB_ISF 1
#define SB_LIB_ISR 2
#define SB_LIB_U 3
#define SB_LIB_SF 4
#define SB_LIB_SR 5
void sb_map_default_params(sb_map_params* p);
/* salmon's Bowtie2-mimicking presets (rule: DESIGN.md section 14), applied to p after the other options so that they
 * override them; set lib_type first.  Both: max_read_occ 1000, consensus_frac 0.5 (consensusSlack 0.5), allow_orphans 0
 * (discardOrphansQuasi) for paired-end library types (a single-end read is a left orphan here and stays), and softclip
 * mode 1 (--softclipOverhangs) back to 0; mode 2 (--softclip) stays.
 * strict = 0 (--mimicBT2): ma 2, mp -4, go 5, ge 3.  strict != 0 (--mimicStrictBT2): min_score_fraction 0.8, ma 1,
 * mp 0, go 25, ge 25.  Returns 0, or SB_ERR_INVALID for a null p. */
int sb_map_mimic_bt2(sb_map_params* p, int strict);

typedef struct sb_map_batch_stats {
  uint32_t n_pairs;
  uint32_t gpu_launches;
  uint64_t mapped, lookups, postings, seeds, candidates, kept, label_entries, n_batch_classes;
  float device_ms;            /* H2D of the reads + all kernels of the batch (CUDA events) */
  uint32_t reserved;
  uint64_t full_dp;           /* mate alignments that needed the banded DP (the rest: ungapped shortcut) */
  float seed_kernel_ms;       /* device time of the seed/chain kernel launches of this batch (CUDA events) */
  uint32_t seed_kernel_launches;
  /* orphan rescue (recover_orphans): fragments with at least one rescued pair, mate searches run, anchors whose mate
   * was found but whose candidate list had no room; device time of the rescue kernels (CUDA events) */
  uint64_t orphans_rescued, rescue_searches, rescue_no_room;
  float rescue_kernel_ms;
  uint32_t reserved2;
  uint64_t compatible;        /* mapped fragments with at least one kept mapping compatible with lib_type */
} sb_map_batch_stats;

typedef struct sb_map_result {   /* host CSR owned by the context, valid until destroy / next finish */
  uint64_t n_classes;
  const uint64_t* off;        /* [n_classes+1] */
  const uint32_t* tids;       /* label, transcript part */
  const double* weights;      /* normalised (finish()) */
  const uint64_t* counts;
  const uint32_t* bins;       /* range-factorisation part of the label (NULL if range_bins == 0) */
  uint64_t n_mapped, lookups, postings, seeds, candidates, kept, label_entries;
  /* what CollapsedEMOptimizer::optimize reads per transcript (inputs of sb_em_optimize): */
  uint32_t n_txps;
  uint32_t reserved;
  const double* projected_counts;  /* normalizeAlphas (src/util/SalmonUtils.cpp:461-529): Transcript::projectedCounts */
  const double* eff_len;           /* exp(cachedLogEffectiveLength) (CollapsedEMOptimizer.cpp:782-784) */
  const uint64_t* unique_counts;   /* Transcript::uniqueCount() */
  const uint64_t* total_counts;    /* Transcript::totalCount() */
  /* fragments that showed each observed format among their kept mappings (ReadLibrary::libTypeCounts,
   * SalmonQuantify.cpp:765,1000-1002): [0] ISF (pair, left mate forward), [1] ISR, [2] SF (orphan / single-end read
   * mapped forward), [3] SR; [4..7] reserved */
  uint64_t lib_format_counts[8];
  uint64_t orphans_rescued, rescue_searches, rescue_no_room;   /* sums of sb_map_batch_stats' fields since create / reset */
  uint64_t n_compatible;           /* sum of sb_map_batch_stats.compatible (sb_map_reduce_global: over all ranks) */
} sb_map_result;

typedef struct sb_map_ctx sb_map_ctx;
sb_map_ctx* sb_map_create(sb_index* ix, const sb_map_params* p, int device, uint32_t max_pairs_per_batch,
                          uint32_t max_read_len);
void sb_map_destroy(sb_map_ctx* ctx);
/* One batch: H2D, seed/chain, DP scoring, filtering + auxiliary probabilities + labels, online mass / FLD
 * updates (processMiniBatch), per-batch class aggregation.  BATCHED SEMANTICS: the model state (transcript
 * masses, fragment-length distribution, burn-in regime) is frozen for the duration of the batch and the batch's
 * contributions are folded in afterwards (order-independent, bit-reproducible); forgetting-mass timesteps still
 * advance every `mini_batch` reads.  Smaller batches track the reference's per-5000-read dynamics more closely. */
int sb_map_batch(sb_map_ctx* ctx, const uint8_t* left, const uint8_t* right, uint32_t n_pairs,
                 uint32_t read_len, sb_map_batch_stats* stats);
/* ---- multi-GPU Stage A (SURVEY.md 8e): reads sharded over ranks, one context per GPU / process, class tables stay
 * per rank.  After sb_map_finish every rank exports its statistics (sb_map_partial_get); the host layer reduces them
 * over the ranks once -- masses and the FLD by log-sum-exp (the FLD prior counted once), counts by sum, fld_min by min,
 * cluster roots all-gathered -- and calls sb_map_project_global, which redoes normalizeAlphas with the global state:
 * every rank then holds identical projected counts / effective lengths / unique counts for sb_em_optimize
 * (classes sharded, alpha all-reduced per iteration). */
typedef struct sb_map_partial {
  uint32_t n_txps, n_fld;          /* n_fld = max_frag_len + 1 */
  const double* mass;              /* [n_txps] log mass (+inf = none) */
  const double* fld_hist;          /* [n_fld] log histogram */
  double fld_tot;                  /* log total mass */
  const double* fld_prior_hist;    /* [n_fld] the prior every rank started from */
  double fld_prior_tot;
  uint32_t fld_min, reserved;
  const uint64_t* unique_counts;   /* [n_txps] */
  const uint64_t* total_counts;    /* [n_txps] */
  const uint64_t* cluster_hits;    /* [n_txps] fragments whose first transcript this is */
  const uint32_t* cluster_root;    /* [n_txps] smallest transcript id of the transcript's cluster */
  uint64_t assigned;               /* fragments assigned by this rank */
  uint64_t compatible;             /* of those, fragments with a kept mapping compatible with the library type */
} sb_map_partial;
int sb_map_partial_get(sb_map_ctx* ctx, sb_map_partial* out);
int sb_map_project_global(sb_map_ctx* ctx, const sb_map_partial* global_stats, uint32_t n_ranks,
                          const uint32_t* roots_all /* n_ranks x n_txps */, sb_map_result* out);

/* ---- B2: the equivalence-class builder on its own -----------------------------------------------------------------
 * Replaces `void EquivalenceClassBuilder<TGValue>::addGroup(TranscriptGroup&&, std::vector<double>& weights)`,
 * `bool finish()` and `eqVec()` (include/salmon/internal/quant/EquivalenceClassBuilder.hpp:237-250,165-181,210-223;
 * callers src/quant/SalmonQuantify.cpp:855-856,2641) for a caller that forms the labels itself, and the table that
 * `--eqclasses` reads (readEquivCounts, src/util/SalmonUtils.cpp:1024-1122).  Host buffers in, host CSR out (owned by
 * the builder, valid until the next finish / destroy); the aggregation runs on the device (label hash -> radix sort ->
 * segmented reduce, the kernels sb_map_batch uses for its own reads).  sb_map_batch / sb_map_finish keep doing this
 * internally for reads mapped by the library. */
typedef struct sb_eq_builder sb_eq_builder;
typedef struct sb_eq_table {
  uint64_t n_classes;
  uint32_t n_txps, reserved;
  const uint64_t* off;             /* [n_classes+1] into tids / weights */
  const uint32_t* tids;            /* transcript part of every label */
  const double* weights;           /* normalised to sum 1 per class (TGValue::normalizeAux, :114-123) */
  const uint64_t* counts;
  const uint32_t* n_txp_in_label;  /* [n_classes] */
  const uint64_t* label_off;       /* [n_classes+1] into labels: the full labels (transcripts + range-factorisation bins) */
  const uint32_t* labels;
  uint64_t n_groups;               /* addGroup calls so far */
} sb_eq_table;
sb_eq_builder* sb_eq_create(uint32_t n_txps, int device);
void sb_eq_destroy(sb_eq_builder* b);
/* addGroup x n: label i = labels[label_off[i] .. label_off[i+1]) (transcript ids, optionally followed by as many
 * range-factorisation bins), weights[weight_off[i] .. weight_off[i+1]) one per transcript; counts NULL = 1 each. */
int sb_eq_add_batch(sb_eq_builder* b, uint32_t n_groups, const uint64_t* label_off, const uint32_t* labels,
                    const uint64_t* weight_off, const double* weights, const uint64_t* counts);
/* a finished table (e.g. sb_eq_file_read's) as one batch */
int sb_eq_from_host(sb_eq_builder* b, const sb_eq_csr* eq);
int sb_eq_finish(sb_eq_builder* b, sb_eq_table* out);

/* Forget everything mapped so far (class tables, online state, counters) without re-allocating. */
int sb_map_reset(sb_map_ctx* ctx);
/* finish(): merge batch tables, normalise weights, return the CSR (feeds sb_em_optimize). */
int sb_map_finish(sb_map_ctx* ctx, sb_map_result* out);
/* Parity tap: the online state after the last batch.  mass_out[n_txps] (log scale, +inf = none),
 * hist_out[max_frag_len+1] (log FLD histogram), log_eff_out[n_txps],
 * scalars6 = {assigned fragments, fragments seen, timestep, burned in, FLD min, bits of the log total FLD mass}. */
int sb_map_online_state(sb_map_ctx* ctx, double* mass_out, double* hist_out, double* log_eff_out, uint64_t* scalars6);
/* Parity tap of the orphan rescue search (DESIGN.md section 11): case i searches pattern pats[pat_off[i]..pat_off[i+1])
 * (base codes 0..3, 4 = N, 1..256 bases) in window wins[win_off[i]..win_off[i+1]) with edit limit K[i] on `device`,
 * with the kernel's own search; dist[i] = the smallest infix edit distance and end[i] = the leftmost window position
 * where an alignment at that distance ends, both -1 when it exceeds K[i] or the window is empty. */
int sb_rescue_search_tap(int device, uint32_t n, const uint8_t* pats, const uint64_t* pat_off, const uint8_t* wins,
                         const uint64_t* win_off, const int32_t* K, int32_t* dist, int32_t* end);
/* Parity tap: the per-read alignments / labels of the last batch (arrays n*cap; label n*2*cap). */
int sb_map_last_alignments(sb_map_ctx* ctx, uint32_t n, uint32_t* n_aln, uint32_t* tid, int32_t* score,
                           double* prob, int32_t* pos, int32_t* mate_pos, uint8_t* flags, int32_t* flen,
                           uint32_t* label, double* weight);
/* Parity tap: the per-read candidates of the last batch as the seed kernel left them: n_l / n_r [n] (bit 31 of n_l set:
 * the read has no joint hit or more than max_read_occ of them), cand_l / cand_r [n * 64] of 12 bytes each (tid, diag_c,
 * orientation << 31 | coverage).  SB_ERR_STATE when the last batch ran as more than one chunk or with orphan rescue. */
int sb_map_last_candidates(sb_map_ctx* ctx, uint32_t n, uint32_t* n_l, uint32_t* n_r, void* cand_l, void* cand_r);

/* The read stream as [n, L] batches of one read length each (what sb_map_batch takes): a reader thread parses, groups
 * the reads by length into double-buffered (page-locked, when a device is present) matrices and hands full ones to
 * `cb` on the calling thread, so parsing overlaps whatever the callback does (sb_quant_files: sb_map_batch).  A pair
 * whose mates differ in length goes at the shorter length (the longer mate loses its 3' end); pairs shorter than
 * min_len are counted and dropped.  The stream is cut into global batches of `batch` records; this call delivers the
 * batches g with g % shard_count == shard_index (multi-GPU: one process per shard).  A batch of one length -- the usual
 * case -- is translated straight into the bucket, without staging.  cb != 0 aborts and is returned.  Single-end
 * readers deliver right == NULL. */
typedef int (*sb_batch_cb)(void* user, const uint8_t* left, const uint8_t* right, uint32_t n_pairs, uint32_t read_len);
typedef struct sb_bucket_stats {
  uint64_t n_observed, n_delivered, n_too_short, n_trimmed_mates, n_batches;
  uint32_t n_read_lengths, reserved;
} sb_bucket_stats;
int sb_reads_bucketed(sb_reads* rd, uint32_t min_len, uint32_t batch, uint32_t max_read_len, uint32_t threads,
                      uint32_t shard_index, uint32_t shard_count, sb_batch_cb cb, void* user, sb_bucket_stats* stats);

/* ---- the host driver of the path (C++; salmon_b200/csrc/pipeline.cu): `salmon quant -i idx -l IU -1 .. -2 .. -o out`
 * for the hot path.  Mirrors processReadLibrary / quantifyLibrary (src/quant/SalmonQuantify.cpp:2339-2730) and
 * stageFinalizeMappingOutputs (src/quant/pipeline/MappingPipelineStages.cpp:37-206): a reader thread parses and groups
 * reads by length into pinned buffers while the calling thread runs sb_map_batch on the previous ones; then
 * sb_map_finish, sb_em_optimize, optional bootstraps / Gibbs samples, and the output files under out_dir
 * (quant.sf, aux_info/eq_classes.txt.gz, aux_info/bootstrap/{bootstraps.gz,names.tsv.gz}).  One GPU per call. */
typedef struct sb_quant_opts {
  int32_t device;
  uint32_t batch;            /* read pairs per sb_map_batch (262144) */
  uint32_t max_read_len;     /* longest read accepted, 32..256 */
  uint32_t threads;          /* read-file translation threads */
  int32_t dump_eq;           /* --dumpEq */
  int32_t dump_eq_weights;   /* --dumpEqWeights */
  uint32_t num_bootstraps;   /* --numBootstraps */
  uint32_t num_gibbs;        /* --numGibbsSamples */
  uint32_t thinning;         /* --thinningFactor (16) */
  int32_t no_gamma_draw;     /* --noGammaDraw */
  uint32_t shard_index, shard_count;   /* rank / number of ranks of a multi-GPU run (one process per GPU); 0 / 1 on one GPU */
  uint64_t seed;
  const void* nccl_uid;      /* shard_count > 1: the 128 bytes of rank 0's sb_nccl_unique_id(), the same on every rank */
  /* SAM output (one GPU only; NULL / 0 = off): */
  const char* write_mappings;     /* --writeMappings[=FILE]: path of the SAM file, "-" = standard output */
  int32_t write_qualities;        /* --writeQualities: QUAL from the read files instead of '*' */
  int32_t write_unmapped_names;   /* --writeUnmappedNames: out_dir/aux_info/unmapped_names.txt */
  const char* cmdline;            /* the @PG CL: field of the SAM header (may be NULL) */
  int32_t skip_quant;             /* --skipQuant: map and write the run metadata (and the classes with --dumpEq); no
                                     normalizeAlphas, optimiser, quant.sf or samples (MappingPipelineStages.cpp:45-162) */
} sb_quant_opts;
typedef struct sb_quant_summary {
  uint64_t n_observed, n_mapped, n_too_short, n_trimmed_mates, n_classes, n_batches;
  uint32_t n_read_lengths, em_iters, em_converged, reserved;
  double map_seconds, em_seconds, total_seconds;   /* wall clock */
  float map_device_ms;                             /* sum of sb_map_batch_stats.device_ms */
  float map_setup_ms;                              /* the part of map_seconds before the first read is parsed: sb_map_create
                                                      (workspace allocation, index upload if not resident) + opening the files */
  uint64_t orphans_rescued, rescue_searches, rescue_no_room;   /* this rank's orphan rescue counters (sb_map_result) */
} sb_quant_summary;
void sb_quant_default_opts(sb_quant_opts* o);
/* mp / ep / o may be NULL (defaults); out_dir may be NULL (no files); alpha_out[n_txps] may be NULL (decoy entries, the
 * suffix of the id space, are 0: decoys are dropped before the optimiser and the writers, SalmonQuantify.cpp:2479).
 * shard_count > 1: every rank calls this with its shard_index and the same nccl_uid; reads are sharded by global batch,
 * the end-of-mapping statistics are reduced once, the optimiser exchanges alpha inside its kernel, rank 0 writes. */
int sb_quant_files(sb_index* ix, const char* const* mates1, const char* const* mates2, uint32_t n_files,
                   const sb_map_params* mp, const sb_em_params* ep, const sb_quant_opts* o, const char* out_dir,
                   double* alpha_out, sb_quant_summary* summary);

/* ---- host-level communicator of the multi-GPU driver (one process per GPU; NCCL underneath, loaded with dlopen) ----
 * rank / nranks as the launcher gives them; nccl_uid128 = the 128 bytes of sb_nccl_unique_id(), made by rank 0 and
 * handed to the other ranks by the launcher (sb_salmon: a file in the output directory; torchrun: any broadcast).
 * In place over HOST buffers of 8-byte elements: dtype 0 = f64, 1 = u64; op 0 = sum, 2 = max, 3 = min. */
typedef struct sb_comm sb_comm;
sb_comm* sb_comm_create(int rank, int nranks, const void* nccl_uid128, int device);
void sb_comm_destroy(sb_comm* comm);
int sb_comm_rank(const sb_comm* comm);
int sb_comm_size(const sb_comm* comm);
int sb_comm_allreduce(sb_comm* comm, void* buf, size_t n, int dtype, int op);
int sb_comm_allgather(sb_comm* comm, const void* send, void* recv, size_t bytes_per_rank);
/* sb_em_peer_handle + all-gather + sb_em_peer_open on this communicator (fused multi-GPU EM) */
int sb_em_peer_setup(sb_em_ctx* ctx, sb_comm* comm, uint32_t max_txps);
/* End-of-mapping reduction of a sharded run (SURVEY.md 8e), the C++ form of salmon_b200/dist.py: masses and the
 * fragment-length histogram by log-sum-exp over the ranks (the prior counted once), counts by sum, cluster roots
 * all-gathered, then normalizeAlphas with the global state (sb_map_project_global).  On return every rank holds the
 * same projected counts / effective lengths / unique counts in *out; *assigned_out = fragments assigned by all ranks. */
int sb_map_reduce_global(sb_map_ctx* ctx, sb_comm* comm, sb_map_result* out, uint64_t* assigned_out);

/* `salmon quant -e` (processEqClasses, src/alignment/SalmonQuantifyAlignments.cpp:1406-1440): optimiser + samplers over a
 * dumped class table.  shard_count > 1: every rank holds the table, the posterior samples (bootstraps / Gibbs chains,
 * which are independent: CollapsedGibbsSampler.cpp:425-461, CollapsedEMOptimizer.cpp:670-688) are split over the ranks
 * and gathered by rank 0 into aux_info/bootstrap/bootstraps.gz in sample order. */
int sb_quant_eqclasses(const char* eq_path, const sb_em_params* ep, const sb_quant_opts* o, const char* out_dir,
                       sb_quant_summary* summary);

/* Tuning knobs of the mapping context: "variant" (1 = warp-cooperative kernels, 0 = serial-form kernels),
 * "fast_dp" (ungapped shortcut of the DP kernel on/off), "chunk" (reads per pipeline chunk), "input_on_device"
 * (sb_map_batch's read pointers are device pointers: inputs already resident in HBM), "ascii_reads" (the read bytes
 * are sequence characters A/C/G/T/N as the reference's parser delivers them, klibpp::KSeq::seq, instead of base
 * codes).  Results are identical for every setting.  "no_projection" = 1: sb_map_finish and
 * sb_map_project_global skip normalizeAlphas' cluster projection and report projected_counts of 0 (a --skipQuant run,
 * which has no optimiser to start); everything else they report is unchanged. */
int sb_map_set_option(sb_map_ctx* ctx, const char* key, int64_t value);

/* "lib_type" is also a key of sb_map_set_option: the expected library format of the batches that follow (inside the
 * family the context was created with: IU / ISF / ISR or U / SF / SR).
 * sb_map_lib_counts: fragments mapped so far that showed the formats {ISF, ISR, SF, SR} among their kept mappings
 * (cumulative over the batches; no device work).
 * sb_detect_lib_type: LibraryTypeDetector::mostLikelyType for the inward / unmated formats this library maps --
 * fraction of sense-strand fragments below 0.3 -> ISR (SR), below 0.7 -> IU (U), else ISF (SF); -1 when no fragment
 * has shown a strand yet. */
int sb_map_lib_counts(const sb_map_ctx* ctx, uint64_t out4[4]);
int sb_detect_lib_type(int paired, const uint64_t counts4[4]);

/* ---- SAM output of the mapping path (`salmon quant --writeMappings`; format rules: DESIGN.md "SAM output") -------
 * A sink writes the header (@HD, one @SQ per indexed reference with its indexed length, @PG) when it opens.  Attached
 * to a mapping context, every sb_map_batch_sam call also formats the batch's alignments on the GPU (a sizing kernel, a
 * scan, a writing kernel over windows of whole fragments that fit a fixed device buffer) and hands the text to the
 * sink's writer thread, which writes it in batch order.  sam_path "-" = standard output; either path may be NULL
 * (unmapped_path: the `<name> <type>` lines of --writeUnmappedNames). */
typedef struct sb_sam sb_sam;
#define SB_SAM_QUALITIES 1u   /* QUAL from the reads' quality lines (sb_map_batch_sam then needs them) */
sb_sam* sb_sam_open(const char* sam_path, const char* unmapped_path, const sb_index* ix, const char* cmdline, uint32_t flags);
/* waits for the writer, closes the files; < 0 when a write failed */
int sb_sam_close(sb_sam* sam);
/* unmapped-names lines the host writes itself (pairs too short to map), appended in call order */
int sb_sam_write_unmapped(sb_sam* sam, const char* text, size_t len);
typedef struct sb_sam_stats {
  uint64_t records, sam_bytes, unmapped_lines, batches, windows;
  double format_ms;           /* device time of the format kernels (CUDA events), all batches */
  double copy_ms;             /* host wall time of the windows' device->host copies */
  double slot_wait_ms;        /* host wall time the mapping thread waited for a page-locked buffer the writer held */
  double write_ms;            /* writer thread's wall time in fwrite */
} sb_sam_stats;
int sb_sam_get_stats(const sb_sam* sam, sb_sam_stats* out);
/* Attach a sink to a context (NULL detaches).  Without a sink sb_map_batch does exactly what it did before: no side
 * output, no extra kernel.  The device buffer of one window is "sam_window_bytes" (sb_map_set_option, 256 MiB). */
int sb_map_attach_sam(sb_map_ctx* ctx, sb_sam* sam);
/* sb_map_batch + SAM records of the batch.  names: the reads' names (mate 1), concatenated, read i at
 * names[name_off[i] .. name_off[i+1]); qual_left / qual_right: n_pairs x read_len quality characters (only with
 * SB_SAM_QUALITIES; NULL otherwise). */
int sb_map_batch_sam(sb_map_ctx* ctx, const uint8_t* left, const uint8_t* right, uint32_t n_pairs, uint32_t read_len,
                     const char* names, const uint64_t* name_off, const uint8_t* qual_left, const uint8_t* qual_right,
                     sb_map_batch_stats* stats);

/* Reads with their names (and optionally qualities): sb_reads_next that also returns, in *meta, the names of the
 * delivered records of the first mate file (up to the first white space, a trailing "/1" or "/2" removed) and, with
 * want_quals, both mates' quality lines laid out like the bases (stride bytes per read; FASTA records give 'I').
 * The arrays belong to the reader and stay valid until its next call. */
typedef struct sb_read_meta {
  const char* names;
  const uint64_t* name_off;        /* [n+1] */
  const uint8_t* qual_left;        /* NULL unless want_quals */
  const uint8_t* qual_right;
} sb_read_meta;
int64_t sb_reads_next_meta(sb_reads* r, uint32_t max_pairs, uint32_t stride, uint8_t* left, uint8_t* right,
                           uint32_t* len_left, uint32_t* len_right, int want_quals, sb_read_meta* meta);
/* sb_reads_bucketed whose callback also receives the rows' names and qualities (trimmed like the bases, read_len per
 * row).  too_short: called once on the calling thread at the end with the names of the pairs dropped as too short,
 * one per line (may be NULL). */
typedef int (*sb_batch_meta_cb)(void* user, const uint8_t* left, const uint8_t* right, uint32_t n_pairs, uint32_t read_len,
                                const sb_read_meta* meta);
typedef void (*sb_names_cb)(void* user, const char* names, size_t len);
int sb_reads_bucketed_meta(sb_reads* rd, uint32_t min_len, uint32_t batch, uint32_t max_read_len, uint32_t threads,
                           uint32_t shard_index, uint32_t shard_count, int want_quals, sb_batch_meta_cb cb,
                           sb_names_cb too_short, void* user, sb_bucket_stats* stats);

/* Debug: per-warp phase timestamps (ns) of one iteration of the last persistent run:
 * out[n_warps*16] = {P1 start, P1 end, barrier1 end, P2 start, P2 end, reduce end, barrier2 end, P2 home stream end,
 * P1 home stream end, then per phase (slots 9-10 P1, 11-12 P2) what the warp took from the long-row work queue:
 * long rows << 32 | their entries, longest row taken; -}.
 * Returns the number of warps (call with out=NULL to size the buffer). */
int sb_em_debug_timeline(sb_em_ctx* ctx, uint64_t* out, uint32_t iteration);

/* Debug: the library's CUDA resources, process-wide: out3 = {live buffers, streams and events; live buffer bytes;
 * buffers, streams and events made since the library was loaded}.  Leaks and reallocations show here even on a GPU
 * that other processes share. */
int sb_debug_device_memory(uint64_t out3[3]);

/* Tuning knobs (not part of the reference contract).  Unknown keys return SB_ERR_INVALID.
 * key: "variant" (0 = multi-kernel per iteration, 1 = persistent cooperative), "blocks_per_sm" (0 = as many as fit),
 *      "sell_group_cm" / "sell_group_tm" (rows per length-bucketing group, a power of two >= 32), "rebalance" (rounds
 *      of measured re-cutting of the warp ranges), "push_pass" (fused multi-GPU path: -1 by rank count, 0 push from the
 *      row epilogues, 1 coalesced pass), "sample_offset". */
int sb_em_set_option(sb_em_ctx* ctx, const char* key, int64_t value);

/* Figures of the layout sb_em_prepare built (after prepare).  key: "stream_bytes" (bytes one iteration streams:
 * both SELL matrices at 10 bytes per entry, padding included, + the long rows' CSR at 12), or per matrix with the
 * suffix "_cm" (class-major) / "_tm" (transcript-major): "stream_bytes", "sell_cols" (SELL columns of 32 entries),
 * "long_rows", "long_entries", "fallback_rows" (rows on the long-row path only because their slice's indices span
 * more than 16 bits); "warps" (warps of the iteration grid, which the slice ranges were cut for), "ring_cols" (columns
 * one warp's stream ring holds), "sum_scale_log2" (s: the iteration sums alpha' + prior in fixed point, in units
 * of 2^-s; 20, or less when the class counts and priors are large enough to need it). */
int sb_em_get_info(sb_em_ctx* ctx, const char* key, int64_t* value);

/* ---- multi-GPU: classes stay sharded per rank, alpha is all-reduced once per
 * iteration (the only collective; SURVEY.md section 8e).  The caller provides
 * the NCCL unique id (128 bytes, from sb_nccl_unique_id on rank 0, broadcast
 * by whatever the host uses -- bench.py uses torch.distributed). */
int sb_nccl_unique_id(void* out128);
int sb_em_comm_init(sb_em_ctx* ctx, int rank, int nranks, const void* unique_id128);
int sb_em_comm_destroy(sb_em_ctx* ctx);
/* Fused all-reduce (GPUs of one box, NVLink P2P): every rank allocates an exchange block (sb_em_peer_handle returns
 * its 64-byte CUDA IPC handle), the host layer all-gathers the handles, sb_em_peer_open maps the peers' blocks.  From
 * then on sb_em_optimize / sb_em_run iterate inside ONE persistent kernel per rank that all-reduces alpha' over peer
 * memory (reduce-scatter + all-gather with in-kernel GPU-to-GPU barriers) instead of calling NCCL per iteration.
 * Without peers the NCCL path (sb_em_comm_init) is used. */
int sb_em_peer_handle(sb_em_ctx* ctx, uint32_t max_txps, void* out64);
int sb_em_peer_open(sb_em_ctx* ctx, int rank, int nranks, const void* handles /* nranks x 64 bytes */);

/* Write a buffer larger than L2 (bench hygiene between timed steps). */
int sb_flush_l2(sb_em_ctx* ctx);

/* Page-lock / unlock a host buffer the caller will pass to sb_em_optimize / sb_em_upload
 * repeatedly (cudaHostRegister), so the host->device copies run at full PCIe rate. */
int sb_host_register(void* ptr, size_t bytes);
int sb_host_unregister(void* ptr);

#ifdef __cplusplus
}
#endif
#endif /* SALMON_B200_H */
