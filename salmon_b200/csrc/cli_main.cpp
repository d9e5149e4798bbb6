// sb_salmon -- thin command-line front end over the C ABI (include/salmon_b200.h), keeping the `salmon index` /
// `salmon quant` invocations of the hot path (option names from src/core/ProgramOptionsGenerator.cpp:85-289 and
// src/index/BuildSalmonIndex.cpp:72-124).  No logic of its own: argument parsing, then sb_txome_read_fasta +
// sb_index_build + sb_index_save, or sb_index_load + sb_quant_files, or sb_eq_file_read + sb_em_optimize.
// Options outside the hot path (bias models, alignment mode, SAM output, ...) are rejected with a message.
#include <signal.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <sys/stat.h>
#include <sys/wait.h>
#include <unistd.h>

#include <algorithm>
#include <string>
#include <thread>
#include <vector>

#include "../../include/salmon_b200.h"

static double now_wall() {
  timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}
static const double T_PROCESS_START = now_wall();

// the per-rank child processes of `quant --gpus N`: a signal that ends the parent ends them too
static pid_t g_kids[64];
static volatile sig_atomic_t g_n_kids = 0;
static void forward_signal(int sig) {
  for (int i = 0; i < g_n_kids; ++i) if (g_kids[i] > 0) kill(g_kids[i], SIGTERM);
  _exit(128 + sig);
}

namespace {

int die(const char* what) {
  fprintf(stderr, "sb_salmon: %s: %s\n", what, sb_last_error());
  return 1;
}

struct Args {
  std::vector<std::string> v;
  std::vector<std::string> all;    // the arguments as given (cmd_info.json, re-execution per rank)
  std::string argv0;
  size_t i = 0;
  bool more() const { return i < v.size(); }
  const std::string& peek() const { return v[i]; }
  std::string next() { return v[i++]; }
  bool value(std::string& out) {
    if (!more()) return false;
    out = next();
    return true;
  }
  // file lists: everything up to the next option
  void list(std::vector<std::string>& out) {
    while (more() && !(peek().size() > 1 && peek()[0] == '-')) {
      std::string a = next();
      size_t b = 0;   // also accept comma-separated lists
      while (b <= a.size()) {
        size_t e = a.find(',', b);
        if (e == std::string::npos) e = a.size();
        if (e > b) out.push_back(a.substr(b, e - b));
        b = e + 1;
      }
    }
  }
};

int usage() {
  fprintf(stderr,
          "sb_salmon (salmon-b200 %d): H100-native hot path of salmon\n"
          "  sb_salmon index -t transcripts.fa[.gz] -i index_dir [-k 31] [--gencode] [-d decoys.txt] [--keepDuplicates] [--no-clip]\n"
          "  sb_salmon quant -i index_dir -l IU|ISF|ISR -1 r1.fq[.gz] ... -2 r2.fq[.gz] ... | -l U|SF|SR -r reads.fq[.gz] ...  -o out_dir [--gpus N]\n"
          "                  [-p threads] [--dumpEq] [--dumpEqWeights] [--writeMappings[=FILE] | -z] [--writeQualities] [--writeUnmappedNames]\n"
          "                  [--recoverOrphans] [--softclip] [--softclipOverhangs] [--incompatPrior 0] [--noSingleFragProb]\n"
          "                  [--mimicBT2 | --mimicStrictBT2] [--minAlnProb 1e-5]\n"
          "                  [--noFragLengthDist --noEffectiveLengthCorrection | --noEffectiveLengthCorrection]\n"
          "                  [--numBootstraps N | --numGibbsSamples N] [--thinningFactor 16] [--noGammaDraw] [--useEM] [--vbPrior 0.01]\n"
          "                  [--bootstrapReproject] [--meta] [--alternativeInitMode] [--skipQuant]\n"
          "                  [--perNucleotidePrior] [--maxReadOcc 200] [--maxOccsPerHit 1000] [--minScoreFraction 0.65] [--consensusSlack 0.35]\n"
          "                  [--preMergeChainSubThresh 0.75] [--postMergeChainSubThresh 0.9] [--orphanChainSubThresh 0.95] [--allowDovetail]\n"
          "                  [--discardOrphansQuasi] [--hardFilter] [--rangeFactorizationBins 4] [--fldMean 250] [--fldSD 25] [--fldMax 1000] [--scoreExp 1]\n"
          "                  [--numPreAuxModelSamples 5000] [--numAuxModelSamples 5000000] [--gpu 0] [--batch 262144] [--maxReadLen 256] [--seed 42]\n"
          "  sb_salmon quant -e eq_classes.txt[.gz] -o out_dir [--useEM] [--numBootstraps N] [--bootstrapReproject] [--meta]\n"
          "                  [--alternativeInitMode]\n",
          sb_version());
  return 1;
}

int cmd_index(Args& a) {
  std::string fasta, dir, decoys, v;
  uint32_t k = 31;
  int gencode = 0, keep_dup = 0, no_clip = 0;
  while (a.more()) {
    const std::string o = a.next();
    if (o == "-t" || o == "--transcripts") { if (!a.value(fasta)) return usage(); }
    else if (o == "-i" || o == "--index") { if (!a.value(dir)) return usage(); }
    else if (o == "-k" || o == "--kmerLen") { if (!a.value(v)) return usage(); k = (uint32_t)atoi(v.c_str()); }
    else if (o == "-d" || o == "--decoys") { if (!a.value(decoys)) return usage(); }
    else if (o == "--gencode") gencode = 1;
    else if (o == "--keepDuplicates") keep_dup = 1;
    else if (o == "-n" || o == "--no-clip") no_clip = 1;
    else if (o == "-p" || o == "--threads" || o == "--type" || o == "-m" || o == "--minimizerLen" || o == "-f" ||
             o == "--filterSize" || o == "--tmpdir") { a.value(v); /* accepted, not needed by this index */ }
    else if (o == "--keepFixedFasta" || o == "--features") { fprintf(stderr, "sb_salmon index: %s is not supported\n", o.c_str()); return 1; }
    else { fprintf(stderr, "sb_salmon index: unknown option %s\n", o.c_str()); return usage(); }
  }
  if (fasta.empty() || dir.empty()) return usage();
  if (k == 0) k = 31;
  if ((k & 1) == 0) { fprintf(stderr, "Error: k must be an odd value, you chose %u.\n", k); return 1; }   // BuildSalmonIndex.cpp:206-211
  if (k > 31) { fprintf(stderr, "Error: k must not be larger than 31, you chose %u.\n", k); return 1; }
  sb_txome* t = nullptr;
  if (sb_txome_read_fasta(fasta.c_str(), k, gencode, decoys.empty() ? nullptr : decoys.c_str(), no_clip, keep_dup, &t) != 0)
    return die("reading the transcripts");
  fprintf(stderr, "read %u sequences (%u decoys), %llu bases; %u duplicates removed, %u poly-A tails clipped, %u shorter than k\n",
          t->n_txps, t->n_txps - t->first_decoy, (unsigned long long)t->seq_off[t->n_txps], t->n_duplicates_removed, t->n_clipped,
          t->n_short);
  sb_index* ix = sb_index_build(t->n_txps, t->seq_off, t->codes, k);
  if (!ix) return die("building the index");
  sb_index_set_meta(ix, t->names, t->complete_len, t->first_decoy);
  mkdir(dir.c_str(), 0777);
  if (sb_index_save(ix, (dir + "/sb_index.bin").c_str()) != 0) return die("writing the index");
  uint64_t info[4] = {0, 0, 0, 0};
  sb_index_info(ix, info);
  if (FILE* f = fopen((dir + "/info.json").c_str(), "w")) {
    fprintf(f, "{\n  \"index_type\": \"sb_kmer_table\",\n  \"k\": %u,\n  \"num_references\": %u,\n  \"first_decoy\": %u,\n"
               "  \"num_kmers\": %llu,\n  \"num_postings\": %llu,\n  \"table_capacity\": %llu,\n  \"bytes\": %llu\n}\n",
            k, t->n_txps, t->first_decoy, (unsigned long long)info[0], (unsigned long long)info[1], (unsigned long long)info[2],
            (unsigned long long)info[3]);
    fclose(f);
  }
  fprintf(stderr, "index: %llu distinct %u-mers, %llu postings, %.1f MB -> %s\n", (unsigned long long)info[0], k,
          (unsigned long long)info[1], (double)info[3] / 1e6, dir.c_str());
  sb_index_free(ix);
  sb_txome_free(t);
  return 0;
}

int quant_eqclasses(const std::string& eqfile, const std::string& out, const sb_em_params& ep, const sb_quant_opts& qo) {
  sb_quant_summary sum;
  if (sb_quant_eqclasses(eqfile.c_str(), &ep, &qo, out.c_str(), &sum) != 0) return die("quant -e");
  if (qo.shard_index == 0)
    fprintf(stderr, "%llu classes: %u iterations (%s) in %.2f s, total %.2f s on %u GPU(s)\n", (unsigned long long)sum.n_classes,
            sum.em_iters, sum.em_converged ? "converged" : "iteration limit", sum.em_seconds, sum.total_seconds, qo.shard_count ? qo.shard_count : 1);
  return 0;
}

// cmd_info.json (salmon::utils::writeCmdInfo): the options as given
void write_cmd_info(const std::string& out, const std::vector<std::string>& argv_all) {
  FILE* f = fopen((out + "/cmd_info.json").c_str(), "w");
  if (!f) return;
  fprintf(f, "{\n    \"salmon_version\": \"1.11.4-sb%d\"", sb_version());
  std::string key;
  std::vector<std::string> vals;
  auto flush = [&]() {
    if (key.empty()) return;
    fprintf(f, ",\n    \"%s\": ", key.c_str());
    if (vals.empty()) fprintf(f, "[]");
    else if (vals.size() == 1) fprintf(f, "\"%s\"", vals[0].c_str());
    else { fprintf(f, "["); for (size_t i = 0; i < vals.size(); ++i) fprintf(f, "%s\"%s\"", i ? ", " : "", vals[i].c_str()); fprintf(f, "]"); }
  };
  static const char* const short_names[][2] = {{"i", "index"}, {"l", "libType"}, {"1", "mates1"}, {"2", "mates2"},
                                                {"o", "output"}, {"p", "threads"}, {"r", "unmatedReads"}, {"e", "eqclasses"},
                                                {"d", "dumpEqWeights"}, {"q", "quiet"}};
  for (const std::string& a : argv_all) {
    const bool is_opt = a.size() > 1 && a[0] == '-' && (a == "-1" || a == "-2" || !(a[1] >= '0' && a[1] <= '9'));
    if (is_opt) {
      flush();
      key = a.substr(a.find_first_not_of('-'));
      for (auto& sn : short_names) if (key == sn[0]) key = sn[1];
      if (key.size() > 1 && key[0] == '_') key.clear();       // the per-rank re-execution's own options
      vals.clear();
    } else if (!key.empty()) {
      vals.push_back(a);
    }
  }
  flush();
  fprintf(f, "\n}\n");
  fclose(f);
}

// rank 0 writes the communicator id into the output directory, the other ranks wait for it
bool exchange_uid(const std::string& out, int rank, const std::string& tag, unsigned char* uid) {
  const std::string path = out + "/.sb_nccl_uid_" + tag;
  if (rank == 0) {
    if (sb_nccl_unique_id(uid) != 0) return false;
    const std::string tmp = path + ".tmp";
    FILE* f = fopen(tmp.c_str(), "wb");
    if (!f || fwrite(uid, 1, 128, f) != 128) { if (f) fclose(f); return false; }
    fclose(f);
    return rename(tmp.c_str(), path.c_str()) == 0;
  }
  for (int tries = 0; tries < 6000; ++tries) {       // up to 60 s
    FILE* f = fopen(path.c_str(), "rb");
    if (f) {
      const size_t n = fread(uid, 1, 128, f);
      fclose(f);
      if (n == 128) return true;
    }
    usleep(10000);
  }
  return false;
}

int cmd_quant(Args& a) {
  std::string dir, out, lib = "A", eqfile, v;
  std::vector<std::string> m1, m2, unmated;
  sb_map_params mp;
  sb_em_params ep;
  sb_quant_opts qo;
  sb_map_default_params(&mp);
  sb_em_default_params(&ep);
  sb_quant_default_opts(&qo);
  auto num = [&](double& d) { if (!a.value(v)) return false; d = atof(v.c_str()); return true; };
  double d = 0;
  bool vb_prior_given = false, pre_merge_given = false, threads_given = false, mimic = false, mimic_strict = false;
  bool meta = false;
  int n_gpus = 1, my_rank = -1;
  std::string run_tag, sam_path;
  while (a.more()) {
    const std::string o = a.next();
    if (o == "-i" || o == "--index") { if (!a.value(dir)) return usage(); }
    else if (o == "-o" || o == "--output") { if (!a.value(out)) return usage(); }
    else if (o == "-l" || o == "--libType") { if (!a.value(lib)) return usage(); }
    else if (o == "-1" || o == "--mates1") a.list(m1);
    else if (o == "-2" || o == "--mates2") a.list(m2);
    else if (o == "-r" || o == "--unmatedReads") a.list(unmated);
    else if (o == "-e" || o == "--eqclasses") { if (!a.value(eqfile)) return usage(); }
    else if (o == "-p" || o == "--threads") { if (!num(d)) return usage(); qo.threads = (uint32_t)d; threads_given = true; }
    else if (o == "--dumpEq") qo.dump_eq = 1;
    else if (o == "-d" || o == "--dumpEqWeights") qo.dump_eq_weights = 1;
    else if (o == "--numBootstraps") { if (!num(d)) return usage(); qo.num_bootstraps = (uint32_t)d; }
    else if (o == "--numGibbsSamples") { if (!num(d)) return usage(); qo.num_gibbs = (uint32_t)d; }
    else if (o == "--thinningFactor") { if (!num(d)) return usage(); qo.thinning = (uint32_t)d; }
    else if (o == "--noGammaDraw") qo.no_gamma_draw = 1;
    else if (o == "--useEM") ep.use_vbem = 0;
    else if (o == "--useVBOpt") ep.use_vbem = 1;
    else if (o == "--vbPrior") { if (!num(ep.vb_prior)) return usage(); vb_prior_given = true; }
    else if (o == "--perNucleotidePrior") ep.per_txp_prior = 0;
    else if (o == "--perTranscriptPrior") ep.per_txp_prior = 1;
    else if (o == "--initUniform") ep.init_uniform = 1;
    else if (o == "--noLengthCorrection") ep.no_length_correction = 1;
    else if (o == "--noRichEqClasses") ep.no_rich_eq = 1;
    else if (o == "--meta") meta = true;
    else if (o == "--alternativeInitMode") ep.alt_init = 1;
    else if (o == "--bootstrapReproject") ep.bootstrap_reproject = 1;
    else if (o == "--skipQuant") qo.skip_quant = 1;
    else if (o == "--maxReadOcc") { if (!num(d)) return usage(); mp.max_read_occ = (uint32_t)d; }
    else if (o == "--maxOccsPerHit") { if (!num(d)) return usage(); mp.max_occs_per_hit = (uint32_t)d; }
    else if (o == "--minScoreFraction") { if (!num(mp.min_score_fraction)) return usage(); }
    else if (o == "--consensusSlack") { if (!num(d)) return usage(); mp.consensus_frac = 1.0 - d; }
    else if (o == "--hardFilter") mp.hard_filter = 1;
    else if (o == "--preMergeChainSubThresh") { if (!num(mp.pre_merge_thresh)) return usage(); pre_merge_given = true; }
    else if (o == "--postMergeChainSubThresh") { if (!num(mp.post_merge_thresh)) return usage(); }
    else if (o == "--orphanChainSubThresh") { if (!num(mp.orphan_thresh)) return usage(); }
    else if (o == "--allowDovetail") mp.allow_dovetail = 1;
    else if (o == "--discardOrphansQuasi") mp.allow_orphans = 0;
    else if (o == "--rangeFactorizationBins") { if (!num(d)) return usage(); mp.range_bins = (uint32_t)d; }
    else if (o == "--fldMean") { if (!num(mp.fld_mean)) return usage(); }
    else if (o == "--fldSD") { if (!num(mp.fld_sd)) return usage(); }
    else if (o == "--fldMax") { if (!num(d)) return usage(); mp.max_frag_len = (uint32_t)d; }
    else if (o == "--scoreExp") { if (!num(mp.score_exp)) return usage(); }
    else if (o == "--decoyThreshold") { if (!num(mp.decoy_threshold)) return usage(); }
    else if (o == "--ma") { if (!num(d)) return usage(); mp.ma = (int32_t)d; }
    else if (o == "--mp") { if (!num(d)) return usage(); mp.mp = (int32_t)d; }
    else if (o == "--go") { if (!num(d)) return usage(); mp.go = (int32_t)d; }
    else if (o == "--ge") { if (!num(d)) return usage(); mp.ge = (int32_t)d; }
    else if (o == "--bandwidth") { if (!num(d)) return usage(); mp.band = (uint32_t)d; }
    else if (o == "--numPreAuxModelSamples") { if (!num(d)) return usage(); mp.num_pre_burnin = (uint64_t)d; }
    else if (o == "--numAuxModelSamples") { if (!num(d)) return usage(); mp.num_burnin = (uint64_t)d; }
    else if (o == "--gpu") { if (!num(d)) return usage(); qo.device = (int32_t)d; }
    else if (o == "--gpus" || o == "--numGpus") { if (!num(d)) return usage(); n_gpus = (int)d; }
    else if (o == "--_rank") { if (!num(d)) return usage(); my_rank = (int)d; }
    else if (o == "--_tag") { if (!a.value(run_tag)) return usage(); }
    else if (o == "--batch") { if (!num(d)) return usage(); qo.batch = (uint32_t)d; }
    else if (o == "--maxReadLen") { if (!num(d)) return usage(); qo.max_read_len = (uint32_t)d; }
    else if (o == "--seed") { if (!num(d)) return usage(); qo.seed = (uint64_t)d; mp.seed = (uint64_t)d; }
    else if (o == "--validateMappings" || o == "-q" || o == "--quiet") { /* default behaviour / no-op */ }
    else if (o == "--softclipOverhangs") { if (mp.softclip < 1) mp.softclip = 1; }   // --softclip includes it
    else if (o == "--softclip") mp.softclip = 2;
    else if (o == "--writeMappings" || o == "-z") sam_path = "-";   // (SAM on standard output)
    else if (o.rfind("--writeMappings=", 0) == 0) sam_path = o.substr(16);
    else if (o == "--writeQualities") qo.write_qualities = 1;
    else if (o == "--writeUnmappedNames") qo.write_unmapped_names = 1;
    else if (o == "--recoverOrphans") mp.recover_orphans = 1;
    else if (o == "--incompatPrior") {
      if (!a.value(v)) return usage();
      char* end = nullptr;
      const double x = strtod(v.c_str(), &end);
      if (v.empty() || *end != '\0' || !(x >= 0.0 && x <= 1.0)) {
        fprintf(stderr, "sb_salmon quant: --incompatPrior takes a probability in [0, 1], got '%s'\n", v.c_str());
        return 1;
      }
      // 0 or below 1e-100: incompatible mappings are ignored (QuantOptionsUtils.cpp:608-616)
      mp.incompat_prior = (x == 0.0 || x < 1e-100) ? 0.0 : x;
    }
    else if (o == "--minAlnProb") {
      if (!a.value(v)) return usage();
      char* end = nullptr;
      const double x = strtod(v.c_str(), &end);
      if (v.empty() || *end != '\0' || !(x >= 0.0 && x <= 1.0)) {
        fprintf(stderr, "sb_salmon quant: --minAlnProb takes a probability in [0, 1], got '%s'\n", v.c_str());
        return 1;
      }
      mp.min_aln_prob = x;
    }
    else if (o == "--mimicBT2") mimic = true;
    else if (o == "--mimicStrictBT2") mimic_strict = true;
    else if (o == "--noSingleFragProb") mp.no_single_frag_prob = 1;
    else if (o == "--noFragLengthDist") mp.no_frag_len_dist = 1;
    else if (o == "--noEffectiveLengthCorrection") mp.no_eff_len_correction = 1;
    else if (o == "--seqBias" || o == "--gcBias" || o == "--posBias" || o == "-a" ||
             o == "--alignments" || o == "-g" || o == "--geneMap" || o == "--sketchMode") {
      fprintf(stderr, "sb_salmon quant: %s is outside the hot path this build replaces (DESIGN.md, out of scope)\n", o.c_str());
      return 1;
    } else { fprintf(stderr, "sb_salmon quant: unknown option %s\n", o.c_str()); return usage(); }
  }
  if (out.empty()) return usage();
  if (meta) {   // a preset over the options given, whatever their order (QuantOptionsUtils.cpp:449-454)
    ep.init_uniform = 1;
    ep.no_rich_eq = 1;
    ep.use_vbem = 0;
    ep.alt_init = 1;   // (metaGenomeMode, CollapsedEMOptimizer.cpp:800-810; no effect beside initUniform)
    if (my_rank <= 0)
      fprintf(stderr, "[info] --meta sets --useEM --initUniform --noRichEqClasses, whatever else the command line says "
                      "about them.\n");
  }
  if (qo.skip_quant && !eqfile.empty()) {
    fprintf(stderr, "sb_salmon quant: --skipQuant applies to mapping mode; with --eqclasses there is nothing to skip to\n");
    return 1;
  }
  if (mimic && mimic_strict) {   // QuantOptionsUtils.cpp:250-254
    fprintf(stderr, "sb_salmon quant: You passed both the --mimicBT2 and --mimicStrictBT2 parameters.  These are mutually "
                    "exclusive. Please select only one of these flags.\n");
    return 1;
  }
  if (mp.no_frag_len_dist && !mp.no_eff_len_correction) {   // QuantOptionsUtils.cpp:641-647
    fprintf(stderr, "sb_salmon quant: You cannot enable --noFragLengthDist without also enabling --noEffectiveLengthCorrection\n");
    return 1;
  }
  if (n_gpus > 1 && (!sam_path.empty() || qo.write_unmapped_names)) {
    fprintf(stderr, "sb_salmon quant: --writeMappings / --writeUnmappedNames are written by a one-GPU run only: a read-sharded "
                    "--gpus %d run cannot write them\n", n_gpus);
    return 1;
  }
  if (sam_path.empty() && qo.write_qualities) { fprintf(stderr, "sb_salmon quant: --writeQualities needs --writeMappings\n"); return 1; }
  std::string cmdline = "sb_salmon quant";
  for (const std::string& arg : a.all) cmdline += " " + arg;
  if (!sam_path.empty()) qo.write_mappings = sam_path.c_str();
  qo.cmdline = cmdline.c_str();
  if (!threads_given) {   // host threads for the reader (inflate, scan, translate): half the hardware threads, 32 at most
    const unsigned hw = std::thread::hardware_concurrency();
    qo.threads = std::max(2u, std::min(32u, hw / 2 / (unsigned)std::max(1, n_gpus)));   // (per rank)
  }
  // --perNucleotidePrior without an explicit --vbPrior: the reference switches the default to 1e-5
  // (src/cli/QuantOptionsUtils.cpp:569-572)
  if (ep.use_vbem && !ep.per_txp_prior && !vb_prior_given) ep.vb_prior = 1e-5;
  mkdir(out.c_str(), 0777);
  // ---- multi-GPU: one process per GPU.  The parent re-executes itself once per rank; rank r uses GPU r.
  if (n_gpus > 1 && my_rank < 0) {
    const int have = sb_device_count();
    if (have < n_gpus) { fprintf(stderr, "sb_salmon quant: --gpus %d but %d CUDA device(s) visible\n", n_gpus, have); return 1; }
    char tag[64];
    snprintf(tag, sizeof tag, "%ld_%d", (long)time(nullptr), (int)getpid());
    std::vector<pid_t> kids;
    for (int r = 0; r < n_gpus; ++r) {
      pid_t pid = fork();
      if (pid < 0) { perror("fork"); return 1; }
      if (pid == 0) {
        std::vector<std::string> av = a.all;
        av.push_back("--_rank"); av.push_back(std::to_string(r));
        av.push_back("--_tag"); av.push_back(tag);
        std::vector<char*> cv;
        cv.push_back(const_cast<char*>(a.argv0.c_str()));
        cv.push_back(const_cast<char*>("quant"));
        for (auto& x : av) cv.push_back(const_cast<char*>(x.c_str()));
        cv.push_back(nullptr);
        execv(a.argv0.c_str(), cv.data());
        perror("execv");
        _exit(127);
      }
      kids.push_back(pid);
      if (g_n_kids < 64) { g_kids[g_n_kids] = pid; g_n_kids = g_n_kids + 1; }
    }
    signal(SIGTERM, forward_signal);
    signal(SIGINT, forward_signal);
    // a rank that fails leaves the others waiting in a collective: the first failure ends the run for all of them
    int bad = 0;
    size_t left = kids.size();
    while (left > 0) {
      int st = 0;
      const pid_t k = wait(&st);
      if (k < 0) break;
      bool ours = false;
      for (size_t i = 0; i < kids.size(); ++i)
        if (kids[i] == k) { ours = true; kids[i] = -1; }
      if (!ours) continue;
      --left;
      if (!WIFEXITED(st) || WEXITSTATUS(st) != 0) {
        if (!bad) {
          fprintf(stderr, "sb_salmon quant: a rank failed (%s %d); stopping the other ranks\n", WIFEXITED(st) ? "exit code" : "signal",
                  WIFEXITED(st) ? WEXITSTATUS(st) : WTERMSIG(st));
          for (pid_t o : kids) if (o > 0) kill(o, SIGTERM);
        }
        bad = 1;
      }
    }
    unlink((out + "/.sb_nccl_uid_" + tag).c_str());
    return bad;
  }
  unsigned char uid[128];
  if (n_gpus > 1) {
    qo.shard_index = (uint32_t)my_rank; qo.shard_count = (uint32_t)n_gpus; qo.device = my_rank;
    if (!exchange_uid(out, my_rank, run_tag, uid)) { fprintf(stderr, "sb_salmon quant: rank %d could not obtain the communicator id\n", my_rank); return 1; }
    qo.nccl_uid = uid;
  }
  if (qo.shard_index == 0) write_cmd_info(out, a.all);
  if (!eqfile.empty()) return quant_eqclasses(eqfile, out, ep, qo);
  if (dir.empty()) return usage();
  // library type (-l): IU / ISF / ISR for mate files, U / SF / SR for unmated reads; A = the unstranded type of the input
  static const struct { const char* name; int id; } lib_names[] = {{"IU", SB_LIB_IU}, {"ISF", SB_LIB_ISF}, {"ISR", SB_LIB_ISR},
                                                                   {"U", SB_LIB_U}, {"SF", SB_LIB_SF}, {"SR", SB_LIB_SR}};
  const bool se_input = !unmated.empty();
  if (se_input ? (!m1.empty() || !m2.empty()) : (m1.empty() || m1.size() != m2.size())) {
    fprintf(stderr, "sb_salmon quant: give either mate files (-1 / -2, the same number of each) or unmated reads (-r)\n");
    return 1;
  }
  int lib_id = -1;
  if (lib == "A") lib_id = se_input ? SB_LIB_AUTO_SINGLE : SB_LIB_AUTO_PAIRED;   // detected from the first 50 000 stranded fragments
  for (auto& ln : lib_names) if (lib == ln.name) lib_id = ln.id;
  if (lib_id < 0 || ((lib_id >= SB_LIB_U && lib_id != SB_LIB_AUTO_PAIRED) != se_input)) {
    fprintf(stderr, "sb_salmon quant: library type %s does not fit the input (IU / ISF / ISR with -1 -2, U / SF / SR with -r; "
                    "outward and same-strand types are not supported)\n", lib.c_str());
    return 1;
  }
  mp.lib_type = lib_id;
  if (mimic || mimic_strict) {   // the presets override the values given for the same options (:256-289)
    const bool overhangs = mp.softclip == 1;
    sb_map_mimic_bt2(&mp, mimic_strict ? 1 : 0);
    if (my_rank <= 0) {
      fprintf(stderr, "[info] The --mimicBT2 and --mimicStrictBT2 flags increases maxReadOccs to %u.\n", mp.max_read_occ);
      fprintf(stderr, "[info] The --mimicBT2 and --mimicStrictBT2 flags increases consensusSlack to %g.\n", 1.0 - mp.consensus_frac);
      fprintf(stderr, mimic_strict ? "[info] Usage of --mimicStrictBT2 overrides other settings for mapping validation. Setting "
                                     "strict RSEM+Bowtie2-like parameters now.\n"
                                   : "[info] Usage of --mimicBT2 overrides other settings for mapping validation. Setting "
                                     "Bowtie2-like parameters now.\n");
      if (overhangs)
        fprintf(stderr, "[info] Softclipping of overhangs is not allowed in %s mode; setting to false.\n",
                mimic_strict ? "mimicStrictBT2" : "mimicBT2");
    }
  }
  if (se_input && !pre_merge_given) mp.pre_merge_thresh = 1.0;    // single-end default (QuantOptionsUtils.cpp:215-218)
  if (se_input) mp.recover_orphans = 0;   // a single-end read has no mate to rescue: accepted, no effect (as in salmon)
  // the CUDA context comes up (seconds) while the index is read from disk
  const double t_start = now_wall();
  std::thread ctx_thread([&] { sb_device_init(qo.device); });
  sb_index* ix = sb_index_load((dir + "/sb_index.bin").c_str());
  const double t_loaded = now_wall();
  ctx_thread.join();
  if (!ix) return die("loading the index");
  if (qo.shard_index == 0)
    fprintf(stderr, "index loaded in %.2f s (CUDA context ready after %.2f s)\n", t_loaded - t_start, now_wall() - t_start);
  std::vector<const char*> p1, p2;
  for (auto& s : (se_input ? unmated : m1)) p1.push_back(s.c_str());
  for (auto& s : m2) p2.push_back(s.c_str());
  sb_quant_summary sum;
  if (sb_quant_files(ix, p1.data(), se_input ? nullptr : p2.data(), (uint32_t)p1.size(), &mp, &ep, &qo, out.c_str(), nullptr, &sum) != 0)
    return die("quant");
  if (qo.shard_index == 0) {
    const double rate = sum.n_observed ? 100.0 * (double)sum.n_mapped / (double)sum.n_observed : 0.0;
    fprintf(stderr, "%llu fragments observed, %llu mapped (%.4f%%), %llu equivalence classes%s; %u read lengths, %llu batches%s\n",
            (unsigned long long)sum.n_observed, (unsigned long long)sum.n_mapped, rate, (unsigned long long)sum.n_classes,
            n_gpus > 1 ? " on rank 0" : "", sum.n_read_lengths, (unsigned long long)sum.n_batches, n_gpus > 1 ? " on rank 0" : "");
    fprintf(stderr, "mapping %.2f s (%.1f ms on the device, %.2f M fragments/s end to end, %d GPU(s)), optimiser %u iterations in %.2f s, total %.2f s; mapping set-up %.2f s\n",
            sum.map_seconds, sum.map_device_ms, sum.map_seconds > 0 ? (double)sum.n_observed / sum.map_seconds / 1e6 : 0.0, n_gpus, sum.em_iters,
            sum.em_seconds, sum.total_seconds, (double)sum.map_setup_ms * 1e-3);
    if (mp.recover_orphans)
      fprintf(stderr, "Number of orphans recovered using orphan rescue : %llu%s (%llu mate searches, %llu without room)\n",
              (unsigned long long)sum.orphans_rescued, n_gpus > 1 ? " on rank 0" : "", (unsigned long long)sum.rescue_searches,
              (unsigned long long)sum.rescue_no_room);
  }
  if (qo.shard_index == 0) fprintf(stderr, "done %.2f s after the process started\n", now_wall() - T_PROCESS_START);
  // the outputs are written and closed: leave without tearing down 10+ GB of host and device state piece by piece
  fflush(nullptr);
  _exit(0);
}

}  // namespace

int main(int argc, char** argv) {
  if (argc < 2) return usage();
  Args a;
  for (int i = 2; i < argc; ++i) a.v.push_back(argv[i]);
  a.all = a.v;
  {   // the executable's own path, for the per-rank re-execution
    char self[4096];
    const ssize_t n = readlink("/proc/self/exe", self, sizeof self - 1);
    a.argv0 = n > 0 ? std::string(self, (size_t)n) : std::string(argv[0]);
  }
  const std::string cmd = argv[1];
  if (cmd == "index") return cmd_index(a);
  if (cmd == "quant") return cmd_quant(a);
  if (cmd == "--version" || cmd == "-v") { printf("sb_salmon %d\n", sb_version()); return 0; }
  return usage();
}
