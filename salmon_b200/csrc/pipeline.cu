// pipeline.cu -- the host driver of the hot path (C++, no kernels of its own): what processReadLibrary / quantifyLibrary
// / stageFinalizeMappingOutputs do around the seams in the reference (src/quant/SalmonQuantify.cpp:2339-2730 spawn the
// parser + worker threads; src/quant/pipeline/MappingPipelineStages.cpp:37-206 optimise and write), here as
//
//     reader thread:  sb_reads_next -> rows grouped by read length into pinned [n, L] buffers   (host cores)
//     caller thread:  sb_map_batch per full buffer                                              (GPU)
//     then:           sb_map_finish -> sb_em_optimize -> (sb_bootstrap | sb_gibbs) -> quant.sf, eq_classes, bootstraps.gz
//
// so parsing / packing of the next batch overlaps the kernels of the current one.  One GPU per call; multi-GPU runs
// shard the read stream over processes (shard_index / shard_count) and do the once-per-run reduction in the host layer
// (salmon_b200/dist.py).  sb_map_batch takes one read length per call: a pair whose mates differ in length is mapped
// at the shorter length (documented deviation until the kernels take per-mate lengths).
#include <errno.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/stat.h>
#include <time.h>
#include <zlib.h>

#include <cmath>
#include <condition_variable>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <random>
#include <string>
#include <thread>
#include <vector>

#include "common.cuh"

namespace {

double now_s() {
  timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

struct HostBuf {   // pinned [cap, L] byte matrix pair
  uint8_t* left = nullptr;
  uint8_t* right = nullptr;
  uint32_t cap = 0, L = 0, n = 0;
  bool busy = false;   // handed to the consumer side
  bool pinned = false;
  // sb_reads_bucketed_meta: the rows' names (concatenated, name_off[row]) and quality lines ([cap, L] per mate)
  std::string names;
  std::vector<uint64_t> name_off;
  std::vector<uint8_t> qual[2];
  int alloc(uint32_t cap_, uint32_t L_) {
    cap = cap_; L = L_; n = 0;
    const size_t bytes = (size_t)cap * L;
    // page-locked when a CUDA device is there (the consumer copies these to the GPU), plain memory otherwise
    if (cudaMallocHost(&left, bytes) == cudaSuccess && cudaMallocHost(&right, bytes) == cudaSuccess) { pinned = true; return SB_OK; }
    cudaGetLastError();
    if (left) { cudaFreeHost(left); left = nullptr; }
    left = (uint8_t*)malloc(bytes ? bytes : 1);
    right = (uint8_t*)malloc(bytes ? bytes : 1);
    if (!left || !right) { sb::set_error("cannot allocate %zu bytes of host memory", 2 * bytes); return SB_ERR_NOMEM; }
    return SB_OK;
  }
  void release() {
    if (pinned) { if (left) cudaFreeHost(left); if (right) cudaFreeHost(right); }
    else { free(left); free(right); }
    left = right = nullptr;
  }
};

struct Bucket {   // reads of one length: two buffers, the reader fills one while the GPU consumes the other
  HostBuf buf[2];
  int fill = 0;
  uint32_t cnt = 0;        // rows in buf[fill] (reader-private; HostBuf::n is set at submit)
  bool checked = true;     // buf[fill] is known to be released by the GPU side
};

struct Job {
  HostBuf* b;
};

struct Pipe {
  std::mutex mu;
  std::condition_variable cv_job, cv_free;
  std::deque<Job> jobs;
  bool reader_done = false;
  bool abort = false;
  std::string err;
  uint64_t n_observed = 0, n_too_short = 0, n_trimmed_mates = 0;
};

struct BootUser {
  sb_bootstrap_writer* w;
  int rc;
};
int boot_cb(const double* alpha, uint32_t n, void* user) {
  BootUser* u = (BootUser*)user;
  u->rc = sb_bootstrap_writer_write(u->w, alpha, n);
  return u->rc;
}

bool make_dirs(const std::string& path) {
  std::string cur;
  for (size_t i = 0; i <= path.size(); ++i) {
    if (i == path.size() || path[i] == '/') {
      if (!cur.empty() && cur != "/") {
        if (mkdir(cur.c_str(), 0777) != 0 && errno != EEXIST) return false;
      }
    }
    if (i < path.size()) cur += path[i];
  }
  return true;
}

}  // namespace

// meta: the meta variant -- names (and with want_quals qualities) travel with their rows to mcb; too-short pairs' names go
// to too_short at the end
static int reads_bucketed(sb_reads* rd, uint32_t min_len, uint32_t batch, uint32_t max_read_len, uint32_t threads,
                          uint32_t shard_index, uint32_t shard_count, sb_batch_cb cb, bool meta, bool want_quals,
                          sb_batch_meta_cb mcb, sb_names_cb too_short, void* user, sb_bucket_stats* stats) {
  if (!rd || !(cb || mcb)) { sb::set_error("sb_reads_bucketed: null argument"); return SB_ERR_INVALID; }
  if (batch < 1) batch = 1;
  if (max_read_len < 1) { sb::set_error("sb_reads_bucketed: max_read_len must be positive"); return SB_ERR_INVALID; }
  if (shard_count == 0 || shard_index >= shard_count) { sb::set_error("bad shard index / count"); return SB_ERR_INVALID; }
  if (threads == 0) threads = 1;
  const bool paired = sb_reads_paired(rd) != 0;
  Pipe P;
  std::map<uint32_t, std::unique_ptr<Bucket>> buckets;
  const uint32_t stride = max_read_len;
  // ---- reader side ---------------------------------------------------------------------------------------------
  auto submit = [&](HostBuf* b) {   // hand a filled buffer to the consumer side
    std::unique_lock<std::mutex> lk(P.mu);
    b->busy = true;
    P.jobs.push_back(Job{b});
    P.cv_job.notify_one();
  };
  std::string dropped_names;             // (meta) pairs too short to map, one name per line
  auto reader = [&]() {
    std::vector<uint8_t> sl, sr;          // staging for batches of mixed lengths (allocated on first use)
    std::vector<uint32_t> ll(batch), lr(batch);
    std::string err;
    sb_read_meta md{};
    // (meta) rows [i0, i0 + cnt) of the last delivery (quality rows `src_stride` apart) -> rows [row0, ..) of b
    auto put_meta = [&](HostBuf* b, uint32_t row0, int64_t i0, int64_t cnt, uint32_t src_stride) {
      if (row0 == 0) { b->names.clear(); b->name_off.assign(1, 0); }
      for (int64_t q = 0; q < cnt; ++q) {
        b->names.append(md.names + md.name_off[i0 + q], md.name_off[i0 + q + 1] - md.name_off[i0 + q]);
        b->name_off.push_back(b->names.size());
      }
      if (!want_quals) return;
      const uint8_t* src[2] = {md.qual_left, md.qual_right};
      for (int m = 0; m < (paired ? 2 : 1); ++m) {
        if (b->qual[m].size() < (size_t)b->cap * b->L) b->qual[m].resize((size_t)b->cap * b->L);
        for (int64_t q = 0; q < cnt; ++q)
          memcpy(b->qual[m].data() + (size_t)(row0 + q) * b->L, src[m] + (size_t)(i0 + q) * src_stride, b->L);
      }
    };
    auto next = [&](uint32_t n, uint32_t st, uint8_t* l, uint8_t* r) -> int64_t {
      return meta ? sb_reads_next_meta(rd, n, st, l, r, ll.data(), lr.data(), want_quals ? 1 : 0, &md)
                  : sb_reads_next(rd, n, st, l, r, ll.data(), lr.data());
    };
    // the bucket of length L with room for at least one row; nullptr on error / abort
    auto bucket_for = [&](uint32_t L) -> Bucket* {
      std::unique_ptr<Bucket>& bp = buckets[L];
      if (!bp) {
        bp.reset(new Bucket());
        // the first length seen gets full-size buffers; rarer lengths smaller ones
        const uint32_t cap = buckets.size() == 1 ? batch : std::max<uint32_t>(batch / 8, std::min<uint32_t>(batch, 4096));
        if (bp->buf[0].alloc(cap, L) != SB_OK || bp->buf[1].alloc(cap, L) != SB_OK) { err = sb_last_error(); return nullptr; }
      }
      HostBuf* b = &bp->buf[bp->fill];
      if (!bp->checked) {   // first row after a flip: the consumer must have released this buffer
        std::unique_lock<std::mutex> lk(P.mu);
        P.cv_free.wait(lk, [&] { return !b->busy || P.abort; });
        if (P.abort) { err = "aborted"; return nullptr; }
        bp->checked = true;
      }
      return bp.get();
    };
    auto filled = [&](Bucket* bp, uint32_t rows) {
      HostBuf* b = &bp->buf[bp->fill];
      bp->cnt += rows;
      if (bp->cnt == b->cap) { b->n = bp->cnt; submit(b); bp->fill ^= 1; bp->cnt = 0; bp->checked = false; }
    };
    // rows [i0, i1) of the staging buffers -> the bucket of length L (copied by an OpenMP team when it is a run)
    auto put_rows = [&](uint32_t L, int64_t i0, int64_t i1) {
      while (i0 < i1 && err.empty()) {
        Bucket* bp = bucket_for(L);
        if (!bp) return;
        HostBuf* b = &bp->buf[bp->fill];
        const int64_t take = std::min<int64_t>(i1 - i0, (int64_t)(b->cap - bp->cnt));
        const int nt = (int)std::max<int64_t>(1, std::min<int64_t>(threads, take / 4096));
#pragma omp parallel for schedule(static) num_threads(nt)
        for (int64_t q = 0; q < take; ++q) {
          memcpy(b->left + (size_t)(bp->cnt + q) * L, sl.data() + (size_t)(i0 + q) * stride, L);
          if (paired) memcpy(b->right + (size_t)(bp->cnt + q) * L, sr.data() + (size_t)(i0 + q) * stride, L);
        }
        if (meta) put_meta(b, bp->cnt, i0, take, stride);
        i0 += take;
        filled(bp, (uint32_t)take);
      }
    };
    // the read stream is cut into global batches of `batch` records; batch g belongs to shard g % shard_count
    for (uint64_t g = 0; err.empty(); ++g) {
      { std::lock_guard<std::mutex> lk(P.mu); if (P.abort) break; }
      uint32_t L0 = 0;
      int64_t n = sb_reads_peek(rd, batch, &L0);
      if (n < 0) { err = sb_last_error(); break; }
      if (n == 0) break;
      P.n_observed += (uint64_t)n;
      if (g % shard_count != shard_index) {
        if (sb_reads_skip(rd, (uint32_t)n) != n) { err = sb_last_error(); break; }
        continue;
      }
      if (L0 >= min_len && L0 > 0 && L0 <= stride) {
        // one length (the usual case): translated straight into the bucket buffer, no staging, no copy
        int64_t left_n = n;
        while (left_n > 0 && err.empty()) {
          Bucket* bp = bucket_for(L0);
          if (!bp) break;
          HostBuf* b = &bp->buf[bp->fill];
          const uint32_t take = (uint32_t)std::min<int64_t>(left_n, (int64_t)(b->cap - bp->cnt));
          const int64_t got = next(take, L0, b->left + (size_t)bp->cnt * L0, b->right + (size_t)bp->cnt * L0);
          if (got != (int64_t)take) { err = got < 0 ? sb_last_error() : "short read from the parser"; break; }
          if (meta) put_meta(b, bp->cnt, 0, take, L0);
          left_n -= take;
          filled(bp, take);
        }
        continue;
      }
      if (sl.empty()) { sl.resize((size_t)batch * stride); sr.resize((size_t)batch * stride); }
      const int64_t got = next((uint32_t)n, stride, sl.data(), sr.data());
      if (got != n) { err = got < 0 ? sb_last_error() : "short read from the parser"; break; }
      // runs of equal length go in one piece
      int64_t run0 = 0;
      uint32_t runL = 0;
      for (int64_t i = 0; i <= n && err.empty(); ++i) {
        uint32_t L = 0;
        if (i < n) {
          L = paired ? std::min(ll[i], lr[i]) : ll[i];
          if (paired && ll[i] != lr[i]) ++P.n_trimmed_mates;
          if (L < min_len || L == 0) {   // cannot hold a k-mer: observed, never delivered
            ++P.n_too_short;
            L = 0;
            if (meta) { dropped_names.append(md.names + md.name_off[i], md.name_off[i + 1] - md.name_off[i]); dropped_names += '\n'; }
          }
        }
        if (i == n || L != runL) {
          if (runL != 0 && i > run0) put_rows(runL, run0, i);
          run0 = i; runL = L;
        }
      }
    }
    if (err == "aborted") err.clear();
    if (err.empty())
      for (auto& kv : buckets) {   // ascending read length
        Bucket& bk = *kv.second;
        if (bk.cnt > 0) { HostBuf* b = &bk.buf[bk.fill]; b->n = bk.cnt; bk.cnt = 0; submit(b); }
      }
    std::lock_guard<std::mutex> lk(P.mu);
    if (!err.empty()) P.err = err;
    P.reader_done = true;
    P.cv_job.notify_all();
  };
  std::thread rt(reader);
  // ---- consumer side (the calling thread) ------------------------------------------------------------------------
  int rc = SB_OK;
  std::string cb_err;
  uint64_t n_batches = 0, n_delivered = 0;
  double t_wait_job = 0, t_cb = 0;
  for (;;) {
    Job j{nullptr};
    {
      const double tw = now_s();
      std::unique_lock<std::mutex> lk(P.mu);
      P.cv_job.wait(lk, [&] { return !P.jobs.empty() || P.reader_done; });
      t_wait_job += now_s() - tw;
      if (P.jobs.empty()) break;
      j = P.jobs.front();
      P.jobs.pop_front();
    }
    if (rc == SB_OK) {
      const double tc = now_s();
      if (meta) {
        sb_read_meta m{j.b->names.data(), j.b->name_off.data(), want_quals ? j.b->qual[0].data() : nullptr,
                       (want_quals && paired) ? j.b->qual[1].data() : nullptr};
        rc = mcb(user, j.b->left, paired ? j.b->right : nullptr, j.b->n, j.b->L, &m);
      } else {
        rc = cb(user, j.b->left, paired ? j.b->right : nullptr, j.b->n, j.b->L);
      }
      t_cb += now_s() - tc;
      if (rc != SB_OK) {
        cb_err = sb_last_error();
        std::lock_guard<std::mutex> lk(P.mu);
        P.abort = true;
      } else {
        ++n_batches;
        n_delivered += j.b->n;
      }
    }
    {
      std::lock_guard<std::mutex> lk(P.mu);
      j.b->n = 0;
      j.b->busy = false;
    }
    P.cv_free.notify_all();
  }
  rt.join();
  if (getenv("SB_READS_PROFILE"))
    fprintf(stderr, "sb_reads_bucketed: consumer waited %.3f s for batches, spent %.3f s in the callback (%llu batches)\n", t_wait_job, t_cb,
            (unsigned long long)n_batches);
  const uint32_t n_lengths = (uint32_t)buckets.size();
  for (auto& kv : buckets) { kv.second->buf[0].release(); kv.second->buf[1].release(); }
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->n_observed = P.n_observed; stats->n_delivered = n_delivered; stats->n_too_short = P.n_too_short;
    stats->n_trimmed_mates = P.n_trimmed_mates; stats->n_batches = n_batches; stats->n_read_lengths = n_lengths;
  }
  if (rc != SB_OK) { sb::set_error("%s", cb_err.c_str()); return rc > 0 ? SB_ERR_STATE : rc; }
  if (!P.err.empty()) { sb::set_error("%s", P.err.c_str()); return SB_ERR_INVALID; }
  if (meta && too_short && !dropped_names.empty()) too_short(user, dropped_names.data(), dropped_names.size());
  return SB_OK;
}

extern "C" int sb_reads_bucketed(sb_reads* rd, uint32_t min_len, uint32_t batch, uint32_t max_read_len, uint32_t threads,
                                 uint32_t shard_index, uint32_t shard_count, sb_batch_cb cb, void* user,
                                 sb_bucket_stats* stats) {
  if (!cb) { sb::set_error("sb_reads_bucketed: null argument"); return SB_ERR_INVALID; }
  return reads_bucketed(rd, min_len, batch, max_read_len, threads, shard_index, shard_count, cb, false, false, nullptr,
                        nullptr, user, stats);
}

extern "C" int sb_reads_bucketed_meta(sb_reads* rd, uint32_t min_len, uint32_t batch, uint32_t max_read_len, uint32_t threads,
                                      uint32_t shard_index, uint32_t shard_count, int want_quals, sb_batch_meta_cb cb,
                                      sb_names_cb too_short, void* user, sb_bucket_stats* stats) {
  if (!cb) { sb::set_error("sb_reads_bucketed_meta: null argument"); return SB_ERR_INVALID; }
  return reads_bucketed(rd, min_len, batch, max_read_len, threads, shard_index, shard_count, nullptr, true, want_quals != 0,
                        cb, too_short, user, stats);
}

extern "C" void sb_quant_default_opts(sb_quant_opts* o) {
  if (!o) return;
  memset(o, 0, sizeof(*o));
  o->device = 0;
  o->batch = 262144;
  o->max_read_len = 256;
  o->threads = 8;
  o->shard_index = 0;
  o->shard_count = 1;
  o->thinning = 16;
  o->seed = 42;
}

namespace {
// ---- run metadata of the drop-in contract (src/output/GZipWriter.cpp:294-640 writeMeta, ReadExperiment.inl:219-350
// summarizeLibraryTypeCounts, MappingPipelineStages.cpp:164-173 flenDist.txt) -----------------------------------------
struct MetaIn {
  const sb_quant_opts* o; const sb_em_params* ep; const sb_map_params* mp;
  uint32_t n_valid, n_decoy;
  uint64_t n_observed, n_mapped, n_classes;
  const std::vector<double>* fld_log;     // log histogram of the fragment-length distribution
  const uint64_t* uniq; const uint64_t* total;
  std::string files, start_time, end_time;
  int n_ranks;
  uint64_t lib_counts[4];     // fragments that showed ISF / ISR / SF / SR among their kept mappings
  uint64_t orphans_rescued;   // over all ranks
  uint64_t n_compatible;      // assigned fragments with a kept mapping compatible with the library type, over all ranks
};
std::string time_string() {
  time_t t = time(nullptr);
  char buf[64];
  struct tm tmv;
  localtime_r(&t, &tmv);
  strftime(buf, sizeof buf, "%a %b %e %H:%M:%S %Y", &tmv);
  return buf;
}
bool write_text(const std::string& path, const std::string& text) {
  FILE* f = fopen(path.c_str(), "w");
  if (!f) return false;
  const bool ok = fwrite(text.data(), 1, text.size(), f) == text.size();
  return (fclose(f) == 0) && ok;
}
bool write_gz(const std::string& path, const void* data, size_t bytes) {
  gzFile g = gzopen(path.c_str(), "wb");
  if (!g) return false;
  const bool ok = bytes == 0 || gzwrite(g, data, (unsigned)bytes) == (int)bytes;
  return (gzclose(g) == Z_OK) && ok;
}
int write_run_metadata(const std::string& outs, const MetaIn& m) {
  if (!make_dirs(outs + "/aux_info") || !make_dirs(outs + "/libParams") || !make_dirs(outs + "/logs")) {
    sb::set_error("cannot create the output sub-directories of %s", outs.c_str());
    return SB_ERR_INVALID;
  }
  // normalised pmf of the fragment-length distribution, its mean / sd (DistributionUtils.cpp:57-101)
  const std::vector<double>& lh = *m.fld_log;
  std::vector<double> pmf(lh.size(), 0.0);
  double mx = -INFINITY;
  for (double v : lh) if (std::isfinite(v)) mx = std::max(mx, v);
  double tot = 0.0;
  if (std::isfinite(mx)) for (size_t i = 0; i < lh.size(); ++i) { pmf[i] = std::isfinite(lh[i]) ? std::exp(lh[i] - mx) : 0.0; tot += pmf[i]; }
  double mean = 0.0, var = 0.0;
  if (tot > 0) for (size_t i = 0; i < pmf.size(); ++i) { pmf[i] /= tot; mean += pmf[i] * (double)i; var += pmf[i] * (double)i * (double)i; }
  var -= mean * mean;
  const double sd = var > 0 ? std::sqrt(var) : 0.0;
  // aux_info/fld.gz: int32 counts of 10000 draws from the pmf (the reference seeds from random_device; here --seed)
  std::vector<int32_t> samples(pmf.size(), 0);
  if (tot > 0) {
    std::mt19937 gen((uint32_t)m.o->seed);
    std::discrete_distribution<int32_t> dist(pmf.begin(), pmf.end());
    for (int i = 0; i < 10000; ++i) ++samples[dist(gen)];
  }
  bool ok = write_gz(outs + "/aux_info/fld.gz", samples.data(), samples.size() * 4);
  if (!m.mp->no_frag_len_dist) {   // libParams/flenDist.txt: exp(pmf(i)), tab separated, ostream precision
    std::string t;
    char buf[48];
    for (size_t i = 0; i < pmf.size(); ++i) { snprintf(buf, sizeof buf, "%g", pmf[i]); t += buf; t += (i + 1 < pmf.size()) ? "\t" : "\n"; }
    t += "\n";
    ok = write_text(outs + "/libParams/flenDist.txt", t) && ok;
  }
  {   // aux_info/ambig_info.tsv (GZipWriter.cpp:603-616)
    std::string t = "UniqueCount\tAmbigCount\n";
    for (uint32_t i = 0; i < m.n_valid; ++i)
      t += std::to_string(m.uniq[i]) + "\t" + std::to_string(m.total[i] >= m.uniq[i] ? m.total[i] - m.uniq[i] : 0) + "\n";
    ok = write_text(outs + "/aux_info/ambig_info.tsv", t) && ok;
  }
  const uint32_t n_samp = m.o->num_bootstraps ? m.o->num_bootstraps : m.o->num_gibbs;
  const double pct = m.n_observed ? 100.0 * (double)m.n_mapped / (double)m.n_observed : 0.0;
  {
    char buf[4096];
    snprintf(buf, sizeof buf,
             "{\n    \"salmon_version\": \"1.11.4-sb%d\",\n    \"samp_type\": \"%s\",\n    \"opt_type\": \"%s\",\n    \"quant_errors\": [],\n"
             "    \"num_libraries\": 1,\n    \"library_types\": [\n        \"%s\"\n    ],\n    \"frag_dist_length\": %zu,\n"
             "    \"frag_length_mean\": %.6f,\n    \"frag_length_sd\": %.6f,\n    \"seq_bias_correct\": false,\n    \"gc_bias_correct\": false,\n"
             "    \"num_bias_bins\": 0,\n    \"mapping_type\": \"mapping\",\n    \"keep_duplicates\": false,\n    \"num_valid_targets\": %u,\n"
             "    \"num_decoy_targets\": %u,\n    \"num_eq_classes\": %llu,\n    \"serialized_eq_classes\": %s,\n    \"eq_class_properties\": [%s],\n"
             "    \"length_classes\": [],\n    \"index_seq_hash\": \"\",\n    \"index_name_hash\": \"\",\n    \"num_bootstraps\": %u,\n"
             "    \"num_processed\": %llu,\n    \"num_mapped\": %llu,\n    \"num_decoy_fragments\": 0,\n    \"num_dovetail_fragments\": 0,\n"
             "    \"num_fragments_filtered_vm\": 0,\n    \"num_alignments_below_threshold_for_mapped_fragments_vm\": 0,\n"
             "    \"percent_mapped\": %.6f,\n    \"call\": \"quant\",\n    \"start_time\": \"%s\",\n    \"end_time\": \"%s\",\n    \"sb_num_gpus\": %d,\n"
             "    \"sb_num_orphans_rescued\": %llu,\n"
             "    \"sb_mapping_params\": {\"max_read_occ\": %u, \"consensus_slack\": %.15g, \"min_score_fraction\": %.15g, "
             "\"min_aln_prob\": %.15g, \"ma\": %d, \"mp\": %d, \"go\": %d, \"ge\": %d, \"discard_orphans\": %s, "
             "\"softclip\": %s, \"softclip_overhangs\": %s}\n}\n",
             sb_version(), m.o->num_bootstraps ? "bootstrap" : (m.o->num_gibbs ? "gibbs" : "none"), m.ep->use_vbem ? "vb" : "em",
             (m.mp->lib_type >= 0 && m.mp->lib_type <= 5) ? (const char* const[]){"IU", "ISF", "ISR", "U", "SF", "SR"}[m.mp->lib_type] : "IU",
             pmf.size(), mean, sd, m.n_valid, m.n_decoy, (unsigned long long)m.n_classes,
             (m.o->dump_eq || m.o->dump_eq_weights) ? "true" : "false",
             m.mp->range_bins ? "\n        \"range_factorized\"\n    " : "", n_samp, (unsigned long long)m.n_observed,
             (unsigned long long)m.n_mapped, pct, m.start_time.c_str(), m.end_time.c_str(), m.n_ranks,
             (unsigned long long)m.orphans_rescued, m.mp->max_read_occ, 1.0 - m.mp->consensus_frac, m.mp->min_score_fraction,
             m.mp->min_aln_prob, m.mp->ma, m.mp->mp, m.mp->go, m.mp->ge, m.mp->allow_orphans ? "false" : "true",
             m.mp->softclip == 2 ? "true" : "false", m.mp->softclip >= 1 ? "true" : "false");
    ok = write_text(outs + "/aux_info/meta_info.json", buf) && ok;
  }
  {   // lib_format_counts.json (ReadExperiment.inl:219-350): compatible = assigned fragments with at least one kept mapping
      // compatible with the expected format (all of them unless --incompatPrior keeps incompatible ones); the per-format
      // counts are what the fragments showed; strand_mapping_bias = first strand variant / both, as
      // summarizeLibraryTypeCounts computes it
    static const char* const lib_names[] = {"IU", "ISF", "ISR", "U", "SF", "SR"};
    const int lt = m.mp->lib_type;
    const bool pe = lt < 3;
    const uint64_t f1 = pe ? m.lib_counts[0] : m.lib_counts[2], f2 = pe ? m.lib_counts[1] : m.lib_counts[3];
    const bool unstranded = lt == 0 || lt == 3;
    const uint64_t agree = unstranded ? f1 + f2 : ((lt == 1 || lt == 4) ? f1 : f2);
    const uint64_t other = pe ? m.lib_counts[2] + m.lib_counts[3] : 0;          // orphans of a paired-end library
    const double ratio = (f1 + f2) ? (double)f1 / (double)(f1 + f2) : 0.0;
    char buf[2048];
    snprintf(buf, sizeof buf,
             "{\n    \"read_files\": \"%s\",\n    \"expected_format\": \"%s\",\n    \"compatible_fragment_ratio\": %.6f,\n"
             "    \"num_compatible_fragments\": %llu,\n    \"num_assigned_fragments\": %llu,\n"
             "    \"num_frags_with_concordant_consistent_mappings\": %llu,\n    \"num_frags_with_inconsistent_or_orphan_mappings\": %llu,\n"
             "    \"strand_mapping_bias\": %.6f,\n    \"ISF\": %llu,\n    \"ISR\": %llu,\n    \"SF\": %llu,\n    \"SR\": %llu\n}\n",
             m.files.c_str(), lib_names[lt < 0 || lt > 5 ? 0 : lt],
             m.n_mapped ? (double)m.n_compatible / (double)m.n_mapped : 0.0, (unsigned long long)m.n_compatible,
             (unsigned long long)m.n_mapped, (unsigned long long)agree, (unsigned long long)other, ratio,
             (unsigned long long)m.lib_counts[0], (unsigned long long)m.lib_counts[1], (unsigned long long)m.lib_counts[2],
             (unsigned long long)m.lib_counts[3]);
    ok = write_text(outs + "/lib_format_counts.json", buf) && ok;
  }
  if (!ok) { sb::set_error("write error on the run metadata under %s", outs.c_str()); return SB_ERR_INVALID; }
  return SB_OK;
}

// posterior samples split over the ranks (chains restart independently, CollapsedGibbsSampler.cpp:425-461; bootstrap
// replicates are independent, CollapsedEMOptimizer.cpp:670-688): rank r draws samples [lo_r, hi_r) with their own
// counter-RNG streams, rank 0 gathers them in sample order
struct GatherUser { std::vector<double>* buf; };
int gather_cb(const double* sample, uint32_t n, void* user) {
  GatherUser* g = (GatherUser*)user;
  g->buf->insert(g->buf->end(), sample, sample + n);
  return 0;
}
int run_samples(sb_em_ctx* em, const sb_em_params& ep, const sb_quant_opts& o, const double* alpha, uint32_t M, double n_mapped,
                sb_comm* comm, const std::string& outs, const char* const* names) {
  const uint32_t n_total = o.num_bootstraps ? o.num_bootstraps : o.num_gibbs;
  const int G = comm ? sb_comm_size(comm) : 1, r = comm ? sb_comm_rank(comm) : 0;
  const uint32_t lo = (uint32_t)((uint64_t)n_total * r / G), hi = (uint32_t)((uint64_t)n_total * (r + 1) / G);
  std::vector<double> mine;
  mine.reserve((size_t)(hi - lo) * M);
  GatherUser gu{&mine};
  int rc = SB_OK;
  if (hi > lo) {
    // the samplers key their counter RNG by (seed, sample index): a rank's share starts at index lo, so a split run
    // draws exactly the bootstrap replicates of the one-GPU run; a Gibbs share is a chain of its own from alphasInit
    SB_TRY(sb_em_set_option(em, "sample_offset", lo));
    if (o.num_bootstraps) {
      sb_em_params bp = ep;
      bp.min_iter = 50;   // CollapsedEMOptimizer.cpp:411
      rc = sb_bootstrap(em, &bp, n_mapped, hi - lo, o.seed, gather_cb, &gu);
    } else {
      rc = sb_gibbs(em, alpha, ep.use_vbem, ep.per_txp_prior, ep.vb_prior, hi - lo, o.thinning ? o.thinning : 16,
                    o.no_gamma_draw, n_mapped, o.seed, gather_cb, &gu);
    }
    sb_em_set_option(em, "sample_offset", 0);
    if (rc < 0) return rc;
  }
  // gather: equal-sized slots of ceil(n/G) samples
  const uint32_t slot = (n_total + G - 1) / G;
  std::vector<double> all;
  if (G > 1) {
    mine.resize((size_t)slot * M, 0.0);
    all.resize((size_t)slot * M * G);
    SB_TRY(sb_comm_allgather(comm, mine.data(), all.data(), (size_t)slot * M * 8));
  }
  if (r != 0 || outs.empty()) return SB_OK;
  if (!make_dirs(outs + "/aux_info/bootstrap")) { sb::set_error("cannot create the bootstrap directory"); return SB_ERR_INVALID; }
  sb_bootstrap_writer* w = sb_bootstrap_writer_open((outs + "/aux_info/bootstrap/bootstraps.gz").c_str());
  if (!w) return SB_ERR_INVALID;
  for (int q = 0; q < G && rc >= 0; ++q) {
    const uint32_t qlo = (uint32_t)((uint64_t)n_total * q / G), qhi = (uint32_t)((uint64_t)n_total * (q + 1) / G);
    const double* base = G > 1 ? all.data() + (size_t)q * slot * M : mine.data();
    for (uint32_t k = 0; k < qhi - qlo && rc >= 0; ++k) rc = sb_bootstrap_writer_write(w, base + (size_t)k * M, M);
  }
  const int rc2 = sb_bootstrap_writer_close(w);
  if (rc < 0 || rc2 < 0) return rc < 0 ? rc : rc2;
  std::string nm;
  for (uint32_t t = 0; t < M; ++t) { nm += names[t]; nm += (t + 1 < M) ? '\t' : '\n'; }
  if (!write_gz(outs + "/aux_info/bootstrap/names.tsv.gz", nm.data(), nm.size())) {
    sb::set_error("write error on %s/aux_info/bootstrap/names.tsv.gz", outs.c_str());
    return SB_ERR_INVALID;
  }
  return SB_OK;
}
}  // namespace

// `salmon quant` (mapping mode) for one library, on one GPU or -- shard_count > 1, one process per GPU -- on several:
// processReadLibrary -> quantifyLibrary -> stageFinalizeMappingOutputs (SalmonQuantify.cpp:2340-2480,
// pipeline/MappingPipelineStages.cpp:21-175).  Rank r maps the global batches g with g % shard_count == r and keeps
// their classes; the end-of-mapping statistics are reduced once (sb_map_reduce_global), the EM runs over the sharded
// classes with the per-iteration exchange inside the kernel, rank 0 writes the outputs.
extern "C" int sb_quant_files(sb_index* ix, const char* const* mates1, const char* const* mates2, uint32_t n_files,
                              const sb_map_params* mp_in, const sb_em_params* ep_in, const sb_quant_opts* o_in,
                              const char* out_dir, double* alpha_out, sb_quant_summary* sum) {
  if (!ix || !mates1 || !n_files) { sb::set_error("sb_quant_files: null argument"); return SB_ERR_INVALID; }
  sb_quant_opts o;
  if (o_in) o = *o_in; else sb_quant_default_opts(&o);
  if (o.batch < 1024) o.batch = 1024;
  if (o.max_read_len < 32 || o.max_read_len > 256) { sb::set_error("max_read_len must be in 32..256"); return SB_ERR_INVALID; }
  if (o.shard_count == 0) o.shard_count = 1;
  if (o.shard_index >= o.shard_count) { sb::set_error("shard_index must be below shard_count"); return SB_ERR_INVALID; }
  const bool multi = o.shard_count > 1;
  if (multi && !o.nccl_uid) {
    sb::set_error("sb_quant_files: a sharded run needs the communicator id (sb_quant_opts.nccl_uid, sb_nccl_unique_id of rank 0): "
                  "a shard's classes alone are not a quantification");
    return SB_ERR_INVALID;
  }
  if (o.num_bootstraps && o.num_gibbs) { sb::set_error("choose bootstraps or Gibbs samples, not both"); return SB_ERR_INVALID; }
  const bool sam_out = o.write_mappings || o.write_unmapped_names;
  if (multi && sam_out) {
    sb::set_error("--writeMappings / --writeUnmappedNames are written by a one-GPU run only: a read-sharded run (--gpus N) "
                  "cannot write them");
    return SB_ERR_INVALID;
  }
  if (o.write_unmapped_names && !out_dir) { sb::set_error("--writeUnmappedNames needs an output directory"); return SB_ERR_INVALID; }
  if (multi && (o.num_bootstraps || o.num_gibbs || o.dump_eq || o.dump_eq_weights)) {
    sb::set_error("posterior samples / --dumpEq need the whole class table on one GPU: run them on one GPU, or sample from a dumped table "
                  "with `quant -e` (which splits the samples over the GPUs)");
    return SB_ERR_INVALID;
  }
  sb_map_params mp;
  if (mp_in) mp = *mp_in; else sb_map_default_params(&mp);
  sb_em_params ep;
  if (ep_in) ep = *ep_in; else sb_em_default_params(&ep);
  // -l A: start unstranded (nothing is incompatible before the type is known, SalmonQuantify.cpp:496-501), decide from
  // the first 50 000 fragments that show a strand, checked after every batch
  bool auto_lib = false;
  if (mp.lib_type == SB_LIB_AUTO_PAIRED || mp.lib_type == SB_LIB_AUTO_SINGLE) {
    auto_lib = !multi;   // (with the reads sharded the ranks would decide at different points: the run stays unstranded)
    mp.lib_type = mp.lib_type == SB_LIB_AUTO_PAIRED ? SB_LIB_IU : SB_LIB_U;
  }
  // single-end libraries (-r, library types U / SF / SR) come with mates2 == NULL
  const bool single_end = mp.lib_type >= SB_LIB_U;
  if (single_end != (mates2 == nullptr)) {
    sb::set_error(single_end ? "a single-end library type takes unmated reads only (mates2 == NULL)"
                             : "a paired-end library type needs both mate files");
    return SB_ERR_INVALID;
  }
  uint32_t M = 0, k = 0, first_decoy = 0;
  const char* const* names = nullptr;
  const uint32_t* complete_len = nullptr;
  sb_index_get_meta(ix, &M, &k, &first_decoy, &names, &complete_len);
  if (first_decoy < M) mp.first_decoy = (int32_t)first_decoy;
  // decoys are dropped before normalizeAlphas / the optimiser / the writers (readExp.dropDecoyTranscripts(),
  // SalmonQuantify.cpp:2479, ReadExperiment.hpp:120): they are the suffix of the id space and never appear in a label
  const uint32_t Mq = first_decoy < M ? first_decoy : M;
  const double t0 = now_s();
  const std::string start_time = time_string();

  struct Scope {   // everything acquired below, released on every exit path
    sb_map_ctx* ctx = nullptr; sb_em_ctx* em = nullptr; sb_comm* comm = nullptr; sb_reads* rd = nullptr; sb_sam* sam = nullptr;
    ~Scope() {
      if (rd) sb_reads_close(rd);
      if (em) sb_em_destroy(em);
      if (ctx) sb_map_destroy(ctx);
      if (sam) sb_sam_close(sam);
      if (comm) sb_comm_destroy(comm);
    }
  } S;
  if (multi) {
    S.comm = sb_comm_create((int)o.shard_index, (int)o.shard_count, o.nccl_uid, o.device);
    if (!S.comm) return SB_ERR_NCCL;
  }
  S.ctx = sb_map_create(ix, &mp, o.device, o.batch, o.max_read_len);
  if (!S.ctx) return SB_ERR_CUDA;
  if (getenv("SB_READS_PROFILE")) fprintf(stderr, "sb_quant_files: sb_map_create %.3f s\n", now_s() - t0);
  if (sam_out) {
    std::string un;
    if (o.write_unmapped_names) {
      un = std::string(out_dir) + "/aux_info";
      if (!make_dirs(un)) { sb::set_error("cannot create %s", un.c_str()); return SB_ERR_INVALID; }
      un += "/unmapped_names.txt";
    }
    S.sam = sb_sam_open(o.write_mappings, o.write_unmapped_names ? un.c_str() : nullptr, ix, o.cmdline,
                        o.write_qualities ? SB_SAM_QUALITIES : 0u);
    if (!S.sam) return SB_ERR_INVALID;
    SB_TRY(sb_map_attach_sam(S.ctx, S.sam));
  }
  S.rd = sb_reads_open(mates1, mates2, n_files, o.threads);
  if (!S.rd) return SB_ERR_INVALID;
  const double t_setup = now_s();

  struct MapUser {
    sb_map_ctx* ctx; float device_ms; bool detect; bool paired; int detected; uint64_t at_fragment, seen;
    // bookkeeping after a mapped batch: device time, library-type detection
    int after(const sb_map_batch_stats& st, uint32_t n) {
      device_ms += st.device_ms;
      seen += n;
      int rc = SB_OK;
      if (detect) {
        uint64_t c4[4];
        rc = sb_map_lib_counts(ctx, c4);
        if (rc == SB_OK && (paired ? c4[0] + c4[1] : c4[2] + c4[3]) >= 50000) {   // numSamplesNeeded_, LibraryTypeDetector.hpp:171
          detected = sb_detect_lib_type(paired ? 1 : 0, c4);
          at_fragment = seen;
          detect = false;
          if (detected >= 0) rc = sb_map_set_option(ctx, "lib_type", detected);
        }
      }
      return rc;
    }
  } mu{S.ctx, 0.0f, auto_lib, !single_end, -1, 0, 0};
  sb_batch_cb map_cb = [](void* user, const uint8_t* l, const uint8_t* r, uint32_t n, uint32_t L) -> int {
    MapUser* u = (MapUser*)user;
    sb_map_batch_stats st;
    const int rc = sb_map_batch(u->ctx, l, r, n, L, &st);
    return rc != SB_OK ? rc : u->after(st, n);
  };
  sb_bucket_stats bs;
  int rc;
  if (S.sam) {
    // the same per-batch work, with the rows' names (and qualities) for the SAM records; pairs too short to map are
    // listed as unmapped by the host
    struct SamUser { MapUser* mu; sb_sam* sam; int rc; } su{&mu, S.sam, SB_OK};
    sb_batch_meta_cb sam_cb = [](void* user, const uint8_t* l, const uint8_t* r, uint32_t n, uint32_t L,
                                 const sb_read_meta* m) -> int {
      SamUser* u = (SamUser*)user;
      sb_map_batch_stats st;
      const int rc = sb_map_batch_sam(u->mu->ctx, l, r, n, L, m->names, m->name_off, m->qual_left, m->qual_right, &st);
      return rc != SB_OK ? rc : u->mu->after(st, n);
    };
    sb_names_cb short_cb = [](void* user, const char* names, size_t len) {
      SamUser* u = (SamUser*)user;
      std::string t;
      for (size_t i = 0, b = 0; i < len; ++i)
        if (names[i] == '\n') { t.append(names + b, i - b); t += " u\n"; b = i + 1; }
      if (u->rc == SB_OK) u->rc = sb_sam_write_unmapped(u->sam, t.data(), t.size());
    };
    rc = sb_reads_bucketed_meta(S.rd, mp.k, o.batch, o.max_read_len, o.threads, o.shard_index, o.shard_count,
                                o.write_qualities ? 1 : 0, sam_cb, short_cb, &su, &bs);
    if (rc == SB_OK) rc = su.rc;
    if (rc == SB_OK) rc = sb_map_attach_sam(S.ctx, nullptr);
    const int rc2 = sb_sam_close(S.sam);
    S.sam = nullptr;
    if (rc == SB_OK) rc = rc2;
  } else {
    rc = sb_reads_bucketed(S.rd, mp.k, o.batch, o.max_read_len, o.threads, o.shard_index, o.shard_count, map_cb, &mu, &bs);
  }
  sb_reads_close(S.rd);
  S.rd = nullptr;
  if (rc != SB_OK) return rc;
  const float device_ms = mu.device_ms;
  const double t_map = now_s();
  if (auto_lib && o.shard_index == 0) {
    static const char* const nm[6] = {"IU", "ISF", "ISR", "U", "SF", "SR"};
    if (mu.detected >= 0) {
      mp.lib_type = mu.detected;       // what the run metadata reports as the expected format
      fprintf(stderr, "Automatically detected most likely library type as %s (after %llu fragments)\n", nm[mu.detected],
              (unsigned long long)mu.at_fragment);
    } else {
      fprintf(stderr, "library type not detected (fewer than 50000 stranded fragments): the run stayed %s\n", nm[mp.lib_type]);
    }
  }

  // ---- classes -> (global statistics) -> EM -> outputs -----------------------------------------------------------
  // --skipQuant: no normalizeAlphas (MappingPipelineStages.cpp:45-47), so finish without the cluster projection
  if (o.skip_quant) SB_TRY(sb_map_set_option(S.ctx, "no_projection", 1));
  sb_map_result res;
  rc = sb_map_finish(S.ctx, &res);
  if (rc != SB_OK) return rc;
  sb_map_result glob = res;          // per-transcript inputs of the optimiser
  uint64_t n_mapped_u = res.n_mapped, n_observed = bs.n_observed;
  if (multi) SB_TRY(sb_map_reduce_global(S.ctx, S.comm, &glob, &n_mapped_u));   // (every rank's reader sees the whole stream: n_observed is global already)
  sb_eq_csr eq;
  eq.n_classes = res.n_classes; eq.n_txps = Mq; eq.off = res.off; eq.tids = res.tids; eq.weights = res.weights; eq.counts = res.counts;
  std::vector<double> alpha(M, 0.0);
  sb_em_stats est;
  memset(&est, 0, sizeof est);
  // --skipQuant --dumpEqWeights: the dumped weights are the combined weights (MappingPipelineStages.cpp:112-162)
  std::vector<double> combined;
  if (!o.skip_quant || o.dump_eq_weights) {
    S.em = sb_em_create(o.device);
    if (!S.em) return SB_ERR_CUDA;
  }
  if (!o.skip_quant) {
    if (multi) SB_TRY(sb_em_peer_setup(S.em, S.comm, Mq));
    rc = sb_em_optimize(S.em, &eq, &ep, glob.projected_counts, glob.eff_len, glob.unique_counts, alpha.data(), &est);
    if (rc < 0) return rc;
    if (rc == 1) { sb::set_error("The optimization algorithm failed (total alpha weight too small)"); return SB_ERR_STATE; }
  } else if (o.dump_eq_weights && out_dir && o.shard_index == 0) {
    combined.resize((res.n_classes ? res.off[res.n_classes] : 0) + 1);   // (+1: a table with no entries still has weights)
    SB_TRY(sb_eq_combined_weights(S.em, &eq, glob.eff_len, ep.no_rich_eq, combined.data()));
  }
  const double n_mapped = (double)n_mapped_u;
  std::string outs = out_dir ? out_dir : "";
  const double t_em = now_s();
  std::vector<std::string> gen;
  std::vector<const char*> np;
  if (!names) {
    for (uint32_t t = 0; t < M; ++t) gen.push_back("t" + std::to_string(t));
    for (auto& sname : gen) np.push_back(sname.c_str());
    names = np.data();
  }
  // (a collective: every rank takes part, whether it writes the outputs or not)
  uint64_t libc[5] = {res.lib_format_counts[0], res.lib_format_counts[1], res.lib_format_counts[2], res.lib_format_counts[3],
                      res.orphans_rescued};
  if (multi) SB_TRY(sb_comm_allreduce(S.comm, libc, 5, 1, 0));   // (glob.n_compatible is global already)
  if (!outs.empty() && o.shard_index == 0) {
    if (!make_dirs(outs + "/aux_info")) { sb::set_error("cannot create %s/aux_info", outs.c_str()); return SB_ERR_INVALID; }
    std::vector<uint32_t> lens;
    if (!complete_len) {
      const uint64_t* off = nullptr;
      sb_index_host_arrays(ix, &off, nullptr, nullptr, nullptr, nullptr, nullptr);
      for (uint32_t t = 0; t < M; ++t) lens.push_back((uint32_t)(off[t + 1] - off[t]));
      complete_len = lens.data();
    }
    rc = o.skip_quant ? SB_OK
                      : sb_write_quant_sf((outs + "/quant.sf").c_str(), Mq, names, complete_len, glob.eff_len, alpha.data(),
                                          n_mapped, 3);
    if (rc == SB_OK && (o.dump_eq || o.dump_eq_weights))
      rc = sb_write_eq_classes((outs + "/aux_info/eq_classes.txt.gz").c_str(), Mq, names, res.n_classes, res.off, res.tids,
                               o.dump_eq_weights ? (o.skip_quant ? combined.data() : res.weights) : nullptr, res.counts);
    if (rc != SB_OK) return rc;
    // run metadata
    std::vector<double> hist((size_t)mp.max_frag_len + 1, 0.0);
    SB_TRY(sb_map_online_state(S.ctx, nullptr, hist.data(), nullptr, nullptr));
    std::string files = "[ ";
    for (uint32_t f = 0; f < n_files; ++f)
      files += std::string(f ? ", " : "") + (mates2 ? std::string("( ") + mates1[f] + ", " + mates2[f] + " )" : std::string(mates1[f]));
    files += " ]";
    MetaIn mi{&o, &ep, &mp, Mq, M - Mq, n_observed, n_mapped_u, res.n_classes, &hist, glob.unique_counts, glob.total_counts,
              files, start_time, time_string(), (int)o.shard_count, {libc[0], libc[1], libc[2], libc[3]}, libc[4],
              glob.n_compatible};
    SB_TRY(write_run_metadata(outs, mi));
  }
  if ((o.num_bootstraps || o.num_gibbs) && !o.skip_quant) {   // --skipQuant draws no samples (its help text)
    rc = run_samples(S.em, ep, o, alpha.data(), Mq, n_mapped, nullptr, o.shard_index == 0 ? outs : std::string(), names);
    if (rc < 0) return rc;
  }
  if (alpha_out) memcpy(alpha_out, alpha.data(), (size_t)M * 8);
  if (sum) {
    memset(sum, 0, sizeof(*sum));
    sum->n_observed = n_observed; sum->n_mapped = n_mapped_u; sum->n_too_short = bs.n_too_short;
    sum->n_trimmed_mates = bs.n_trimmed_mates;
    sum->n_classes = res.n_classes; sum->n_batches = bs.n_batches; sum->n_read_lengths = bs.n_read_lengths;
    sum->em_iters = est.iters; sum->em_converged = est.converged;
    sum->map_seconds = t_map - t0; sum->em_seconds = t_em - t_map; sum->total_seconds = now_s() - t0;
    sum->map_device_ms = device_ms;
    sum->map_setup_ms = (float)((t_setup - t0) * 1e3);
    sum->orphans_rescued = res.orphans_rescued; sum->rescue_searches = res.rescue_searches; sum->rescue_no_room = res.rescue_no_room;
  }
  return SB_OK;
}

// `salmon quant -e` (processEqClasses, SalmonQuantifyAlignments.cpp:1406-1440): the optimiser and the samplers over a
// dumped class table.  With shard_count > 1 (one process per GPU, every rank holding the whole table) the posterior
// samples are split over the ranks -- BASELINE.json configs[4] -- and gathered by rank 0.
extern "C" int sb_quant_eqclasses(const char* eq_path, const sb_em_params* ep_in, const sb_quant_opts* o_in,
                                  const char* out_dir, sb_quant_summary* sum) {
  if (!eq_path) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  sb_quant_opts o;
  if (o_in) o = *o_in; else sb_quant_default_opts(&o);
  if (o.shard_count == 0) o.shard_count = 1;
  const bool multi = o.shard_count > 1;
  if (multi && !o.nccl_uid) { sb::set_error("sb_quant_eqclasses: a multi-GPU run needs sb_quant_opts.nccl_uid"); return SB_ERR_INVALID; }
  if (o.num_bootstraps && o.num_gibbs) { sb::set_error("choose bootstraps or Gibbs samples, not both"); return SB_ERR_INVALID; }
  sb_em_params ep;
  if (ep_in) ep = *ep_in; else sb_em_default_params(&ep);
  const double t0 = now_s();
  struct Scope {
    sb_eq_file* f = nullptr; sb_em_ctx* em = nullptr; sb_comm* comm = nullptr;
    ~Scope() { if (em) sb_em_destroy(em); if (f) sb_eq_file_free(f); if (comm) sb_comm_destroy(comm); }
  } S;
  if (sb_eq_file_read(eq_path, &S.f) != SB_OK) return SB_ERR_INVALID;
  const sb_eq_file* f = S.f;
  if (multi) {
    S.comm = sb_comm_create((int)o.shard_index, (int)o.shard_count, o.nccl_uid, o.device);
    if (!S.comm) return SB_ERR_NCCL;
  }
  if (!f->has_weights) { sb::set_error("--eqclasses needs the weights (write the file with --dumpEqWeights)"); return SB_ERR_INVALID; }
  const uint32_t M = f->n_txps;
  std::vector<double> zeros(M, 0.0), alpha(M, 0.0);
  std::vector<uint64_t> uniq(M, 0);
  double n_frags = 0.0;
  for (uint64_t c = 0; c < f->n_classes; ++c) n_frags += (double)f->counts[c];
  // processEqClasses: uniform initialisation, eq-class mode (the weights of the file are the combined weights)
  ep.init_uniform = 1;
  ep.eq_class_mode = 1;
  sb_eq_csr eqv;
  eqv.n_classes = f->n_classes; eqv.n_txps = M; eqv.off = f->off; eqv.tids = f->tids; eqv.weights = f->weights; eqv.counts = f->counts;
  S.em = sb_em_create(o.device);
  if (!S.em) return SB_ERR_CUDA;
  sb_em_stats st;
  memset(&st, 0, sizeof st);
  int rc = sb_em_optimize(S.em, &eqv, &ep, zeros.data(), f->eff_len, uniq.data(), alpha.data(), &st);
  if (rc < 0) return rc;
  if (rc == 1) { sb::set_error("The optimization algorithm failed (total alpha weight too small)"); return SB_ERR_STATE; }
  const double t_em = now_s();
  const std::string outs = out_dir ? out_dir : "";
  if (!outs.empty() && o.shard_index == 0) {
    if (!make_dirs(outs + "/aux_info")) { sb::set_error("cannot create %s/aux_info", outs.c_str()); return SB_ERR_INVALID; }
    std::vector<uint32_t> lens(M);
    for (uint32_t t = 0; t < M; ++t) lens[t] = (uint32_t)(f->eff_len[t] < 1.0 ? 1.0 : f->eff_len[t]);   // the table carries no lengths
    SB_TRY(sb_write_quant_sf((outs + "/quant.sf").c_str(), M, f->names, lens.data(), f->eff_len, alpha.data(), n_frags, 3));
  }
  if (o.num_bootstraps || o.num_gibbs) {
    rc = run_samples(S.em, ep, o, alpha.data(), M, n_frags, S.comm, o.shard_index == 0 ? outs : std::string(), f->names);
    if (rc < 0) return rc;
  }
  if (sum) {
    memset(sum, 0, sizeof(*sum));
    sum->n_observed = (uint64_t)n_frags; sum->n_mapped = (uint64_t)n_frags; sum->n_classes = f->n_classes;
    sum->em_iters = st.iters; sum->em_converged = st.converged;
    sum->em_seconds = t_em - t0; sum->total_seconds = now_s() - t0;
  }
  return SB_OK;
}

// ---- end-of-mapping reduction of a sharded run, C++ form of salmon_b200/dist.py::reduce_partials --------------------
extern "C" int sb_map_reduce_global(sb_map_ctx* ctx, sb_comm* comm, sb_map_result* out, uint64_t* assigned_out) {
  if (!ctx || !comm || !out) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  sb_map_partial p;
  SB_TRY(sb_map_partial_get(ctx, &p));
  const int G = sb_comm_size(comm);
  const uint32_t M = p.n_txps, nf = p.n_fld;
  if (G == 1) {
    if (assigned_out) *assigned_out = p.assigned;
    out->n_compatible = p.compatible;
    return sb_map_project_global(ctx, &p, 1, p.cluster_root, out);
  }
  // log-sum-exp over the ranks; +inf = no mass (salmon's LOG_0); `prior` (counted by every rank) is kept once
  auto lse = [&](const double* vals, size_t n, const double* prior, std::vector<double>& res) -> int {
    res.assign(vals, vals + n);
    double ref = -INFINITY;
    for (size_t i = 0; i < n; ++i) if (std::isfinite(vals[i])) ref = std::max(ref, vals[i]);
    SB_TRY(sb_comm_allreduce(comm, &ref, 1, 0, 2));
    if (!std::isfinite(ref)) return SB_OK;
    std::vector<double> lin(n);
    for (size_t i = 0; i < n; ++i) {
      double v = std::isfinite(vals[i]) ? std::exp(vals[i] - ref) : 0.0;
      if (prior) v = std::max(v - std::exp(prior[i] - ref), 0.0);
      lin[i] = v;
    }
    SB_TRY(sb_comm_allreduce(comm, lin.data(), n, 0, 0));
    for (size_t i = 0; i < n; ++i) {
      const double tot = lin[i] + (prior ? std::exp(prior[i] - ref) : 0.0);
      res[i] = tot > 0.0 ? ref + std::log(tot) : INFINITY;
    }
    return SB_OK;
  };
  std::vector<double> mass, hist, tot1;
  SB_TRY(lse(p.mass, M, nullptr, mass));
  SB_TRY(lse(p.fld_hist, nf, p.fld_prior_hist, hist));
  SB_TRY(lse(&p.fld_tot, 1, &p.fld_prior_tot, tot1));
  std::vector<uint64_t> uniq(p.unique_counts, p.unique_counts + M), total(p.total_counts, p.total_counts + M),
      hits(p.cluster_hits, p.cluster_hits + M);
  SB_TRY(sb_comm_allreduce(comm, uniq.data(), M, 1, 0));
  SB_TRY(sb_comm_allreduce(comm, total.data(), M, 1, 0));
  SB_TRY(sb_comm_allreduce(comm, hits.data(), M, 1, 0));
  uint64_t scal[3] = {p.fld_min, p.assigned, p.compatible};
  SB_TRY(sb_comm_allreduce(comm, &scal[0], 1, 1, 3));
  SB_TRY(sb_comm_allreduce(comm, &scal[1], 2, 1, 0));
  std::vector<uint32_t> roots((size_t)G * std::max<uint32_t>(M, 1));
  SB_TRY(sb_comm_allgather(comm, p.cluster_root, roots.data(), (size_t)M * 4));
  sb_map_partial g = p;
  g.mass = mass.data(); g.fld_hist = hist.data(); g.fld_tot = tot1[0];
  g.unique_counts = uniq.data(); g.total_counts = total.data(); g.cluster_hits = hits.data();
  g.fld_min = (uint32_t)scal[0]; g.assigned = scal[1]; g.compatible = scal[2];
  if (assigned_out) *assigned_out = scal[1];
  out->n_compatible = scal[2];
  return sb_map_project_global(ctx, &g, (uint32_t)G, roots.data(), out);
}
