// ingest.cu -- the input seam of the hot path (host code, no device work): what sits immediately before seam B1 and
// B3 in the reference (SURVEY.md 8f-1 and 3.4/3.5):
//   * sb_reads_*   : FASTQ / FASTA (plain or gzip) -> batches of base codes.  Replaces FQFeeder's
//                    fastx_parser<ReadPair> / <ReadSeq> as salmon drives it (src/quant/SalmonQuantify.cpp:2357-2373
//                    parser construction, :2419-2430 start(), :1118-1141 the per-thread ReadGroup loop).
//   * sb_eq_file_* : the --eqclasses reader (src/util/SalmonUtils.cpp:1024-1122 readEquivCounts).
//   * sb_bootstrap_writer_* : aux_info/bootstrap/bootstraps.gz (src/output/GZipWriter.cpp:765-789 writeBootstrap).
//   * sb_txome_*   : transcript FASTA -> names / base codes / decoy boundary, the input of sb_index_build
//                    (src/index/BuildSalmonIndex.cpp:72-124 options; the FASTA "fixing" itself is pufferfish code that is
//                    not in the reference tree, the rules here follow the option help strings).
//
// Design: one splitter thread per mate stream inflates / reads 8 MiB chunks and cuts them at record boundaries (three
// memchr per record), queueing blocks with a (offset, length) list of the sequence lines; sb_reads_next() hands the
// records of a batch to an OpenMP team that translates bytes to codes straight into the caller's (pinned) buffers.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <time.h>
#include <zlib.h>

#include <condition_variable>
#include <deque>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "common.cuh"
#include "pgzip.h"

namespace {

// base byte -> code (0..3 = A,C,G,T; everything else 4 = N).  U is read as T.
struct CodeLut {
  uint8_t t[256];
  CodeLut() {
    memset(t, 4, sizeof t);
    t['A'] = t['a'] = 0; t['C'] = t['c'] = 1; t['G'] = t['g'] = 2; t['T'] = t['t'] = 3; t['U'] = t['u'] = 3;
  }
};
const CodeLut LUT;

struct RecBlock {               // recycled through Stream::pool: no allocation / page faults in steady state
  char* buf = nullptr;         // raw text of whole records
  size_t cap = 0, len = 0;
  std::vector<uint32_t> seq;   // 2 per record: offset, length of the sequence line
  uint32_t n = 0;
  bool borrowed = false;       // buf points into a memory-mapped file or an inflated piece: not ours to free or reuse
  std::shared_ptr<void> keep;  // (inflated piece: released with the last block that points into it)
  ~RecBlock() { if (!borrowed) free(buf); }
  bool reserve(size_t need) {
    if (need <= cap) return true;
    char* nb = (char*)realloc(buf, need);
    if (!nb) return false;
    buf = nb; cap = need;
    return true;
  }
};

// SB_READS_PROFILE=1: where the reader's time goes (printed by sb_reads_close)
struct Prof {
  double t_read = 0, t_scan = 0, t_push_wait = 0, t_alloc = 0;
};
inline double wall() {
  timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

struct Stream {
  std::vector<std::string> files;
  std::thread th;
  std::mutex mu;
  std::condition_variable cv_put, cv_get;
  std::deque<std::unique_ptr<RecBlock>> q;
  std::vector<std::unique_ptr<RecBlock>> pool;   // consumed blocks, reused by the splitter
  std::vector<std::pair<void*, size_t>> maps;     // memory-mapped plain files (unmapped by sb_reads_close)
  int scanners = 1;                               // plain files: threads that cut sub-ranges of a wave in parallel
  int inflaters = 1;                              // gzip files: inflate threads (pgzip.h); 1 = zlib's gzread
  bool done = false, stop = false;
  std::string err;
  Prof prof;
  // consumer side
  std::deque<std::unique_ptr<RecBlock>> held;   // blocks taken from the queue, not yet fully delivered
  uint32_t front_pos = 0;                        // records of held.front() already delivered
  uint64_t held_recs = 0;                        // records in `held` still to deliver
  bool drained = false;                          // the splitter is done and its queue is empty
};

constexpr size_t CHUNK = 8u << 20;
constexpr size_t MAX_QUEUED = 8;            // blocks of the serial splitter (each owns CHUNK bytes)
constexpr size_t MAX_QUEUED_BORROWED = 96;  // blocks that point into a mapping / an inflated piece

bool push_block(Stream* s, std::unique_ptr<RecBlock> b) {
  std::unique_lock<std::mutex> lk(s->mu);
  s->cv_put.wait(lk, [&] { return s->q.size() < MAX_QUEUED || s->stop; });
  if (s->stop) return false;
  s->q.push_back(std::move(b));
  s->cv_get.notify_one();
  return true;
}
// the blocks of one wave at once: one lock, one wake-up (a thread hand-over costs far more than a block's scan)
bool push_blocks(Stream* s, std::vector<std::unique_ptr<RecBlock>>& bs) {
  std::unique_lock<std::mutex> lk(s->mu);
  s->cv_put.wait(lk, [&] { return s->q.size() < MAX_QUEUED_BORROWED || s->stop; });
  if (s->stop) return false;
  for (auto& b : bs)
    if (b && b->n) s->q.push_back(std::move(b));
  s->cv_get.notify_one();
  return true;
}

void finish_stream(Stream* s, const std::string& err) {
  std::lock_guard<std::mutex> lk(s->mu);
  if (!err.empty()) s->err = err;
  s->done = true;
  s->cv_get.notify_all();
}

inline size_t line_len(const char* b, const char* e) {   // length without a trailing '\r'
  size_t n = (size_t)(e - b);
  if (n && b[n - 1] == '\r') --n;
  return n;
}

// Cut `len` bytes at buf into whole records.  Returns the number of bytes consumed; records are appended to blk->seq
// with offsets relative to buf.  eof: no more data follows (the last line may lack its newline).
size_t scan_records(const char* buf, size_t len, bool eof, RecBlock* blk, std::string& err) {
  size_t p = 0, cut = 0;
  while (p < len) {
    const char c = buf[p];
    if (c == '\n' || c == '\r') { ++p; cut = p; continue; }
    if (c != '@' && c != '>') { err = "malformed read file: record does not start with '@' or '>'"; return cut; }
    const char* nl1 = (const char*)memchr(buf + p, '\n', len - p);
    if (!nl1) break;
    const size_t s0 = (size_t)(nl1 - buf) + 1;
    const char* nl2 = (const char*)memchr(buf + s0, '\n', len - s0);
    if (c == '>') {
      size_t send, next;
      if (nl2) { send = (size_t)(nl2 - buf); next = send + 1; }
      else if (eof) { send = len; next = len; }
      else break;
      if (next >= len && !eof) break;          // cannot see whether the sequence continues on another line
      if (next < len && buf[next] != '>' && buf[next] != '\n' && buf[next] != '\r') {
        err = "multi-line FASTA reads are not supported";
        return cut;
      }
      blk->seq.push_back((uint32_t)s0);
      blk->seq.push_back((uint32_t)line_len(buf + s0, buf + send));
      p = next; cut = p;
      continue;
    }
    if (!nl2) break;
    const size_t slen = line_len(buf + s0, nl2);
    const size_t p3 = (size_t)(nl2 - buf) + 1;
    if (p3 >= len) break;
    if (buf[p3] != '+') { err = "malformed FASTQ: third line of a record does not start with '+' (multi-line FASTQ is not supported)"; return cut; }
    const char* nl3 = (p3 + 1 < len && buf[p3 + 1] == '\n') ? buf + p3 + 1 : (const char*)memchr(buf + p3, '\n', len - p3);
    if (!nl3) break;
    const size_t q0 = (size_t)(nl3 - buf) + 1;
    // the quality line is as long as the sequence line: look for its newline there first
    const size_t raw = (size_t)(nl2 - buf) - s0;
    const char* nl4 = (q0 + raw < len && buf[q0 + raw] == '\n') ? buf + q0 + raw
                      : ((q0 < len) ? (const char*)memchr(buf + q0, '\n', len - q0) : nullptr);
    size_t qend, next;
    if (nl4) { qend = (size_t)(nl4 - buf); next = qend + 1; }
    else if (eof && q0 <= len) { qend = len; next = len; }
    else break;
    if (line_len(buf + q0, buf + qend) != slen) { err = "malformed FASTQ: quality and sequence lengths differ"; return cut; }
    blk->seq.push_back((uint32_t)s0);
    blk->seq.push_back((uint32_t)slen);
    p = next; cut = p;
  }
  return cut;
}

// plain or gzip input behind one read call (gzread's transparent mode costs a copy: plain files are read() directly)
struct Input {
  gzFile g = nullptr;
  FILE* f = nullptr;
  bool open(const char* path) {
    FILE* t = fopen(path, "rb");
    if (!t) return false;
    unsigned char m[2] = {0, 0};
    const size_t k = fread(m, 1, 2, t);
    if (k == 2 && m[0] == 0x1f && m[1] == 0x8b) {
      fclose(t);
      g = gzopen(path, "rb");
      if (g) gzbuffer(g, 1u << 20);
      return g != nullptr;
    }
    rewind(t);
    setvbuf(t, nullptr, _IONBF, 0);
    f = t;
    return true;
  }
  long read(char* dst, size_t n, std::string& err) {
    if (g) {
      const int got = gzread(g, dst, (unsigned)n);
      if (got < 0) { int e; err = gzerror(g, &e); }
      return got;
    }
    const size_t got = fread(dst, 1, n, f);
    if (got < n && ferror(f)) { err = "read error"; return -1; }
    return (long)got;
  }
  void close() { if (g) gzclose(g); if (f) fclose(f); g = nullptr; f = nullptr; }
};

std::unique_ptr<RecBlock> take_block(Stream* s) {
  {
    std::lock_guard<std::mutex> lk(s->mu);
    if (!s->pool.empty()) {
      std::unique_ptr<RecBlock> b = std::move(s->pool.back());
      s->pool.pop_back();
      b->seq.clear(); b->n = 0; b->len = 0;
      return b;
    }
  }
  return std::unique_ptr<RecBlock>(new RecBlock());
}

// ---- plain files: memory-mapped, cut by several threads ------------------------------------------------------------
// One splitter thread per mate file tops out near 12 M records/s (read + scan), a third of what the GPU maps.  A plain
// file is therefore mapped, and a wave of `scanners` x CHUNK bytes is cut into sub-ranges at validated record starts and
// scanned by a thread each; the blocks point into the mapping (no copy) and are queued in file order.
// A FASTQ record start inside the file: a line that begins with '@' whose third line begins with '+' and whose second
// and fourth lines are equally long (a quality line may begin with '@', but then the "third line" is a sequence line).
bool fastq_record_at(const char* buf, size_t p, size_t len) {
  if (p >= len || buf[p] != '@') return false;
  const char* nl1 = (const char*)memchr(buf + p, '\n', len - p);
  if (!nl1) return false;
  const size_t s0 = (size_t)(nl1 - buf) + 1;
  const char* nl2 = (s0 < len) ? (const char*)memchr(buf + s0, '\n', len - s0) : nullptr;
  if (!nl2) return false;
  const size_t p3 = (size_t)(nl2 - buf) + 1;
  if (p3 >= len || buf[p3] != '+') return false;
  const char* nl3 = (const char*)memchr(buf + p3, '\n', len - p3);
  if (!nl3) return false;
  const size_t q0 = (size_t)(nl3 - buf) + 1;
  const char* nl4 = (q0 < len) ? (const char*)memchr(buf + q0, '\n', len - q0) : nullptr;
  const size_t qend = nl4 ? (size_t)(nl4 - buf) : len;
  return line_len(buf + q0, buf + qend) == line_len(buf + s0, nl2);
}
// first record start at or after `from` (a line start), or len
size_t next_record_start(const char* buf, size_t from, size_t len, bool fasta) {
  size_t p = from;
  if (p > 0 && p < len && buf[p - 1] != '\n') {   // move to the next line start
    const char* nl = (const char*)memchr(buf + p, '\n', len - p);
    if (!nl) return len;
    p = (size_t)(nl - buf) + 1;
  }
  while (p < len) {
    if (fasta ? buf[p] == '>' : fastq_record_at(buf, p, len)) return p;
    const char* nl = (const char*)memchr(buf + p, '\n', len - p);
    if (!nl) return len;
    p = (size_t)(nl - buf) + 1;
  }
  return len;
}

// returns false (and leaves the file to the serial path) when the file cannot be mapped
bool split_mapped(Stream* s, const std::string& path, std::string& err) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return false;
  struct stat sb;
  if (fstat(fileno(f), &sb) != 0 || !S_ISREG(sb.st_mode) || sb.st_size == 0) { fclose(f); return false; }
  const size_t len = (size_t)sb.st_size;
  void* mp = mmap(nullptr, len, PROT_READ, MAP_PRIVATE, fileno(f), 0);
  fclose(f);
  if (mp == MAP_FAILED) return false;
  madvise(mp, len, MADV_SEQUENTIAL);
  { std::lock_guard<std::mutex> lk(s->mu); s->maps.emplace_back(mp, len); }
  const char* buf = (const char*)mp;
  size_t pos = 0;
  while (pos < len && (buf[pos] == '\n' || buf[pos] == '\r')) ++pos;
  if (pos >= len) return true;
  if (buf[pos] != '@' && buf[pos] != '>') { err = "malformed read file: record does not start with '@' or '>' (" + path + ")"; return true; }
  const bool fasta = buf[pos] == '>';
  const int W = std::max(1, s->scanners);
  while (pos < len && err.empty()) {
    double t0 = wall();
    // sub-range boundaries of this wave
    std::vector<size_t> b(1, pos);
    for (int i = 1; i <= W; ++i) {
      const size_t target = pos + (size_t)i * CHUNK;
      if (target >= len) { b.push_back(len); break; }
      const size_t q = next_record_start(buf, target, len, fasta);
      if (q > b.back()) b.push_back(q);
      if (q >= len) break;
    }
    const int nr = (int)b.size() - 1;
    std::vector<std::unique_ptr<RecBlock>> blks(nr);
    std::vector<std::string> errs(nr);
    for (int i = 0; i < nr; ++i) {
      blks[i].reset(new RecBlock());
      blks[i]->borrowed = true;
    }
#pragma omp parallel for schedule(static, 1) num_threads(std::min(W, nr))
    for (int i = 0; i < nr; ++i) {
      RecBlock* k = blks[i].get();
      k->buf = const_cast<char*>(buf + b[i]);
      k->len = b[i + 1] - b[i];
      k->seq.reserve(2 * (k->len / 200 + 16));
      // every sub-range holds whole records by construction: the scanner may treat its end like the end of a file
      const size_t cut = scan_records(k->buf, k->len, true, k, errs[i]);
      if (errs[i].empty() && cut != k->len) {
        // bytes after the last whole record: only white space is fine (end of the file)
        for (size_t x = cut; x < k->len; ++x)
          if (k->buf[x] != '\n' && k->buf[x] != '\r' && k->buf[x] != ' ' && k->buf[x] != '\t') {
            errs[i] = (b[i + 1] == len) ? "truncated record at the end of " + path : "malformed record (" + path + ")";
            break;
          }
      }
      k->n = (uint32_t)(k->seq.size() / 2);
    }
    s->prof.t_scan += wall() - t0;
    for (int i = 0; i < nr && err.empty(); ++i)
      if (!errs[i].empty()) { err = errs[i]; if (err.find(path) == std::string::npos) err += " (" + path + ")"; }
    if (err.empty()) {
      t0 = wall();
      const bool pushed = push_blocks(s, blks);
      s->prof.t_push_wait += wall() - t0;
      if (!pushed) { err = "stopped"; break; }
    }
    pos = b.back();
  }
  return true;
}

// Cut [buf, buf+len) -- text that starts at a record start -- into whole records with up to `scanners` threads and queue
// the blocks in order (they point into buf; `keep` keeps it alive).  eof: nothing follows this text.  Returns the bytes
// consumed (the rest is the beginning of a record that continues in the next piece).
size_t scan_wave(Stream* s, const std::shared_ptr<void>& keep, const char* buf, size_t len, bool eof, bool fasta,
                 const std::string& path, std::string& err) {
  const int W = std::max(1, std::min(s->scanners, (int)(len >> 21) + 1));
  std::vector<size_t> b(1, 0);
  for (int i = 1; i < W; ++i) {
    const size_t q = next_record_start(buf, len / W * i, len, fasta);
    if (q > b.back() && q < len) b.push_back(q);
  }
  b.push_back(len);
  const int nr = (int)b.size() - 1;
  std::vector<std::unique_ptr<RecBlock>> blks(nr);
  std::vector<std::string> errs(nr);
  std::vector<size_t> cuts(nr, 0);
  for (int i = 0; i < nr; ++i) { blks[i].reset(new RecBlock()); blks[i]->borrowed = true; blks[i]->keep = keep; }
#pragma omp parallel for schedule(static, 1) num_threads(nr)
  for (int i = 0; i < nr; ++i) {
    RecBlock* k = blks[i].get();
    k->buf = const_cast<char*>(buf + b[i]);
    k->len = b[i + 1] - b[i];
    k->seq.reserve(2 * (k->len / 200 + 16));
    const bool last = i == nr - 1;
    cuts[i] = scan_records(k->buf, k->len, last ? eof : true, k, errs[i]);
    if (errs[i].empty() && cuts[i] != k->len && (!last || eof)) {
      for (size_t x = cuts[i]; x < k->len; ++x)
        if (k->buf[x] != '\n' && k->buf[x] != '\r' && k->buf[x] != ' ' && k->buf[x] != '\t') {
          errs[i] = last ? "truncated record at the end of " + path : "malformed record (" + path + ")";
          break;
        }
    }
    k->n = (uint32_t)(k->seq.size() / 2);
  }
  for (int i = 0; i < nr; ++i)
    if (!errs[i].empty()) { err = errs[i]; if (err.find(path) == std::string::npos) err += " (" + path + ")"; return 0; }
  const double t0 = wall();
  const bool pushed = push_blocks(s, blks);
  s->prof.t_push_wait += wall() - t0;
  if (!pushed) { err = "stopped"; return 0; }
  return b[nr - 1] + cuts[nr - 1];
}

// ---- gzip files: inflated by several threads (pgzip.h), cut like the mapped plain files -------------------------------
// returns false (and leaves the file to the serial gzread path) when the file cannot be mapped or is not gzip
bool split_gz_parallel(Stream* s, const std::string& path, std::string& err) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return false;
  struct stat stt;
  if (fstat(fileno(f), &stt) != 0 || !S_ISREG(stt.st_mode) || stt.st_size == 0) { fclose(f); return false; }
  const size_t flen = (size_t)stt.st_size;
  void* mp = mmap(nullptr, flen, PROT_READ, MAP_PRIVATE, fileno(f), 0);
  fclose(f);
  if (mp == MAP_FAILED) return false;
  madvise(mp, flen, MADV_SEQUENTIAL);
  struct Unmap { void* p; size_t n; ~Unmap() { munmap(p, n); } } unmap{mp, flen};
  sb::pgz::ParallelGz pg((const uint8_t*)mp, flen, s->inflaters);
  std::string perr;
  if (!pg.start(perr)) return false;
  std::vector<char> carry;
  bool first = true, fasta = false;
  sb::pgz::Piece pc;
  for (;;) {
    double t0 = wall();
    const bool more = pg.next(pc, perr);
    s->prof.t_read += wall() - t0;
    if (!more) break;
    std::shared_ptr<void> keep = pc.keep;
    char* data = (char*)pc.data;
    size_t len = pc.len;
    if (!carry.empty()) {
      if (carry.size() <= sb::pgz::HEAD) {             // the piece's head room takes the carried partial record
        data -= carry.size();
        memcpy(data, carry.data(), carry.size());
        len += carry.size();
      } else {
        char* nb = (char*)malloc(carry.size() + len);
        if (!nb) { err = "out of memory"; return true; }
        memcpy(nb, carry.data(), carry.size());
        memcpy(nb + carry.size(), pc.data, len);
        keep = std::shared_ptr<void>(nb, free);
        data = nb;
        len += carry.size();
      }
      carry.clear();
    }
    if (first) {
      size_t p0 = 0;
      while (p0 < len && (data[p0] == '\n' || data[p0] == '\r')) ++p0;
      if (p0 == len) continue;                           // only blank lines so far
      if (data[p0] != '@' && data[p0] != '>') { err = "malformed read file: record does not start with '@' or '>' (" + path + ")"; return true; }
      fasta = data[p0] == '>';
      data += p0; len -= p0;
      first = false;
    }
    t0 = wall();
    const size_t used = scan_wave(s, keep, data, len, false, fasta, path, err);
    s->prof.t_scan += wall() - t0;
    if (!err.empty()) return true;
    carry.assign(data + used, data + len);
  }
  if (!perr.empty()) { err = "read error in " + path + ": " + perr; return true; }
  if (!carry.empty()) {                                  // the last record(s): nothing follows
    char* nb = (char*)malloc(carry.size());
    if (!nb) { err = "out of memory"; return true; }
    memcpy(nb, carry.data(), carry.size());
    std::shared_ptr<void> keep(nb, free);
    if (first) {
      size_t p0 = 0;
      while (p0 < carry.size() && (nb[p0] == '\n' || nb[p0] == '\r')) ++p0;
      if (p0 == carry.size()) return true;
      if (nb[p0] != '@' && nb[p0] != '>') { err = "malformed read file: record does not start with '@' or '>' (" + path + ")"; return true; }
      fasta = nb[p0] == '>';
    }
    scan_wave(s, keep, nb, carry.size(), true, fasta, path, err);
  }
  return true;
}

void split_stream(Stream* s) {
  std::string err;
  for (const std::string& path : s->files) {
    Input in;
    if (!in.open(path.c_str())) { err = "cannot open " + path; break; }
    if (in.f && s->scanners > 0) {   // plain file: mapped and cut in parallel (falls through when it cannot be mapped)
      if (split_mapped(s, path, err)) {
        in.close();
        if (err == "stopped") { finish_stream(s, ""); return; }
        if (!err.empty()) break;
        continue;
      }
    }
    if (in.g && s->inflaters > 1) {   // gzip file: inflated by several threads (falls through when it cannot be mapped)
      if (split_gz_parallel(s, path, err)) {
        in.close();
        if (err == "stopped") { finish_stream(s, ""); return; }
        if (!err.empty()) break;
        continue;
      }
    }
    std::vector<char> carry;
    bool eof = false;
    while (!eof && err.empty()) {
      double t0 = wall();
      std::unique_ptr<RecBlock> blk = take_block(s);
      // slack for the carried-over partial record, so that recycled blocks are not re-allocated
      if (!blk->reserve(std::max<size_t>(carry.size(), 1u << 20) + CHUNK)) { err = "out of memory"; break; }
      if (!carry.empty()) memcpy(blk->buf, carry.data(), carry.size());
      double t1 = wall();
      s->prof.t_alloc += t1 - t0;
      std::string rerr;
      const long got = in.read(blk->buf + carry.size(), CHUNK, rerr);
      t0 = wall();
      s->prof.t_read += t0 - t1;
      if (got < 0) { err = "read error in " + path + ": " + rerr; break; }
      const size_t len = carry.size() + (size_t)got;
      eof = (size_t)got < CHUNK;
      const size_t cut = scan_records(blk->buf, len, eof, blk.get(), err);
      t1 = wall();
      s->prof.t_scan += t1 - t0;
      if (!err.empty()) { err += " (" + path + ")"; break; }
      carry.assign(blk->buf + cut, blk->buf + len);
      blk->len = cut;
      blk->n = (uint32_t)(blk->seq.size() / 2);
      if (eof) {
        for (char ch : carry)
          if (ch != '\n' && ch != '\r' && ch != ' ' && ch != '\t') { err = "truncated record at the end of " + path; break; }
      }
      t0 = wall();
      const bool pushed = !(blk->n && err.empty()) || push_block(s, std::move(blk));
      s->prof.t_push_wait += wall() - t0;
      if (!pushed) { in.close(); finish_stream(s, ""); return; }
    }
    in.close();
    if (!err.empty()) break;
  }
  finish_stream(s, err);
}

// bytes -> base codes, 32 at a time: the low nibble of A C G T U (1 3 7 4 5) indexes a code table and a table of the
// expected upper-case letter; a byte whose upper-case form is not the expected letter is N (4).
#if defined(__x86_64__)
#include <immintrin.h>
__attribute__((target("avx2"))) void translate_avx2(const uint8_t* src, uint8_t* dst, uint32_t n) {
  const __m256i code_tab = _mm256_setr_epi8(4, 0, 4, 1, 3, 3, 4, 2, 4, 4, 4, 4, 4, 4, 4, 4, 4, 0, 4, 1, 3, 3, 4, 2, 4, 4, 4, 4, 4, 4, 4, 4);
  const __m256i chr_tab = _mm256_setr_epi8(0, 'A', 0, 'C', 'T', 'U', 0, 'G', 0, 0, 0, 0, 0, 0, 0, 0, 0, 'A', 0, 'C', 'T', 'U', 0, 'G', 0, 0, 0, 0, 0, 0,
                                           0, 0);
  const __m256i up = _mm256_set1_epi8((char)0xDF), lo = _mm256_set1_epi8(0x0F), four = _mm256_set1_epi8(4);
  uint32_t j = 0;
  for (; j + 32 <= n; j += 32) {
    const __m256i c = _mm256_loadu_si256((const __m256i*)(src + j));
    const __m256i u = _mm256_and_si256(c, up);
    const __m256i nib = _mm256_and_si256(c, lo);
    const __m256i code = _mm256_shuffle_epi8(code_tab, nib);
    const __m256i want = _mm256_shuffle_epi8(chr_tab, nib);
    const __m256i ok = _mm256_cmpeq_epi8(u, want);
    _mm256_storeu_si256((__m256i*)(dst + j), _mm256_blendv_epi8(four, code, ok));
  }
  for (; j < n; ++j) dst[j] = LUT.t[src[j]];
}
const bool HAVE_AVX2 = __builtin_cpu_supports("avx2");
#else
const bool HAVE_AVX2 = false;
inline void translate_avx2(const uint8_t*, uint8_t*, uint32_t) {}
#endif
inline void translate(const uint8_t* src, uint8_t* dst, uint32_t n) {
  if (HAVE_AVX2) { translate_avx2(src, dst, n); return; }
  for (uint32_t j = 0; j < n; ++j) dst[j] = LUT.t[src[j]];
}

// consumer side: make sure `want` undelivered records are held (or the stream has ended)
bool hold(Stream& s, uint64_t want, std::string& err) {
  while (s.held_recs < want && !s.drained) {
    std::unique_lock<std::mutex> lk(s.mu);
    s.cv_get.wait(lk, [&] { return !s.q.empty() || s.done; });
    if (!s.err.empty()) { err = s.err; return false; }
    if (s.q.empty()) { s.drained = true; break; }
    s.held_recs += s.q.front()->n;
    s.held.push_back(std::move(s.q.front()));
    s.q.pop_front();
    s.cv_put.notify_one();
  }
  return true;
}
// n records have been delivered (or skipped): drop them, hand fully consumed blocks back to the splitter
void consume(Stream& s, uint64_t n) {
  s.held_recs -= n;
  while (n > 0) {
    RecBlock* b = s.held.front().get();
    const uint64_t take = std::min<uint64_t>(n, b->n - s.front_pos);
    s.front_pos += (uint32_t)take;
    n -= take;
    if (s.front_pos == b->n) {
      std::unique_ptr<RecBlock> done = std::move(s.held.front());
      s.held.pop_front();
      s.front_pos = 0;
      std::lock_guard<std::mutex> lk(s.mu);
      if (!done->borrowed && s.pool.size() < 2 * MAX_QUEUED) s.pool.push_back(std::move(done));
    }
  }
}

struct Task {
  const RecBlock* blk;
  uint32_t from, cnt;
  uint64_t dst;
  int mate;
};

}  // namespace

struct sb_reads {
  Stream st[2];
  int n_streams = 0;
  uint32_t n_threads = 1;
  uint64_t n_delivered = 0;
  uint32_t max_len_seen = 0;
  bool failed = false;
  double t_wait_blocks = 0, t_translate = 0;
  // sb_reads_next_meta: names / qualities of the last delivery
  std::vector<const char*> name_src;
  std::vector<uint32_t> name_len;
  std::string names;
  std::vector<uint64_t> name_off;
  std::vector<uint8_t> qual[2];
};

namespace {
// The header line of the record whose sequence line starts at buf + seq_off: it ends just before the sequence line
// and starts at the block's start or after a newline.
inline const char* record_header(const char* buf, uint32_t seq_off) {
  int64_t i = (int64_t)seq_off - 2;   // (buf[seq_off - 1] is the header's newline)
  while (i >= 0 && buf[i] != '\n') --i;
  return buf + i + 1;
}
// QNAME: the header after '@' / '>' up to the first white space, a trailing "/1" or "/2" removed
inline uint32_t read_name(const char* hdr, const char** start) {
  const char* p = hdr + 1;
  uint32_t n = 0;
  while (p[n] != '\n' && p[n] != '\r' && p[n] != ' ' && p[n] != '\t') ++n;
  if (n >= 2 && p[n - 2] == '/' && (p[n - 1] == '1' || p[n - 1] == '2')) n -= 2;
  *start = p;
  return n;
}
// the quality line of a FASTQ record (sequence line at seq_off, len characters before its line end)
inline const char* record_quality(const char* buf, uint32_t seq_off, uint32_t len) {
  const char* p = buf + seq_off + len;
  if (*p == '\r') ++p;
  ++p;                                         // '\n'; now at the '+' line
  while (*p != '\n') ++p;
  return p + 1;
}
}  // namespace

extern "C" sb_reads* sb_reads_open(const char* const* files1, const char* const* files2, uint32_t n_files,
                                   uint32_t n_threads) {
  if (!files1 || !n_files) { sb::set_error("sb_reads_open: no input files"); return nullptr; }
  sb_reads* r = new sb_reads();
  r->n_streams = files2 ? 2 : 1;
  r->n_threads = n_threads ? n_threads : 1;
  for (uint32_t i = 0; i < n_files; ++i) {
    if (!files1[i] || (files2 && !files2[i])) { delete r; sb::set_error("sb_reads_open: null file name"); return nullptr; }
    r->st[0].files.push_back(files1[i]);
    if (files2) r->st[1].files.push_back(files2[i]);
  }
  // plain files are cut by several scanner threads per stream (SB_READS_SCANNERS overrides; 0 = serial splitter)
  int scanners = (int)std::max<uint32_t>(1, std::min<uint32_t>(8, r->n_threads / 4));
  if (const char* e = getenv("SB_READS_SCANNERS")) scanners = atoi(e);
  // gzip files: inflate threads per stream (SB_READS_INFLATERS overrides; 1 = zlib's gzread on the splitter thread)
  int inflaters = (int)std::max<uint32_t>(1, std::min<uint32_t>(32, r->n_threads / (uint32_t)r->n_streams));
  if (const char* e = getenv("SB_READS_INFLATERS")) inflaters = std::max(1, atoi(e));
  for (int m = 0; m < r->n_streams; ++m) { r->st[m].scanners = scanners; r->st[m].inflaters = inflaters; }
  for (int m = 0; m < r->n_streams; ++m) r->st[m].th = std::thread(split_stream, &r->st[m]);
  return r;
}

extern "C" void sb_reads_close(sb_reads* r) {
  if (!r) return;
  for (int m = 0; m < r->n_streams; ++m) {
    { std::lock_guard<std::mutex> lk(r->st[m].mu); r->st[m].stop = true; }
    r->st[m].cv_put.notify_all();
    if (r->st[m].th.joinable()) r->st[m].th.join();
  }
  for (int m = 0; m < r->n_streams; ++m) {   // blocks that point into the mappings go first
    r->st[m].held.clear(); r->st[m].q.clear(); r->st[m].pool.clear();
    for (auto& mp : r->st[m].maps) munmap(mp.first, mp.second);
    r->st[m].maps.clear();
  }
  if (getenv("SB_READS_PROFILE")) {
    for (int m = 0; m < r->n_streams; ++m)
      fprintf(stderr, "sb_reads: stream %d splitter: alloc %.3f s, read/inflate %.3f s, scan %.3f s, waiting for the consumer %.3f s\n", m,
              r->st[m].prof.t_alloc, r->st[m].prof.t_read, r->st[m].prof.t_scan, r->st[m].prof.t_push_wait);
    fprintf(stderr, "sb_reads: consumer: waiting for blocks %.3f s, translating %.3f s, %llu records\n", r->t_wait_blocks, r->t_translate,
            (unsigned long long)r->n_delivered);
  }
  delete r;
}

static int64_t reads_next(sb_reads* r, uint32_t max_pairs, uint32_t stride, uint8_t* left, uint8_t* right,
                          uint32_t* len_left, uint32_t* len_right, bool want_names, bool want_quals) {
  if (!r || !left || !len_left || !stride || (r->n_streams == 2 && (!right || !len_right))) {
    sb::set_error("sb_reads_next: null argument"); return SB_ERR_INVALID;
  }
  if (r->failed) { sb::set_error("sb_reads_next: the reader is in a failed state"); return SB_ERR_INVALID; }
  std::vector<Task> tasks;
  uint64_t filled[2] = {0, 0};
  const double tw0 = wall();
  for (int m = 0; m < r->n_streams; ++m) {
    Stream& s = r->st[m];
    std::string err;
    if (!hold(s, max_pairs, err)) { r->failed = true; sb::set_error("%s", err.c_str()); return SB_ERR_INVALID; }
    size_t bi = 0;
    uint32_t pos = s.front_pos;
    while (filled[m] < max_pairs && bi < s.held.size()) {
      RecBlock* b = s.held[bi].get();
      const uint32_t take = (uint32_t)std::min<uint64_t>(b->n - pos, max_pairs - filled[m]);
      for (uint32_t o = 0; o < take; o += 2048)
        tasks.push_back(Task{b, pos + o, std::min(2048u, take - o), filled[m] + o, m});
      filled[m] += take;
      pos += take;
      if (pos == b->n) { ++bi; pos = 0; }
    }
  }
  if (r->n_streams == 2 && filled[0] != filled[1]) {
    r->failed = true;
    sb::set_error("the mate files hold different numbers of records (after %llu pairs)",
                  (unsigned long long)(r->n_delivered + std::min(filled[0], filled[1])));
    return SB_ERR_INVALID;
  }
  uint32_t maxlen = 0;
  const double tw1 = wall();
  r->t_wait_blocks += tw1 - tw0;
  const int nt = (int)std::max<size_t>(1, std::min<size_t>(r->n_threads, tasks.size()));
  if (want_names) { r->name_src.resize(filled[0]); r->name_len.resize(filled[0]); }
  if (want_quals)
    for (int m = 0; m < r->n_streams; ++m) r->qual[m].resize((size_t)filled[m] * stride);
#pragma omp parallel for schedule(dynamic, 1) num_threads(nt) reduction(max : maxlen)
  for (long ti = 0; ti < (long)tasks.size(); ++ti) {
    const Task& t = tasks[ti];
    uint8_t* out = t.mate ? right : left;
    uint32_t* lens = t.mate ? len_right : len_left;
    for (uint32_t i = 0; i < t.cnt; ++i) {
      const uint32_t off = t.blk->seq[2 * (size_t)(t.from + i)], len = t.blk->seq[2 * (size_t)(t.from + i) + 1];
      maxlen = std::max(maxlen, len);
      lens[t.dst + i] = len;
      const uint32_t n = std::min(len, stride);
      const uint8_t* src = (const uint8_t*)t.blk->buf + off;
      uint8_t* d = out + (t.dst + i) * (size_t)stride;
      translate(src, d, n);
      if (n < stride) memset(d + n, 4, stride - n);
      if (want_names || want_quals) {
        const char* hdr = record_header(t.blk->buf, off);
        if (want_names && t.mate == 0) r->name_len[t.dst + i] = read_name(hdr, &r->name_src[t.dst + i]);
        if (want_quals) {
          uint8_t* q = r->qual[t.mate].data() + (t.dst + i) * (size_t)stride;
          if (hdr[0] == '@') memcpy(q, record_quality(t.blk->buf, off, len), n);
          else memset(q, 'I', n);
        }
      }
    }
  }
  if (want_names) {
    const uint64_t nn = filled[0];
    r->name_off.resize(nn + 1);
    r->name_off[0] = 0;
    for (uint64_t i = 0; i < nn; ++i) r->name_off[i + 1] = r->name_off[i] + r->name_len[i];
    r->names.resize(r->name_off[nn]);
#pragma omp parallel for schedule(static) num_threads(nt)
    for (int64_t i = 0; i < (int64_t)nn; ++i) memcpy(&r->names[r->name_off[i]], r->name_src[i], r->name_len[i]);
  }
  r->t_translate += wall() - tw1;
  for (int m = 0; m < r->n_streams; ++m) consume(r->st[m], filled[m]);
  r->max_len_seen = std::max(r->max_len_seen, maxlen);
  if (maxlen > stride) {
    r->failed = true;
    sb::set_error("a read of %u bases exceeds the buffer stride of %u", maxlen, stride);
    return SB_ERR_INVALID;
  }
  r->n_delivered += filled[0];
  return (int64_t)filled[0];
}

extern "C" int64_t sb_reads_next(sb_reads* r, uint32_t max_pairs, uint32_t stride, uint8_t* left, uint8_t* right,
                                 uint32_t* len_left, uint32_t* len_right) {
  return reads_next(r, max_pairs, stride, left, right, len_left, len_right, false, false);
}

extern "C" int64_t sb_reads_next_meta(sb_reads* r, uint32_t max_pairs, uint32_t stride, uint8_t* left, uint8_t* right,
                                      uint32_t* len_left, uint32_t* len_right, int want_quals, sb_read_meta* meta) {
  if (!meta) { sb::set_error("sb_reads_next_meta: null argument"); return SB_ERR_INVALID; }
  const int64_t got = reads_next(r, max_pairs, stride, left, right, len_left, len_right, true, want_quals != 0);
  if (got < 0) return got;
  meta->names = r->names.data();
  meta->name_off = r->name_off.data();
  meta->qual_left = want_quals ? r->qual[0].data() : nullptr;
  meta->qual_right = (want_quals && r->n_streams == 2) ? r->qual[1].data() : nullptr;
  return got;
}

// Look at the lengths of the next records without delivering them: returns how many records (pairs) the next call can
// deliver, up to max_pairs (fewer only at the end of the input), and in *uniform_len their common length when every
// read of both mates has the same one (else 0).  Lets a caller that groups reads by length take the usual case --
// one length -- straight into its [n, L] buffer with sb_reads_next(..., stride = L, ...).
extern "C" int64_t sb_reads_peek(sb_reads* r, uint32_t max_pairs, uint32_t* uniform_len) {
  if (!r) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  if (r->failed) { sb::set_error("sb_reads_peek: the reader is in a failed state"); return SB_ERR_INVALID; }
  uint64_t n = max_pairs;
  const double tw0 = wall();
  for (int m = 0; m < r->n_streams; ++m) {
    std::string err;
    if (!hold(r->st[m], max_pairs, err)) { r->failed = true; sb::set_error("%s", err.c_str()); return SB_ERR_INVALID; }
    n = std::min<uint64_t>(n, r->st[m].held_recs);
  }
  r->t_wait_blocks += wall() - tw0;
  if (uniform_len) {
    uint32_t L = 0;
    bool uni = n > 0;
    for (int m = 0; m < r->n_streams && uni; ++m) {
      const Stream& s = r->st[m];
      uint64_t left = n;
      uint32_t pos = s.front_pos;
      for (size_t bi = 0; bi < s.held.size() && left > 0 && uni; ++bi, pos = 0) {
        const RecBlock* b = s.held[bi].get();
        const uint64_t take = std::min<uint64_t>(left, b->n - pos);
        if (m == 0 && bi == 0 && take > 0) L = b->seq[2 * (size_t)pos + 1];
        for (uint64_t i = 0; i < take; ++i)
          if (b->seq[2 * (size_t)(pos + i) + 1] != L) { uni = false; break; }
        left -= take;
      }
    }
    *uniform_len = uni ? L : 0;
  }
  return (int64_t)n;
}

extern "C" int sb_reads_paired(const sb_reads* r) { return (r && r->n_streams == 2) ? 1 : 0; }

// Drop the next n records (pairs) unread (another shard's batch).  Returns the number dropped.
extern "C" int64_t sb_reads_skip(sb_reads* r, uint32_t n) {
  if (!r) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  if (r->failed) { sb::set_error("sb_reads_skip: the reader is in a failed state"); return SB_ERR_INVALID; }
  uint64_t k = n;
  for (int m = 0; m < r->n_streams; ++m) {
    std::string err;
    if (!hold(r->st[m], n, err)) { r->failed = true; sb::set_error("%s", err.c_str()); return SB_ERR_INVALID; }
    k = std::min<uint64_t>(k, r->st[m].held_recs);
  }
  if (r->n_streams == 2 && k < n && r->st[0].held_recs != r->st[1].held_recs) {
    r->failed = true;
    sb::set_error("the mate files hold different numbers of records (after %llu pairs)", (unsigned long long)(r->n_delivered + k));
    return SB_ERR_INVALID;
  }
  for (int m = 0; m < r->n_streams; ++m) consume(r->st[m], k);
  r->n_delivered += k;
  return (int64_t)k;
}

// ---------------------------------------------------------------------------------------------------------------------
// --eqclasses reader
// ---------------------------------------------------------------------------------------------------------------------
namespace {
// a whole text file (plain or gzip) into memory; a regular gzip file of some size is inflated by several threads
bool slurp(const char* path, std::string& out, std::string& err) {
  {
    FILE* f = fopen(path, "rb");
    struct stat stt;
    if (f && fstat(fileno(f), &stt) == 0 && S_ISREG(stt.st_mode) && stt.st_size > (8 << 20)) {
      const size_t flen = (size_t)stt.st_size;
      void* mp = mmap(nullptr, flen, PROT_READ, MAP_PRIVATE, fileno(f), 0);
      if (mp != MAP_FAILED) {
        bool handled = false, ok = true;
        {
          sb::pgz::ParallelGz pg((const uint8_t*)mp, flen, 8);
          std::string perr;
          if (pg.start(perr)) {     // (not gzip: the plain path below reads it)
            handled = true;
            sb::pgz::Piece pc;
            while (pg.next(pc, perr)) out.append((const char*)pc.data, pc.len);
            if (!perr.empty()) { err = std::string("read error in ") + path + ": " + perr; ok = false; }
          }
        }
        munmap(mp, flen);
        if (handled) { fclose(f); return ok; }
      }
    }
    if (f) fclose(f);
  }
  gzFile g = gzopen(path, "rb");
  if (!g) { err = std::string("cannot open ") + path; return false; }
  gzbuffer(g, 1u << 20);
  std::vector<char> buf(4u << 20);
  for (;;) {
    const int got = gzread(g, buf.data(), (unsigned)buf.size());
    if (got < 0) { int e; err = std::string("read error in ") + path + ": " + gzerror(g, &e); gzclose(g); return false; }
    out.append(buf.data(), (size_t)got);
    if ((size_t)got < buf.size()) break;
  }
  gzclose(g);
  return true;
}
struct Tok {   // whitespace tokenizer that also knows where lines end
  const char* p; const char* e;
  void skip_ws() { while (p < e && (*p == ' ' || *p == '\t' || *p == '\n' || *p == '\r')) ++p; }
  bool next(const char*& b, size_t& n) {
    skip_ws();
    if (p >= e) return false;
    b = p;
    while (p < e && !(*p == ' ' || *p == '\t' || *p == '\n' || *p == '\r')) ++p;
    n = (size_t)(p - b);
    return true;
  }
};
struct EqFileStore {
  sb_eq_file pub;
  std::vector<std::string> names;
  std::vector<const char*> name_ptrs;
  std::vector<uint64_t> off, counts;
  std::vector<uint32_t> tids;
  std::vector<double> weights, eff;
};
}  // namespace

extern "C" int sb_eq_file_read(const char* path, sb_eq_file** out) {
  if (!path || !out) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  std::string text, err;
  if (!slurp(path, text, err)) { sb::set_error("%s", err.c_str()); return SB_ERR_INVALID; }
  std::unique_ptr<EqFileStore> S(new EqFileStore());
  Tok tk{text.data(), text.data() + text.size()};
  const char* b; size_t n;
  auto bad = [&](const char* what) { sb::set_error("%s: %s", path, what); return SB_ERR_INVALID; };
  auto get_u64 = [&](uint64_t& v) {
    if (!tk.next(b, n)) return false;
    if (n == 0 || *b == '-' || *b == '+') return false;     // strtoull would wrap a negative number
    char* endp = nullptr;
    v = strtoull(b, &endp, 10);
    return endp == b + n;
  };
  uint64_t numTxps = 0, numEq = 0;
  if (!get_u64(numTxps) || !get_u64(numEq)) return bad("missing transcript / class counts");
  if (numTxps > 0xffffffffull) return bad("too many transcripts");
  // every name / class takes at least two bytes of the file: header values beyond that are corrupt (and would make
  // the reservations below throw through the C boundary)
  if (numTxps > text.size() / 2 + 1 || numEq > text.size() / 2 + 1) return bad("header counts exceed the file size");
  try {
  S->names.reserve(numTxps);
  std::unordered_map<std::string, uint32_t> nameToIndex;
  nameToIndex.reserve(numTxps * 2);
  for (uint64_t i = 0; i < numTxps; ++i) {
    if (!tk.next(b, n)) return bad("truncated transcript name list");
    S->names.emplace_back(b, n);
    nameToIndex[S->names.back()] = (uint32_t)i;
  }
  S->off.reserve(numEq + 1);
  S->off.push_back(0);
  S->counts.reserve(numEq);
  int has_w = -1;
  for (uint64_t c = 0; c < numEq; ++c) {
    uint64_t k = 0;
    if (!get_u64(k) || k == 0) return bad("bad class size");
    for (uint64_t i = 0; i < k; ++i) {
      uint64_t t;
      if (!get_u64(t) || t >= numTxps) return bad("bad transcript id in a class");
      S->tids.push_back((uint32_t)t);
    }
    // the rest of the line: either `count` or `w_1 .. w_k count` (--dumpEqWeights, what readEquivCounts expects)
    const char* line_end = (const char*)memchr(tk.p, '\n', (size_t)(tk.e - tk.p));
    if (!line_end) line_end = tk.e;
    size_t ntok = 0;
    { Tok t2{tk.p, line_end}; const char* bb; size_t nn; while (t2.next(bb, nn)) ++ntok; }
    const int w_here = (ntok == k + 1) ? 1 : (ntok == 1 ? 0 : -1);
    if (w_here < 0) return bad("class line has neither `count` nor `weights count` after the ids");
    if (has_w < 0) has_w = w_here;
    if (has_w != w_here) return bad("classes with and without weights are mixed");
    if (w_here)
      for (uint64_t i = 0; i < k; ++i) {
        if (!tk.next(b, n)) return bad("truncated class");
        char* endp = nullptr;
        const double w = strtod(b, &endp);
        if (endp != b + n) return bad("bad weight");
        S->weights.push_back(w);
      }
    uint64_t cnt;
    if (!get_u64(cnt)) return bad("bad class count");
    S->counts.push_back(cnt);
    S->off.push_back(S->tids.size());
  }
  // optional trailer: `name effective_length` lines; missing ones are set to 100.0 (SalmonUtils.cpp:1109-1116)
  S->eff.assign(numTxps, 100.0);
  std::vector<uint8_t> seen(numTxps, 0);
  uint32_t n_seen = 0;
  while (tk.next(b, n)) {
    std::string nm(b, n);
    if (!tk.next(b, n)) return bad("effective-length trailer: name without a value");
    char* endp = nullptr;
    const double v = strtod(b, &endp);
    if (endp != b + n) return bad("effective-length trailer: bad value");
    auto it = nameToIndex.find(nm);
    if (it == nameToIndex.end()) return bad("effective-length trailer names an unknown transcript");
    if (!seen[it->second]) { seen[it->second] = 1; ++n_seen; }
    S->eff[it->second] = v;
  }
  S->name_ptrs.resize(numTxps);
  for (uint64_t i = 0; i < numTxps; ++i) S->name_ptrs[i] = S->names[i].c_str();
  sb_eq_file& P = S->pub;
  memset(&P, 0, sizeof P);
  P.n_txps = (uint32_t)numTxps;
  P.has_weights = has_w > 0 ? 1u : 0u;
  P.n_classes = numEq;
  P.names = S->name_ptrs.data();
  P.off = S->off.data();
  P.tids = S->tids.data();
  P.weights = P.has_weights ? S->weights.data() : nullptr;
  P.counts = S->counts.data();
  P.eff_len = S->eff.data();
  P.n_missing_eff_len = (uint32_t)(numTxps - n_seen);
  *out = &S.release()->pub;
  return SB_OK;
  } catch (const std::bad_alloc&) {
    sb::set_error("%s: out of memory", path);
    return SB_ERR_NOMEM;
  } catch (const std::exception& ex) {
    sb::set_error("%s: %s", path, ex.what());
    return SB_ERR_INVALID;
  }
}

extern "C" void sb_eq_file_free(sb_eq_file* f) {
  if (f) delete reinterpret_cast<EqFileStore*>(f);   // pub is the first member
}

// ---------------------------------------------------------------------------------------------------------------------
// bootstraps.gz
// ---------------------------------------------------------------------------------------------------------------------
// bootstraps.gz is one gzip member, as the reference writes it (zstr::ofstream at level 6, GZipWriter.cpp:774-783), but
// deflated by a team of threads the way pigz does it: every 128 KiB slice of a sample is a raw deflate stream of its own that
// ends on a byte boundary (Z_SYNC_FLUSH), the slices are written back to back, the member's CRC is combined from the
// slices' CRCs.  (One zlib thread writes ~40 MB/s of doubles: 100 samples at human scale took longer than sampling them.)
struct sb_bootstrap_writer {
  FILE* f = nullptr;
  std::mutex mu;
  uint64_t n_written = 0;
  uint32_t crc = 0;
  uint64_t total = 0;
  bool failed = false;
};

extern "C" sb_bootstrap_writer* sb_bootstrap_writer_open(const char* path) {
  if (!path) { sb::set_error("null argument"); return nullptr; }
  FILE* f = fopen(path, "wb");
  if (!f) { sb::set_error("cannot open %s", path); return nullptr; }
  static const unsigned char hdr[10] = {0x1f, 0x8b, 8, 0, 0, 0, 0, 0, 0, 3};   // deflate, no name / time, OS = Unix
  if (fwrite(hdr, 1, 10, f) != 10) { fclose(f); sb::set_error("write error (bootstraps)"); return nullptr; }
  sb_bootstrap_writer* w = new sb_bootstrap_writer();
  w->f = f;
  return w;
}

// One sample = n raw native-endian doubles appended to the stream (GZipWriter.cpp:779-783); callable from several
// threads like the reference's writeBootstrap (serialised by a mutex, :766-771).
extern "C" int sb_bootstrap_writer_write(sb_bootstrap_writer* w, const double* sample, uint32_t n) {
  if (!w || !sample) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  std::lock_guard<std::mutex> lk(w->mu);
  if (w->failed) { sb::set_error("write error (bootstraps)"); return SB_ERR_INVALID; }
  const size_t bytes = (size_t)n * sizeof(double);
  constexpr size_t SLICE = (size_t)128 << 10;   // (pigz's block size)
  const long ns = (long)((bytes + SLICE - 1) / SLICE);
  std::vector<std::vector<unsigned char>> outs((size_t)ns);
  std::vector<uint32_t> crcs((size_t)ns, 0);
  int bad = 0;
#pragma omp parallel for schedule(dynamic, 1) num_threads((int)std::max<long>(1, std::min<long>(8, ns))) reduction(| : bad)
  for (long i = 0; i < ns; ++i) {
    const unsigned char* src = (const unsigned char*)sample + (size_t)i * SLICE;
    const size_t len = std::min(SLICE, bytes - (size_t)i * SLICE);
    z_stream zs;
    memset(&zs, 0, sizeof zs);
    if (deflateInit2(&zs, 6, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY) != Z_OK) { bad = 1; continue; }
    outs[(size_t)i].resize(deflateBound(&zs, (uLong)len) + 64);
    zs.next_in = const_cast<Bytef*>(src); zs.avail_in = (uInt)len;
    zs.next_out = outs[(size_t)i].data(); zs.avail_out = (uInt)outs[(size_t)i].size();
    const int rc = deflate(&zs, Z_SYNC_FLUSH);
    if (rc != Z_OK || zs.avail_in != 0 || zs.avail_out == 0) bad = 1;
    outs[(size_t)i].resize(outs[(size_t)i].size() - zs.avail_out);
    deflateEnd(&zs);
    crcs[(size_t)i] = (uint32_t)crc32(0, src, (uInt)len);
  }
  if (bad) { w->failed = true; sb::set_error("deflate failed (bootstraps)"); return SB_ERR_INVALID; }
  for (long i = 0; i < ns; ++i) {
    if (fwrite(outs[(size_t)i].data(), 1, outs[(size_t)i].size(), w->f) != outs[(size_t)i].size()) {
      w->failed = true; sb::set_error("write error (bootstraps)"); return SB_ERR_INVALID;
    }
    const size_t len = std::min(SLICE, bytes - (size_t)i * SLICE);
    w->crc = (uint32_t)crc32_combine(w->crc, crcs[(size_t)i], (z_off_t)len);
    w->total += len;
  }
  ++w->n_written;
  return SB_OK;
}

// returns the number of samples written, or a negative code when the file could not be completed
extern "C" int64_t sb_bootstrap_writer_close(sb_bootstrap_writer* w) {
  if (!w) return 0;
  int64_t n = (int64_t)w->n_written;
  // the final (empty, fixed-code) block, then CRC-32 and the length modulo 2^32
  unsigned char tail[10] = {0x03, 0x00, 0, 0, 0, 0, 0, 0, 0, 0};
  const uint32_t c = w->crc, l = (uint32_t)w->total;
  for (int i = 0; i < 4; ++i) { tail[2 + i] = (unsigned char)(c >> (8 * i)); tail[6 + i] = (unsigned char)(l >> (8 * i)); }
  bool ok = !w->failed && fwrite(tail, 1, 10, w->f) == 10;
  ok = (fclose(w->f) == 0) && ok;
  if (!ok) { sb::set_error("write error (bootstraps)"); n = SB_ERR_INVALID; }
  delete w;
  return n;
}

// ---------------------------------------------------------------------------------------------------------------------
// transcript FASTA -> sb_txome
// ---------------------------------------------------------------------------------------------------------------------
namespace {
struct TxomeStore {
  sb_txome pub;
  std::vector<std::string> names;
  std::vector<const char*> name_ptrs;
  std::vector<uint64_t> seq_off;
  std::vector<uint8_t> codes;
  std::vector<uint32_t> complete_len;
};
inline uint64_t fnv1a(const uint8_t* p, size_t n) {
  uint64_t h = 1469598103934665603ull;
  for (size_t i = 0; i < n; ++i) { h ^= p[i]; h *= 1099511628211ull; }
  return h;
}
}  // namespace

extern "C" int sb_txome_read_fasta(const char* path, uint32_t k, int gencode, const char* decoys_path, int no_clip,
                                   int keep_duplicates, sb_txome** out) {
  if (!path || !out) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  std::string text, err;
  if (!slurp(path, text, err)) { sb::set_error("%s", err.c_str()); return SB_ERR_INVALID; }
  std::unordered_set<std::string> decoys;
  if (decoys_path && *decoys_path) {
    std::string dtext;
    if (!slurp(decoys_path, dtext, err)) { sb::set_error("%s", err.c_str()); return SB_ERR_INVALID; }
    Tok tk{dtext.data(), dtext.data() + dtext.size()};
    const char* b; size_t n;
    while (tk.next(b, n)) decoys.emplace(b, n);
  }
  std::unique_ptr<TxomeStore> S(new TxomeStore());
  S->seq_off.push_back(0);
  std::unordered_map<uint64_t, std::vector<uint32_t>> by_hash;
  uint32_t n_dup = 0, n_clipped = 0, n_short = 0, first_decoy = 0xffffffffu;
  const char* p = text.data();
  const char* e = p + text.size();
  std::vector<uint8_t> seq;
  while (p < e) {
    while (p < e && (*p == '\n' || *p == '\r')) ++p;
    if (p >= e) break;
    if (*p != '>') { sb::set_error("%s: expected '>' at the start of a record", path); return SB_ERR_INVALID; }
    const char* nl = (const char*)memchr(p, '\n', (size_t)(e - p));
    if (!nl) nl = e;
    const char* hb = p + 1;
    const char* he = hb;
    // the name ends at the first white space (or, with --gencode, at the first '|'; BuildSalmonIndex.cpp:82-88)
    while (he < nl && *he != ' ' && *he != '\t' && *he != '\r' && !(gencode && *he == '|')) ++he;
    std::string name(hb, he);
    p = (nl < e) ? nl + 1 : e;
    seq.clear();
    while (p < e && *p != '>') {
      const char* l2 = (const char*)memchr(p, '\n', (size_t)(e - p));
      if (!l2) l2 = e;
      for (const char* q = p; q < l2; ++q)
        if (*q != '\r' && *q != ' ') seq.push_back(LUT.t[(uint8_t)*q]);
      p = (l2 < e) ? l2 + 1 : e;
    }
    const uint32_t complete = (uint32_t)seq.size();
    const bool is_decoy = decoys.count(name) != 0;
    if (is_decoy) {
      if (first_decoy == 0xffffffffu) first_decoy = (uint32_t)S->names.size();
    } else if (first_decoy != 0xffffffffu) {
      sb::set_error("%s: the non-decoy sequence %s follows a decoy; decoys must come last", path, name.c_str());
      return SB_ERR_INVALID;
    }
    // poly-A clipping (--no-clip turns it off): a run of more than 10 trailing A's is removed
    if (!no_clip && !is_decoy) {
      size_t a = seq.size();
      while (a > 0 && seq[a - 1] == 0) --a;
      if (seq.size() - a > 10) { seq.resize(a); ++n_clipped; }
    }
    if (seq.size() < k) ++n_short;
    if (!keep_duplicates && !is_decoy) {
      const uint64_t h = fnv1a(seq.data(), seq.size());
      auto& cand = by_hash[h];
      bool dup = false;
      for (uint32_t t : cand) {
        const uint64_t b0 = S->seq_off[t], n0 = S->seq_off[t + 1] - b0;
        if (n0 == seq.size() && (n0 == 0 || memcmp(S->codes.data() + b0, seq.data(), n0) == 0)) { dup = true; break; }
      }
      if (dup) { ++n_dup; continue; }
      cand.push_back((uint32_t)S->names.size());
    }
    // a decoy longer than the index's per-reference limit (2^21 - 1 bases; chromosomes are 100x that) is stored as
    // overlapping pieces: a decoy only matters as "the best hit of a read is in a decoy" (SalmonMappingUtils.hpp:
    // 268-283), and with an overlap above the longest read every read that lies in the chromosome lies in one piece
    constexpr size_t PIECE = 2000000, OVERLAP = 1024;
    if (is_decoy && seq.size() > PIECE) {
      size_t part = 0;
      for (size_t a = 0; a < seq.size(); a += PIECE - OVERLAP, ++part) {
        const size_t b = std::min(seq.size(), a + PIECE);
        S->names.push_back(name + ":" + std::to_string(part));
        S->complete_len.push_back((uint32_t)(b - a));
        S->codes.insert(S->codes.end(), seq.begin() + (long)a, seq.begin() + (long)b);
        S->seq_off.push_back(S->codes.size());
        if (b == seq.size()) break;
      }
      continue;
    }
    S->names.push_back(std::move(name));
    S->complete_len.push_back(complete);
    S->codes.insert(S->codes.end(), seq.begin(), seq.end());
    S->seq_off.push_back(S->codes.size());
  }
  S->name_ptrs.resize(S->names.size());
  for (size_t i = 0; i < S->names.size(); ++i) S->name_ptrs[i] = S->names[i].c_str();
  sb_txome& P = S->pub;
  memset(&P, 0, sizeof P);
  P.n_txps = (uint32_t)S->names.size();
  P.first_decoy = (first_decoy == 0xffffffffu) ? P.n_txps : first_decoy;
  P.names = S->name_ptrs.data();
  P.seq_off = S->seq_off.data();
  P.codes = S->codes.data();
  P.complete_len = S->complete_len.data();
  P.n_duplicates_removed = n_dup;
  P.n_clipped = n_clipped;
  P.n_short = n_short;
  *out = &S.release()->pub;
  return SB_OK;
}

extern "C" void sb_txome_free(sb_txome* t) {
  if (t) delete reinterpret_cast<TxomeStore*>(t);
}
