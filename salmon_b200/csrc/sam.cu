// sam.cu -- SAM output of the mapping path (`salmon quant --writeMappings`), formatted on the GPU.
//
//   k_sam_size   one thread per fragment: bytes of its records and of its unmapped-names line
//   cub scan     exclusive sums -> each fragment's offset in the batch's text
//   k_sam_write  one warp per fragment: writes the text of a window of fragments that fits the device buffer
//
// The per-record rules live in sam_core.h (shared with the host build the tests use).  Each window is copied into one
// of two page-locked buffers and written out by the sink's writer thread in batch order, so the file writes overlap
// the mapping of the next batch.
#include <string.h>
#include <time.h>

#include <condition_variable>
#include <cub/cub.cuh>
#include <deque>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "sam_core.h"
#include "resources.h"
#include "sam_internal.h"

using namespace sbsam;

struct sb_sam {
  FILE* sam = nullptr;
  FILE* un = nullptr;
  bool sam_is_stdout = false;
  uint32_t flags = 0;
  uint32_t n_txps = 0;
  std::vector<uint32_t> ref_len;
  std::vector<uint64_t> rname_off;
  std::string rnames;
  // writer thread: jobs in batch order; a job is a page-locked slot or a string of its own
  struct Job { int slot; size_t len; bool unmapped; std::string own; };
  std::thread th;
  std::mutex mu;
  std::condition_variable cv_job, cv_free;
  std::deque<Job> q;
  bool stop = false, failed = false;
  char* pin[2] = {nullptr, nullptr};
  size_t pin_cap = 0;
  bool pin_busy[2] = {false, false};
  int next_slot = 0;
  sb_sam_stats st{};
};

namespace {

double now_ms() {
  timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return 1e3 * (double)ts.tv_sec + 1e-6 * (double)ts.tv_nsec;
}

void writer_main(sb_sam* s) {
  for (;;) {
    sb_sam::Job j;
    {
      std::unique_lock<std::mutex> lk(s->mu);
      s->cv_job.wait(lk, [&] { return !s->q.empty() || s->stop; });
      if (s->q.empty()) return;
      j = std::move(s->q.front());
      s->q.pop_front();
    }
    FILE* f = j.unmapped ? s->un : s->sam;
    const char* data = j.slot >= 0 ? s->pin[j.slot] : j.own.data();
    const double t0 = now_ms();
    const bool ok = !f || j.len == 0 || fwrite(data, 1, j.len, f) == j.len;
    std::lock_guard<std::mutex> lk(s->mu);
    s->st.write_ms += now_ms() - t0;
    if (!ok) s->failed = true;
    if (j.slot >= 0) s->pin_busy[j.slot] = false;
    s->cv_free.notify_all();
  }
}

void enqueue(sb_sam* s, sb_sam::Job&& j) {
  std::lock_guard<std::mutex> lk(s->mu);
  s->q.push_back(std::move(j));
  s->cv_job.notify_one();
}

// a free page-locked slot of at least `bytes`
int take_slot(sb_sam* s, size_t bytes) {
  std::unique_lock<std::mutex> lk(s->mu);
  if (bytes > s->pin_cap) {   // (re)allocate both: wait until the writer holds neither
    s->cv_free.wait(lk, [&] { return !s->pin_busy[0] && !s->pin_busy[1]; });
    for (int i = 0; i < 2; ++i) { if (s->pin[i]) cudaFreeHost(s->pin[i]); s->pin[i] = nullptr; }
    s->pin_cap = 0;
    for (int i = 0; i < 2; ++i)
      if (cudaMallocHost(&s->pin[i], bytes) != cudaSuccess) { sb::set_error("cannot page-lock %zu bytes", bytes); return -1; }
    s->pin_cap = bytes;
  }
  const int k = s->next_slot;
  s->cv_free.wait(lk, [&] { return !s->pin_busy[k]; });
  s->pin_busy[k] = true;
  s->next_slot ^= 1;
  return k;
}

struct SamArgs {
  SamBatch b;
  sbmap::SamSide side;
  const uint8_t* codes[2];
  const uint8_t* qual[2];        // nullptr: QUAL is '*'
  const char* names;
  const uint64_t* name_off;      // the caller's offsets; names holds name_base onwards
  uint64_t name_base;
  const uint32_t* ref_len;
  const uint64_t* rname_off;
  const char* rnames;
  int write_sam, write_un;
};

__device__ __forceinline__ Aln load_aln(const SamArgs& A, uint32_t r, uint32_t a) {
  const size_t i = (size_t)r * A.b.cap + a;
  Aln x;
  x.tid = A.b.tid[i]; x.pos = A.b.pos[i]; x.mate_pos = A.b.mate_pos[i]; x.flags = A.b.flags[i]; x.flen = A.b.flen[i];
  x.score1 = A.side.score1[i]; x.score2 = A.side.score2[i];
  return x;
}

__global__ void k_sam_size(SamArgs A, uint64_t* __restrict__ sam_bytes, uint64_t* __restrict__ un_bytes,
                           unsigned long long* __restrict__ records) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= A.b.n) return;
  const uint32_t nout = A.side.n_out[r];
  const uint32_t name_len = (uint32_t)(A.name_off[r + 1] - A.name_off[r]);
  const uint32_t nm = A.b.paired ? 2 : 1;
  uint64_t bytes = 0;
  if (A.write_sam)
    for (uint32_t a = 0; a < nout; ++a) {
      const Aln x = load_aln(A, r, a);
      const uint32_t rl = (uint32_t)(A.rname_off[x.tid + 1] - A.rname_off[x.tid]);
      for (uint32_t m = 0; m < nm; ++m)
        bytes += rec_len(sam_record(x, m, a, nout, A.b.paired, A.b.L, A.ref_len[x.tid]), name_len, rl, A.b.L, A.qual[m] != nullptr);
    }
  sam_bytes[r] = bytes;
  if (A.write_sam && nout) atomicAdd(records, (unsigned long long)nout * nm);
  uint64_t ub = 0;
  if (A.write_un) {
    const char* t = unmapped_type(nout, A.side.decoy[r] != 0, A.b.flags[(size_t)r * A.b.cap], A.b.paired);
    if (t) ub = name_len + 1 + str_len(t) + 1;
  }
  un_bytes[r] = ub;
}

// one warp per fragment of [f0, f1); text at sam_off[r] - sam_off[f0] of `out`, unmapped lines at un_off[r] of `un`
__global__ void __launch_bounds__(256) k_sam_write(SamArgs A, uint32_t f0, uint32_t f1, const uint64_t* __restrict__ sam_off,
                                                   const uint64_t* __restrict__ un_off, char* __restrict__ out,
                                                   char* __restrict__ un) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const uint64_t base = sam_off[f0];
  const uint32_t L = A.b.L;
  for (uint32_t r = f0 + w; r < f1; r += nw) {
    const uint32_t nout = A.side.n_out[r];
    const char* name = A.names + (A.name_off[r] - A.name_base);
    const uint32_t name_len = (uint32_t)(A.name_off[r + 1] - A.name_off[r]);
    if (A.write_sam) {
      char* o = out + (sam_off[r] - base);
      const uint32_t nm = A.b.paired ? 2 : 1;
      for (uint32_t a = 0; a < nout; ++a) {
        const Aln x = load_aln(A, r, a);
        const char* rname = A.rnames + A.rname_off[x.tid];
        const uint32_t rl = (uint32_t)(A.rname_off[x.tid + 1] - A.rname_off[x.tid]);
        for (uint32_t m = 0; m < nm; ++m) {
          const Rec rec = sam_record(x, m, a, nout, A.b.paired, L, A.ref_len[x.tid]);
          const uint8_t* codes = A.codes[m] + (size_t)r * L;
          const uint8_t* q = A.qual[m] ? A.qual[m] + (size_t)r * L : nullptr;
          const uint32_t hl = head_len(rec, name_len, rl), bl = body_len(L, q != nullptr);
          if (lane == 0) head_write(o, rec, name, name_len, rname, rl);
          for (uint32_t i = lane; i < bl; i += 32) o[hl + i] = body_char(i, L, rec.rev, codes, q, A.b.ascii != 0);
          if (lane == 0) tail_write(o + hl + bl, rec);
          o += hl + bl + tail_len(rec);
        }
      }
    }
    if (A.write_un && lane == 0 && un_off[r + 1] > un_off[r]) {
      const char* t = unmapped_type(nout, A.side.decoy[r] != 0, A.b.flags[(size_t)r * A.b.cap], A.b.paired);
      char* o = un + un_off[r];
      uint32_t k = put_s(o, name, name_len);
      o[k++] = ' ';
      k += put_s(o + k, t, str_len(t));
      o[k] = '\n';
    }
  }
}

}  // namespace

struct SamDev {
  sb::Resources res;              // every buffer and event below, made and released on the mapping context's device
  sb_sam* s = nullptr;
  uint32_t B = 0, Lcap = 0, cap = 0;
  sbmap::SamSide side{};
  uint8_t* codes[2] = {nullptr, nullptr};
  uint8_t* qual[2] = {nullptr, nullptr};
  char* names = nullptr;
  uint64_t* name_off = nullptr;
  uint64_t *sam_bytes = nullptr, *sam_off = nullptr, *un_bytes = nullptr, *un_off = nullptr;
  uint64_t* h_off = nullptr;     // page-locked copy of sam_off
  unsigned long long* records = nullptr;   // [0]: records of the batch (device), [1]: its page-locked copy
  char* win = nullptr;
  char* un = nullptr;
  uint32_t* ref_len = nullptr; uint64_t* rname_off = nullptr; char* rnames = nullptr;
  void* tmp = nullptr; size_t tmp_bytes = 0;
  cudaEvent_t ev[2] = {nullptr, nullptr};
};

int sam_dev_create(SamDev** out, sb_sam* s, uint32_t B, uint32_t Lcap, uint32_t cap) {
  SamDev* d = new SamDev();
  *out = d;
  d->s = s; d->B = B; d->Lcap = Lcap; d->cap = cap;
  const size_t BC = (size_t)B * cap;
  sb::Resources& r = d->res;
  SB_TRY(r.alloc(&d->side.n_out, B));
  SB_TRY(r.alloc(&d->side.decoy, B));
  SB_TRY(r.alloc(&d->side.score1, BC));
  SB_TRY(r.alloc(&d->side.score2, BC));
  for (int m = 0; m < 2; ++m) SB_TRY(r.alloc(&d->codes[m], (size_t)B * Lcap));
  if (s->flags & SB_SAM_QUALITIES)
    for (int m = 0; m < 2; ++m) SB_TRY(r.alloc(&d->qual[m], (size_t)B * Lcap));
  SB_TRY(r.alloc(&d->name_off, (size_t)B + 1));
  SB_TRY(r.alloc(&d->sam_bytes, (size_t)B + 1)); SB_TRY(r.alloc(&d->sam_off, (size_t)B + 1));
  SB_TRY(r.alloc(&d->un_bytes, (size_t)B + 1)); SB_TRY(r.alloc(&d->un_off, (size_t)B + 1));
  SB_TRY(r.alloc_host(&d->h_off, (size_t)B + 2));
  SB_TRY(r.alloc(&d->records, 1));
  const uint32_t M = s->n_txps;
  SB_TRY(r.alloc(&d->ref_len, M));
  SB_TRY(r.alloc(&d->rname_off, (size_t)M + 1));
  SB_TRY(r.alloc(&d->rnames, s->rnames.size()));
  SB_CUDA(cudaMemcpy(d->ref_len, s->ref_len.data(), (size_t)M * 4, cudaMemcpyHostToDevice));
  SB_CUDA(cudaMemcpy(d->rname_off, s->rname_off.data(), ((size_t)M + 1) * 8, cudaMemcpyHostToDevice));
  SB_CUDA(cudaMemcpy(d->rnames, s->rnames.data(), s->rnames.size(), cudaMemcpyHostToDevice));
  SB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, d->tmp_bytes, d->sam_bytes, d->sam_off, (int)B + 1));
  SB_TRY(r.alloc((unsigned char**)&d->tmp, d->tmp_bytes));
  for (int i = 0; i < 2; ++i) SB_TRY(r.event(&d->ev[i], cudaEventDefault));
  return SB_OK;
}

void sam_dev_destroy(SamDev* d) { delete d; }

sbmap::SamSide sam_dev_side(SamDev* d) { return d->side; }

int sam_dev_format(SamDev* d, cudaStream_t st, const SamBatch& b, const uint8_t* left, const uint8_t* right,
                   const char* names, const uint64_t* name_off, const uint8_t* ql, const uint8_t* qr,
                   uint64_t window_bytes, float* format_ms) {
  sb_sam* s = d->s;
  const uint32_t n = b.n, L = b.L;
  *format_ms = 0;
  if (n == 0) return SB_OK;
  const bool want_q = (s->flags & SB_SAM_QUALITIES) != 0;
  if (want_q && (!ql || (b.paired && !qr))) { sb::set_error("the SAM sink writes qualities: the batch needs them"); return SB_ERR_INVALID; }
  // inputs of the pass: reads, names, qualities (the reads may already be on the device)
  SB_CUDA(cudaMemcpyAsync(d->codes[0], left, (size_t)n * L, cudaMemcpyDefault, st));
  if (b.paired) SB_CUDA(cudaMemcpyAsync(d->codes[1], right, (size_t)n * L, cudaMemcpyDefault, st));
  if (want_q) {
    SB_CUDA(cudaMemcpyAsync(d->qual[0], ql, (size_t)n * L, cudaMemcpyHostToDevice, st));
    if (b.paired) SB_CUDA(cudaMemcpyAsync(d->qual[1], qr, (size_t)n * L, cudaMemcpyHostToDevice, st));
  }
  const uint64_t name_bytes = name_off[n] - name_off[0];
  SB_TRY(d->res.grow(&d->names, name_bytes));
  SB_CUDA(cudaMemcpyAsync(d->names, names + name_off[0], name_bytes, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(d->name_off, name_off, ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, st));
  SamArgs A;
  A.b = b; A.side = d->side;
  A.codes[0] = d->codes[0]; A.codes[1] = b.paired ? d->codes[1] : d->codes[0];
  A.qual[0] = want_q ? d->qual[0] : nullptr; A.qual[1] = (want_q && b.paired) ? d->qual[1] : nullptr;
  A.names = d->names; A.name_off = d->name_off; A.name_base = name_off[0];
  A.ref_len = d->ref_len; A.rname_off = d->rname_off; A.rnames = d->rnames;
  A.write_sam = s->sam != nullptr; A.write_un = s->un != nullptr;
  float ms = 0;
  SB_CUDA(cudaEventRecord(d->ev[0], st));
  SB_CUDA(cudaMemsetAsync(d->sam_bytes + n, 0, 8, st));
  SB_CUDA(cudaMemsetAsync(d->un_bytes + n, 0, 8, st));
  SB_CUDA(cudaMemsetAsync(d->records, 0, 8, st));
  k_sam_size<<<(n + 255) / 256, 256, 0, st>>>(A, d->sam_bytes, d->un_bytes, d->records);
  size_t tb = d->tmp_bytes;
  SB_CUDA(cub::DeviceScan::ExclusiveSum(d->tmp, tb, d->sam_bytes, d->sam_off, (int)n + 1, st));
  tb = d->tmp_bytes;
  SB_CUDA(cub::DeviceScan::ExclusiveSum(d->tmp, tb, d->un_bytes, d->un_off, (int)n + 1, st));
  SB_CUDA(cudaEventRecord(d->ev[1], st));
  SB_CUDA(cudaMemcpyAsync(d->h_off, d->sam_off, ((size_t)n + 1) * 8, cudaMemcpyDeviceToHost, st));
  uint64_t un_total = 0;
  SB_CUDA(cudaMemcpyAsync(&un_total, d->un_off + n, 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(d->h_off + n + 1, d->records, 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  const uint64_t n_records = d->h_off[n + 1];
  SB_CUDA(cudaEventElapsedTime(&ms, d->ev[0], d->ev[1]));
  *format_ms += ms;
  SB_TRY(d->res.grow(&d->un, un_total));
  // windows of whole fragments that fit the device buffer (a fragment larger than the buffer gets a window of its own,
  // and the buffer grows to hold it)
  const uint64_t W = std::max<uint64_t>(window_bytes, 1);
  for (uint32_t f0 = 0; f0 < n;) {
    uint32_t f1 = f0 + 1;
    {   // largest f1 with h_off[f1] - h_off[f0] <= W (binary search; at least one fragment)
      uint32_t lo = f0 + 1, hi = n;
      while (lo < hi) {
        const uint32_t mid = lo + (hi - lo + 1) / 2;
        if (d->h_off[mid] - d->h_off[f0] <= W) lo = mid; else hi = mid - 1;
      }
      f1 = lo;
    }
    const uint64_t bytes = d->h_off[f1] - d->h_off[f0], want = std::max<uint64_t>(bytes, std::min<uint64_t>(W, d->h_off[n]));
    SB_TRY(d->res.grow(&d->win, want));
    SB_CUDA(cudaEventRecord(d->ev[0], st));
    const uint32_t warps = f1 - f0, blocks = std::min<uint32_t>((warps + 7) / 8, 65535u);
    k_sam_write<<<blocks, 256, 0, st>>>(A, f0, f1, d->sam_off, d->un_off, d->win, d->un);
    SB_CUDA(cudaEventRecord(d->ev[1], st));
    if (bytes) {
      const double t0 = now_ms();
      const int slot = take_slot(s, want);
      if (slot < 0) return SB_ERR_NOMEM;
      const double t1 = now_ms();
      SB_CUDA(cudaMemcpyAsync(s->pin[slot], d->win, bytes, cudaMemcpyDeviceToHost, st));
      SB_CUDA(cudaStreamSynchronize(st));
      s->st.slot_wait_ms += t1 - t0;
      s->st.copy_ms += now_ms() - t1;
      enqueue(s, sb_sam::Job{slot, (size_t)bytes, false, std::string()});
    } else {
      SB_CUDA(cudaStreamSynchronize(st));
    }
    SB_CUDA(cudaEventElapsedTime(&ms, d->ev[0], d->ev[1]));
    *format_ms += ms;
    s->st.windows++;
    s->st.sam_bytes += bytes;
    f0 = f1;
  }
  if (un_total) {
    std::string t(un_total, '\0');
    SB_CUDA(cudaMemcpy(&t[0], d->un, un_total, cudaMemcpyDeviceToHost));
    uint64_t lines = 0;
    for (char c : t) lines += c == '\n';
    s->st.unmapped_lines += lines;
    enqueue(s, sb_sam::Job{-1, (size_t)un_total, true, std::move(t)});
  }
  s->st.records += n_records;
  s->st.batches++;
  s->st.format_ms += *format_ms;
  return SB_OK;
}

// ---- the sink ---------------------------------------------------------------------------------------------------
extern "C" sb_sam* sb_sam_open(const char* sam_path, const char* unmapped_path, const sb_index* ix, const char* cmdline,
                               uint32_t flags) {
  if (!ix || (!sam_path && !unmapped_path)) { sb::set_error("sb_sam_open: needs an index and at least one output path"); return nullptr; }
  uint32_t M = 0, k = 0, first_decoy = 0;
  const char* const* names = nullptr;
  const uint32_t* complete = nullptr;
  if (sb_index_get_meta(ix, &M, &k, &first_decoy, &names, &complete) != SB_OK) return nullptr;
  const uint64_t* tx_off = nullptr;
  if (sb_index_host_arrays(ix, &tx_off, nullptr, nullptr, nullptr, nullptr, nullptr) != SB_OK) return nullptr;
  sb_sam* s = new sb_sam();
  s->flags = flags;
  s->n_txps = M;
  s->ref_len.resize(M);
  s->rname_off.assign((size_t)M + 1, 0);
  for (uint32_t t = 0; t < M; ++t) {
    s->ref_len[t] = (uint32_t)(tx_off[t + 1] - tx_off[t]);   // the indexed length (after poly-A clipping)
    s->rnames += names ? std::string(names[t]) : "t" + std::to_string(t);
    s->rname_off[t + 1] = s->rnames.size();
  }
  if (sam_path) {
    s->sam_is_stdout = !strcmp(sam_path, "-");
    s->sam = s->sam_is_stdout ? stdout : fopen(sam_path, "w");
    if (!s->sam) { sb::set_error("cannot open %s for writing", sam_path); delete s; return nullptr; }
    std::string h = "@HD\tVN:1.0\tSO:unknown\n";
    for (uint32_t t = 0; t < M; ++t)
      h += "@SQ\tSN:" + s->rnames.substr(s->rname_off[t], s->rname_off[t + 1] - s->rname_off[t]) + "\tLN:" +
           std::to_string(s->ref_len[t]) + "\n";
    h += "@PG\tID:salmon\tPN:salmon\tVN:1.11.4-sb" + std::to_string(sb_version());
    if (cmdline && *cmdline) h += std::string("\tCL:") + cmdline;
    h += "\n";
    if (fwrite(h.data(), 1, h.size(), s->sam) != h.size()) {
      sb::set_error("write error on %s", sam_path);
      if (!s->sam_is_stdout) fclose(s->sam);
      delete s;
      return nullptr;
    }
    s->st.sam_bytes = h.size();
  }
  if (unmapped_path) {
    s->un = fopen(unmapped_path, "w");
    if (!s->un) {
      sb::set_error("cannot open %s for writing", unmapped_path);
      if (s->sam && !s->sam_is_stdout) fclose(s->sam);
      delete s;
      return nullptr;
    }
  }
  s->th = std::thread(writer_main, s);
  return s;
}

extern "C" int sb_sam_write_unmapped(sb_sam* s, const char* text, size_t len) {
  if (!s || (len && !text)) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  if (!s->un || len == 0) return SB_OK;
  uint64_t lines = 0;
  for (size_t i = 0; i < len; ++i) lines += text[i] == '\n';
  s->st.unmapped_lines += lines;
  enqueue(s, sb_sam::Job{-1, len, true, std::string(text, len)});
  return SB_OK;
}

extern "C" int sb_sam_get_stats(const sb_sam* s, sb_sam_stats* out) {
  if (!s || !out) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  *out = s->st;
  return SB_OK;
}

extern "C" int sb_sam_close(sb_sam* s) {
  if (!s) return SB_OK;
  {
    std::lock_guard<std::mutex> lk(s->mu);
    s->stop = true;
    s->cv_job.notify_all();
  }
  if (s->th.joinable()) s->th.join();
  bool ok = !s->failed;
  if (s->sam) ok = (s->sam_is_stdout ? fflush(s->sam) == 0 : fclose(s->sam) == 0) && ok;
  if (s->un) ok = fclose(s->un) == 0 && ok;
  for (int i = 0; i < 2; ++i) if (s->pin[i]) cudaFreeHost(s->pin[i]);
  delete s;
  if (!ok) { sb::set_error("write error on the SAM / unmapped-names output"); return SB_ERR_INVALID; }
  return SB_OK;
}
