// map.cu -- Stage A on the GPU: index (host build, HBM resident), per-read mapping kernels, banded
// affine DP scoring (one warp per mate alignment, lanes = band cells), alignment filtering +
// auxiliary probabilities + labels, and the equivalence-class builder (hash -> radix sort ->
// segmented reduce).  C ABI at the reference's seams B1 (processReads, src/quant/
// SalmonQuantify.cpp:1026-1874) and B2 (EquivalenceClassBuilder, include/salmon/internal/quant/
// EquivalenceClassBuilder.hpp:165-181,237-250).  See map_core.h for MAPSPEC.
#include <cub/cub.cuh>
#include <math.h>
#include <string.h>
#include <time.h>

#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <memory>
#include <parallel/algorithm>
#include <vector>
#include <new>
#include <string>

#include "common.cuh"
#include "map_core.h"
#include "map_kernels.cuh"
#include "rescue.cuh"
#include "resources.h"
#include "sam_internal.h"

using namespace sbmap;

// std::vector without the zero fill of resize(): the big index arrays are overwritten right away (by parallel preads on
// load), and first-touch by one thread costs seconds at human scale
template <class T>
struct NoInit {
  using value_type = T;
  NoInit() = default;
  template <class U> NoInit(const NoInit<U>&) {}
  T* allocate(size_t n) { T* p = (T*)malloc(n * sizeof(T)); if (!p) throw std::bad_alloc(); return p; }
  void deallocate(T* p, size_t) { free(p); }
  template <class U> void construct(U* p) { ::new ((void*)p) U; }                                   // default-init: no store
  template <class U, class A0, class... A> void construct(U* p, A0&& a0, A&&... a) { ::new ((void*)p) U(std::forward<A0>(a0), std::forward<A>(a)...); }
  template <class U> bool operator==(const NoInit<U>&) const { return true; }
  template <class U> bool operator!=(const NoInit<U>&) const { return false; }
};
template <class T> using BigVec = std::vector<T, NoInit<T>>;

// ---------------------------------------------------------------------------------------------
// index (host build)
// ---------------------------------------------------------------------------------------------
struct sb_index {
  uint32_t n_txps = 0, k = 0;
  std::vector<uint64_t> tx_off;
  BigVec<uint8_t> codes;
  BigVec<TableEntry> table;
  BigVec<Posting> post;
  BigVec<uint64_t> packed;     // 2-bit packed codes with PACK_GUARD_BASES of guard on both sides
  std::vector<uint8_t> tx_has_n;
  uint64_t n_kmers = 0;
  // what `salmon quant` needs besides the sequence: names, lengths before clipping, first decoy (optional)
  std::vector<std::string> names;
  std::vector<const char*> name_ptrs;
  std::vector<uint32_t> complete_len;
  uint32_t first_decoy = 0xffffffffu;   // clamped to n_txps by set_meta / build
  // device copies (one device)
  int device = -1;
  std::unique_ptr<sb::Resources> dev;   // owns them
  uint64_t* d_tx_off = nullptr;
  uint8_t* d_codes = nullptr;
  TableEntry* d_table = nullptr;
  Posting* d_post = nullptr;
  uint64_t* d_packed = nullptr;
  uint8_t* d_tx_has_n = nullptr;
};

namespace {
struct KP {
  uint64_t km;
  uint32_t tid, tpos_rc;
};
IndexView dev_view(const sb_index* ix) {
  IndexView v;
  v.n_txps = ix->n_txps; v.k = ix->k; v.mask = ix->table.size() - 1;
  v.tx_off = ix->d_tx_off; v.codes = ix->d_codes; v.table = ix->d_table; v.post = ix->d_post;
  v.packed = ix->d_packed; v.tx_has_n = ix->d_tx_has_n;
  return v;
}
}  // namespace

extern "C" sb_index* sb_index_build(uint32_t n_txps, const uint64_t* seq_off, const uint8_t* codes, uint32_t k) {
  if (!seq_off || (!codes && seq_off[n_txps]) || k < 3 || k > 31 || (k & 1) == 0) {
    sb::set_error("sb_index_build: bad arguments (k must be odd, 3..31)");
    return nullptr;
  }
  for (uint32_t t = 0; t < n_txps; ++t)
    if (seq_off[t + 1] - seq_off[t] >= (1u << 21)) {
      sb::set_error("sb_index_build: reference %u longer than 2^21 bases (seed key layout)", t);
      return nullptr;
    }
  sb_index* ix = new sb_index();
  ix->n_txps = n_txps; ix->k = k; ix->first_decoy = n_txps;
  ix->tx_off.assign(seq_off, seq_off + n_txps + 1);
  ix->codes.assign(codes, codes + seq_off[n_txps]);
  std::vector<KP> kp;
  uint64_t cap = 0;
  for (uint32_t t = 0; t < n_txps; ++t) { uint64_t L = seq_off[t + 1] - seq_off[t]; if (L >= k) cap += L - k + 1; }
  kp.reserve(cap);
  const uint64_t kmask = (k == 32) ? ~0ull : ((1ull << (2 * k)) - 1);
  for (uint32_t t = 0; t < n_txps; ++t) {
    const uint64_t b = seq_off[t], e = seq_off[t + 1];
    uint64_t fw = 0, rc = 0;
    uint32_t valid = 0;   // consecutive valid bases ending at p
    for (uint64_t p = b; p < e; ++p) {
      const uint8_t c = codes[p];
      if (c > 3) { valid = 0; fw = rc = 0; continue; }
      fw = ((fw << 2) | c) & kmask;
      rc = (rc >> 2) | ((uint64_t)(3 - c) << (2 * (k - 1)));
      if (++valid >= k) kp.push_back({fw < rc ? fw : rc, t, (uint32_t)(p + 1 - k - b) | (fw < rc ? 0u : 0x80000000u)});
    }
  }
  // (k-mer, transcript, offset) order; the orientation flag (bit 31) is a function of the other three
  __gnu_parallel::sort(kp.begin(), kp.end(), [](const KP& a, const KP& b) {
    if (a.km != b.km) return a.km < b.km;
    if (a.tid != b.tid) return a.tid < b.tid;
    return (a.tpos_rc & 0x7fffffffu) < (b.tpos_rc & 0x7fffffffu);
  });
  // 2-bit packed reference (DP windows, exact-match tests); transcripts with N keep using the byte codes
  {
    const uint64_t total = seq_off[n_txps];
    ix->packed.assign((total + 2 * (uint64_t)PACK_GUARD_BASES + 31) / 32 + 2, 0);
    ix->tx_has_n.assign(std::max<uint32_t>(n_txps, 1), 0);
    for (uint32_t t = 0; t < n_txps; ++t)
      for (uint64_t g = seq_off[t]; g < seq_off[t + 1]; ++g) {
        const uint8_t c = codes[g];
        if (c > 3) { ix->tx_has_n[t] = 1; continue; }
        const uint64_t q = g + PACK_GUARD_BASES;
        ix->packed[q >> 5] |= (uint64_t)c << (2 * (q & 31));
      }
  }
  uint64_t nk = 0;
  for (size_t i = 0; i < kp.size(); ++i) if (i == 0 || kp[i].km != kp[i - 1].km) ++nk;
  ix->n_kmers = nk;
  uint64_t capt = 1024;
  while (capt < 2 * nk) capt <<= 1;
  ix->table.assign(capt, TableEntry{EMPTY_KEY, 0, 0});
  ix->post.resize(kp.size());
  const uint64_t mask = capt - 1;
  for (size_t i = 0; i < kp.size();) {
    size_t j = i;
    while (j < kp.size() && kp[j].km == kp[i].km) { ix->post[j] = Posting{kp[j].tid, kp[j].tpos_rc}; ++j; }
    uint64_t h = mix64(kp[i].km) & mask;
    while (ix->table[h].key != EMPTY_KEY) h = (h + 1) & mask;
    ix->table[h] = TableEntry{kp[i].km, (uint32_t)i, (uint32_t)(j - i)};
    i = j;
  }
  return ix;
}

extern "C" void sb_index_free(sb_index* ix) {
  delete ix;
}

extern "C" int sb_index_info(const sb_index* ix, uint64_t* out4) {
  if (!ix || !out4) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  out4[0] = ix->n_kmers; out4[1] = ix->post.size(); out4[2] = ix->table.size();
  out4[3] = ix->table.size() * sizeof(TableEntry) + ix->post.size() * sizeof(Posting) + ix->codes.size() +
            ix->tx_off.size() * 8 + ix->packed.size() * 8 + ix->tx_has_n.size();
  return SB_OK;
}

// raw views of the host-side arrays (serialisation; also lets tests run map_core.h on the CPU)
extern "C" int sb_index_host_arrays(const sb_index* ix, const uint64_t** tx_off, const uint8_t** codes,
                                    const void** table, uint64_t* table_capacity, const void** postings,
                                    uint64_t* n_postings) {
  if (!ix) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  if (tx_off) *tx_off = ix->tx_off.data();
  if (codes) *codes = ix->codes.data();
  if (table) *table = ix->table.data();
  if (table_capacity) *table_capacity = ix->table.size();
  if (postings) *postings = ix->post.data();
  if (n_postings) *n_postings = ix->post.size();
  return SB_OK;
}

// ---- on-disk form of the index (own format; `salmon index` writes a directory, so do we: <dir>/sb_index.bin).
// Header + the host arrays verbatim + the reference names / complete lengths / decoy boundary that `salmon quant`
// needs for quant.sf.  Not the pufferfish / SSHash format (SURVEY.md 8f-2; that source is not in the reference tree).
namespace {
constexpr uint64_t INDEX_MAGIC = 0x3130584449324253ull;   // "SB2IDX01"
struct IndexHeader {
  uint64_t magic;
  uint32_t version, k, n_txps, first_decoy;
  uint64_t n_codes, n_table, n_post, n_packed, n_kmers, names_bytes;
};
template <typename T>
bool wr(FILE* f, const T* p, size_t n) { return n == 0 || fwrite(p, sizeof(T), n, f) == n; }
template <typename T>
bool rd(FILE* f, T* p, size_t n) { return n == 0 || fread(p, sizeof(T), n, f) == n; }
}  // namespace

extern "C" int sb_index_set_meta(sb_index* ix, const char* const* names, const uint32_t* complete_len, uint32_t first_decoy) {
  if (!ix) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  ix->names.clear(); ix->complete_len.clear();
  if (names) for (uint32_t t = 0; t < ix->n_txps; ++t) ix->names.emplace_back(names[t] ? names[t] : "");
  if (complete_len) ix->complete_len.assign(complete_len, complete_len + ix->n_txps);
  ix->first_decoy = first_decoy > ix->n_txps ? ix->n_txps : first_decoy;
  ix->name_ptrs.clear();
  for (auto& n : ix->names) ix->name_ptrs.push_back(n.c_str());
  return SB_OK;
}

extern "C" int sb_index_get_meta(const sb_index* ix, uint32_t* n_txps, uint32_t* k, uint32_t* first_decoy,
                                 const char* const** names, const uint32_t** complete_len) {
  if (!ix) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  if (n_txps) *n_txps = ix->n_txps;
  if (k) *k = ix->k;
  if (first_decoy) *first_decoy = ix->first_decoy;
  if (names) *names = ix->name_ptrs.empty() ? nullptr : ix->name_ptrs.data();
  if (complete_len) *complete_len = ix->complete_len.empty() ? nullptr : ix->complete_len.data();
  return SB_OK;
}

extern "C" int sb_index_save(const sb_index* ix, const char* path) {
  if (!ix || !path) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  FILE* f = fopen(path, "wb");
  if (!f) { sb::set_error("cannot open %s for writing", path); return SB_ERR_INVALID; }
  std::string names;
  for (auto& n : ix->names) { names += n; names += '\n'; }
  IndexHeader h{};
  h.magic = INDEX_MAGIC; h.version = 1; h.k = ix->k; h.n_txps = ix->n_txps; h.first_decoy = ix->first_decoy;
  h.n_codes = ix->codes.size(); h.n_table = ix->table.size(); h.n_post = ix->post.size(); h.n_packed = ix->packed.size();
  h.n_kmers = ix->n_kmers; h.names_bytes = names.size();
  const uint32_t has_len = ix->complete_len.empty() ? 0u : 1u;
  bool ok = wr(f, &h, 1) && wr(f, &has_len, 1) && wr(f, ix->tx_off.data(), ix->tx_off.size()) &&
            wr(f, ix->codes.data(), ix->codes.size()) && wr(f, ix->table.data(), ix->table.size()) &&
            wr(f, ix->post.data(), ix->post.size()) && wr(f, ix->packed.data(), ix->packed.size()) &&
            wr(f, ix->tx_has_n.data(), ix->tx_has_n.size()) && wr(f, names.data(), names.size()) &&
            (!has_len || wr(f, ix->complete_len.data(), ix->complete_len.size()));
  ok = (fclose(f) == 0) && ok;
  if (!ok) { sb::set_error("write error on %s", path); return SB_ERR_INVALID; }
  return SB_OK;
}

extern "C" sb_index* sb_index_load(const char* path) {
  if (!path) { sb::set_error("null argument"); return nullptr; }
  FILE* f = fopen(path, "rb");
  if (!f) { sb::set_error("cannot open %s", path); return nullptr; }
  IndexHeader h{};
  uint32_t has_len = 0;
  if (!rd(f, &h, 1) || h.magic != INDEX_MAGIC || h.version != 1 || !rd(f, &has_len, 1)) {
    fclose(f); sb::set_error("%s is not an sb index (bad header)", path); return nullptr;
  }
  if (h.n_table == 0 || (h.n_table & (h.n_table - 1)) || h.k < 3 || h.k > 31 || h.first_decoy > h.n_txps) {
    fclose(f); sb::set_error("%s: corrupt header", path); return nullptr;
  }
  {   // the arrays the header announces must fit in the file (a corrupt count must not drive the allocations)
    struct stat stt;
    const uint64_t need = (uint64_t)(h.n_txps + 1ull) * 8 + h.n_codes + (uint64_t)h.n_table * sizeof(TableEntry) +
                          (uint64_t)h.n_post * sizeof(Posting) + h.names_bytes;
    if (fstat(fileno(f), &stt) != 0 || need > (uint64_t)stt.st_size) {
      fclose(f); sb::set_error("%s: truncated or corrupt index (the header announces more data than the file holds)", path); return nullptr;
    }
  }
  sb_index* ix = new sb_index();
  ix->n_txps = h.n_txps; ix->k = h.k; ix->n_kmers = h.n_kmers; ix->first_decoy = h.first_decoy;
  bool ok = true;
  try {
    ix->tx_off.resize((size_t)h.n_txps + 1); ix->codes.resize(h.n_codes); ix->table.resize(h.n_table);
    ix->post.resize(h.n_post); ix->packed.resize(h.n_packed); ix->tx_has_n.resize(std::max<uint32_t>(h.n_txps, 1));
    std::string names(h.names_bytes, '\0');
    // the big arrays: read by a team of threads (pread on disjoint slices; each thread first-touches what it reads)
    ok = rd(f, ix->tx_off.data(), ix->tx_off.size());
    if (ok) {
      const int fd = fileno(f);
      off_t pos = ftello(f);
      struct Part { void* dst; size_t bytes; off_t off; };
      Part parts[4] = {{ix->codes.data(), ix->codes.size(), 0}, {ix->table.data(), ix->table.size() * sizeof(TableEntry), 0},
                       {ix->post.data(), ix->post.size() * sizeof(Posting), 0}, {ix->packed.data(), ix->packed.size() * 8, 0}};
      struct Slice { char* dst; size_t bytes; off_t off; };
      std::vector<Slice> slices;
      constexpr size_t SL = (size_t)16 << 20;
      for (Part& pt : parts) {
        pt.off = pos;
        for (size_t o = 0; o < pt.bytes; o += SL) slices.push_back(Slice{(char*)pt.dst + o, std::min(SL, pt.bytes - o), pos + (off_t)o});
        pos += (off_t)pt.bytes;
      }
      int bad = 0;
      const int nt = (int)std::max<size_t>(1, std::min<size_t>(16, slices.size()));
#pragma omp parallel for schedule(dynamic, 1) num_threads(nt) reduction(| : bad)
      for (long i = 0; i < (long)slices.size(); ++i) {
        size_t done = 0;
        while (done < slices[i].bytes) {
          const ssize_t got = pread(fd, slices[i].dst + done, slices[i].bytes - done, slices[i].off + (off_t)done);
          if (got <= 0) { bad = 1; break; }
          done += (size_t)got;
        }
      }
      ok = !bad && fseeko(f, pos, SEEK_SET) == 0;
    }
    ok = ok && rd(f, ix->tx_has_n.data(), ix->tx_has_n.size()) && rd(f, &names[0], names.size());
    if (ok && has_len) { ix->complete_len.resize(h.n_txps); ok = rd(f, ix->complete_len.data(), ix->complete_len.size()); }
    if (ok) {
      size_t b = 0;
      while (b < names.size()) {
        size_t e = names.find('\n', b);
        if (e == std::string::npos) e = names.size();
        ix->names.emplace_back(names, b, e - b);
        b = e + 1;
      }
      if (!ix->names.empty() && ix->names.size() != h.n_txps) ok = false;
      for (auto& n : ix->names) ix->name_ptrs.push_back(n.c_str());
      ok = ok && ix->tx_off[h.n_txps] == h.n_codes && ix->tx_off[0] == 0;
      for (uint32_t t = 0; t < h.n_txps && ok; ++t) ok = ix->tx_off[t] <= ix->tx_off[t + 1];   // monotonic offsets
      // every table entry points inside the posting array, every posting inside its transcript (these go to the GPU)
      if (ok) {
        int bad = 0;
        const TableEntry* tb = ix->table.data();
        const Posting* po = ix->post.data();
        const uint64_t* txo = ix->tx_off.data();
        const size_t nt_ = ix->table.size(), np_ = ix->post.size();
#pragma omp parallel for schedule(static) num_threads(16) reduction(| : bad)
        for (long i = 0; i < (long)nt_; ++i)
          if (tb[i].key != EMPTY_KEY && (uint64_t)tb[i].off + tb[i].cnt > np_) bad = 1;
#pragma omp parallel for schedule(static) num_threads(16) reduction(| : bad)
        for (long i = 0; i < (long)np_; ++i) {
          const Posting& q = po[i];
          if (q.tid >= h.n_txps || (uint64_t)(q.tpos_rc & 0x7fffffffu) + h.k > txo[q.tid + 1] - txo[q.tid]) bad = 1;
        }
        ok = !bad;
      }
    }
  } catch (const std::exception&) { ok = false; }   // bad_alloc, length_error from a corrupt count
  fclose(f);
  if (!ok) { delete ix; sb::set_error("%s: truncated or corrupt index", path); return nullptr; }
  return ix;
}

// host (pageable) -> device for the index arrays: slices are copied into two page-locked staging buffers by a team of
// threads while the previous slice is on the wire
static int upload_big(void* dst, const void* src, size_t bytes) {
  constexpr size_t SL = (size_t)64 << 20;
  if (bytes < 2 * SL) { SB_CUDA(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice)); return SB_OK; }
  sb::Resources res;   // on the current device
  char* stage[2] = {nullptr, nullptr};
  cudaEvent_t ev[2] = {nullptr, nullptr};
  cudaStream_t st = nullptr;
  int rc = SB_OK;
  if (res.alloc_host(&stage[0], SL) != SB_OK || res.alloc_host(&stage[1], SL) != SB_OK ||
      res.stream(&st, cudaStreamNonBlocking) != SB_OK ||
      res.event(&ev[0], cudaEventDisableTiming) != SB_OK || res.event(&ev[1], cudaEventDisableTiming) != SB_OK) {
    cudaGetLastError();
    rc = cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice) == cudaSuccess ? SB_OK : SB_ERR_CUDA;   // plain copy instead
  } else {
    int b = 0;
    for (size_t o = 0; o < bytes && rc == SB_OK; o += SL, b ^= 1) {
      const size_t n = std::min(SL, bytes - o);
      if (o >= 2 * SL && cudaEventSynchronize(ev[b]) != cudaSuccess) { rc = SB_ERR_CUDA; break; }
      const char* sp = (const char*)src + o;
      char* dp = stage[b];
#pragma omp parallel for schedule(static) num_threads(8)
      for (long q = 0; q < (long)((n + (1 << 20) - 1) >> 20); ++q) {
        const size_t a = (size_t)q << 20;
        memcpy(dp + a, sp + a, std::min<size_t>((size_t)1 << 20, n - a));
      }
      if (cudaMemcpyAsync((char*)dst + o, dp, n, cudaMemcpyHostToDevice, st) != cudaSuccess || cudaEventRecord(ev[b], st) != cudaSuccess) rc = SB_ERR_CUDA;
    }
    if (cudaStreamSynchronize(st) != cudaSuccess) rc = SB_ERR_CUDA;
  }
  if (rc != SB_OK) sb::set_error("index upload failed: %s", cudaGetErrorString(cudaGetLastError()));
  return rc;
}

// Creates the CUDA context of `device` (seconds on a large GPU): a front end calls this from a thread of its own while
// it loads the index from disk, so that the two overlap.
extern "C" int sb_device_init(int device) {
  SB_CUDA(cudaSetDevice(device));
  SB_CUDA(cudaFree(nullptr));
  return SB_OK;
}

static int index_to_device(sb_index* ix, int device) {
  if (ix->device == device) return SB_OK;
  if (ix->device >= 0) { sb::set_error("index already resident on device %d", ix->device); return SB_ERR_STATE; }
  SB_CUDA(cudaSetDevice(device));
  // on any failure `res` releases what was made so far and the index stays host-only, so that a retry starts clean
  auto res = std::make_unique<sb::Resources>(device);
  SB_TRY(res->alloc(&ix->d_tx_off, ix->tx_off.size()));
  SB_TRY(res->alloc(&ix->d_codes, std::max<size_t>(ix->codes.size(), 1) + 64));
  SB_TRY(res->alloc(&ix->d_table, ix->table.size()));
  SB_TRY(res->alloc(&ix->d_post, ix->post.size()));
  SB_CUDA(cudaMemcpy(ix->d_tx_off, ix->tx_off.data(), ix->tx_off.size() * 8, cudaMemcpyHostToDevice));
  SB_TRY(upload_big(ix->d_codes, ix->codes.data(), ix->codes.size()));
  SB_TRY(upload_big(ix->d_table, ix->table.data(), ix->table.size() * sizeof(TableEntry)));
  SB_TRY(upload_big(ix->d_post, ix->post.data(), ix->post.size() * sizeof(Posting)));
  SB_TRY(res->alloc(&ix->d_packed, ix->packed.size()));
  SB_TRY(res->alloc(&ix->d_tx_has_n, ix->tx_has_n.size()));
  SB_TRY(upload_big(ix->d_packed, ix->packed.data(), ix->packed.size() * 8));
  SB_CUDA(cudaMemcpy(ix->d_tx_has_n, ix->tx_has_n.data(), ix->tx_has_n.size(), cudaMemcpyHostToDevice));
  ix->dev = std::move(res);
  ix->device = device;
  return SB_OK;
}

// ---------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------
namespace {

struct BatchBufs {
  // per read
  uint32_t* n_l; uint32_t* n_r;      // candidates per mate
  Cand* cand_l; Cand* cand_r;        // [B*MAXCAND]
  int32_t* score_l; int32_t* score_r;// [B*MAXCAND]
  uint64_t* keys;                    // [MAXSEEDS * T] interleaved seed scratch, T = threads of K1
  // DP task list
  uint32_t* n_tasks; uint32_t* tasks;  // task = read<<7 | mate<<6 | cand
  // outputs (cap per read)
  uint32_t* n_aln; uint32_t* tid; int32_t* score; double* prob; int32_t* pos; int32_t* mate_pos;
  uint8_t* flags; int32_t* flen; uint32_t* label; double* weight;
  // scratch for assign
  int32_t* sc; int32_t* perm_idx; int32_t* perm_tid; int32_t* bs_tid; int32_t* bs_score; int32_t* bs_idx;
  Joint* jh;
  double* lp;                        // per-thread scratch: alignment log-probabilities
  Counters* ctr;
};

__device__ __forceinline__ void add_counters(Counters* g, const Counters& c) {
  if (c.lookups) atomicAdd(&g->lookups, c.lookups);
  if (c.postings) atomicAdd(&g->postings, c.postings);
  if (c.seeds) atomicAdd(&g->seeds, c.seeds);
  if (c.candidates) atomicAdd(&g->candidates, c.candidates);
  if (c.kept) atomicAdd(&g->kept, c.kept);
  if (c.label_entries) atomicAdd(&g->label_entries, c.label_entries);
  if (c.mapped) atomicAdd(&g->mapped, c.mapped);
  for (int i = 0; i < 4; ++i) if (c.lib_mask_sum[i]) atomicAdd(&g->lib_mask_sum[i], c.lib_mask_sum[i]);
  if (c.compatible) atomicAdd(&g->compatible, c.compatible);
}

// K1: one thread per read pair -- seeds, chains, candidates, DP task list
__global__ void k_seed_chain(IndexView ix, Params p, const uint8_t* __restrict__ left,
                             const uint8_t* __restrict__ right, uint32_t n, uint32_t L, BatchBufs b) {
  const uint32_t T = gridDim.x * blockDim.x;
  const uint32_t tid0 = blockIdx.x * blockDim.x + threadIdx.x;
  Counters ctr;
  memset(&ctr, 0, sizeof(ctr));
  uint64_t* keys = b.keys + tid0;
  for (uint32_t r = tid0; r < n; r += T) {
    Cand* lc = b.cand_l + (size_t)r * MAXCAND;
    Cand* rc = b.cand_r + (size_t)r * MAXCAND;
    const uint32_t nl = mate_candidates(ix, p, left + (size_t)r * L, L, keys, T, lc, ctr);
    const uint32_t nr = mate_candidates(ix, p, right + (size_t)r * L, L, keys, T, rc, ctr);
    b.n_l[r] = nl;
    b.n_r[r] = nr;
    // which candidates take part in a joint hit (=> need a DP score)
    unsigned long long used_l = 0, used_r = 0;
    const uint32_t nj = for_each_joint(p, lc, nl, rc, nr, L, [&](const Joint& j, uint32_t) {
      if (j.li >= 0) used_l |= 1ull << j.li;
      if (j.ri >= 0) used_r |= 1ull << j.ri;
    });
    if (nj == 0 || nj > p.max_read_occ) { b.n_l[r] |= 0x80000000u; continue; }   // unmapped / too many places
    const uint32_t cnt = (uint32_t)(__popcll(used_l) + __popcll(used_r));
    uint32_t slot = atomicAdd(b.n_tasks, cnt);
    for (uint32_t a = 0; a < nl; ++a) if (used_l >> a & 1) b.tasks[slot++] = (r << 7) | a;
    for (uint32_t a = 0; a < nr; ++a) if (used_r >> a & 1) b.tasks[slot++] = (r << 7) | 64u | a;
    ctr.candidates += cnt;
  }
  add_counters(b.ctr, ctr);
}

// K2: one warp per mate alignment.  Lane j <-> band cell j (W = 2*band+1 <= 32): for read row i
// the cell is reference position diag_c + i + (j - band).  Same recurrences as dp_score_serial:
//   M = H(i-1,j) + s ; E = max(H(i-1,j+1) - go - ge, E(i-1,j+1) - ge) ; F = max_{k<j} (H'(i,k) - go - (j-k) ge)
// with H' = max(M, E): opening a gap from an F-derived H never beats extending that F (go >= 0),
// so the in-row dependency of F is a max-plus prefix scan (5 shuffle steps).
__global__ void k_dp_score(IndexView ix, Params p, const uint8_t* __restrict__ left,
                           const uint8_t* __restrict__ right, uint32_t L, BatchBufs b) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t ntasks = *b.n_tasks;
  const int32_t B = (int32_t)p.band, W = 2 * B + 1;
  for (uint32_t t = warp; t < ntasks; t += nwarps) {
    const uint32_t task = b.tasks[t];
    const uint32_t r = task >> 7, mate = (task >> 6) & 1u, ci = task & 63u;
    const Cand c = mate ? b.cand_r[(size_t)r * MAXCAND + ci] : b.cand_l[(size_t)r * MAXCAND + ci];
    const uint8_t* read = (mate ? right : left) + (size_t)r * L;
    const uint32_t ori = c.ori_cov >> 31;
    const int64_t tlen = (int64_t)(ix.tx_off[c.tid + 1] - ix.tx_off[c.tid]);
    const uint8_t* ref = ix.codes + ix.tx_off[c.tid];
    const bool in_band = (int32_t)lane < W;
    int32_t H = in_band ? 0 : NEG_SCORE, E = NEG_SCORE;
    // the reference base of lane j for row i is ref[diag_c + i + j - B]: lane j's base for row i+1
    // is lane j+1's base of row i, so each row needs ONE new base (for the last lane)
    int64_t rpos = (int64_t)c.diag_c + ((int32_t)lane - B);
    uint8_t rbase = (rpos >= 0 && rpos < tlen) ? ref[rpos] : (uint8_t)255;
    for (uint32_t i = 0; i < L; ++i) {
      const uint8_t cc = ori ? read[L - 1 - i] : read[i];
      const uint8_t rb = ori ? (uint8_t)(cc > 3 ? 4 : 3 - cc) : cc;
      const bool valid = in_band && rbase != 255;
      const int32_t Hup = __shfl_down_sync(0xffffffffu, H, 1);
      const int32_t Eup = __shfl_down_sync(0xffffffffu, E, 1);
      int32_t m = NEG_SCORE, e = NEG_SCORE;
      if (valid) {
        m = H + ((rb < 4 && rb == rbase) ? p.ma : p.mp);
        if ((int32_t)lane + 1 < W) e = max(Hup - p.go - p.ge, Eup - p.ge);
        if (e < NEG_SCORE) e = NEG_SCORE;
      }
      const int32_t hp = valid ? max(m, e) : NEG_SCORE;
      // F_j = max_{k<j} (hp_k + k*ge) - go - j*ge  (exclusive max-prefix over lanes)
      int32_t x = (hp <= NEG_SCORE) ? NEG_SCORE : hp + (int32_t)lane * p.ge;
      int32_t pref = __shfl_up_sync(0xffffffffu, x, 1);
      if (lane == 0) pref = NEG_SCORE;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int32_t y = __shfl_up_sync(0xffffffffu, pref, o);
        if ((int)lane >= o) pref = max(pref, y);
      }
      int32_t f = (pref <= NEG_SCORE) ? NEG_SCORE : pref - p.go - (int32_t)lane * p.ge;
      if (f < NEG_SCORE) f = NEG_SCORE;
      int32_t h = NEG_SCORE;
      if (valid) { h = max(hp, f); if (h < NEG_SCORE) h = NEG_SCORE; }
      H = h;
      E = valid ? e : NEG_SCORE;
      // advance the reference window by one base
      const uint8_t nb = __shfl_down_sync(0xffffffffu, rbase, 1);
      ++rpos;
      if ((int32_t)lane == W - 1) rbase = (rpos >= 0 && rpos < tlen) ? ref[rpos] : (uint8_t)255;
      else rbase = nb;
    }
    int32_t best = in_band ? H : NEG_SCORE;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
    if (lane == 0) (mate ? b.score_r : b.score_l)[(size_t)r * MAXCAND + ci] = best;
  }
}

// K3: one thread per read pair -- salmon's alignment filtering, auxiliary probabilities, label
// work estimate of a read for k_assign (joint hits to walk): reads are handed to threads in this order so that the
// threads of a warp run loops of similar length
__global__ void k_assign_work(uint32_t n, const uint32_t* __restrict__ n_l, const uint32_t* __restrict__ n_r,
                              uint32_t* __restrict__ work, uint32_t* __restrict__ ids) {
  uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const uint32_t nl = n_l[r], nr = n_r[r];
  uint32_t w = 0;
  if (!(nl & 0x80000000u)) { w = 1 + nl * nr + nl + nr; if (w > 255u) w = 255u; }
  work[r] = w; ids[r] = r;
}

// SAM: a sink is attached -- also fill the side output (per-mate scores, decoy alignments); `side` holds the chunk's
// base pointers.  RESCUE: orphan rescue ran on the chunk -- a read with rescued pairs takes them (rb) instead of the
// join.  The instance without either is the default path, unchanged.
template <bool SAM, bool RESCUE>
__global__ void k_assign(IndexView ix, Params p, FldView fld, int useAux, int burnedIn, uint32_t n, uint32_t L,
                         BatchBufs b, OnlineView on, uint32_t chunk_first_read, const uint32_t* __restrict__ order,
                         SamSide side, RescueBufs rb) {
  const uint32_t T = gridDim.x * blockDim.x;
  const uint32_t tid0 = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t cap = p.max_read_occ;
  Counters ctr;
  memset(&ctr, 0, sizeof(ctr));
  for (uint32_t q = tid0; q < n; q += T) {
    const uint32_t r = order ? order[q] : q;
    ReadOut o;
    o.n_aln = b.n_aln + r;
    o.tid = b.tid + (size_t)r * cap; o.score = b.score + (size_t)r * cap; o.prob = b.prob + (size_t)r * cap;
    o.pos = b.pos + (size_t)r * cap; o.mate_pos = b.mate_pos + (size_t)r * cap; o.flags = b.flags + (size_t)r * cap;
    o.flen = b.flen + (size_t)r * cap; o.label = b.label + (size_t)r * 2 * cap; o.weight = b.weight + (size_t)r * cap;
    SamSide sd;
    const SamSide* sdp = nullptr;
    if (SAM) {
      sd.n_out = side.n_out + r; sd.decoy = side.decoy + r;
      sd.score1 = side.score1 + (size_t)r * cap; sd.score2 = side.score2 + (size_t)r * cap;
      sdp = &sd;
    }
    const uint32_t nlr = b.n_l[r];
    if (nlr & 0x80000000u) {
      *o.n_aln = 0;
      if (SAM) { *sd.n_out = 0; *sd.decoy = 0; }
      continue;
    }
    const uint32_t nl = nlr, nr = b.n_r[r];
    if (nl * nr <= 32u && nl + nr <= 32u) {
      // common case: few joint hits -> per-thread scratch in local memory (interleaved across threads, L1-cached)
      int32_t sc[32], pi[32], pt[32], b1[32], b2[32], b3[32];
      Joint jh[32];
      double lp[32];
      // candidates and their scores first, with independent loads (the logic below re-reads them many times)
      Cand lcl[32], rcl[32];
      int32_t sl[32], sr[32];
      const Cand* gl = b.cand_l + (size_t)r * MAXCAND;
      const Cand* gr = b.cand_r + (size_t)r * MAXCAND;
      for (uint32_t a = 0; a < nl; ++a) { lcl[a] = gl[a]; sl[a] = b.score_l[(size_t)r * MAXCAND + a]; }
      for (uint32_t a = 0; a < nr; ++a) { rcl[a] = gr[a]; sr[a] = b.score_r[(size_t)r * MAXCAND + a]; }
      // rescued pairs (at most one per appended candidate, so <= 32 here) are built in place in jh
      const uint32_t npre = RESCUE ? rescued_joints(p, rb, r, lcl, rcl, L, jh) : 0;
      assign_read(ix, p, fld, useAux != 0, burnedIn != 0, lcl, nl, rcl, nr, sl, sr, L, sc, pi, pt, b1, b2, b3, jh, o, ctr,
                  &on, chunk_first_read + r, lp, sdp, npre ? jh : nullptr, npre);
    } else {
      const size_t so = (size_t)tid0 * cap;
      const Cand* gl = b.cand_l + (size_t)r * MAXCAND;
      const Cand* gr = b.cand_r + (size_t)r * MAXCAND;
      const uint32_t npre = RESCUE ? rescued_joints(p, rb, r, gl, gr, L, b.jh + so) : 0;   // <= anchors <= cap
      assign_read(ix, p, fld, useAux != 0, burnedIn != 0, gl, nl, gr, nr, b.score_l + (size_t)r * MAXCAND,
                  b.score_r + (size_t)r * MAXCAND, L, b.sc + so, b.perm_idx + so, b.perm_tid + so, b.bs_tid + so,
                  b.bs_score + so, b.bs_idx + so, b.jh + so, o, ctr, &on, chunk_first_read + r, b.lp + so, sdp,
                  npre ? b.jh + so : nullptr, npre);
    }
  }
  add_counters(b.ctr, ctr);
}

// ---- online state: initialisation, end-of-batch fold, burn-in, effective lengths ---------------------------
struct OnlineState {
  double *mass = nullptr, *prior = nullptr, *log_eff = nullptr;   // [M]
  double *hist = nullptr;             // [nf] log histogram of the FLD
  double *tot = nullptr;              // [1] log total mass
  double *cf = nullptr;               // [nf] correction factors (effective lengths)
  unsigned long long *mass_acc = nullptr, *fld_acc = nullptr;
  unsigned int *mins = nullptr;       // [0] this batch's smallest FLD length, [1] FragmentLengthDistribution::min_
  double *fm_rel = nullptr; unsigned long long *tap_q = nullptr;   // per-batch tables
  uint32_t table_cap = 0;
};

__global__ void k_online_init(uint32_t M, const uint64_t* __restrict__ tx_off, double* mass, double* prior, double* log_eff) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= M) return;
  const double len = (double)(tx_off[t + 1] - tx_off[t]);
  mass[t] = log0();
  prior[t] = sbm_det_log(0.005 * len);      // Transcript(id, name, len, alpha = 0.005), Transcript.hpp:51
  log_eff[t] = sbm_det_log(len);
}
__global__ void k_online_fold_mass(uint32_t M, double ref, double* __restrict__ mass, unsigned long long* __restrict__ acc) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= M) return;
  const unsigned long long a = acc[t];
  if (!a) return;
  mass[t] = log_add(mass[t], ref + sbm_det_log((double)a * (1.0 / MASS_SCALE)));
  acc[t] = 0;
}
// one block: FLD histogram, total mass, min, live pmf table
__global__ void k_online_fold_fld(uint32_t nf, double ref, OnlineState S, double* __restrict__ pmf_live) {
  __shared__ unsigned long long s_tot[32];
  unsigned long long mine = 0;
  for (uint32_t j = threadIdx.x; j < nf; j += blockDim.x) {
    const unsigned long long a = S.fld_acc[j];
    if (a) {
      S.hist[j] = log_add(S.hist[j], ref + sbm_det_log((double)a * (1.0 / MASS_SCALE)));
      mine += a;
      S.fld_acc[j] = 0;
    }
  }
  for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
  if ((threadIdx.x & 31) == 0) s_tot[threadIdx.x >> 5] = mine;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long tot_acc = 0;
    for (uint32_t w = 0; w < (blockDim.x + 31) / 32; ++w) tot_acc += s_tot[w];
    if (tot_acc) {
      *S.tot = log_add(*S.tot, ref + sbm_det_log((double)tot_acc * (1.0 / MASS_SCALE)));
      if (S.mins[0] < S.mins[1]) S.mins[1] = S.mins[0];
    }
  }
  __syncthreads();
  const double tot = *S.tot;
  for (uint32_t j = threadIdx.x; j < nf; j += blockDim.x) pmf_live[j] = S.hist[j] - tot;
}
// ReadExperiment::updateTranscriptLengthsAtomic (ReadExperiment.inl:61-94) + correctionFactorsFromMass
// (DistributionUtils.cpp:9-31): one thread, nf sequential steps.  With cache != 0 also FragmentLengthDistribution::
// cacheCMF (getLockedPMF + cmf(pmf), FragmentLengthDistribution.cpp:159-201) into pmf_cached / cmf_cached.
__global__ void k_online_correction(uint32_t nf, OnlineState S, int cache, double* __restrict__ scratch /* nf */,
                                    double* __restrict__ pmf_cached, double* __restrict__ cmf_cached) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  const uint32_t maxV = nf - 1;
  const uint32_t minV = (S.mins[1] == nf - 1) ? 1u : S.mins[1];
  const double tot = *S.tot;
  double sum = log0();
  for (uint32_t i = minV; i <= maxV; ++i) sum = log_add(sum, S.hist[i] - tot);
  for (uint32_t i = 0; i < nf; ++i) scratch[i] = 0.0;
  for (uint32_t i = minV; i < maxV; ++i) scratch[i] = 100.0 * sbm_det_exp((S.hist[i] - tot) - sum);
  double vals = 0.0, mult = scratch[0];
  S.cf[0] = 0.0;
  for (uint32_t i = 1; i < nf; ++i) {
    const double v = scratch[i];
    vals = __dmul_rn(v, (double)i) + vals;       // no FMA: the product rounds as the reference's does
    mult = v + mult;
    S.cf[i] = (mult > 0) ? vals / mult : 0.0;
  }
  if (cache) {
    double tm = log0(), cum = log0();
    for (uint32_t j = 0; j < nf; ++j) tm = log_add(tm, S.hist[j] - tot);
    for (uint32_t j = 0; j < nf; ++j) {
      pmf_cached[j] = (S.hist[j] - tot) - tm;
      cum = log_add(cum, pmf_cached[j]);
      cmf_cached[j] = cum;
    }
  }
}
// computeSmoothedEffectiveLengths (DistributionUtils.cpp:33-56)
__global__ void k_online_eff_len(uint32_t M, uint32_t nf, const uint64_t* __restrict__ tx_off, const double* __restrict__ cf,
                                 double* __restrict__ log_eff) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= M) return;
  const double origLen = (double)(tx_off[t + 1] - tx_off[t]);
  const double c = (origLen >= (double)nf) ? cf[nf - 1] : cf[(uint32_t)origLen];
  double effLen = origLen - c;
  if (effLen < 1.0) effLen = origLen;
  log_eff[t] = sbm_det_log(effLen);
}

// ---- normalizeAlphas (src/util/SalmonUtils.cpp:461-529) over the finished classes -------------------------
__device__ __forceinline__ uint32_t uf_find(const uint32_t* parent, uint32_t x) {
  for (;;) { const uint32_t q = ((const volatile uint32_t*)parent)[x]; if (q == x) return x; x = q; }
}
// per class: unique / total counts, cluster hits (at the first transcript), unions (ClusterForest::mergeClusters)
__global__ void k_cls_accumulate(uint64_t n_classes, const uint64_t* __restrict__ loff, const uint64_t* __restrict__ woff,
                                 const uint32_t* __restrict__ labels, const uint64_t* __restrict__ counts,
                                 unsigned long long* uniq, unsigned long long* total, unsigned long long* hits,
                                 uint32_t* parent) {
  uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_classes) return;
  const uint32_t ntx = (uint32_t)(woff[c + 1] - woff[c]);
  if (ntx == 0) return;
  const uint32_t* t = labels + loff[c];
  const unsigned long long cnt = counts[c];
  atomicAdd(hits + t[0], cnt);
  if (ntx == 1) atomicAdd(uniq + t[0], cnt);
  for (uint32_t j = 0; j < ntx; ++j) {
    atomicAdd(total + t[j], cnt);
    uint32_t a = t[0], b = t[j];
    for (;;) {   // hook the larger root under the smaller: the root of a cluster is its smallest member
      a = uf_find(parent, a); b = uf_find(parent, b);
      if (a == b) break;
      if (a < b) { const uint32_t x = a; a = b; b = x; }
      if (atomicCAS(parent + a, a, b) == a) break;
    }
  }
}
__global__ void k_iota(uint32_t n, uint32_t* a) { uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; if (i < n) a[i] = i; }
__global__ void k_roots(uint32_t M, const uint32_t* __restrict__ parent, uint32_t* __restrict__ root, uint32_t* __restrict__ ids) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= M) return;
  root[t] = uf_find(parent, t); ids[t] = t;
}
__global__ void k_cluster_heads(uint32_t M, const uint32_t* __restrict__ root_sorted, uint32_t* __restrict__ head) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > M) return;
  head[i] = (i < M && (i == 0 || root_sorted[i] != root_sorted[i - 1])) ? 1u : 0u;
}
__global__ void k_cluster_starts(uint32_t M, const uint32_t* __restrict__ head, const uint32_t* __restrict__ head_scan,
                                 uint32_t* __restrict__ start) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < M && head[i]) start[head_scan[i]] = i;
}
// one warp per cluster (members ascending by transcript id): projected counts + TranscriptCluster::projectToPolytope
__global__ void k_cluster_project(uint32_t n_clusters, uint32_t M, const uint32_t* __restrict__ start,
                                  const uint32_t* __restrict__ memb, const double* __restrict__ mass,
                                  const unsigned long long* __restrict__ hits, const unsigned long long* __restrict__ uniq,
                                  const unsigned long long* __restrict__ total, double* __restrict__ projected,
                                  uint8_t* __restrict__ bound) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (c >= n_clusters) return;
  const uint32_t b = start[c], e = (c + 1 < n_clusters) ? start[c + 1] : M;
  const uint32_t cs = e - b;
  unsigned long long h = 0;
  double mx = -log0();
  for (uint32_t q = b + lane; q < e; q += 32) {
    const uint32_t t = memb[q];
    h += hits[t];
    const double m = mass[t];
    if (m != log0() && m > mx) mx = m;
  }
  for (int o = 16; o > 0; o >>= 1) { h += __shfl_xor_sync(0xffffffffu, h, o); mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o)); }
  if (mx == -log0()) {   // no mass anywhere in the cluster: projectedCounts = 0 (SalmonUtils.cpp:497-498)
    for (uint32_t q = b + lane; q < e; q += 32) projected[memb[q]] = 0.0;
    return;
  }
  double se = 0.0;
  for (uint32_t q = b + lane; q < e; q += 32) { const double m = mass[memb[q]]; if (m != log0()) se += sbm_det_exp(m - mx); }
  se = sb::warp_sum(se);
  const double logClusterMass = mx + sbm_det_log(se);
  const double clusterHits = (double)h;
  const double logClusterCount = sbm_det_log(clusterHits);
  int req = 0;
  for (uint32_t q = b + lane; q < e; q += 32) {
    const uint32_t t = memb[q];
    const double m = mass[t];
    double pc = 0.0;
    if (m != log0()) {
      pc = sbm_det_exp((m - logClusterMass) + logClusterCount);
      req |= (pc > (double)total[t]) || (pc < (double)uniq[t]);
    }
    projected[t] = pc;
    bound[q] = 0;
  }
  req = __any_sync(0xffffffffu, req);
  if (cs <= 1 || !req) return;
  __syncwarp();
  for (uint32_t round = 0;;) {
    double ub = 0.0, bd = 0.0;
    for (uint32_t q = b + lane; q < e; q += 32) {
      const uint32_t t = memb[q];
      double pc = projected[t];
      if (pc > (double)total[t]) { pc = (double)total[t]; bound[q] = 1; projected[t] = pc; }
      else if (pc < (double)uniq[t]) { pc = (double)uniq[t]; bound[q] = 1; projected[t] = pc; }
      if (bound[q]) bd += pc; else ub += pc;
    }
    ub = sb::warp_sum(ub); bd = sb::warp_sum(bd);
    if (fabs(ub + bd - clusterHits) <= 0.375e-10) break;     // approxEqual, SalmonMath.hpp:51-53
    if (ub == 0) {
      for (uint32_t q = b + lane; q < e; q += 32) bound[q] = 0;
      ub = bd; bd = 0;
    }
    const double normalizer = (clusterHits - bd) / ub;
    __syncwarp();
    for (uint32_t q = b + lane; q < e; q += 32) if (!bound[q]) projected[memb[q]] *= normalizer;
    __syncwarp();
    if (++round > 5000) break;
  }
}
// transcript lengths as effective lengths (--noEffectiveLengthCorrection)
__global__ void k_tx_len(uint32_t M, const uint64_t* __restrict__ tx_off, double* __restrict__ out) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < M) out[t] = (double)(tx_off[t + 1] - tx_off[t]);
}
__global__ void k_exp_vec(uint32_t n, const double* __restrict__ in, double* __restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = sbm_det_exp(in[i]);
}

// ---- equivalence-class builder: records (label, weights, count) -> classes ----------------
// A record i is (labels[lstart[i] .. +llen[i]), weights[wstart[i] .. +wlen[i]), counts[i] or 1).
// hash of a label (64-bit FNV-1a over the 32-bit words; the value is never persisted, like the
// reference's XXH64 in TranscriptGroup::hash, src/model/TranscriptGroup.cpp:10-15)
struct Records {
  uint32_t n;
  const uint64_t* lstart; const uint32_t* llen;
  const uint64_t* wstart; const uint32_t* wlen;
  const uint32_t* labels; const double* weights; const uint64_t* counts;
};

// per-read slots of a batch as records: read i owns labels[i*2cap ..), weights[i*cap ..)
__global__ void k_read_records(uint32_t n, uint32_t cap, int binned, const uint32_t* __restrict__ n_aln,
                               uint64_t* __restrict__ lstart, uint32_t* __restrict__ llen,
                               uint64_t* __restrict__ wstart, uint32_t* __restrict__ wlen) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t na = n_aln[i];
  lstart[i] = (uint64_t)i * 2 * cap; llen[i] = na * (binned ? 2u : 1u);
  wstart[i] = (uint64_t)i * cap; wlen[i] = na;
}
__global__ void k_label_hash(Records R, uint64_t* __restrict__ hash, uint32_t* __restrict__ idx) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R.n) return;
  uint64_t h = 1469598103934665603ull;
  const uint32_t* lab = R.labels + R.lstart[i];
  const uint32_t len = R.llen[i];
  for (uint32_t j = 0; j < len; ++j) { h ^= lab[j]; h *= 1099511628211ull; }
  h ^= len;
  h = mix64(h);
  hash[i] = h;
  idx[i] = i;
}
__global__ void k_label_heads(Records R, const uint64_t* __restrict__ hash_sorted, const uint32_t* __restrict__ idx,
                              uint32_t* __restrict__ head) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > R.n) return;
  if (i == R.n) { head[i] = 0; return; }
  uint32_t h = 1;
  if (i > 0 && hash_sorted[i] == hash_sorted[i - 1]) {
    const uint32_t a = idx[i], b = idx[i - 1];
    const uint32_t la = R.llen[a], lb = R.llen[b];
    if (la == lb) {
      h = 0;
      const uint32_t* pa = R.labels + R.lstart[a];
      const uint32_t* pb = R.labels + R.lstart[b];
      for (uint32_t j = 0; j < la; ++j) if (pa[j] != pb[j]) { h = 1; break; }
    }
  }
  head[i] = h;
}
// per class: position of its first record in the sorted order, label / weight lengths
__global__ void k_class_sizes(Records R, const uint32_t* __restrict__ head, const uint32_t* __restrict__ head_scan,
                              const uint32_t* __restrict__ idx, uint32_t* __restrict__ first,
                              uint64_t* __restrict__ cls_llen, uint64_t* __restrict__ cls_wlen) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R.n || !head[i]) return;
  const uint32_t c = head_scan[i];
  const uint32_t r = idx[i];
  first[c] = i;
  cls_llen[c] = R.llen[r];
  cls_wlen[c] = R.wlen[r];
}
// per class (one warp): count and weights summed over its records IN RECORD ORDER
// (EquivalenceClassBuilder.hpp:237-250: count++, weights[i] += w_i); lanes = label / weight entries
__global__ void k_class_reduce(Records R, uint32_t n_classes, const uint32_t* __restrict__ first,
                               const uint32_t* __restrict__ idx, const uint64_t* __restrict__ out_loff,
                               const uint64_t* __restrict__ out_woff, uint32_t* __restrict__ out_labels,
                               double* __restrict__ out_weights, uint64_t* __restrict__ out_counts) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (c >= n_classes) return;
  const uint32_t b = first[c], e = (c + 1 < n_classes) ? first[c + 1] : R.n;
  const uint32_t r0 = idx[b];
  const uint32_t ll = R.llen[r0], wl = R.wlen[r0];
  const uint32_t* lab = R.labels + R.lstart[r0];
  for (uint32_t j = lane; j < ll; j += 32) out_labels[out_loff[c] + j] = lab[j];
  for (uint32_t j = lane; j < wl; j += 32) {
    double s = 0.0;
    for (uint32_t q = b; q < e; ++q) s = __dadd_rn(s, R.weights[R.wstart[idx[q]] + j]);
    out_weights[out_woff[c] + j] = s;
  }
  if (lane == 0) {
    uint64_t cnt = 0;
    if (R.counts) for (uint32_t q = b; q < e; ++q) cnt += R.counts[idx[q]];
    else cnt = e - b;
    out_counts[c] = cnt;
  }
}
// finish(): TGValue::normalizeAux (EquivalenceClassBuilder.hpp:114-123)
__global__ void k_normalize(uint64_t n_classes, const uint64_t* __restrict__ woff, double* __restrict__ w) {
  uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_classes) return;
  double s = 0.0;
  for (uint64_t j = woff[c]; j < woff[c + 1]; ++j) s = __dadd_rn(s, w[j]);
  const double norm = __ddiv_rn(1.0, s);
  for (uint64_t j = woff[c]; j < woff[c + 1]; ++j) w[j] = __dmul_rn(w[j], norm);
}
// CSR store -> record descriptors (finish: the class tables of all batches become records)
__global__ void k_store_records(uint64_t n, const uint64_t* __restrict__ loff, const uint64_t* __restrict__ woff,
                                uint64_t lbase, uint64_t wbase, uint64_t* __restrict__ lstart, uint32_t* __restrict__ llen,
                                uint64_t* __restrict__ wstart, uint32_t* __restrict__ wlen) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  lstart[i] = lbase + loff[i]; llen[i] = (uint32_t)(loff[i + 1] - loff[i]);
  wstart[i] = wbase + woff[i]; wlen[i] = (uint32_t)(woff[i + 1] - woff[i]);
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// host driver
// ---------------------------------------------------------------------------------------------
// Class tables live in a growing device arena (no cudaMalloc / cudaFree per batch: with peer access enabled -- any
// multi-GPU run -- every allocation is mapped into all peers and becomes expensive).  A store = one table.
struct Arena {
  uint32_t* labels = nullptr; double* weights = nullptr; uint64_t* counts = nullptr;
  uint64_t *loff = nullptr, *woff = nullptr;        // per store n+1 entries, relative to the store's label / weight base
  uint64_t n_l = 0, n_w = 0, n_c = 0, n_o = 0;           // cursors
};
struct EqStore {   // a CSR table inside the arena
  uint64_t n = 0, n_lab = 0, n_w = 0;
  uint64_t base_l = 0, base_w = 0, base_c = 0, base_o = 0;
};

struct AggScratch {   // sized for `cap` records
  uint64_t cap = 0;
  uint64_t *lstart = nullptr, *wstart = nullptr, *hash = nullptr, *hash2 = nullptr, *cls_llen = nullptr, *cls_wlen = nullptr;
  uint32_t *llen = nullptr, *wlen = nullptr, *idx = nullptr, *idx2 = nullptr, *head = nullptr, *head_scan = nullptr, *first = nullptr;
  void* tmp = nullptr;
  size_t tmp_bytes = 0;
};

struct FinBufs {   // normalizeAlphas scratch, [M] each
  unsigned long long *uniq = nullptr, *total = nullptr, *hits = nullptr;
  uint32_t *parent = nullptr, *root = nullptr, *root2 = nullptr, *ids = nullptr, *memb = nullptr, *head = nullptr,
           *head_scan = nullptr, *start = nullptr;
  double *proj = nullptr, *eff = nullptr;
  uint8_t* bound = nullptr;
  void* tmp = nullptr;
  size_t tmp_bytes = 0;
};

struct sb_map_ctx {
  int device = 0;
  sb::Resources res;                 // every buffer, stream and event below (the SAM formatter's are samd's)
  explicit sb_map_ctx(int dev) : device(dev), res(dev) {}
  int n_sm = 0;
  cudaStream_t stream = nullptr, copy_stream = nullptr;
  sb_index* index = nullptr;
  Params p{};
  uint32_t batch_cap = 0, read_len_cap = 0, chunk = 0, chunk_cap = 0;
  int variant = 1;                   // 1 = warp kernels (map_kernels.cuh), 0 = serial-form kernels
  int input_dev = 0;                 // sb_map_batch's read pointers are device pointers (bench: inputs resident in HBM)
  int ascii = 0;                     // reads are sequence characters (ACGTN...) instead of base codes
  int fast_ok = 1;
  int no_projection = 0;             // finish without normalizeAlphas' cluster projection (--skipQuant)
  uint32_t k1_threads = 0, seed_blocks = 0, dp_blocks = 0;
  BatchBufs b{};                     // cand/score/task buffers: one chunk; outputs: whole batch
  // k_assign of chunk i runs on its own stream next to the seed / DP kernels of chunk i+1 (it is latency-bound at
  // low issue utilisation, they are issue-bound): the buffers both sides touch exist twice
  int profile = 0;          // SB_MAP_PROFILE: per-batch host / device times on stderr
  int overlap_assign = 1;   // results are bit-identical either way
  cudaStream_t assign_stream = nullptr;
  cudaEvent_t ev_dp[2] = {nullptr, nullptr}, ev_asg[2] = {nullptr, nullptr};
  uint32_t *alt_n_l = nullptr, *alt_n_r = nullptr;
  Cand *alt_cand_l = nullptr, *alt_cand_r = nullptr;
  int32_t *alt_score_l = nullptr, *alt_score_r = nullptr;
  uint8_t* d_in[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};   // [slot][mate]
  cudaEvent_t ev_in[2] = {nullptr, nullptr}, ev_free[2] = {nullptr, nullptr};
  PackedReads pr{};
  uint64_t* d_overflow = nullptr;
  uint32_t* d_next_task = nullptr;     // [0] task counter, [4..6] list sizes
  uint32_t *d_list_int = nullptr, *d_list_edge = nullptr, *d_list_n = nullptr;
  uint32_t *d_work = nullptr, *d_work2 = nullptr, *d_ids = nullptr, *d_order = nullptr;   // k_assign read order
  unsigned long long* d_full_dp = nullptr;
  // FLD tables
  double* d_fld = nullptr;
  FldView fld{};
  AggScratch agg;
  FinBufs fin;
  // multi-GPU: this rank's partial statistics on the host (sb_map_partial_get)
  std::vector<double> hp_mass, hp_hist;
  std::vector<uint64_t> hp_uniq, hp_total, hp_hits;
  std::vector<uint32_t> hp_root;
  // online state (masses, FLD, effective lengths)
  OnlineState on;
  uint32_t M = 0, nf = 0;
  uint64_t frags_seen = 0, timestep = 0;
  int burned_in = 0;
  std::vector<double> fm;                 // log forgetting masses by timestep
  std::vector<double> h_fm_rel; std::vector<unsigned long long> h_tap_q;
  double* d_scratch_nf = nullptr;
  unsigned int h_bm = 0;
  std::vector<double> init_tables;     // FLD tables of the prior (sb_map_reset)
  std::vector<cudaEvent_t> ev_seed;    // pairs of events around the seed kernel of each chunk
  std::vector<double> h_proj, h_eff;
  std::vector<uint64_t> h_uniq, h_total;
  // eq-class store: one EqStore per processed batch, merged at finish
  Arena arena;
  std::vector<EqStore> stores;
  uint64_t frag_counter = 0;     // fragments assigned so far (batched semantics)
  Counters totals{};
  uint8_t* d_dummy_mate = nullptr;     // single-end libraries: the absent second mate (N codes)
  uint64_t full_dp_total = 0;
  uint32_t launches = 0;
  float last_ms = 0;
  uint32_t last_chunks = 0;            // the last batch: chunks it ran as, whether orphan rescue ran (candidate tap)
  int last_rescue = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  // finished result (host)
  std::vector<uint64_t> h_off, h_counts;
  std::vector<uint32_t> h_tids, h_ntx, h_bins;
  std::vector<double> h_w;
  // SAM output (sb_map_attach_sam): the sink, the formatter's device buffers, the size of one output window
  sb_sam* sam = nullptr;
  SamDev* samd = nullptr;
  uint64_t sam_window = 256ull << 20;
  // orphan rescue (p.recover_orphans): task lists of one chunk; the pair lists k_assign reads exist twice (alt set)
  RescueBufs rb{};
  uint32_t* alt_rs_n_pairs = nullptr;
  uint16_t* alt_rs_pairs = nullptr;
  uint64_t rescued_total = 0, rescue_searches_total = 0, rescue_no_room_total = 0;
  std::vector<cudaEvent_t> ev_rescue;   // pairs of events around the rescue kernels of each chunk
};

static inline unsigned nblk(uint64_t n, unsigned t) { return (unsigned)((n + t - 1) / t); }

// the ungapped shortcut of k_dp_classify is exact only when no cell scores above ma and gaps cost something; under
// other scores set_option("fast_dp", 1) leaves it off
static inline int fast_dp_exact(const Params& p) { return (p.ma >= 0 && p.mp <= p.ma && p.go >= 0 && p.ge >= 0) ? 1 : 0; }

// gapless settlement of k_dp_classify (DESIGN.md section 14): in scoring mode 0, when every gapped path scores below the
// lowest mate score that can change an outcome, the best ungapped diagonal settles every alignment.  The thresholds are
// evaluated exactly as assign_read and rescue_mate_passes evaluate them, at the highest score a gapped path can reach
// (G = ma*L - go - ge) and, for a pair, with a perfect partner.  Decided per launch: it depends on L.
static inline int gapless_settles(const Params& p, uint32_t L) {
  if (p.softclip != 0) return 0;
  const int32_t perfect = p.ma * (int32_t)L, G = perfect - p.go - p.ge;
  if (!((double)G < p.min_score_fraction * (double)perfect)) return 0;   // orphans, single-end reads, rescue
  if (p.lib_type < 3 && !((double)(G + perfect) < p.min_score_fraction * (double)(2 * perfect))) return 0;   // pairs
  return 1;
}

// the three DP kernels of one chunk for scoring mode MODE (Params::softclip); the same launches in every mode
template <int NWR, int MODE>
static void launch_dp(const sb_map_ctx* c, cudaStream_t st, const IndexView& ix, const Params& p, uint32_t L,
                      const uint8_t* dl, const uint8_t* dr, const DpIo& io) {
  const int gapless = (c->fast_ok && gapless_settles(p, L)) ? 1 : 0;
  k_dp_classify<NWR, MODE><<<c->n_sm * 3, 256, 0, st>>>(ix, p, c->pr, L, c->fast_ok, gapless, io);
  k_dp_pair<NWR, MODE == 2 ? 2 : 0><<<c->n_sm * (NWR == 4 ? 3 : 2), 256, 0, st>>>(ix, p, c->pr, L, io);
  k_dp_general<NWR, MODE><<<c->n_sm * 3, 256, 0, st>>>(ix, p, c->pr, dl, dr, L, c->ascii, io);
}

extern "C" void sb_map_default_params(sb_map_params* q) {
  memset(q, 0, sizeof(*q));
  q->k = 31; q->stride = 4; q->max_occs_per_hit = 1000; q->max_read_occ = 200; q->max_frag_len = 1000;
  q->band = 15; q->chain_gap = 8; q->range_bins = 4; q->ma = 2; q->mp = -4; q->go = 6; q->ge = 2;
  q->hard_filter = 0; q->first_decoy = 0x7fffffff; q->consensus_frac = 0.65; q->min_score_fraction = 0.65;
  q->score_exp = 1.0; q->min_aln_prob = 1e-5; q->decoy_threshold = 1.0; q->fld_mean = 250.0; q->fld_sd = 25.0;
  q->num_pre_burnin = 5000; q->num_burnin = 5000000;
  q->seed = 42; q->mini_batch = 5000;
  q->pre_merge_thresh = 0.75; q->post_merge_thresh = 0.9; q->orphan_thresh = 0.95;   // SalmonDefaults.hpp:28-30
  q->allow_dovetail = 0; q->allow_orphans = 1;                                         // :46, discardOrphansQuasi = false
}

// --mimicBT2 / --mimicStrictBT2 (QuantOptionsUtils.cpp:250-289), applied after the other options so that it overrides them
extern "C" int sb_map_mimic_bt2(sb_map_params* q, int strict) {
  if (!q) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  q->max_read_occ = 1000;
  q->consensus_frac = 1.0 - 0.5;        // consensusSlack 0.5
  // discardOrphansQuasi concerns the mates of pairs: a single-end read is a left orphan in this mapper, so it stays
  const bool single_end = (q->lib_type >= SB_LIB_U && q->lib_type <= SB_LIB_SR) || q->lib_type == SB_LIB_AUTO_SINGLE;
  if (!single_end) q->allow_orphans = 0;
  if (q->softclip == 1) q->softclip = 0;   // softclipOverhangs off; --softclip (mode 2) stays
  if (strict) { q->min_score_fraction = 0.8; q->ma = 1; q->mp = 0; q->go = 25; q->ge = 25; }
  else { q->ma = 2; q->mp = -4; q->go = 5; q->ge = 3; }
  return SB_OK;
}

static void build_fld_host(const Params& p, std::vector<double>& t) {
  // FragmentLengthDistribution ctor / pmf / cmf / cached tables (FragmentLengthDistribution.cpp:22-78,
  // :122-132, :163-201) and LogCMFCache's pre-burn-in table (DistributionUtils.cpp:103-116); host libm.
  const uint32_t n = p.max_frag_len + 1;
  const double LOG_0 = HUGE_VAL, LOG_EPSILON = log(0.375e-10);
  auto logAdd = [&](double x, double y) {
    if (fabs(x) == LOG_0) return y;
    if (fabs(y) == LOG_0) return x;
    if (y > x) std::swap(x, y);
    return x + log(1 + exp(y - x));
  };
  auto ncdf = [&](double x) { return 0.5 * erfc(-(x - p.fld_mean) / (p.fld_sd * sqrt(2.0))); };
  t.assign((size_t)5 * n + 1, 0.0);
  double* pmf_live = t.data(); double* pmf_cached = t.data() + n; double* cmf_cached = t.data() + 2 * n;
  double* cmf_quirk = t.data() + 3 * n;
  double* hist = t.data() + 4 * n;     // [4n, 5n): log histogram; [5n]: log total mass
  double tot = LOG_0;
  for (uint32_t i = 0; i < n; ++i) {
    const double nm = ncdf(i + 0.5) - ncdf(i - 0.5);
    double mass = LOG_EPSILON;
    if (nm != 0) mass = 0.0 + log(nm);
    hist[i] = mass;
    tot = logAdd(tot, mass);
  }
  double tm = LOG_0;
  for (uint32_t i = 0; i < n; ++i) { pmf_live[i] = hist[i] - tot; tm = logAdd(tm, pmf_live[i]); }
  double cum = LOG_0, cq = LOG_0;
  for (uint32_t i = 0; i < n; ++i) {
    pmf_cached[i] = pmf_live[i] - tm;
    cum = logAdd(cum, pmf_cached[i]);
    cmf_cached[i] = cum;
    cq = logAdd(cq, LOG_EPSILON);
    cmf_quirk[i] = cq;
  }
  t[(size_t)5 * n] = tot;
}

// ForgettingMassCalculator (ForgettingMassCalculator.hpp:24-40), forgettingFactor 0.65
static double forgetting_mass(std::vector<double>& fm, uint64_t t) {
  const double ff = 0.65;
  while (fm.size() <= t) {
    const uint64_t j = fm.size();
    if (j == 0) fm.push_back(0.0);
    else fm.push_back(fm[j - 1] + ff * log((double)j) - log(pow((double)(j + 1), ff) - 1));
  }
  return fm[t];
}

static int agg_reserve(sb_map_ctx* c, uint64_t n) {
  AggScratch& a = c->agg;
  sb::Resources& r = c->res;
  if (n <= a.cap) return SB_OK;
  a.cap = 0;   // until every buffer holds the new size
  const uint64_t cap = std::max<uint64_t>(n, 1024);
  SB_TRY(r.grow(&a.lstart, cap)); SB_TRY(r.grow(&a.wstart, cap)); SB_TRY(r.grow(&a.hash, cap)); SB_TRY(r.grow(&a.hash2, cap));
  SB_TRY(r.grow(&a.cls_llen, cap + 1)); SB_TRY(r.grow(&a.cls_wlen, cap + 1));
  SB_TRY(r.grow(&a.llen, cap)); SB_TRY(r.grow(&a.wlen, cap)); SB_TRY(r.grow(&a.idx, cap)); SB_TRY(r.grow(&a.idx2, cap));
  SB_TRY(r.grow(&a.head, cap + 1)); SB_TRY(r.grow(&a.head_scan, cap + 1)); SB_TRY(r.grow(&a.first, cap + 1));
  size_t tb = 0, tb2 = 0, tb3 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tb, a.hash, a.hash2, a.idx, a.idx2, (int)cap, 0, 64, (cudaStream_t)0);
  cub::DeviceScan::ExclusiveSum(nullptr, tb2, a.head, a.head_scan, (int)cap + 1, (cudaStream_t)0);
  cub::DeviceScan::ExclusiveSum(nullptr, tb3, a.cls_llen, a.cls_llen, (int)cap + 1, (cudaStream_t)0);
  a.tmp_bytes = std::max(tb, std::max(tb2, tb3));
  SB_TRY(r.grow((unsigned char**)&a.tmp, a.tmp_bytes));
  a.cap = cap;
  return SB_OK;
}

static inline double wall_s() {
  timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

extern "C" sb_map_ctx* sb_map_create(sb_index* ix, const sb_map_params* q, int device, uint32_t batch_cap,
                                     uint32_t max_read_len) {
  if (!ix || !q) { sb::set_error("null argument"); return nullptr; }
  if (q->softclip < 0 || q->softclip > 2) {
    sb::set_error("sb_map_create: unsupported softclip mode %d (0 end-to-end, 1 overhangs, 2 soft-clip)", q->softclip);
    return nullptr;
  }
  if (!(q->incompat_prior >= 0.0 && q->incompat_prior <= 1.0)) {
    sb::set_error("sb_map_create: incompat_prior must be a probability in [0, 1], got %g", q->incompat_prior);
    return nullptr;
  }
  if (q->max_read_occ > MAX_READ_OCC) {
    sb::set_error("sb_map_create: max_read_occ %u is above the supported %u (--maxReadOcc)", q->max_read_occ, MAX_READ_OCC);
    return nullptr;
  }
  if (q->no_frag_len_dist && !q->no_eff_len_correction) {   // QuantOptionsUtils.cpp:641-647
    sb::set_error("sb_map_create: no_frag_len_dist needs no_eff_len_correction (--noFragLengthDist without "
                  "--noEffectiveLengthCorrection)");
    return nullptr;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
    cudaGetLastError();
    sb::set_error("no CUDA device available (libsalmon_b200 has no CPU fallback)");
    return nullptr;
  }
  if (q->band > 15 || max_read_len > 256 || q->k != ix->k || batch_cap == 0 ||
      batch_cap > (1u << 24) || q->stride == 0 || max_read_len < q->k ||
      (max_read_len - q->k) / q->stride + 2 > MAX_LOOKUPS) {
    sb::set_error("sb_map_create: unsupported parameters (band<=15, read_len<=256, k must match "
                  "the index, at most %u seed positions per mate)", MAX_LOOKUPS);
    return nullptr;
  }
  if (index_to_device(ix, device) != SB_OK) return nullptr;
  sb_map_ctx* c = new sb_map_ctx(device);
  c->index = ix; c->batch_cap = batch_cap; c->read_len_cap = max_read_len;
  Params& p = c->p;
  p.k = q->k; p.stride = q->stride; p.max_occs_per_hit = q->max_occs_per_hit; p.max_read_occ = q->max_read_occ;
  p.max_frag_len = q->max_frag_len; p.band = q->band; p.chain_gap = q->chain_gap; p.range_bins = q->range_bins;
  p.ma = q->ma; p.mp = q->mp; p.go = q->go; p.ge = q->ge; p.hard_filter = q->hard_filter; p.first_decoy = q->first_decoy;
  p.consensus_frac = q->consensus_frac; p.min_score_fraction = q->min_score_fraction; p.score_exp = q->score_exp;
  p.min_aln_prob = q->min_aln_prob; p.decoy_threshold = q->decoy_threshold; p.fld_mean = q->fld_mean; p.fld_sd = q->fld_sd;
  p.num_pre_burnin = q->num_pre_burnin; p.num_burnin = q->num_burnin;
  p.seed = q->seed; p.mini_batch = q->mini_batch ? q->mini_batch : 5000; p.reserved = 0;
  p.pre_merge_thresh = q->pre_merge_thresh; p.post_merge_thresh = q->post_merge_thresh; p.orphan_thresh = q->orphan_thresh;
  p.allow_dovetail = q->allow_dovetail; p.allow_orphans = q->allow_orphans;
  p.lib_type = q->lib_type; p.recover_orphans = q->recover_orphans ? 1 : 0; p.softclip = q->softclip;
  p.no_single_frag_prob = q->no_single_frag_prob ? 1 : 0; p.no_frag_len_dist = q->no_frag_len_dist ? 1 : 0;
  p.no_eff_len_correction = q->no_eff_len_correction ? 1 : 0; p.incompat_prior = q->incompat_prior;
  if (p.lib_type < 0 || p.lib_type > 5) { sb::set_error("unsupported library type %d (IU, ISF, ISR, U, SF, SR)", p.lib_type); delete c; return nullptr; }
  if (!(p.pre_merge_thresh >= 0 && p.pre_merge_thresh <= 1) || !(p.post_merge_thresh >= 0 && p.post_merge_thresh <= 1) ||
      !(p.orphan_thresh >= 0 && p.orphan_thresh <= 1)) {
    sb::set_error("the chain sub-thresholds must be in [0, 1]");    // QuantOptionsUtils.cpp:234-247
    delete c;
    return nullptr;
  }
  c->fast_ok = fast_dp_exact(p);
  cudaDeviceProp prop;
  const cudaError_t de = cudaSetDevice(device);
  if (de != cudaSuccess || cudaGetDeviceProperties(&prop, device) != cudaSuccess) {
    sb::set_error("sb_map_create: cannot use device %d: %s", device, cudaGetErrorString(de != cudaSuccess ? de : cudaGetLastError()));
    delete c;
    return nullptr;
  }
  c->n_sm = prop.multiProcessorCount;
  if (const char* e = getenv("SB_MAP_OVERLAP")) c->overlap_assign = atoi(e) ? 1 : 0;
  c->profile = getenv("SB_MAP_PROFILE") ? 1 : 0;
  int rc = SB_OK;
  auto E = [&](cudaEvent_t* ev, unsigned flags) { if (rc == SB_OK) rc = c->res.event(ev, flags); };
  auto A = [&](auto** ptr, size_t n) { if (rc == SB_OK) rc = c->res.alloc(ptr, n); };
  for (cudaStream_t* st : {&c->stream, &c->copy_stream, &c->assign_stream}) if (rc == SB_OK) rc = c->res.stream(st, cudaStreamNonBlocking);
  E(&c->ev0, cudaEventDefault); E(&c->ev1, cudaEventDefault);
  for (int s = 0; s < 2; ++s) {
    E(&c->ev_dp[s], cudaEventDisableTiming); E(&c->ev_asg[s], cudaEventDisableTiming);
    E(&c->ev_in[s], cudaEventDisableTiming); E(&c->ev_free[s], cudaEventDisableTiming);
  }
  const uint32_t cap = p.max_read_occ;
  const size_t B = batch_cap;
  // reads per pipeline chunk: the per-chunk buffers are sized for chunk_cap; SB_MAP_CHUNK raises it for sweeps
  size_t chunk_cap = 131072;
  if (const char* e = getenv("SB_MAP_CHUNK")) { const long v = atol(e); if (v >= 1024 && v <= (1 << 24)) chunk_cap = (size_t)v; }
  c->chunk = c->chunk_cap = (uint32_t)std::min<size_t>(B, chunk_cap);
  const size_t CH = c->chunk;
  c->k1_threads = (uint32_t)std::min<size_t>((size_t)c->n_sm * 1024, (CH + 127) / 128 * 128);
  c->seed_blocks = (uint32_t)c->n_sm * 4;
  c->dp_blocks = (uint32_t)c->n_sm * 4;
  BatchBufs& b = c->b;
  // per chunk
  A(&b.n_l, CH); A(&b.n_r, CH); A(&b.cand_l, CH * MAXCAND); A(&b.cand_r, CH * MAXCAND);
  A(&b.score_l, CH * MAXCAND); A(&b.score_r, CH * MAXCAND);
  A(&c->alt_n_l, CH); A(&c->alt_n_r, CH); A(&c->alt_cand_l, CH * MAXCAND); A(&c->alt_cand_r, CH * MAXCAND);
  A(&c->alt_score_l, CH * MAXCAND); A(&c->alt_score_r, CH * MAXCAND);
  A(&b.keys, (size_t)MAXSEEDS * c->k1_threads);
  A(&b.n_tasks, 4); A(&b.tasks, CH * 2 * MAXCAND);
  const size_t S = (size_t)c->k1_threads * cap;
  A(&b.sc, S); A(&b.perm_idx, S); A(&b.perm_tid, S); A(&b.bs_tid, S); A(&b.bs_score, S); A(&b.bs_idx, S); A(&b.jh, S);
  A(&b.lp, S);
  A(&b.ctr, 1);
  // online state
  c->M = ix->n_txps; c->nf = p.max_frag_len + 1;
  {
    OnlineState& o = c->on;
    const size_t M = std::max<uint32_t>(c->M, 1), nf = c->nf;
    o.table_cap = (uint32_t)((B + p.mini_batch - 1) / p.mini_batch + 1);
    A(&o.mass, M); A(&o.prior, M); A(&o.log_eff, M); A(&o.hist, nf); A(&o.tot, 1); A(&o.cf, nf);
    A(&o.mass_acc, M); A(&o.fld_acc, nf); A(&o.mins, 2); A(&o.fm_rel, o.table_cap); A(&o.tap_q, (size_t)o.table_cap * 5);
    A(&c->d_scratch_nf, nf);
    FinBufs& f = c->fin;
    A(&f.uniq, M); A(&f.total, M); A(&f.hits, M); A(&f.parent, M); A(&f.root, M); A(&f.root2, M); A(&f.ids, M); A(&f.memb, M);
    A(&f.head, M + 1); A(&f.head_scan, M + 1); A(&f.start, M + 1); A(&f.proj, M); A(&f.eff, M); A(&f.bound, M);
    size_t tb = 0, tb2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tb, f.root, f.root2, f.ids, f.memb, (int)M, 0, 32, (cudaStream_t)0);
    cub::DeviceScan::ExclusiveSum(nullptr, tb2, f.head, f.head_scan, (int)M + 1, (cudaStream_t)0);
    f.tmp_bytes = std::max(tb, tb2);
    A((unsigned char**)&f.tmp, f.tmp_bytes);
  }
  A(&c->d_overflow, (size_t)c->seed_blocks * SEED_WARPS * MAXSEEDS);
  A(&c->d_next_task, 8); A(&c->d_full_dp, 1);
  A(&c->d_list_int, CH * 2 * MAXCAND); A(&c->d_list_edge, CH * 2 * MAXCAND); A(&c->d_list_n, CH * 2 * MAXCAND);
  A(&c->d_work, CH); A(&c->d_work2, CH); A(&c->d_ids, CH); A(&c->d_order, CH);
  for (int s = 0; s < 2; ++s) for (int m = 0; m < 2; ++m) A(&c->d_in[s][m], CH * max_read_len);
  c->pr.wpr = (max_read_len + 31) / 32 + 1; c->pr.mpr = (max_read_len + 63) / 64 + 1;
  A(&c->pr.bits, 2 * CH * c->pr.wpr); A(&c->pr.nmask, 2 * CH * c->pr.mpr);
  // per batch (outputs)
  A(&b.n_aln, B); A(&b.tid, B * cap); A(&b.score, B * cap); A(&b.prob, B * cap); A(&b.pos, B * cap);
  A(&b.mate_pos, B * cap); A(&b.flags, B * cap); A(&b.flen, B * cap); A(&b.label, B * 2 * cap); A(&b.weight, B * cap);
  std::vector<double>& t = c->init_tables;
  build_fld_host(p, t);
  A(&c->d_fld, (size_t)4 * (p.max_frag_len + 1));
  if (p.recover_orphans) {
    RescueBufs& r = c->rb;
    const size_t NT = CH * 2 * MAXCAND;
    A(&r.n_tasks, 1); A(&r.tasks, NT); A(&r.first, CH); A(&r.n_anchor, CH); A(&r.diag, NT); A(&r.score, NT);
    A(&r.pairs, NT); A(&r.n_pairs, CH); A(&r.ctr, 3); A(&c->alt_rs_pairs, NT); A(&c->alt_rs_n_pairs, CH);
  }
  if (rc == SB_OK) rc = agg_reserve(c, B);
  if (rc == SB_OK) rc = [&]() -> int {
    SB_CUDA(cudaMemcpy(c->d_fld, t.data(), (size_t)4 * c->nf * 8, cudaMemcpyHostToDevice));
    SB_CUDA(cudaMemcpy(c->on.hist, t.data() + (size_t)4 * c->nf, (size_t)c->nf * 8, cudaMemcpyHostToDevice));
    SB_CUDA(cudaMemcpy(c->on.tot, t.data() + (size_t)5 * c->nf, 8, cudaMemcpyHostToDevice));
    SB_CUDA(cudaMemset(c->on.mass_acc, 0, std::max<uint32_t>(c->M, 1) * 8));
    SB_CUDA(cudaMemset(c->on.fld_acc, 0, (size_t)c->nf * 8));
    const unsigned int mins[2] = {p.max_frag_len, p.max_frag_len};   // FragmentLengthDistribution::min_ starts at max_val
    SB_CUDA(cudaMemcpy(c->on.mins, mins, 8, cudaMemcpyHostToDevice));
    if (c->M) k_online_init<<<nblk(c->M, 256), 256>>>(c->M, ix->d_tx_off, c->on.mass, c->on.prior, c->on.log_eff);
    SB_CUDA(cudaGetLastError());
    SB_CUDA(cudaDeviceSynchronize());
    SB_CUDA(cudaMemset(c->pr.nmask, 0, 2 * CH * c->pr.mpr * 8));
    SB_CUDA(cudaMemset(b.ctr, 0, sizeof(Counters)));
    SB_CUDA(cudaMemset(c->d_full_dp, 0, 8));
    return SB_OK;
  }();
  if (rc != SB_OK) { sb_map_destroy(c); return nullptr; }
  const uint32_t n = p.max_frag_len + 1;
  c->fld.max_val = p.max_frag_len; c->fld.pmf_live = c->d_fld; c->fld.pmf_cached = c->d_fld + n;
  c->fld.cmf_cached = c->d_fld + 2 * n; c->fld.cmf_quirk = c->d_fld + 3 * n;
  return c;
}

extern "C" void sb_map_destroy(sb_map_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  sam_dev_destroy(c->samd);
  delete c;
}

extern "C" int sb_map_set_option(sb_map_ctx* c, const char* key, int64_t value) {
  if (!c || !key) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  if (!strcmp(key, "variant")) {
    if (value == 0 && c->p.recover_orphans) { sb::set_error("recover_orphans needs the warp kernels (variant 1)"); return SB_ERR_INVALID; }
    if (value == 0 && c->p.softclip) { sb::set_error("softclip modes 1 and 2 need the warp kernels (variant 1)"); return SB_ERR_INVALID; }
    c->variant = (int)value;
    return SB_OK;
  }
  if (!strcmp(key, "fast_dp")) { c->fast_ok = (value && fast_dp_exact(c->p)) ? 1 : 0; return SB_OK; }
  if (!strcmp(key, "input_on_device")) { c->input_dev = value ? 1 : 0; return SB_OK; }
  if (!strcmp(key, "ascii_reads")) {
    if (value && c->variant == 0) { sb::set_error("ascii_reads needs the warp kernels (variant 1)"); return SB_ERR_INVALID; }
    c->ascii = value ? 1 : 0;
    c->res.release(c->d_dummy_mate);   // its N codes depend on the encoding
    c->d_dummy_mate = nullptr;
    return SB_OK;
  }
  if (!strcmp(key, "no_projection")) { c->no_projection = value ? 1 : 0; return SB_OK; }
  if (!strcmp(key, "overlap_assign")) { c->overlap_assign = value ? 1 : 0; return SB_OK; }
  if (!strcmp(key, "sam_window_bytes")) {
    if (value < 1) { sb::set_error("sam_window_bytes must be positive"); return SB_ERR_INVALID; }
    c->sam_window = (uint64_t)value;
    return SB_OK;
  }
  if (!strcmp(key, "lib_type")) {   // the expected format of the batches that follow, inside the context's family
    if (value < 0 || value > 5 || (value >= 3) != (c->p.lib_type >= 3)) {
      sb::set_error("lib_type %lld does not fit this context (paired-end: 0..2, single-end: 3..5)", (long long)value);
      return SB_ERR_INVALID;
    }
    c->p.lib_type = (int32_t)value;
    return SB_OK;
  }
  if (!strcmp(key, "chunk")) {   // reads per pipeline chunk (<= the size the context was created with)
    const uint32_t mx = c->chunk_cap;
    if (value < 1 || value > (int64_t)mx) { sb::set_error("chunk must be in 1..%u", mx); return SB_ERR_INVALID; }
    c->chunk = (uint32_t)value;
    return SB_OK;
  }
  sb::set_error("sb_map_set_option: unknown key %s", key);
  return SB_ERR_INVALID;
}

// records -> classes (per batch over the read slots, and at finish over all batch classes); the table is appended to
// the arena
static int aggregate(sb_map_ctx* c, Records R, EqStore& out) {
  cudaStream_t st = c->stream;
  AggScratch& a = c->agg;
  Arena& ar = c->arena;
  out = EqStore();
  const uint32_t n = R.n;
  if (n == 0) return SB_OK;
  k_label_hash<<<nblk(n, 256), 256, 0, st>>>(R, a.hash, a.idx);
  size_t t = a.tmp_bytes;
  SB_CUDA(cub::DeviceRadixSort::SortPairs(a.tmp, t, a.hash, a.hash2, a.idx, a.idx2, (int)n, 0, 64, st));   // stable
  k_label_heads<<<nblk((uint64_t)n + 1, 256), 256, 0, st>>>(R, a.hash2, a.idx2, a.head);
  t = a.tmp_bytes;
  SB_CUDA(cub::DeviceScan::ExclusiveSum(a.tmp, t, a.head, a.head_scan, (int)n + 1, st));
  uint32_t nc = 0;
  SB_CUDA(cudaMemcpyAsync(&nc, a.head_scan + n, 4, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  SB_CUDA(cudaMemsetAsync(a.cls_llen + nc, 0, 8, st)); SB_CUDA(cudaMemsetAsync(a.cls_wlen + nc, 0, 8, st));
  k_class_sizes<<<nblk(n, 256), 256, 0, st>>>(R, a.head, a.head_scan, a.idx2, a.first, a.cls_llen, a.cls_wlen);
  out.base_o = ar.n_o; out.base_c = ar.n_c;
  {
    // R may be the arena's own tables (finish): growing moves them, so remember the offsets of its arrays
    const bool in_arena = R.labels && R.labels == ar.labels;
    const uint64_t ro_l = in_arena ? (uint64_t)(R.labels - ar.labels) : 0, ro_w = in_arena ? (uint64_t)(R.weights - ar.weights) : 0,
                   ro_c = (in_arena && R.counts) ? (uint64_t)(R.counts - ar.counts) : 0;
    SB_TRY(c->res.grow_keep(&ar.loff, ar.n_o, ar.n_o + nc + 1, st));
    SB_TRY(c->res.grow_keep(&ar.woff, ar.n_o, ar.n_o + nc + 1, st));
    SB_TRY(c->res.grow_keep(&ar.counts, ar.n_c, ar.n_c + nc, st));
    t = a.tmp_bytes;
    SB_CUDA(cub::DeviceScan::ExclusiveSum(a.tmp, t, a.cls_llen, ar.loff + out.base_o, (int)nc + 1, st));
    t = a.tmp_bytes;
    SB_CUDA(cub::DeviceScan::ExclusiveSum(a.tmp, t, a.cls_wlen, ar.woff + out.base_o, (int)nc + 1, st));
    uint64_t tl = 0, tw = 0;
    SB_CUDA(cudaMemcpyAsync(&tl, ar.loff + out.base_o + nc, 8, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaMemcpyAsync(&tw, ar.woff + out.base_o + nc, 8, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    out.base_l = ar.n_l; out.base_w = ar.n_w;
    SB_TRY(c->res.grow_keep(&ar.labels, ar.n_l, ar.n_l + tl, st));
    SB_TRY(c->res.grow_keep(&ar.weights, ar.n_w, ar.n_w + tw, st));
    if (in_arena) { R.labels = ar.labels + ro_l; R.weights = ar.weights + ro_w; if (R.counts) R.counts = ar.counts + ro_c; }
    k_class_reduce<<<nblk((uint64_t)nc * 32, 256), 256, 0, st>>>(R, nc, a.first, a.idx2, ar.loff + out.base_o,
                                                                ar.woff + out.base_o, ar.labels + out.base_l,
                                                                ar.weights + out.base_w, ar.counts + out.base_c);
    out.n = nc; out.n_lab = tl; out.n_w = tw;
    ar.n_o += (uint64_t)nc + 1; ar.n_c += nc; ar.n_l += tl; ar.n_w += tw;
  }
  c->launches += 10;
  return SB_OK;
}

// sam: the batch's side output for the attached SAM sink is filled (sb_map_batch_sam formats it afterwards)
static int map_batch(sb_map_ctx* c, const uint8_t* left, const uint8_t* right, uint32_t n, uint32_t L,
                     sb_map_batch_stats* stats, bool sam) {
  if (!c || (n && !left)) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  const bool single_end = c->p.lib_type >= 3;
  if (n && single_end != (right == nullptr)) {
    sb::set_error(single_end ? "single-end library type: sb_map_batch takes right == NULL" : "paired-end library type: both mates are needed");
    return SB_ERR_INVALID;
  }
  if (n > c->batch_cap || L > c->read_len_cap || L < c->p.k) { sb::set_error("batch larger than the context was created for"); return SB_ERR_INVALID; }
  SB_CUDA(cudaSetDevice(c->device));
  const double t_begin = wall_s();
  double t_agg = t_begin;
  cudaStream_t st = c->stream, cs = c->copy_stream;
  if (single_end) {
    // single-end reads (processReads SE, SalmonQuantify.cpp:1880-2325) travel through the paired kernels with an absent
    // second mate: a device buffer of N codes -- no k-mer, no seed, no candidate -- so every mapping is a left "orphan",
    // which is exactly how the auxiliary model treats a single-end read (getAmbigFragLengthProb, :642-650 / :2186-2200)
    if (!c->d_dummy_mate) {
      SB_TRY(c->res.alloc(&c->d_dummy_mate, (size_t)c->batch_cap * c->read_len_cap));
      SB_CUDA(cudaMemset(c->d_dummy_mate, c->ascii ? 'N' : 4, (size_t)c->batch_cap * c->read_len_cap));
    }
  }
  BatchBufs b = c->b;
  const Params& p = c->p;
  const uint32_t cap = p.max_read_occ;
  const IndexView ix = dev_view(c->index);
  const int useAux = c->frag_counter >= p.num_pre_burnin, burnedIn = c->burned_in;
  // forgetting masses of the batch's mini-batches, relative to the largest (the last); FLD kernel taps
  const uint64_t nsteps = ((uint64_t)n + p.mini_batch - 1) / p.mini_batch;
  const double fm_ref = forgetting_mass(c->fm, c->timestep + (nsteps ? nsteps - 1 : 0));
  {
    static const double kern_lin[5] = {1.0 / 16, 4.0 / 16, 6.0 / 16, 4.0 / 16, 1.0 / 16};   // binomial(4, 1/2)
    c->h_fm_rel.assign(std::max<uint64_t>(nsteps, 1), 0.0);
    c->h_tap_q.assign(std::max<uint64_t>(nsteps, 1) * 5, 0ull);
    for (uint64_t s2 = 0; s2 < nsteps; ++s2) {
      c->h_fm_rel[s2] = forgetting_mass(c->fm, c->timestep + s2) - fm_ref;
      for (int i = 0; i < 5; ++i)
        c->h_tap_q[s2 * 5 + i] = (unsigned long long)llrint(sbm_det_exp(c->h_fm_rel[s2] + sbm_det_log(kern_lin[i])) * MASS_SCALE);
    }
    SB_CUDA(cudaMemcpyAsync(c->on.fm_rel, c->h_fm_rel.data(), c->h_fm_rel.size() * 8, cudaMemcpyHostToDevice, st));
    SB_CUDA(cudaMemcpyAsync(c->on.tap_q, c->h_tap_q.data(), c->h_tap_q.size() * 8, cudaMemcpyHostToDevice, st));
    c->h_bm = p.max_frag_len;
    SB_CUDA(cudaMemcpyAsync(c->on.mins, &c->h_bm, 4, cudaMemcpyHostToDevice, st));
  }
  OnlineView onv;
  onv.mass = c->on.mass; onv.prior = c->on.prior; onv.log_eff = c->on.log_eff; onv.mass_acc = c->on.mass_acc;
  onv.fld_acc = c->on.fld_acc; onv.batch_min = c->on.mins; onv.fm_rel = c->on.fm_rel; onv.tap_q = c->on.tap_q;
  onv.mini_batch = p.mini_batch; onv.max_frag_len = p.max_frag_len; onv.frag_base = c->frags_seen; onv.seed = p.seed;
  SB_CUDA(cudaEventRecord(c->ev0, st));
  SB_CUDA(cudaMemsetAsync(c->b.ctr, 0, sizeof(Counters), st));
  SB_CUDA(cudaMemsetAsync(c->d_full_dp, 0, 8, st));
  if (c->rb.ctr) SB_CUDA(cudaMemsetAsync(c->rb.ctr, 0, 24, st));
  // chunks: the host->device copy of chunk i+1 (copy stream) overlaps the kernels of chunk i
  const uint32_t CH = c->chunk;
  const uint32_t nch = (n + CH - 1) / CH;
  SB_CUDA(cudaStreamWaitEvent(cs, c->ev0, 0));
  for (uint32_t ch = 0; ch < nch; ++ch) {
    const uint32_t c0 = ch * CH, cn = std::min(CH, n - c0);
    const int s = (int)(ch & 1);
    const uint8_t* dl = c->d_in[s][0];
    const uint8_t* dr = c->d_in[s][1];
    if (c->input_dev) {
      dl = left + (size_t)c0 * L; dr = single_end ? c->d_dummy_mate : right + (size_t)c0 * L;
    } else {
      if (ch >= 2) SB_CUDA(cudaStreamWaitEvent(cs, c->ev_free[s], 0));
      SB_CUDA(cudaMemcpyAsync(c->d_in[s][0], left + (size_t)c0 * L, (size_t)cn * L, cudaMemcpyHostToDevice, cs));
      if (!single_end) SB_CUDA(cudaMemcpyAsync(c->d_in[s][1], right + (size_t)c0 * L, (size_t)cn * L, cudaMemcpyHostToDevice, cs));
      SB_CUDA(cudaEventRecord(c->ev_in[s], cs));
      SB_CUDA(cudaStreamWaitEvent(st, c->ev_in[s], 0));
      if (single_end) dr = c->d_dummy_mate;
    }
    SB_CUDA(cudaMemsetAsync(c->b.n_tasks, 0, 16, st));
    SB_CUDA(cudaMemsetAsync(c->d_next_task, 0, 32, st));
    // outputs of this chunk inside the batch-wide arrays
    BatchBufs bc = c->b;
    const bool ovl = c->overlap_assign && c->variant != 0;
    const int set = (int)(ch & 1);
    if (ovl && set) {
      bc.n_l = c->alt_n_l; bc.n_r = c->alt_n_r; bc.cand_l = c->alt_cand_l; bc.cand_r = c->alt_cand_r;
      bc.score_l = c->alt_score_l; bc.score_r = c->alt_score_r;
    }
    if (ovl && ch >= 2) SB_CUDA(cudaStreamWaitEvent(st, c->ev_asg[set], 0));   // k_assign of chunk ch-2 still reads this set
    bc.n_aln += c0; bc.tid += (size_t)c0 * cap; bc.score += (size_t)c0 * cap; bc.prob += (size_t)c0 * cap;
    bc.pos += (size_t)c0 * cap; bc.mate_pos += (size_t)c0 * cap; bc.flags += (size_t)c0 * cap; bc.flen += (size_t)c0 * cap;
    bc.label += (size_t)c0 * 2 * cap; bc.weight += (size_t)c0 * cap;
    const uint32_t T = c->k1_threads;
    if (c->variant == 0) {
      k_seed_chain<<<T / 128, 128, 0, st>>>(ix, p, dl, dr, cn, L, bc);
      k_dp_score<<<c->n_sm * 8, 256, 0, st>>>(ix, p, dl, dr, L, bc);
      c->launches += 2;
    } else {
      k_pack_reads<<<nblk((uint64_t)2 * cn * c->pr.wpr, 256), 256, 0, st>>>(dl, dr, cn, L, c->pr, c->ascii);
      SeedOut so{bc.n_l, bc.n_r, bc.cand_l, bc.cand_r, bc.n_tasks, bc.tasks, c->d_overflow, bc.ctr};
      DpIo io{bc.n_tasks, bc.tasks, bc.cand_l, bc.cand_r, bc.score_l, bc.score_r, c->d_next_task, c->d_next_task + 4,
              c->d_list_int, c->d_list_edge, c->d_list_n, c->d_full_dp};
      const uint32_t npos = (L - p.k) / p.stride + 1 + (((L - p.k) % p.stride) ? 1u : 0u);   // seed positions per mate
      while (c->ev_seed.size() < 2 * (size_t)(ch + 1)) { cudaEvent_t e; SB_TRY(c->res.event(&e, cudaEventDefault)); c->ev_seed.push_back(e); }
      SB_CUDA(cudaEventRecord(c->ev_seed[2 * ch], st));
      if (c->read_len_cap <= 128) {
        if (npos <= 32) k_seed_chain_w<2, 1><<<c->seed_blocks, SeedCfg<2>::WARPS * 32, 0, st>>>(ix, p, c->pr, cn, L, so);
        else k_seed_chain_w<2, 2><<<c->seed_blocks, SeedCfg<2>::WARPS * 32, 0, st>>>(ix, p, c->pr, cn, L, so);
        SB_CUDA(cudaEventRecord(c->ev_seed[2 * ch + 1], st));
        switch (p.softclip) {
          case 0: launch_dp<4, 0>(c, st, ix, p, L, dl, dr, io); break;
          case 1: launch_dp<4, 1>(c, st, ix, p, L, dl, dr, io); break;
          default: launch_dp<4, 2>(c, st, ix, p, L, dl, dr, io); break;
        }
      } else {
        if (npos <= 32) k_seed_chain_w<4, 1><<<c->seed_blocks, SeedCfg<4>::WARPS * 32, 0, st>>>(ix, p, c->pr, cn, L, so);
        else k_seed_chain_w<4, 2><<<c->seed_blocks, SeedCfg<4>::WARPS * 32, 0, st>>>(ix, p, c->pr, cn, L, so);
        SB_CUDA(cudaEventRecord(c->ev_seed[2 * ch + 1], st));
        switch (p.softclip) {
          case 0: launch_dp<8, 0>(c, st, ix, p, L, dl, dr, io); break;
          case 1: launch_dp<8, 1>(c, st, ix, p, L, dl, dr, io); break;
          default: launch_dp<8, 2>(c, st, ix, p, L, dl, dr, io); break;
        }
      }
      c->launches += 5;
    }
    // orphan rescue: after the DP scores, before k_assign (and before the input buffers are handed back)
    const bool resc = p.recover_orphans && !single_end;
    RescueBufs rb = c->rb;
    if (resc) {
      if (ovl && set) { rb.pairs = c->alt_rs_pairs; rb.n_pairs = c->alt_rs_n_pairs; }
      while (c->ev_rescue.size() < 2 * (size_t)(ch + 1)) { cudaEvent_t e; SB_TRY(c->res.event(&e, cudaEventDefault)); c->ev_rescue.push_back(e); }
      SB_CUDA(cudaEventRecord(c->ev_rescue[2 * ch], st));
      SB_CUDA(cudaMemsetAsync(rb.n_tasks, 0, 4, st));
      k_rescue_select<<<nblk(cn, 128), 128, 0, st>>>(p, cn, L, bc.n_l, bc.n_r, bc.cand_l, bc.cand_r, bc.score_l, bc.score_r, rb);
      const unsigned sb = c->n_sm * 8;
      switch ((L + 63) / 64) {
        case 1: k_rescue_search<1><<<sb, 128, 0, st>>>(ix, p, c->pr, L, bc.cand_l, bc.cand_r, rb); break;
        case 2: k_rescue_search<2><<<sb, 128, 0, st>>>(ix, p, c->pr, L, bc.cand_l, bc.cand_r, rb); break;
        case 3: k_rescue_search<3><<<sb, 128, 0, st>>>(ix, p, c->pr, L, bc.cand_l, bc.cand_r, rb); break;
        default: k_rescue_search<4><<<sb, 128, 0, st>>>(ix, p, c->pr, L, bc.cand_l, bc.cand_r, rb); break;
      }
      switch (p.softclip) {
        case 0: k_rescue_score<0><<<c->n_sm * 4, 256, 0, st>>>(ix, p, dl, dr, L, c->ascii, bc.cand_l, bc.cand_r, rb); break;
        case 1: k_rescue_score<1><<<c->n_sm * 4, 256, 0, st>>>(ix, p, dl, dr, L, c->ascii, bc.cand_l, bc.cand_r, rb); break;
        default: k_rescue_score<2><<<c->n_sm * 4, 256, 0, st>>>(ix, p, dl, dr, L, c->ascii, bc.cand_l, bc.cand_r, rb); break;
      }
      k_rescue_commit<<<nblk(cn, 128), 128, 0, st>>>(p, cn, L, bc.n_l, bc.n_r, bc.cand_l, bc.cand_r, bc.score_l, bc.score_r, rb);
      SB_CUDA(cudaEventRecord(c->ev_rescue[2 * ch + 1], st));
      c->launches += 4;
    }
    cudaStream_t as = st;
    if (ovl) {   // the input staging buffers are free once the DP kernels are done; k_assign moves to its own stream
      SB_CUDA(cudaEventRecord(c->ev_free[s], st));
      SB_CUDA(cudaEventRecord(c->ev_dp[set], st));
      as = c->assign_stream;
      SB_CUDA(cudaStreamWaitEvent(as, c->ev_dp[set], 0));
    }
    {
      k_assign_work<<<nblk(cn, 256), 256, 0, as>>>(cn, bc.n_l, bc.n_r, c->d_work, c->d_ids);
      size_t tb = c->agg.tmp_bytes;
      SB_CUDA(cub::DeviceRadixSort::SortPairs(c->agg.tmp, tb, c->d_work, c->d_work2, c->d_ids, c->d_order, (int)cn, 0, 8, as));
    }
    if (sam) {
      SamSide sd = sam_dev_side(c->samd);
      sd.n_out += c0; sd.decoy += c0; sd.score1 += (size_t)c0 * cap; sd.score2 += (size_t)c0 * cap;
      if (resc) k_assign<true, true><<<T / 128, 128, 0, as>>>(ix, p, c->fld, useAux, burnedIn, cn, L, bc, onv, c0, c->d_order, sd, rb);
      else k_assign<true, false><<<T / 128, 128, 0, as>>>(ix, p, c->fld, useAux, burnedIn, cn, L, bc, onv, c0, c->d_order, sd, rb);
    } else {
      if (resc) k_assign<false, true><<<T / 128, 128, 0, as>>>(ix, p, c->fld, useAux, burnedIn, cn, L, bc, onv, c0, c->d_order, SamSide{}, rb);
      else k_assign<false, false><<<T / 128, 128, 0, as>>>(ix, p, c->fld, useAux, burnedIn, cn, L, bc, onv, c0, c->d_order, SamSide{}, rb);
    }
    c->launches += 3;
    if (ovl) SB_CUDA(cudaEventRecord(c->ev_asg[set], as));
    else SB_CUDA(cudaEventRecord(c->ev_free[s], st));
  }
  if (c->overlap_assign && c->variant != 0)   // the batch-level kernels below read what the last k_assign launches wrote
    for (int set = 0; set < 2 && (uint32_t)set < nch; ++set) SB_CUDA(cudaStreamWaitEvent(st, c->ev_asg[set], 0));
  // fold the batch into the online state (masses, FLD)
  if (n) {
    if (c->M) k_online_fold_mass<<<nblk(c->M, 256), 256, 0, st>>>(c->M, fm_ref, c->on.mass, c->on.mass_acc);
    k_online_fold_fld<<<1, 1024, 0, st>>>(c->nf, fm_ref, c->on, c->d_fld);
    c->launches += 2;
  }
  // eq-class records of this batch: the per-read slots themselves (no compaction)
  EqStore es;
  if (n) {
    AggScratch& a = c->agg;
    const int binned = p.range_bins > 0;
    k_read_records<<<nblk(n, 256), 256, 0, st>>>(n, cap, binned, b.n_aln, a.lstart, a.llen, a.wstart, a.wlen);
    c->launches += 1;
    // reads without alignments have empty labels: they all hash alike and form one "empty"
    // class; aggregate() keeps it and finish() drops it.
    Records R{n, a.lstart, a.llen, a.wstart, a.wlen, b.label, b.weight, nullptr};
    t_agg = wall_s();
    SB_TRY(aggregate(c, R, es));
    c->stores.push_back(es);
  }
  Counters h;
  unsigned long long full_dp = 0;
  SB_CUDA(cudaMemcpyAsync(&h, b.ctr, sizeof(Counters), cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(&full_dp, c->d_full_dp, 8, cudaMemcpyDeviceToHost, st));
  unsigned long long rctr[3] = {0, 0, 0};
  if (c->rb.ctr) SB_CUDA(cudaMemcpyAsync(rctr, c->rb.ctr, 24, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaEventRecord(c->ev1, st));
  const double t_enq = wall_s();
  SB_CUDA(cudaEventSynchronize(c->ev1));
  cudaEventElapsedTime(&c->last_ms, c->ev0, c->ev1);
  if (c->profile) {
    const double t_end = wall_s();
    fprintf(stderr, "sb_map_batch: n %u host enqueue %.2f ms (aggregate %.2f ms), final wait %.2f ms, device %.2f ms\n", n,
            (t_enq - t_begin) * 1e3, (t_enq - t_agg) * 1e3, (t_end - t_enq) * 1e3, c->last_ms);
  }
  c->frag_counter += h.mapped;
  c->frags_seen += n;
  c->last_chunks = nch;
  c->last_rescue = p.recover_orphans && !single_end;
  c->timestep += nsteps;
  c->full_dp_total += full_dp;
  c->rescued_total += rctr[0]; c->rescue_searches_total += rctr[1]; c->rescue_no_room_total += rctr[2];
  if (!c->burned_in && c->frag_counter >= p.num_burnin) {   // SalmonQuantify.cpp:1013-1018
    k_online_correction<<<1, 32, 0, st>>>(c->nf, c->on, 1, c->d_scratch_nf, c->d_fld + c->nf, c->d_fld + 2 * (size_t)c->nf);
    if (c->M) k_online_eff_len<<<nblk(c->M, 256), 256, 0, st>>>(c->M, c->nf, c->index->d_tx_off, c->on.cf, c->on.log_eff);
    SB_CUDA(cudaStreamSynchronize(st));
    c->burned_in = 1;
    c->launches += 2;
  }
  c->totals.lookups += h.lookups; c->totals.postings += h.postings; c->totals.seeds += h.seeds;
  c->totals.candidates += h.candidates; c->totals.kept += h.kept; c->totals.label_entries += h.label_entries;
  c->totals.mapped += h.mapped;
  for (int i = 0; i < 4; ++i) c->totals.lib_mask_sum[i] += h.lib_mask_sum[i];
  c->totals.compatible += h.compatible;
  if (stats) {
    stats->n_pairs = n; stats->mapped = h.mapped; stats->lookups = h.lookups; stats->postings = h.postings;
    stats->seeds = h.seeds; stats->candidates = h.candidates; stats->kept = h.kept; stats->label_entries = h.label_entries;
    stats->device_ms = c->last_ms; stats->gpu_launches = c->launches;
    stats->n_batch_classes = es.n;
    stats->full_dp = full_dp;
    stats->seed_kernel_ms = 0; stats->seed_kernel_launches = 0;
    if (c->variant != 0)
      for (uint32_t ch = 0; ch < nch; ++ch) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, c->ev_seed[2 * ch], c->ev_seed[2 * ch + 1]) == cudaSuccess) {
          stats->seed_kernel_ms += ms; stats->seed_kernel_launches++;
        }
      }
    stats->orphans_rescued = rctr[0]; stats->rescue_searches = rctr[1]; stats->rescue_no_room = rctr[2];
    stats->compatible = h.compatible;
    stats->rescue_kernel_ms = 0;
    if (c->p.recover_orphans && !single_end)
      for (uint32_t ch = 0; ch < nch; ++ch) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, c->ev_rescue[2 * ch], c->ev_rescue[2 * ch + 1]) == cudaSuccess) stats->rescue_kernel_ms += ms;
      }
  }
  return SB_OK;
}

extern "C" int sb_map_batch(sb_map_ctx* c, const uint8_t* left, const uint8_t* right, uint32_t n, uint32_t L,
                            sb_map_batch_stats* stats) {
  return map_batch(c, left, right, n, L, stats, false);
}

extern "C" int sb_map_attach_sam(sb_map_ctx* c, sb_sam* sam) {
  if (!c) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  SB_CUDA(cudaSetDevice(c->device));
  SB_CUDA(cudaDeviceSynchronize());
  sam_dev_destroy(c->samd);
  c->samd = nullptr;
  c->sam = nullptr;
  if (!sam) return SB_OK;
  SamDev* d = nullptr;
  const int rc = sam_dev_create(&d, sam, c->batch_cap, c->read_len_cap, c->p.max_read_occ);
  if (rc != SB_OK) { sam_dev_destroy(d); return rc; }
  c->samd = d;
  c->sam = sam;
  return SB_OK;
}

extern "C" int sb_map_batch_sam(sb_map_ctx* c, const uint8_t* left, const uint8_t* right, uint32_t n, uint32_t L,
                                const char* names, const uint64_t* name_off, const uint8_t* qual_left,
                                const uint8_t* qual_right, sb_map_batch_stats* stats) {
  if (!c || !c->sam) { sb::set_error("sb_map_batch_sam: no SAM sink attached (sb_map_attach_sam)"); return SB_ERR_STATE; }
  if (n && (!names || !name_off)) { sb::set_error("sb_map_batch_sam: the reads' names are needed"); return SB_ERR_INVALID; }
  SB_TRY(map_batch(c, left, right, n, L, stats, true));
  SamBatch sb;
  sb.n = n; sb.L = L; sb.cap = c->p.max_read_occ; sb.paired = c->p.lib_type < 3 ? 1 : 0; sb.ascii = c->ascii;
  sb.tid = c->b.tid; sb.pos = c->b.pos; sb.mate_pos = c->b.mate_pos; sb.flags = c->b.flags; sb.flen = c->b.flen;
  float ms = 0;
  return sam_dev_format(c->samd, c->stream, sb, left, right, names, name_off, qual_left, qual_right, c->sam_window, &ms);
}

extern "C" int sb_map_lib_counts(const sb_map_ctx* c, uint64_t out4[4]) {
  if (!c || !out4) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  for (int i = 0; i < 4; ++i) out4[i] = c->totals.lib_mask_sum[i];
  return SB_OK;
}

// LibraryTypeDetector::mostLikelyType (LibraryTypeDetector.hpp:34-140) for the formats this library maps (inward
// pairs, unmated reads): the fraction of sense-strand fragments decides
extern "C" int sb_detect_lib_type(int paired, const uint64_t counts4[4]) {
  if (!counts4) return -1;
  const uint64_t nf = paired ? counts4[0] : counts4[2], nr = paired ? counts4[1] : counts4[3];
  if (nf + nr == 0) return -1;
  const double ratio = (double)nf / (double)(nf + nr);
  if (ratio < 0.3) return paired ? SB_LIB_ISR : SB_LIB_SR;
  if (ratio < 0.7) return paired ? SB_LIB_IU : SB_LIB_U;
  return paired ? SB_LIB_ISF : SB_LIB_SF;
}

// parity tap of the rescue search: the windows are laid out as the index lays out its reference (2-bit packed behind a
// guard, byte codes for windows with N) and searched by the device function k_rescue_search runs
extern "C" int sb_rescue_search_tap(int device, uint32_t n, const uint8_t* pats, const uint64_t* pat_off,
                                    const uint8_t* wins, const uint64_t* win_off, const int32_t* K, int32_t* dist,
                                    int32_t* end) {
  if (n && (!pats || !pat_off || !wins || !win_off || !K || !dist || !end)) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  for (uint32_t i = 0; i < n; ++i)
    if (pat_off[i + 1] < pat_off[i] || pat_off[i + 1] - pat_off[i] > 64 * RESCUE_MAX_WORDS || win_off[i + 1] < win_off[i]) {
      sb::set_error("sb_rescue_search_tap: case %u: patterns of 0..%u bases", i, 64 * RESCUE_MAX_WORDS);
      return SB_ERR_INVALID;
    }
  if (!n) return SB_OK;
  SB_CUDA(cudaSetDevice(device));
  const uint64_t np = pat_off[n], nw = win_off[n];
  std::vector<uint64_t> packed((nw + 2 * (uint64_t)PACK_GUARD_BASES + 31) / 32 + 2, 0);
  std::vector<uint8_t> has_n(n, 0);
  for (uint32_t i = 0; i < n; ++i)
    for (uint64_t g = win_off[i]; g < win_off[i + 1]; ++g) {
      if (wins[g] > 3) { has_n[i] = 1; continue; }
      const uint64_t q = g + PACK_GUARD_BASES;
      packed[q >> 5] |= (uint64_t)wins[g] << (2 * (q & 31));
    }
  uint8_t *d_p = nullptr, *d_w = nullptr, *d_hn = nullptr;
  uint64_t *d_po = nullptr, *d_wo = nullptr, *d_pk = nullptr;
  int32_t *d_k = nullptr, *d_d = nullptr, *d_e = nullptr;
  sb::Resources res;   // on the current device
  int rc = SB_OK;
  auto A = [&](auto** ptr, size_t m) { if (rc == SB_OK) rc = res.alloc(ptr, m); };
  A(&d_p, np); A(&d_w, nw); A(&d_hn, n); A(&d_po, n + 1); A(&d_wo, n + 1); A(&d_pk, packed.size()); A(&d_k, n);
  A(&d_d, n); A(&d_e, n);
  cudaError_t e = cudaSuccess;
  if (rc == SB_OK) {
    cudaMemcpy(d_p, pats, np, cudaMemcpyHostToDevice); cudaMemcpy(d_w, wins, nw, cudaMemcpyHostToDevice);
    cudaMemcpy(d_hn, has_n.data(), n, cudaMemcpyHostToDevice); cudaMemcpy(d_po, pat_off, (n + 1) * 8, cudaMemcpyHostToDevice);
    cudaMemcpy(d_wo, win_off, (n + 1) * 8, cudaMemcpyHostToDevice);
    cudaMemcpy(d_pk, packed.data(), packed.size() * 8, cudaMemcpyHostToDevice);
    cudaMemcpy(d_k, K, (size_t)n * 4, cudaMemcpyHostToDevice);
    cudaMemset(d_d, 0xff, (size_t)n * 4); cudaMemset(d_e, 0xff, (size_t)n * 4);
    // one launch per word count: each case runs in the instance k_rescue_search uses for its pattern length
    k_rescue_tap<1><<<nblk(n, 128), 128>>>(n, d_p, d_po, d_pk, d_w, d_wo, d_hn, d_k, d_d, d_e);
    k_rescue_tap<2><<<nblk(n, 128), 128>>>(n, d_p, d_po, d_pk, d_w, d_wo, d_hn, d_k, d_d, d_e);
    k_rescue_tap<3><<<nblk(n, 128), 128>>>(n, d_p, d_po, d_pk, d_w, d_wo, d_hn, d_k, d_d, d_e);
    k_rescue_tap<4><<<nblk(n, 128), 128>>>(n, d_p, d_po, d_pk, d_w, d_wo, d_hn, d_k, d_d, d_e);
    e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(dist, d_d, (size_t)n * 4, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(end, d_e, (size_t)n * 4, cudaMemcpyDeviceToHost);
  }
  if (rc != SB_OK) return rc;
  if (e != cudaSuccess) { sb::set_error("sb_rescue_search_tap: %s", cudaGetErrorString(e)); return SB_ERR_CUDA; }
  return SB_OK;
}

// debug / parity tap: per-read alignments of the LAST batch (arrays sized n*cap, label n*2*cap)
extern "C" int sb_map_last_alignments(sb_map_ctx* c, uint32_t n, uint32_t* n_aln, uint32_t* tid, int32_t* score,
                                      double* prob, int32_t* pos, int32_t* mate_pos, uint8_t* flags, int32_t* flen,
                                      uint32_t* label, double* weight) {
  if (!c) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  SB_CUDA(cudaSetDevice(c->device));
  const size_t cap = c->p.max_read_occ;
  BatchBufs& b = c->b;
  if (n_aln) SB_CUDA(cudaMemcpy(n_aln, b.n_aln, (size_t)n * 4, cudaMemcpyDeviceToHost));
  if (tid) SB_CUDA(cudaMemcpy(tid, b.tid, n * cap * 4, cudaMemcpyDeviceToHost));
  if (score) SB_CUDA(cudaMemcpy(score, b.score, n * cap * 4, cudaMemcpyDeviceToHost));
  if (prob) SB_CUDA(cudaMemcpy(prob, b.prob, n * cap * 8, cudaMemcpyDeviceToHost));
  if (pos) SB_CUDA(cudaMemcpy(pos, b.pos, n * cap * 4, cudaMemcpyDeviceToHost));
  if (mate_pos) SB_CUDA(cudaMemcpy(mate_pos, b.mate_pos, n * cap * 4, cudaMemcpyDeviceToHost));
  if (flags) SB_CUDA(cudaMemcpy(flags, b.flags, n * cap, cudaMemcpyDeviceToHost));
  if (flen) SB_CUDA(cudaMemcpy(flen, b.flen, n * cap * 4, cudaMemcpyDeviceToHost));
  if (label) SB_CUDA(cudaMemcpy(label, b.label, n * 2 * cap * 4, cudaMemcpyDeviceToHost));
  if (weight) SB_CUDA(cudaMemcpy(weight, b.weight, n * cap * 8, cudaMemcpyDeviceToHost));
  return SB_OK;
}

// parity tap: per-read candidates of the LAST batch as the seed kernel left them (n_l / n_r [n], cand_l / cand_r
// [n * MAXCAND]; bit 31 of n_l marks a read the seed kernel found unmapped).  The candidate buffers hold one chunk (and
// alternate between two sets from chunk to chunk), and orphan rescue appends to them: such batches are refused.
extern "C" int sb_map_last_candidates(sb_map_ctx* c, uint32_t n, uint32_t* n_l, uint32_t* n_r, void* cand_l,
                                      void* cand_r) {
  if (!c) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  if (c->last_chunks > 1 || c->last_rescue) {
    sb::set_error("sb_map_last_candidates: the last batch ran as %u chunks%s; candidates are kept for one chunk without "
                  "orphan rescue", c->last_chunks, c->last_rescue ? " with orphan rescue" : "");
    return SB_ERR_STATE;
  }
  if (n > c->chunk_cap) { sb::set_error("sb_map_last_candidates: %u reads, the buffers hold %u", n, c->chunk_cap); return SB_ERR_INVALID; }
  SB_CUDA(cudaSetDevice(c->device));
  const BatchBufs& b = c->b;
  if (n_l) SB_CUDA(cudaMemcpy(n_l, b.n_l, (size_t)n * 4, cudaMemcpyDeviceToHost));
  if (n_r) SB_CUDA(cudaMemcpy(n_r, b.n_r, (size_t)n * 4, cudaMemcpyDeviceToHost));
  if (cand_l) SB_CUDA(cudaMemcpy(cand_l, b.cand_l, (size_t)n * MAXCAND * sizeof(Cand), cudaMemcpyDeviceToHost));
  if (cand_r) SB_CUDA(cudaMemcpy(cand_r, b.cand_r, (size_t)n * MAXCAND * sizeof(Cand), cudaMemcpyDeviceToHost));
  return SB_OK;
}

// per-transcript counts and the transcript clusters of this context's classes (device arrays in c->fin)
static int finish_stats(sb_map_ctx* c, uint64_t n_cls, const uint64_t* loff, const uint64_t* woff, const uint32_t* labels,
                        const uint64_t* counts) {
  cudaStream_t st = c->stream;
  const uint32_t M = c->M;
  if (!M) return SB_OK;
  FinBufs& f = c->fin;
  SB_CUDA(cudaMemsetAsync(f.uniq, 0, (size_t)M * 8, st)); SB_CUDA(cudaMemsetAsync(f.total, 0, (size_t)M * 8, st));
  SB_CUDA(cudaMemsetAsync(f.hits, 0, (size_t)M * 8, st));
  k_iota<<<nblk(M, 256), 256, 0, st>>>(M, f.parent);
  if (n_cls)
    k_cls_accumulate<<<nblk(n_cls, 256), 256, 0, st>>>(n_cls, loff, woff, labels, counts, f.uniq, f.total, f.hits, f.parent);
  k_roots<<<nblk(M, 256), 256, 0, st>>>(M, f.parent, f.root, f.ids);
  c->launches += 3;
  return SB_OK;
}
// clusters from f.root, projection with c->on.mass and f.{hits,uniq,total}; results to the host vectors
static int finish_project(sb_map_ctx* c) {
  cudaStream_t st = c->stream;
  const uint32_t M = c->M;
  c->h_proj.assign(M, 0.0); c->h_eff.assign(M, 0.0); c->h_uniq.assign(M, 0); c->h_total.assign(M, 0);
  if (!M) return SB_OK;
  FinBufs& f = c->fin;
  if (!c->no_projection) {
    size_t t2 = f.tmp_bytes;
    SB_CUDA(cub::DeviceRadixSort::SortPairs(f.tmp, t2, f.root, f.root2, f.ids, f.memb, (int)M, 0, 32, st));   // stable: members ascending
    k_cluster_heads<<<nblk((uint64_t)M + 1, 256), 256, 0, st>>>(M, f.root2, f.head);
    t2 = f.tmp_bytes;
    SB_CUDA(cub::DeviceScan::ExclusiveSum(f.tmp, t2, f.head, f.head_scan, (int)M + 1, st));
    uint32_t ncl = 0;
    SB_CUDA(cudaMemcpyAsync(&ncl, f.head_scan + M, 4, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    k_cluster_starts<<<nblk(M, 256), 256, 0, st>>>(M, f.head, f.head_scan, f.start);
    k_cluster_project<<<nblk((uint64_t)ncl * 32, 256), 256, 0, st>>>(ncl, M, f.start, f.memb, c->on.mass, f.hits, f.uniq,
                                                                     f.total, f.proj, f.bound);
    c->launches += 6;
  }
  if (c->p.no_eff_len_correction)   // --noEffectiveLengthCorrection: transcript lengths (CollapsedEMOptimizer.cpp:611-613,786-788)
    k_tx_len<<<nblk(M, 256), 256, 0, st>>>(M, c->index->d_tx_off, f.eff);
  else
    k_exp_vec<<<nblk(M, 256), 256, 0, st>>>(M, c->on.log_eff, f.eff);     // CollapsedEMOptimizer.cpp:782-784
  c->launches += 1;
  if (!c->no_projection) SB_CUDA(cudaMemcpyAsync(c->h_proj.data(), f.proj, (size_t)M * 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(c->h_eff.data(), f.eff, (size_t)M * 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(c->h_uniq.data(), f.uniq, (size_t)M * 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(c->h_total.data(), f.total, (size_t)M * 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return SB_OK;
}

// finish(): merge the per-batch class tables, normalise weights (EquivalenceClassBuilder.hpp:165-181,
// TGValue::normalizeAux :114-123), hand back a host CSR (sb_eq_csr-compatible).
extern "C" int sb_map_finish(sb_map_ctx* c, sb_map_result* out) {
  if (!c || !out) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  SB_CUDA(cudaSetDevice(c->device));
  cudaStream_t st = c->stream;
  // the class tables of all batches, concatenated, become the records of one more aggregation
  uint64_t n = 0, nl = 0, nw = 0;
  for (auto& s : c->stores) { n += s.n; nl += s.n_lab; nw += s.n_w; }
  if (n >= (1ull << 31)) { sb::set_error("sb_map_finish: too many batch classes"); return SB_ERR_INVALID; }
  EqStore merged;
  Arena& ar = c->arena;
  const uint64_t mark_l = ar.n_l, mark_w = ar.n_w, mark_c = ar.n_c, mark_o = ar.n_o;   // the merged table is temporary
  if (n) {
    SB_TRY(agg_reserve(c, n));
    AggScratch& a = c->agg;
    uint64_t i = 0;
    for (auto& s : c->stores) {   // the batch tables are the records: label / weight starts are arena positions
      if (!s.n) continue;
      k_store_records<<<nblk(s.n, 256), 256, 0, st>>>(s.n, ar.loff + s.base_o, ar.woff + s.base_o, s.base_l, s.base_w,
                                                      a.lstart + i, a.llen + i, a.wstart + i, a.wlen + i);
      i += s.n;
    }
    // counts of the batch tables are contiguous in the arena in store order (every store appends)
    Records R{(uint32_t)n, a.lstart, a.llen, a.wstart, a.wlen, ar.labels, ar.weights, ar.counts + c->stores.front().base_c};
    SB_TRY(aggregate(c, R, merged));
  }
  const uint64_t* m_loff = ar.loff + merged.base_o; const uint64_t* m_woff = ar.woff + merged.base_o;
  const uint32_t* m_labels = ar.labels + merged.base_l; double* m_weights = ar.weights + merged.base_w;
  const uint64_t* m_counts = ar.counts + merged.base_c;
  if (merged.n) {
    k_normalize<<<nblk(merged.n, 128), 128, 0, st>>>(merged.n, m_woff, m_weights);
    c->launches++;
  }
  // ---- normalizeAlphas (SalmonUtils.cpp:461-529): initial alphas for the optimiser, plus what optimize() reads
  //      per transcript (effective length, unique count)
  if (!c->burned_in) {   // burn-in never reached: effective lengths from the observed FLD (SalmonQuantify.cpp:2734-2738)
    k_online_correction<<<1, 32, 0, st>>>(c->nf, c->on, 0, c->d_scratch_nf, nullptr, nullptr);
    if (c->M) k_online_eff_len<<<nblk(c->M, 256), 256, 0, st>>>(c->M, c->nf, c->index->d_tx_off, c->on.cf, c->on.log_eff);
    c->launches += 2;
  }
  SB_TRY(finish_stats(c, merged.n, m_loff, m_woff, m_labels, m_counts));
  SB_TRY(finish_project(c));
  // to host (data movement only): drop the empty-label class, split label into tids | bins
  const int binned = c->p.range_bins > 0;
  std::vector<uint64_t> loff(merged.n + 1), woff(merged.n + 1), counts(merged.n);
  std::vector<uint32_t> labels(merged.n_lab);
  std::vector<double> weights(merged.n_w);
  if (merged.n) {
    SB_CUDA(cudaMemcpyAsync(loff.data(), m_loff, (merged.n + 1) * 8, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaMemcpyAsync(woff.data(), m_woff, (merged.n + 1) * 8, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaMemcpyAsync(counts.data(), m_counts, merged.n * 8, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaMemcpyAsync(labels.data(), m_labels, merged.n_lab * 4, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaMemcpyAsync(weights.data(), m_weights, merged.n_w * 8, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
  }
  c->h_off.assign(1, 0); c->h_counts.clear(); c->h_tids.clear(); c->h_ntx.clear(); c->h_bins.clear(); c->h_w.clear();
  c->h_tids.reserve(merged.n_w); c->h_w.reserve(merged.n_w); c->h_counts.reserve(merged.n); c->h_off.reserve(merged.n + 1);
  for (uint64_t q = 0; q < merged.n; ++q) {
    const uint64_t ntx = woff[q + 1] - woff[q];
    if (ntx == 0) continue;
    for (uint64_t a = 0; a < ntx; ++a) {
      c->h_tids.push_back(labels[loff[q] + a]);
      c->h_w.push_back(weights[woff[q] + a]);
      if (binned) c->h_bins.push_back(labels[loff[q] + ntx + a]);
    }
    c->h_off.push_back(c->h_tids.size());
    c->h_counts.push_back(counts[q]);
    c->h_ntx.push_back((uint32_t)ntx);
  }
  ar.n_l = mark_l; ar.n_w = mark_w; ar.n_c = mark_c; ar.n_o = mark_o;     // drop the merged table, keep the batch tables
  out->n_classes = c->h_counts.size();
  out->off = c->h_off.data(); out->tids = c->h_tids.data(); out->weights = c->h_w.data();
  out->counts = c->h_counts.data(); out->bins = binned ? c->h_bins.data() : nullptr;
  out->n_mapped = c->totals.mapped;
  memset(out->lib_format_counts, 0, sizeof(out->lib_format_counts));
  for (int i = 0; i < 4; ++i) out->lib_format_counts[i] = c->totals.lib_mask_sum[i];
  out->orphans_rescued = c->rescued_total; out->rescue_searches = c->rescue_searches_total;
  out->rescue_no_room = c->rescue_no_room_total;
  out->n_compatible = c->totals.compatible;
  out->lookups = c->totals.lookups; out->postings = c->totals.postings; out->seeds = c->totals.seeds;
  out->candidates = c->totals.candidates; out->kept = c->totals.kept; out->label_entries = c->totals.label_entries;
  out->n_txps = c->M;
  out->projected_counts = c->h_proj.data(); out->eff_len = c->h_eff.data();
  out->unique_counts = c->h_uniq.data(); out->total_counts = c->h_total.data();
  return SB_OK;
}

// ---- multi-GPU (SURVEY.md 8e): reads are sharded over ranks, every rank keeps its own class table; what
// normalizeAlphas needs globally -- transcript masses, the FLD, unique / total / cluster-hit counts and the
// transcript clusters -- is reduced over the ranks ONCE at the end of mapping by the host layer (M-sized vectors).
__global__ void k_union_roots(uint32_t M, const uint32_t* __restrict__ root, uint32_t* parent) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= M) return;
  uint32_t a = t, b = root[t];
  for (;;) {
    a = uf_find(parent, a); b = uf_find(parent, b);
    if (a == b) break;
    if (a < b) { const uint32_t x = a; a = b; b = x; }
    if (atomicCAS(parent + a, a, b) == a) break;
  }
}

// this rank's statistics after sb_map_finish (host arrays owned by the context)
extern "C" int sb_map_partial_get(sb_map_ctx* c, sb_map_partial* out) {
  if (!c || !out) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  SB_CUDA(cudaSetDevice(c->device));
  const uint32_t M = c->M, nf = c->nf;
  c->hp_mass.assign(M, 0.0); c->hp_hist.assign((size_t)nf + 1, 0.0); c->hp_uniq.assign(M, 0); c->hp_total.assign(M, 0);
  c->hp_hits.assign(M, 0); c->hp_root.assign(M, 0);
  unsigned int mins[2] = {0, 0};
  if (M) {
    SB_CUDA(cudaMemcpy(c->hp_mass.data(), c->on.mass, (size_t)M * 8, cudaMemcpyDeviceToHost));
    SB_CUDA(cudaMemcpy(c->hp_uniq.data(), c->fin.uniq, (size_t)M * 8, cudaMemcpyDeviceToHost));
    SB_CUDA(cudaMemcpy(c->hp_total.data(), c->fin.total, (size_t)M * 8, cudaMemcpyDeviceToHost));
    SB_CUDA(cudaMemcpy(c->hp_hits.data(), c->fin.hits, (size_t)M * 8, cudaMemcpyDeviceToHost));
    SB_CUDA(cudaMemcpy(c->hp_root.data(), c->fin.root, (size_t)M * 4, cudaMemcpyDeviceToHost));
  }
  SB_CUDA(cudaMemcpy(c->hp_hist.data(), c->on.hist, (size_t)nf * 8, cudaMemcpyDeviceToHost));
  SB_CUDA(cudaMemcpy(c->hp_hist.data() + nf, c->on.tot, 8, cudaMemcpyDeviceToHost));
  SB_CUDA(cudaMemcpy(mins, c->on.mins, 8, cudaMemcpyDeviceToHost));
  out->n_txps = M; out->n_fld = nf; out->mass = c->hp_mass.data(); out->fld_hist = c->hp_hist.data();
  out->fld_tot = c->hp_hist[nf]; out->fld_prior_hist = c->init_tables.data() + (size_t)4 * nf;
  out->fld_prior_tot = c->init_tables[(size_t)5 * nf]; out->fld_min = mins[1];
  out->unique_counts = c->hp_uniq.data(); out->total_counts = c->hp_total.data(); out->cluster_hits = c->hp_hits.data();
  out->cluster_root = c->hp_root.data(); out->assigned = c->frag_counter; out->compatible = c->totals.compatible;
  return SB_OK;
}

// normalizeAlphas with the statistics reduced over all ranks: g holds the GLOBAL masses / FLD / counts, roots_all the
// n_ranks cluster-root arrays (n_ranks x n_txps).  Effective lengths are recomputed from the global FLD.
extern "C" int sb_map_project_global(sb_map_ctx* c, const sb_map_partial* g, uint32_t n_ranks, const uint32_t* roots_all,
                                     sb_map_result* out) {
  if (!c || !g || !out || (n_ranks && !roots_all)) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  if (g->n_txps != c->M || g->n_fld != c->nf) { sb::set_error("sb_map_project_global: size mismatch"); return SB_ERR_INVALID; }
  SB_CUDA(cudaSetDevice(c->device));
  cudaStream_t st = c->stream;
  const uint32_t M = c->M, nf = c->nf;
  if (M) {
    SB_CUDA(cudaMemcpyAsync(c->on.mass, g->mass, (size_t)M * 8, cudaMemcpyHostToDevice, st));
    SB_CUDA(cudaMemcpyAsync(c->fin.uniq, g->unique_counts, (size_t)M * 8, cudaMemcpyHostToDevice, st));
    SB_CUDA(cudaMemcpyAsync(c->fin.total, g->total_counts, (size_t)M * 8, cudaMemcpyHostToDevice, st));
    SB_CUDA(cudaMemcpyAsync(c->fin.hits, g->cluster_hits, (size_t)M * 8, cudaMemcpyHostToDevice, st));
  }
  SB_CUDA(cudaMemcpyAsync(c->on.hist, g->fld_hist, (size_t)nf * 8, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(c->on.tot, &g->fld_tot, 8, cudaMemcpyHostToDevice, st));
  const unsigned int mins[2] = {g->fld_min, g->fld_min};
  SB_CUDA(cudaMemcpyAsync(c->on.mins, mins, 8, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaStreamSynchronize(st));
  if (M) {
    k_iota<<<nblk(M, 256), 256, 0, st>>>(M, c->fin.parent);
    for (uint32_t r = 0; r < n_ranks; ++r) {
      SB_CUDA(cudaMemcpyAsync(c->fin.root, roots_all + (size_t)r * M, (size_t)M * 4, cudaMemcpyHostToDevice, st));
      k_union_roots<<<nblk(M, 256), 256, 0, st>>>(M, c->fin.root, c->fin.parent);
    }
    k_roots<<<nblk(M, 256), 256, 0, st>>>(M, c->fin.parent, c->fin.root, c->fin.ids);
  }
  k_online_correction<<<1, 32, 0, st>>>(nf, c->on, 0, c->d_scratch_nf, nullptr, nullptr);
  if (M) k_online_eff_len<<<nblk(M, 256), 256, 0, st>>>(M, nf, c->index->d_tx_off, c->on.cf, c->on.log_eff);
  c->launches += 4 + n_ranks;
  SB_TRY(finish_project(c));
  out->n_txps = M;
  out->projected_counts = c->h_proj.data(); out->eff_len = c->h_eff.data();
  out->unique_counts = c->h_uniq.data(); out->total_counts = c->h_total.data();
  return SB_OK;
}

// forget everything mapped so far (class tables, online state, counters): a fresh context without re-allocating
extern "C" int sb_map_reset(sb_map_ctx* c) {
  if (!c) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  SB_CUDA(cudaSetDevice(c->device));
  SB_CUDA(cudaDeviceSynchronize());
  c->stores.clear();
  c->arena.n_l = c->arena.n_w = c->arena.n_c = c->arena.n_o = 0;
  c->frag_counter = 0; c->frags_seen = 0; c->timestep = 0; c->burned_in = 0; c->full_dp_total = 0;
  c->rescued_total = 0; c->rescue_searches_total = 0; c->rescue_no_room_total = 0;
  memset(&c->totals, 0, sizeof(c->totals));
  const std::vector<double>& t = c->init_tables;
  SB_CUDA(cudaMemcpy(c->d_fld, t.data(), (size_t)4 * c->nf * 8, cudaMemcpyHostToDevice));
  SB_CUDA(cudaMemcpy(c->on.hist, t.data() + (size_t)4 * c->nf, (size_t)c->nf * 8, cudaMemcpyHostToDevice));
  SB_CUDA(cudaMemcpy(c->on.tot, t.data() + (size_t)5 * c->nf, 8, cudaMemcpyHostToDevice));
  SB_CUDA(cudaMemset(c->on.mass_acc, 0, std::max<uint32_t>(c->M, 1) * 8));
  SB_CUDA(cudaMemset(c->on.fld_acc, 0, (size_t)c->nf * 8));
  const unsigned int mins[2] = {c->p.max_frag_len, c->p.max_frag_len};
  SB_CUDA(cudaMemcpy(c->on.mins, mins, 8, cudaMemcpyHostToDevice));
  if (c->M) k_online_init<<<nblk(c->M, 256), 256>>>(c->M, c->index->d_tx_off, c->on.mass, c->on.prior, c->on.log_eff);
  SB_CUDA(cudaDeviceSynchronize());
  return SB_OK;
}

// parity tap: the online state after the last batch
extern "C" int sb_map_online_state(sb_map_ctx* c, double* mass_out, double* hist_out, double* log_eff_out,
                                   uint64_t* scalars6) {
  if (!c) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  SB_CUDA(cudaSetDevice(c->device));
  if (mass_out && c->M) SB_CUDA(cudaMemcpy(mass_out, c->on.mass, (size_t)c->M * 8, cudaMemcpyDeviceToHost));
  if (hist_out) SB_CUDA(cudaMemcpy(hist_out, c->on.hist, (size_t)c->nf * 8, cudaMemcpyDeviceToHost));
  if (log_eff_out && c->M) SB_CUDA(cudaMemcpy(log_eff_out, c->on.log_eff, (size_t)c->M * 8, cudaMemcpyDeviceToHost));
  if (scalars6) {
    unsigned int mins[2];
    double tot;
    SB_CUDA(cudaMemcpy(mins, c->on.mins, 8, cudaMemcpyDeviceToHost));
    SB_CUDA(cudaMemcpy(&tot, c->on.tot, 8, cudaMemcpyDeviceToHost));
    scalars6[0] = c->frag_counter; scalars6[1] = c->frags_seen; scalars6[2] = c->timestep; scalars6[3] = (uint64_t)c->burned_in;
    scalars6[4] = mins[1]; scalars6[5] = sbm_d2u(tot);
  }
  return SB_OK;
}

// ---------------------------------------------------------------------------------------------
// B2: the equivalence-class builder as a seam of its own (SURVEY.md section 8b).  Replaces
//   void EquivalenceClassBuilder<TGValue>::addGroup(TranscriptGroup&&, std::vector<double>& weights)
//   bool finish();  std::vector<std::pair<const TranscriptGroup, TGValue>>& eqVec()
// (include/salmon/internal/quant/EquivalenceClassBuilder.hpp:237-250,165-181,210-223) for callers that produce the
// labels themselves (e.g. the reference's own mapping loop, SalmonQuantify.cpp:855-856, or `--eqclasses`,
// SalmonUtils.cpp:1024-1122): groups arrive in batches from the host, are hashed / sorted / reduced on the device with
// the kernels sb_map_batch uses for its own reads, and finish() hands back the CSR sb_em_optimize takes.
// ---------------------------------------------------------------------------------------------
struct sb_eq_builder {
  sb_map_ctx* c = nullptr;          // only stream, aggregation scratch and arena are used
  uint32_t n_txps = 0;
  uint64_t n_groups = 0;
  // device staging of one batch (owned by c)
  uint64_t *d_loff = nullptr, *d_woff = nullptr, *d_counts = nullptr;
  uint32_t* d_labels = nullptr;
  double* d_weights = nullptr;
  // host result
  std::vector<uint64_t> h_off, h_counts, h_label_off;
  std::vector<uint32_t> h_tids, h_ntx, h_labels;
  std::vector<double> h_w;
};

extern "C" sb_eq_builder* sb_eq_create(uint32_t n_txps, int device) {
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev <= 0) { cudaGetLastError(); sb::set_error("no CUDA device available"); return nullptr; }
  if (device < 0 || device >= n_dev) { sb::set_error("device %d out of range", device); return nullptr; }
  if (cudaSetDevice(device) != cudaSuccess) { sb::set_error("cudaSetDevice failed"); return nullptr; }
  sb_eq_builder* b = new sb_eq_builder();
  b->c = new sb_map_ctx(device);
  b->n_txps = n_txps;
  if (b->c->res.stream(&b->c->stream, cudaStreamDefault) != SB_OK) { delete b->c; delete b; return nullptr; }
  return b;
}

extern "C" void sb_eq_destroy(sb_eq_builder* b) {
  if (!b) return;
  sb_map_destroy(b->c);
  delete b;
}

namespace {
__global__ void k_eq_records(uint32_t n, const uint64_t* __restrict__ loff, const uint64_t* __restrict__ woff,
                             uint64_t* __restrict__ lstart, uint32_t* __restrict__ llen, uint64_t* __restrict__ wstart,
                             uint32_t* __restrict__ wlen) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  lstart[i] = loff[i]; llen[i] = (uint32_t)(loff[i + 1] - loff[i]);
  wstart[i] = woff[i]; wlen[i] = (uint32_t)(woff[i + 1] - woff[i]);
}
}  // namespace

// n groups: label i = labels[label_off[i] .. label_off[i+1]) -- transcript ids (ascending, as TranscriptGroup holds them),
// optionally followed by the same number of range-factorisation bins -- and weights[weight_off[i] .. weight_off[i+1])
// (one per transcript of the label).  counts == NULL: every group counts once (addGroup); else counts[i] fragments.
extern "C" int sb_eq_add_batch(sb_eq_builder* b, uint32_t n, const uint64_t* label_off, const uint32_t* labels,
                               const uint64_t* weight_off, const double* weights, const uint64_t* counts) {
  if (!b || (n && (!label_off || !labels || !weight_off || !weights))) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  if (n == 0) return SB_OK;
  const uint64_t nl = label_off[n], nw = weight_off[n];
  for (uint32_t i = 0; i < n; ++i) {
    const uint64_t ll = label_off[i + 1] - label_off[i], wl = weight_off[i + 1] - weight_off[i];
    if (label_off[i + 1] < label_off[i] || weight_off[i + 1] < weight_off[i] || wl == 0 || (ll != wl && ll != 2 * wl)) {
      sb::set_error("sb_eq_add_batch: group %u: label of %llu entries with %llu weights", i, (unsigned long long)ll, (unsigned long long)wl);
      return SB_ERR_INVALID;
    }
    for (uint64_t j = 0; j < wl; ++j)
      if (labels[label_off[i] + j] >= b->n_txps) { sb::set_error("sb_eq_add_batch: transcript id out of range in group %u", i); return SB_ERR_INVALID; }
  }
  sb_map_ctx* c = b->c;
  SB_CUDA(cudaSetDevice(c->device));
  cudaStream_t st = c->stream;
  SB_TRY(c->res.grow(&b->d_loff, (size_t)n + 1)); SB_TRY(c->res.grow(&b->d_woff, (size_t)n + 1));
  SB_TRY(c->res.grow(&b->d_counts, (size_t)n + 1));
  SB_TRY(c->res.grow(&b->d_labels, nl));
  SB_TRY(c->res.grow(&b->d_weights, nw));
  SB_CUDA(cudaMemcpyAsync(b->d_loff, label_off, ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(b->d_woff, weight_off, ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(b->d_labels, labels, nl * 4, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(b->d_weights, weights, nw * 8, cudaMemcpyHostToDevice, st));
  if (counts) SB_CUDA(cudaMemcpyAsync(b->d_counts, counts, (size_t)n * 8, cudaMemcpyHostToDevice, st));
  SB_TRY(agg_reserve(c, n));
  AggScratch& a = c->agg;
  k_eq_records<<<nblk(n, 256), 256, 0, st>>>(n, b->d_loff, b->d_woff, a.lstart, a.llen, a.wstart, a.wlen);
  Records R{n, a.lstart, a.llen, a.wstart, a.wlen, b->d_labels, b->d_weights, counts ? b->d_counts : nullptr};
  EqStore s;
  SB_TRY(aggregate(c, R, s));
  SB_CUDA(cudaStreamSynchronize(st));       // the staging buffers are reused by the next batch
  c->stores.push_back(s);
  b->n_groups += n;
  return SB_OK;
}

// --eqclasses (readEquivCounts, SalmonUtils.cpp:1024-1122): a finished table -- weights per class, counts -- as one batch
extern "C" int sb_eq_from_host(sb_eq_builder* b, const sb_eq_csr* eq) {
  if (!b || !eq) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  if (eq->n_txps != b->n_txps) { sb::set_error("sb_eq_from_host: transcript count mismatch"); return SB_ERR_INVALID; }
  if (eq->n_classes >= (1ull << 31)) { sb::set_error("sb_eq_from_host: too many classes"); return SB_ERR_INVALID; }
  return sb_eq_add_batch(b, (uint32_t)eq->n_classes, eq->off, eq->tids, eq->off, eq->weights, eq->counts);
}

// finish(): merge the batch tables (same label -> one class: counts add, weights add in batch order), normalise the
// weights of every class to sum 1 (TGValue::normalizeAux, EquivalenceClassBuilder.hpp:114-123).
extern "C" int sb_eq_finish(sb_eq_builder* b, sb_eq_table* out) {
  if (!b || !out) { sb::set_error("null argument"); return SB_ERR_INVALID; }
  sb_map_ctx* c = b->c;
  SB_CUDA(cudaSetDevice(c->device));
  cudaStream_t st = c->stream;
  uint64_t n = 0;
  for (auto& s : c->stores) n += s.n;
  if (n >= (1ull << 31)) { sb::set_error("sb_eq_finish: too many batch classes"); return SB_ERR_INVALID; }
  EqStore merged;
  Arena& ar = c->arena;
  const uint64_t mark_l = ar.n_l, mark_w = ar.n_w, mark_c = ar.n_c, mark_o = ar.n_o;
  if (n) {
    SB_TRY(agg_reserve(c, n));
    AggScratch& a = c->agg;
    uint64_t i = 0;
    for (auto& s : c->stores) {
      if (!s.n) continue;
      k_store_records<<<nblk(s.n, 256), 256, 0, st>>>(s.n, ar.loff + s.base_o, ar.woff + s.base_o, s.base_l, s.base_w,
                                                      a.lstart + i, a.llen + i, a.wstart + i, a.wlen + i);
      i += s.n;
    }
    Records R{(uint32_t)n, a.lstart, a.llen, a.wstart, a.wlen, ar.labels, ar.weights, ar.counts + c->stores.front().base_c};
    SB_TRY(aggregate(c, R, merged));
    if (merged.n) k_normalize<<<nblk(merged.n, 128), 128, 0, st>>>(merged.n, ar.woff + merged.base_o, ar.weights + merged.base_w);
  }
  std::vector<uint64_t> loff(merged.n + 1, 0), woff(merged.n + 1, 0);
  b->h_counts.assign(merged.n, 0); b->h_labels.assign(merged.n_lab, 0); b->h_w.assign(merged.n_w, 0.0);
  if (merged.n) {
    SB_CUDA(cudaMemcpyAsync(loff.data(), ar.loff + merged.base_o, (merged.n + 1) * 8, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaMemcpyAsync(woff.data(), ar.woff + merged.base_o, (merged.n + 1) * 8, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaMemcpyAsync(b->h_counts.data(), ar.counts + merged.base_c, merged.n * 8, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaMemcpyAsync(b->h_labels.data(), ar.labels + merged.base_l, merged.n_lab * 4, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaMemcpyAsync(b->h_w.data(), ar.weights + merged.base_w, merged.n_w * 8, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
  }
  b->h_off = woff; b->h_label_off = loff;
  b->h_tids.clear(); b->h_ntx.clear();
  b->h_tids.reserve(merged.n_w);
  for (uint64_t q = 0; q < merged.n; ++q) {
    const uint64_t ntx = woff[q + 1] - woff[q];
    b->h_ntx.push_back((uint32_t)ntx);
    for (uint64_t j = 0; j < ntx; ++j) b->h_tids.push_back(b->h_labels[loff[q] + j]);
  }
  ar.n_l = mark_l; ar.n_w = mark_w; ar.n_c = mark_c; ar.n_o = mark_o;   // the merged table is temporary: more batches may follow
  out->n_classes = merged.n; out->n_txps = b->n_txps;
  out->off = b->h_off.data(); out->tids = b->h_tids.data(); out->weights = b->h_w.data(); out->counts = b->h_counts.data();
  out->n_txp_in_label = b->h_ntx.data(); out->label_off = b->h_label_off.data(); out->labels = b->h_labels.data();
  out->n_groups = b->n_groups;
  return SB_OK;
}
