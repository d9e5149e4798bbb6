// pgzip.h -- parallel gzip inflate for the read files (host code, no device work).
//
// The reference reads .fastq.gz through kseq/zlib with one inflate thread per file (FQFeeder, pufferfish/external/
// FastxParser); a single zlib thread delivers far less text than the mapping kernels take in.
// Here one gzip file is inflated by several threads:
//   * BGZF files (bgzip: every member carries its compressed size in a 'BC' extra field): members are independent,
//     a worker inflates a run of members with zlib;
//   * any other gzip file (gzip, pigz, concatenated members): the compressed bytes are cut into chunks; the worker of
//     chunk i > 0 searches the first deflate block header at or after its nominal start (dynamic-Huffman, non-final
//     blocks: the header's code-length code must be complete, the literal/length code complete with an end-of-block
//     symbol, the distance code complete or a single code) and decodes from there WITHOUT knowing the 32 KiB window
//     before it: back-references into the unknown window are written as 16-bit markers (0x8000 + window index).  Once
//     32 KiB of output hold no marker, the worker switches to plain byte output.  The consumer walks the chunks in
//     order: chunk i must end at exactly the bit where chunk j > i started (else j was a false positive and is
//     ignored -- its predecessor simply decodes on); the markers of chunk j are then replaced from the last 32 KiB of
//     the text before it.  Every member's CRC-32 and length are checked (per-part CRCs, crc32_combine), so a mis-decode
//     cannot pass silently.
// The deflate decoder below restates RFC 1951; the technique (marker symbols + block search) is the one published for
// pugz / rapidgzip.  Nothing here comes from the reference tree.
#pragma once
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <zlib.h>
#if defined(__x86_64__)
#include <immintrin.h>
#endif

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <deque>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

namespace sb {
namespace pgz {

constexpr uint32_t WSIZE = 32768;
constexpr size_t HEAD = 65536;          // writable bytes in front of every delivered piece (room for a carried record)
constexpr uint64_t NONE = ~0ull;        // "no block start found in this chunk's range"

// ---- bit reader (LSB first, RFC 1951 3.1.1) ----------------------------------------------------------------------
struct BitReader {
  const uint8_t* base = nullptr;
  const uint8_t* p = nullptr;
  const uint8_t* end = nullptr;
  uint64_t buf = 0;
  int cnt = 0;            // valid bits in buf
  bool overrun = false;   // asked for bits past the end of the input
  void init(const uint8_t* b, const uint8_t* e, uint64_t bitpos) {
    base = b; end = e; p = b + (bitpos >> 3); buf = 0; cnt = 0; overrun = false;
    if (p > end) { p = end; overrun = true; }
    refill();
    const int sh = (int)(bitpos & 7);
    if (sh) { if (cnt < sh) overrun = true; else { buf >>= sh; cnt -= sh; } }
  }
  inline void refill() {
    if (p + 8 <= end) {
      uint64_t v;
      memcpy(&v, p, 8);
      buf |= v << cnt;
      p += (63 - cnt) >> 3;
      cnt |= 56;
    } else {
      while (cnt <= 56 && p < end) { buf |= (uint64_t)(*p++) << cnt; cnt += 8; }
    }
  }
  inline uint32_t peek(int n) const { return (uint32_t)(buf & ((1ull << n) - 1)); }
  inline void consume(int n) {
    if (n > cnt) { overrun = true; buf = 0; cnt = 0; return; }
    buf >>= n; cnt -= n;
  }
  inline uint32_t get(int n) {   // n <= 32
    if (cnt < n) refill();
    const uint32_t v = peek(n);
    consume(n);
    return v;
  }
  inline uint64_t bitpos() const { return (uint64_t)(p - base) * 8 - (uint64_t)cnt; }
  inline void align_byte() { consume(cnt & 7); }
  // after align_byte(): the position as a byte pointer (un-reads the whole bytes held in buf)
  inline const uint8_t* byte_ptr() const { return p - (cnt >> 3); }
};

// ---- Huffman tables (two levels) -----------------------------------------------------------------------------------
struct Ent {
  uint16_t val;   // literal byte / base length / base distance / sub-table offset
  uint8_t len;    // code bits to consume (sub-table link: the primary bits)
  uint8_t opx;    // op << 4 | extra bits (link: sub-table index bits)
};
enum : uint8_t { OP_LIT = 0, OP_EOB = 1, OP_BASE = 2, OP_LINK = 3, OP_BAD = 4 };
constexpr int LIT_BITS = 10, DIST_BITS = 8, CL_BITS = 7;
constexpr int LIT_TAB = (1 << LIT_BITS) + 288 * 32, DIST_TAB = (1 << DIST_BITS) + 32 * 128;

static const uint16_t LEN_BASE[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
static const uint8_t LEN_XB[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
static const uint16_t DIST_BASE[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
static const uint8_t DIST_XB[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};

inline uint32_t rev_bits(uint32_t v, int n) {
  uint32_t r = 0;
  for (int i = 0; i < n; ++i) { r = (r << 1) | (v & 1); v >>= 1; }
  return r;
}

// kind: 0 = code-length code (19 symbols), 1 = literal/length, 2 = distance.
// returns 0 = complete code, 1 = incomplete, 2 = no code at all, -1 = over-subscribed / too many symbols
inline int build_table(Ent* tab, int primary, const uint8_t* lens, int n, int kind) {
  int count[16] = {0};
  for (int i = 0; i < n; ++i) count[lens[i]]++;
  const Ent bad{0, 0, (uint8_t)(OP_BAD << 4)};
  for (int i = 0; i < (1 << primary); ++i) tab[i] = bad;
  if (count[0] == n) return 2;
  int left = 1;
  for (int l = 1; l <= 15; ++l) { left = (left << 1) - count[l]; if (left < 0) return -1; }
  uint32_t next[16];
  uint32_t code = 0;
  count[0] = 0;
  for (int l = 1; l <= 15; ++l) { code = (code + (uint32_t)count[l - 1]) << 1; next[l] = code; }
  // sub-table sizes: the longest code under each primary prefix
  uint8_t sub_bits[1 << LIT_BITS];
  bool any_long = false;
  for (int l = primary + 1; l <= 15; ++l) if (count[l]) any_long = true;
  uint32_t codes[288];
  for (int i = 0; i < n; ++i) {
    const int l = lens[i];
    if (!l) continue;
    codes[i] = rev_bits(next[l]++, l);
  }
  int used = 1 << primary;
  if (any_long) {
    memset(sub_bits, 0, (size_t)1 << primary);
    for (int i = 0; i < n; ++i) {
      const int l = lens[i];
      if (l > primary) {
        const uint32_t pre = codes[i] & ((1u << primary) - 1);
        if (l - primary > sub_bits[pre]) sub_bits[pre] = (uint8_t)(l - primary);
      }
    }
    for (int pre = 0; pre < (1 << primary); ++pre) {
      if (!sub_bits[pre]) continue;
      const int sz = 1 << sub_bits[pre];
      tab[pre] = Ent{(uint16_t)used, (uint8_t)primary, (uint8_t)((OP_LINK << 4) | sub_bits[pre])};
      for (int k = 0; k < sz; ++k) tab[used + k] = bad;
      used += sz;
    }
  }
  for (int i = 0; i < n; ++i) {
    const int l = lens[i];
    if (!l) continue;
    Ent e;
    e.len = (uint8_t)l;
    if (kind == 0) { e.val = (uint16_t)i; e.opx = OP_LIT << 4; }
    else if (kind == 1) {
      if (i < 256) { e.val = (uint16_t)i; e.opx = OP_LIT << 4; }
      else if (i == 256) { e.val = 0; e.opx = OP_EOB << 4; }
      else if (i < 286) { e.val = LEN_BASE[i - 257]; e.opx = (uint8_t)((OP_BASE << 4) | LEN_XB[i - 257]); }
      else { e.val = 0; e.opx = OP_BAD << 4; }            // 286, 287: in the fixed code, never valid in data
    } else {
      if (i < 30) { e.val = DIST_BASE[i]; e.opx = (uint8_t)((OP_BASE << 4) | DIST_XB[i]); }
      else { e.val = 0; e.opx = OP_BAD << 4; }
    }
    if (l <= primary) {
      for (uint32_t k = codes[i]; k < (1u << primary); k += (1u << l)) tab[k] = e;
    } else {
      const uint32_t pre = codes[i] & ((1u << primary) - 1);
      const Ent link = tab[pre];
      const int sb = link.opx & 15;
      e.len = (uint8_t)(l - primary);
      for (uint32_t k = codes[i] >> primary; k < (1u << sb); k += (1u << (l - primary))) tab[link.val + k] = e;
    }
  }
  return left > 0 ? 1 : 0;
}

constexpr int PAIR_BITS = 12;
struct Tables {
  Ent lit[LIT_TAB];
  Ent dist[DIST_TAB];
  // two literals per look-up (FASTQ text is mostly literals: bases in 2-3 bits, qualities in 4-6): indexed by the next
  // PAIR_BITS bits; low 16 bits = first literal | second << 8, bits 16-19 = code bits of both, bits 20-21 = how many
  // literals (0: the window does not start with a directly coded literal -- the general path decodes it)
  uint32_t pair[1 << PAIR_BITS];
  void build_pairs() {
    for (uint32_t w = 0; w < (1u << PAIR_BITS); ++w) {
      const Ent a = lit[w & ((1u << LIT_BITS) - 1)];
      uint32_t v = 0;
      if ((a.opx >> 4) == OP_LIT && a.len <= LIT_BITS) {
        v = a.val | ((uint32_t)a.len << 16) | (1u << 20);
        const Ent b = lit[(w >> a.len) & ((1u << LIT_BITS) - 1)];
        if ((b.opx >> 4) == OP_LIT && a.len + b.len <= PAIR_BITS)
          v = a.val | ((uint32_t)b.val << 8) | ((uint32_t)(a.len + b.len) << 16) | (2u << 20);
      }
      pair[w] = v;
    }
  }
};

// the fixed code of BTYPE 1 (RFC 1951 3.2.6)
inline const Tables& fixed_tables() {
  static const Tables* T = [] {
    Tables* t = new Tables();
    uint8_t l[288];
    for (int i = 0; i < 144; ++i) l[i] = 8;
    for (int i = 144; i < 256; ++i) l[i] = 9;
    for (int i = 256; i < 280; ++i) l[i] = 7;
    for (int i = 280; i < 288; ++i) l[i] = 8;
    build_table(t->lit, LIT_BITS, l, 288, 1);
    uint8_t d[32];
    for (int i = 0; i < 32; ++i) d[i] = 5;
    build_table(t->dist, DIST_BITS, d, 32, 2);
    t->build_pairs();
    return t;
  }();
  return *T;
}

// the header of a dynamic block (after the 3 block bits): 0 = tables built, -1 = not a valid header (zlib's rules:
// inflate.c / inftrees.c -- the code-length code must be complete; the other two complete or a single 1-bit code)
inline int read_dynamic_header(BitReader& br, Tables& T, bool pairs = false) {
  br.refill();
  const uint32_t nlen = br.get(5) + 257, ndist = br.get(5) + 1, ncode = br.get(4) + 4;
  if (nlen > 286 || ndist > 30) return -1;
  static const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
  uint8_t cl[19] = {0};
  for (uint32_t i = 0; i < ncode; ++i) cl[order[i]] = (uint8_t)br.get(3);
  Ent clt[1 << CL_BITS];
  if (build_table(clt, CL_BITS, cl, 19, 0) != 0) return -1;
  uint8_t lens[288 + 32];
  uint32_t i = 0;
  const uint32_t total = nlen + ndist;
  while (i < total) {
    if (br.cnt < 16) br.refill();
    const Ent e = clt[br.peek(CL_BITS)];
    if ((e.opx >> 4) != OP_LIT) return -1;
    br.consume(e.len);
    const uint32_t sym = e.val;
    if (sym < 16) { lens[i++] = (uint8_t)sym; continue; }
    uint32_t rep, v = 0;
    if (sym == 16) { if (i == 0) return -1; v = lens[i - 1]; rep = 3 + br.get(2); }
    else if (sym == 17) rep = 3 + br.get(3);
    else rep = 11 + br.get(7);
    if (i + rep > total) return -1;
    while (rep--) lens[i++] = (uint8_t)v;
  }
  if (br.overrun) return -1;
  if (lens[256] == 0) return -1;
  uint8_t ll[288];
  memcpy(ll, lens, nlen);
  int r = build_table(T.lit, LIT_BITS, ll, (int)nlen, 1);
  if (r < 0 || r == 2) return -1;
  if (r == 1) { int mx = 0; for (uint32_t k = 0; k < nlen; ++k) mx = ll[k] > mx ? ll[k] : mx; if (mx != 1) return -1; }
  r = build_table(T.dist, DIST_BITS, lens + nlen, (int)ndist, 2);
  if (r < 0) return -1;
  if (r == 1) { int mx = 0; for (uint32_t k = 0; k < ndist; ++k) mx = lens[nlen + k] > mx ? lens[nlen + k] : mx; if (mx != 1) return -1; }
  if (pairs) T.build_pairs();
  return 0;
}

// Is there a plausible non-final dynamic block header at this bit?  (cheap tests first: 7 of 8 positions fail on the
// three block bits, most of the rest on the code-length code)
inline bool block_candidate(const uint8_t* data, size_t len, uint64_t bitpos, Tables& scratch) {
  const size_t byte = (size_t)(bitpos >> 3);
  if (byte + 16 > len) return false;      // too close to the end: the last stretch belongs to the previous chunk
  uint64_t v;
  memcpy(&v, data + byte, 8);
  v >>= (bitpos & 7);
  if ((v & 7) != 4) return false;                       // BFINAL = 0, BTYPE = 2 (bits: 0, then 0 1)
  const uint32_t hlit = (v >> 3) & 31, hdist = (v >> 8) & 31, hclen = (v >> 13) & 15;
  if (hlit > 29 || hdist > 29) return false;
  // Kraft sum of the code-length code lengths that fit into these 57 bits
  const uint32_t nc = hclen + 4, vis = nc < 13 ? nc : 13;
  uint32_t kraft = 0;
  uint64_t w = v >> 17;
  for (uint32_t i = 0; i < vis; ++i) { const uint32_t l = (uint32_t)(w & 7); w >>= 3; if (l) kraft += 128u >> l; }
  if (kraft > 128 || (vis == nc && kraft != 128)) return false;
  BitReader br;
  br.init(data, data + len, bitpos + 3);
  return read_dynamic_header(br, scratch) == 0;
}

// first candidate in [from_bit, to_bit), or NONE
inline uint64_t find_block(const uint8_t* data, size_t len, uint64_t from_bit, uint64_t to_bit, Tables& scratch) {
  for (uint64_t b = from_bit; b < to_bit; ++b) {
    const size_t byte = (size_t)(b >> 3);
    if (byte + 16 > len) return NONE;
    // quick reject of all 8 shifts of a byte pair would be possible; the 3-bit test per position is already cheap
    const uint32_t two = (uint32_t)data[byte] | ((uint32_t)data[byte + 1] << 8);
    if (((two >> (b & 7)) & 7) != 4) continue;
    if (block_candidate(data, len, b, scratch)) return b;
  }
  return NONE;
}

// ---- gzip member header (RFC 1952) ---------------------------------------------------------------------------------
// returns the header's length in bytes, 0 when [p, e) does not start with a gzip header; *bgzf_size = the member's
// total size when a BGZF 'BC' field is present (else 0)
inline size_t parse_gzip_header(const uint8_t* p, const uint8_t* e, uint32_t* bgzf_size) {
  if (bgzf_size) *bgzf_size = 0;
  if (e - p < 18 || p[0] != 0x1f || p[1] != 0x8b || p[2] != 8) return 0;
  const uint8_t flg = p[3];
  if (flg & 0xE0) return 0;
  const uint8_t* q = p + 10;
  if (flg & 4) {   // FEXTRA
    if (e - q < 2) return 0;
    const size_t xlen = q[0] | (q[1] << 8);
    q += 2;
    if ((size_t)(e - q) < xlen) return 0;
    const uint8_t* x = q;
    const uint8_t* xe = q + xlen;
    while (xe - x >= 4) {
      const size_t sl = x[2] | (x[3] << 8);
      if ((size_t)(xe - x) < 4 + sl) break;
      if (x[0] == 'B' && x[1] == 'C' && sl == 2 && bgzf_size) *bgzf_size = (uint32_t)(x[4] | (x[5] << 8)) + 1;
      x += 4 + sl;
    }
    q += xlen;
  }
  if (flg & 8) { while (q < e && *q) ++q; if (q >= e) return 0; ++q; }    // FNAME
  if (flg & 16) { while (q < e && *q) ++q; if (q >= e) return 0; ++q; }   // FCOMMENT
  if (flg & 2) { if (e - q < 2) return 0; q += 2; }                        // FHCRC
  return (size_t)(q - p);
}

// ---- one chunk's result ----------------------------------------------------------------------------------------------
struct MemberEnd {     // a gzip member ended inside this chunk
  uint32_t crc8;       // CRC of the member's byte-mode text inside this chunk
  uint64_t len8;
  uint32_t crc_stored, isize_stored;
};
// Recycled buffers: a chunk's text buffers are tens of MB; malloc would mmap / munmap (and page-fault) each of them,
// which serialises the inflate threads in the kernel.
struct BufPool {
  std::mutex mu;
  std::vector<std::pair<void*, size_t>> v;
  size_t max_keep = 8;
  void* get(size_t bytes, size_t* cap) {
    {
      std::lock_guard<std::mutex> lk(mu);
      size_t best = v.size();     // best fit: the marker buffers are twice the size of the text buffers
      for (size_t i = 0; i < v.size(); ++i)
        if (v[i].second >= bytes && (best == v.size() || v[i].second < v[best].second)) best = i;
      if (best < v.size()) { void* p = v[best].first; *cap = v[best].second; v.erase(v.begin() + (long)best); return p; }
      if (v.size() >= max_keep) { free(v.front().first); v.erase(v.begin()); }   // too small for the asker: make room
    }
    *cap = bytes;
    return malloc(bytes);
  }
  void put(void* p, size_t cap) {
    if (!p) return;
    {
      std::lock_guard<std::mutex> lk(mu);
      if (v.size() < max_keep) { v.emplace_back(p, cap); return; }
    }
    free(p);
  }
  ~BufPool() { for (auto& e : v) free(e.first); }
};

struct ChunkOut {
  std::shared_ptr<BufPool> pool;
  uint16_t* s16 = nullptr;      // malloc'ed leading part with markers (m16 symbols; none when the window was known)
  size_t m16 = 0, cap16 = 0;
  uint8_t* buf8 = nullptr;      // malloc'ed: HEAD bytes of head room, then n8 bytes of text
  size_t n8 = 0, cap8 = 0;
  std::vector<MemberEnd> ends;
  uint32_t tail_crc8 = 0;       // byte-mode text after the last member end
  uint64_t tail_len8 = 0;
  uint64_t start_bit = NONE, end_bit = NONE;
  size_t next = 0;              // the chunk whose start this one ended on (>= number of chunks: end of the file)
  bool file_end = false;
  std::string err;
  // marker replacement (a second task, once the window before the chunk is known)
  std::unique_ptr<uint8_t[]> win_in;   // the window before the chunk
  size_t win_in_n = 0;
  uint8_t* text16 = nullptr;           // HEAD + m16 bytes, the marker part as text
  size_t cap_text16 = 0;
  uint32_t crc16 = 0;
  ~ChunkOut() {
    if (pool) { pool->put(s16, cap16 * 2); pool->put(buf8, HEAD + cap8); pool->put(text16, cap_text16); }
    else { free(s16); free(buf8); free(text16); }
  }
};

struct Piece {                   // what the consumer gets: `len` bytes at `data`, HEAD writable bytes in front of it
  std::shared_ptr<void> keep;
  uint8_t* data = nullptr;
  size_t len = 0;
};

#if defined(__x86_64__)
// CRC-32 (the gzip polynomial, reflected) by carry-less multiplication: 64 bytes per step are folded into four 128-bit
// accumulators, then reduced (Gopal et al., "Fast CRC Computation for Generic Polynomials Using PCLMULQDQ Instruction",
// Intel 2009; the constants are the published ones for this polynomial).  `crc` is the running register value
// (zlib's crc32 value, inverted); len >= 64 and a multiple of 16.  Checked against zlib's crc32 in tests/test_pgzip.py.
__attribute__((target("sse4.2,pclmul"))) inline uint32_t crc32_fold(const uint8_t* buf, size_t len, uint32_t crc) {
  alignas(16) static const uint64_t k1k2[2] = {0x0154442bd4ull, 0x01c6e41596ull};
  alignas(16) static const uint64_t k3k4[2] = {0x01751997d0ull, 0x00ccaa009eull};
  alignas(16) static const uint64_t k5k0[2] = {0x0163cd6124ull, 0x0000000000ull};
  alignas(16) static const uint64_t poly[2] = {0x01db710641ull, 0x01f7011641ull};
  __m128i x0, x1, x2, x3, x4, x5, x6, x7, x8, y5, y6, y7, y8;
  x1 = _mm_loadu_si128((const __m128i*)(buf + 0x00));
  x2 = _mm_loadu_si128((const __m128i*)(buf + 0x10));
  x3 = _mm_loadu_si128((const __m128i*)(buf + 0x20));
  x4 = _mm_loadu_si128((const __m128i*)(buf + 0x30));
  x1 = _mm_xor_si128(x1, _mm_cvtsi32_si128((int)crc));
  x0 = _mm_load_si128((const __m128i*)k1k2);
  buf += 64; len -= 64;
  while (len >= 64) {
    x5 = _mm_clmulepi64_si128(x1, x0, 0x00); x6 = _mm_clmulepi64_si128(x2, x0, 0x00);
    x7 = _mm_clmulepi64_si128(x3, x0, 0x00); x8 = _mm_clmulepi64_si128(x4, x0, 0x00);
    x1 = _mm_clmulepi64_si128(x1, x0, 0x11); x2 = _mm_clmulepi64_si128(x2, x0, 0x11);
    x3 = _mm_clmulepi64_si128(x3, x0, 0x11); x4 = _mm_clmulepi64_si128(x4, x0, 0x11);
    y5 = _mm_loadu_si128((const __m128i*)(buf + 0x00)); y6 = _mm_loadu_si128((const __m128i*)(buf + 0x10));
    y7 = _mm_loadu_si128((const __m128i*)(buf + 0x20)); y8 = _mm_loadu_si128((const __m128i*)(buf + 0x30));
    x1 = _mm_xor_si128(_mm_xor_si128(x1, x5), y5); x2 = _mm_xor_si128(_mm_xor_si128(x2, x6), y6);
    x3 = _mm_xor_si128(_mm_xor_si128(x3, x7), y7); x4 = _mm_xor_si128(_mm_xor_si128(x4, x8), y8);
    buf += 64; len -= 64;
  }
  x0 = _mm_load_si128((const __m128i*)k3k4);
  x5 = _mm_clmulepi64_si128(x1, x0, 0x00); x1 = _mm_clmulepi64_si128(x1, x0, 0x11); x1 = _mm_xor_si128(_mm_xor_si128(x1, x2), x5);
  x5 = _mm_clmulepi64_si128(x1, x0, 0x00); x1 = _mm_clmulepi64_si128(x1, x0, 0x11); x1 = _mm_xor_si128(_mm_xor_si128(x1, x3), x5);
  x5 = _mm_clmulepi64_si128(x1, x0, 0x00); x1 = _mm_clmulepi64_si128(x1, x0, 0x11); x1 = _mm_xor_si128(_mm_xor_si128(x1, x4), x5);
  while (len >= 16) {
    x2 = _mm_loadu_si128((const __m128i*)buf);
    x5 = _mm_clmulepi64_si128(x1, x0, 0x00); x1 = _mm_clmulepi64_si128(x1, x0, 0x11); x1 = _mm_xor_si128(_mm_xor_si128(x1, x2), x5);
    buf += 16; len -= 16;
  }
  x2 = _mm_clmulepi64_si128(x1, x0, 0x10);
  x3 = _mm_setr_epi32(~0, 0, ~0, 0);
  x1 = _mm_srli_si128(x1, 8);
  x1 = _mm_xor_si128(x1, x2);
  x0 = _mm_loadl_epi64((const __m128i*)k5k0);
  x2 = _mm_srli_si128(x1, 4);
  x1 = _mm_and_si128(x1, x3);
  x1 = _mm_clmulepi64_si128(x1, x0, 0x00);
  x1 = _mm_xor_si128(x1, x2);
  x0 = _mm_load_si128((const __m128i*)poly);
  x2 = _mm_and_si128(x1, x3);
  x2 = _mm_clmulepi64_si128(x2, x0, 0x10);
  x2 = _mm_and_si128(x2, x3);
  x2 = _mm_clmulepi64_si128(x2, x0, 0x00);
  x1 = _mm_xor_si128(x1, x2);
  return (uint32_t)_mm_extract_epi32(x1, 1);
}
#endif

// zlib's crc32 value of [p, p + n)
inline uint32_t crc_of(const uint8_t* p, uint64_t n) {
  uint32_t c = 0;
#if defined(__x86_64__)
  static const bool have_clmul = __builtin_cpu_supports("pclmul") && __builtin_cpu_supports("sse4.2");
  if (have_clmul && n >= 64) {
    const uint64_t body = n & ~(uint64_t)15;
    c = ~crc32_fold(p, (size_t)body, ~c);
    p += body; n -= body;
  }
#endif
  while (n) { const uInt k = (uInt)std::min<uint64_t>(n, (uint64_t)1 << 30); c = (uint32_t)crc32(c, p, k); p += k; n -= k; }
  return c;
}

// ---- the deflate decoder ---------------------------------------------------------------------------------------------
struct Decoder {
  BitReader br;
  // marker mode
  uint16_t* s16 = nullptr;
  size_t m = 0, cap16 = 0;
  size_t last_marker = 0;      // one past the position of the last marker symbol written
  bool markers = false;
  // byte mode
  uint8_t* out = nullptr;      // -> ChunkOut::buf8
  size_t n = 0, cap = 0;       // text bytes written (after HEAD) / capacity
  size_t valid_back = 0;       // how far before byte 0 a reference may reach (wrapping arithmetic, see the member start)
  size_t seg_start = 0;        // byte-mode text of the current member starts here
  std::string err;
  BufPool* pool = nullptr;
  ~Decoder() {
    if (pool) { pool->put(s16, cap16 * 2); pool->put(out, HEAD + cap); }
    else { free(s16); free(out); }
  }

  bool grow8(size_t need) {
    if (n + need <= cap) return true;
    size_t nc = cap ? cap * 2 : (size_t)1 << 22;
    while (nc < n + need) nc *= 2;
    uint8_t* q;
    if (!out && pool) { size_t got = 0; q = (uint8_t*)pool->get(HEAD + nc, &got); if (q) nc = got - HEAD; }
    else q = (uint8_t*)realloc(out, HEAD + nc);
    if (!q) { err = "out of memory"; return false; }
    out = q; cap = nc;
    return true;
  }
  bool grow16(size_t need) {
    if (m + need <= cap16) return true;
    size_t nc = cap16 ? cap16 * 2 : (size_t)1 << 21;
    while (nc < m + need) nc *= 2;
    uint16_t* q;
    if (!s16 && pool) { size_t got = 0; q = (uint16_t*)pool->get(nc * 2, &got); if (q) nc = got / 2; }
    else q = (uint16_t*)realloc(s16, nc * 2);
    if (!q) { err = "out of memory"; return false; }
    s16 = q; cap16 = nc;
    return true;
  }

  // markers -> bytes: from the next block on the text goes to the byte buffer; its first WSIZE window bytes are the
  // (marker-free) end of the marker part
  bool switch_to_bytes() {
    markers = false;
    if (!grow8(1)) return false;
    const size_t w = m < WSIZE ? m : WSIZE;
    for (size_t i = 0; i < w; ++i) out[HEAD - w + i] = (uint8_t)s16[m - w + i];
    valid_back = w;
    n = 0; seg_start = 0;
    return true;
  }

  // one block's symbols; 0 = end of block, -1 = error.  The fast loop keeps the bit buffer in registers and never checks
  // for the end of the input (it leaves while 16 bytes are still unread); the careful loop below finishes the block.
  template <bool MARK>
  int codes(const Ent* lt, const Ent* dt, const uint32_t* pt) {
    uint64_t buf = br.buf;
    int cnt = br.cnt;
    const uint8_t* p = br.p;
    const uint8_t* const in_end = br.end;
    int status = 2;   // 2 = go on in the careful loop
#define PGZ_REFILL() do { uint64_t v_; memcpy(&v_, p, 8); buf |= v_ << cnt; p += (63 - cnt) >> 3; cnt |= 56; } while (0)
#define PGZ_DROP(nb) do { buf >>= (nb); cnt -= (nb); } while (0)
    while (in_end - p >= 16 && !br.overrun) {
      if (MARK) { if (m + 264 > cap16) { if (!grow16(264)) { status = -1; break; } } }
      else { if (n + 264 > cap) { if (!grow8(264)) { status = -1; break; } } }
      PGZ_REFILL();
      // up to four look-ups of two literals each per refill (4 x PAIR_BITS = 48 of the 56 bits)
      {
        bool more = true;
        for (int r = 0; r < 4; ++r) {
          const uint32_t v = pt[buf & ((1u << PAIR_BITS) - 1)];
          const uint32_t k = v >> 20;
          if (k == 0) { more = false; break; }
          if (MARK) { s16[m] = (uint16_t)(v & 0xff); s16[m + 1] = (uint16_t)((v >> 8) & 0xff); m += k; }
          else { out[HEAD + n] = (uint8_t)v; out[HEAD + n + 1] = (uint8_t)(v >> 8); n += k; }
          PGZ_DROP((v >> 16) & 15);
        }
        if (more) continue;
      }
      Ent e = lt[buf & ((1u << LIT_BITS) - 1)];
      if (cnt < 48) PGZ_REFILL();
      if ((e.opx >> 4) == OP_LINK) {
        const int sb = e.opx & 15;
        e = lt[e.val + ((buf >> LIT_BITS) & ((1u << sb) - 1))];
        PGZ_DROP(LIT_BITS);
      }
      const uint32_t op = e.opx >> 4;
      PGZ_DROP(e.len);
      if (op == OP_LIT) {
        if (MARK) s16[m++] = e.val; else out[HEAD + n++] = (uint8_t)e.val;
        continue;
      }
      if (op == OP_EOB) { status = 0; break; }
      if (op != OP_BASE) { err = "invalid literal/length code"; status = -1; break; }
      const int lxb = e.opx & 15;
      uint32_t len = e.val + (uint32_t)(buf & ((1u << lxb) - 1));
      PGZ_DROP(lxb);
      if (cnt < 32) PGZ_REFILL();
      Ent d = dt[buf & ((1u << DIST_BITS) - 1)];
      if ((d.opx >> 4) == OP_LINK) {
        const int sb = d.opx & 15;
        d = dt[d.val + ((buf >> DIST_BITS) & ((1u << sb) - 1))];
        PGZ_DROP(DIST_BITS);
      }
      if ((d.opx >> 4) != OP_BASE) { err = "invalid distance code"; status = -1; break; }
      PGZ_DROP(d.len);
      const int dxb = d.opx & 15;
      const uint32_t dist = d.val + (uint32_t)(buf & ((1u << dxb) - 1));
      PGZ_DROP(dxb);
      if (!copy_match<MARK>(len, dist)) { status = -1; break; }
    }
#undef PGZ_REFILL
#undef PGZ_DROP
    br.buf = buf; br.cnt = cnt; br.p = p;
    if (status != 2) return status;
    return codes_careful<MARK>(lt, dt);   // (the careful loop needs no pair table)
  }

  template <bool MARK>
  inline bool copy_match(uint32_t len, uint32_t dist) {
    if (MARK) {
      uint16_t* w = s16;
      uint32_t seen = 0;
      if (dist > m) {                      // reaches into the unknown window
        const size_t before = dist - m;    // how far before the chunk's first byte
        if (before > WSIZE) { err = "distance too far back"; return false; }
        size_t widx = WSIZE - before;      // window index of the first byte
        while (len && widx < WSIZE) { w[m++] = (uint16_t)(0x8000u + widx++); --len; seen = 0x8000u; }
      }
      // (the rest, if any, continues at the chunk's own symbols)
      const uint16_t* src = w + (m - dist);
      uint16_t* dst = w + m;
      if (dist >= 8) {
        // 8 symbols at a time; writes up to 7 symbols past the end (room is reserved by the callers)
        for (uint32_t k = 0; k < len; k += 8) {
          uint64_t a, b;
          memcpy(&a, src + k, 8); memcpy(&b, src + k + 4, 8);
          memcpy(dst + k, &a, 8); memcpy(dst + k + 4, &b, 8);
          seen |= (uint32_t)((a | b) >> 32) | (uint32_t)(a | b);
        }
        // symbols past `len` may have contributed to `seen`: a false "marker seen" only delays the switch to bytes
        seen = (seen | (seen >> 16)) & 0x8000u;
      } else {
        for (uint32_t k = 0; k < len; ++k) { const uint16_t sy = src[k]; dst[k] = sy; seen |= sy; }
      }
      m += len;
      if (seen & 0x8000u) last_marker = m;
    } else {
      if (dist > n + valid_back) { err = "invalid distance too far back"; return false; }
      uint8_t* w = out + HEAD + n;
      const uint8_t* src = w - dist;
      if (dist >= 16) {
        for (uint32_t k = 0; k < len; k += 16) memcpy(w + k, src + k, 16);   // up to 15 bytes past the end (reserved)
      } else if (dist >= len) memcpy(w, src, len);
      else for (uint32_t k = 0; k < len; ++k) w[k] = src[k];
      n += len;
    }
    return true;
  }

  template <bool MARK>
  int codes_careful(const Ent* lt, const Ent* dt) {
    for (;;) {
      if (MARK) { if (m + 264 > cap16 && !grow16(264)) return -1; }
      else { if (n + 264 > cap && !grow8(264)) return -1; }
      br.refill();
      Ent e = lt[br.buf & ((1u << LIT_BITS) - 1)];
      // up to three literals per refill (direct entries take at most LIT_BITS bits each)
      for (int r = 0; r < 3 && (e.opx >> 4) == OP_LIT; ++r) {
        br.consume(e.len);
        if (MARK) s16[m++] = e.val; else out[HEAD + n++] = (uint8_t)e.val;
        e = lt[br.buf & ((1u << LIT_BITS) - 1)];
      }
      if (br.overrun) { err = "unexpected end of the compressed data"; return -1; }
      if ((e.opx >> 4) == OP_LIT) continue;
      if (br.cnt < 48) br.refill();
      if ((e.opx >> 4) == OP_LINK) {
        const int sb = e.opx & 15;
        e = lt[e.val + ((br.buf >> LIT_BITS) & ((1u << sb) - 1))];
        br.consume(LIT_BITS);
      }
      const uint32_t op = e.opx >> 4;
      br.consume(e.len);
      if (op == OP_LIT) {
        if (MARK) s16[m++] = e.val; else out[HEAD + n++] = (uint8_t)e.val;
        continue;
      }
      if (op == OP_EOB) return br.overrun ? -1 : 0;
      if (op != OP_BASE) { err = "invalid literal/length code"; return -1; }
      uint32_t len = e.val + br.peek(e.opx & 15);
      br.consume(e.opx & 15);
      if (br.cnt < 32) br.refill();
      Ent d = dt[br.buf & ((1u << DIST_BITS) - 1)];
      if ((d.opx >> 4) == OP_LINK) {
        const int sb = d.opx & 15;
        d = dt[d.val + ((br.buf >> DIST_BITS) & ((1u << sb) - 1))];
        br.consume(DIST_BITS);
      }
      if ((d.opx >> 4) != OP_BASE) { err = "invalid distance code"; return -1; }
      br.consume(d.len);
      const uint32_t dist = d.val + br.peek(d.opx & 15);
      br.consume(d.opx & 15);
      if (br.overrun) { err = "unexpected end of the compressed data"; return -1; }
      if (!copy_match<MARK>(len, dist)) return -1;
    }
  }

  // a stored block (after the 3 block bits)
  int stored() {
    br.align_byte();
    if (br.cnt < 32) br.refill();
    if (br.cnt < 32) { err = "unexpected end of the compressed data"; return -1; }
    const uint32_t len = br.peek(16);
    br.consume(16);
    const uint32_t nlen = br.peek(16);
    br.consume(16);
    if ((len ^ 0xffffu) != nlen) { err = "invalid stored block lengths"; return -1; }
    const uint8_t* src = br.byte_ptr();
    if ((size_t)(br.end - src) < len) { err = "unexpected end of the compressed data"; return -1; }
    if (markers) { if (!grow16(len)) return -1; for (uint32_t k = 0; k < len; ++k) s16[m++] = src[k]; }
    else { if (!grow8(len)) return -1; memcpy(out + HEAD + n, src, len); n += len; }
    br.init(br.base, br.end, (uint64_t)(src + len - br.base) * 8);
    return 0;
  }
};

// ---- the file ---------------------------------------------------------------------------------------------------------
class ParallelGz {
 public:
  // data/len: the whole compressed file (memory mapped by the caller, must outlive this object)
  ParallelGz(const uint8_t* data, size_t len, int threads, size_t chunk_bytes = (size_t)2 << 20)
      : d_(data), len_(len), T_(threads < 1 ? 1 : threads), C_(chunk_bytes < 1024 ? 1024 : chunk_bytes), pool_(new BufPool()) {
    pool_->max_keep = (size_t)T_ * 4 + 8;
  }
  ~ParallelGz() { stop(); }

  // false: not a gzip file (err says why)
  bool start(std::string& err) {
    uint32_t bsz = 0;
    const size_t h = parse_gzip_header(d_, d_ + len_, &bsz);
    if (!h) { err = "not a gzip file"; return false; }
    bgzf_ = bsz != 0;
    if (bgzf_) {
      // member table (each hop reads one header)
      size_t off = 0;
      std::vector<size_t> mem;
      while (off < len_) {
        uint32_t sz = 0;
        const size_t hh = parse_gzip_header(d_ + off, d_ + len_, &sz);
        if (!hh || !sz || off + sz > len_) { bgzf_ = false; break; }
        mem.push_back(off);
        off += sz;
      }
      if (bgzf_) {
        mem.push_back(len_);
        size_t i = 0;
        while (i + 1 < mem.size()) {   // runs of members of about C_ compressed bytes
          size_t j = i + 1;
          while (j + 1 < mem.size() && mem[j] - mem[i] < C_) ++j;
          bg_runs_.push_back({mem[i], mem[j]});
          i = j;
        }
        nchunks_ = bg_runs_.size();
      }
    }
    if (!bgzf_) {
      first_bit_ = (uint64_t)h * 8;
      nchunks_ = (len_ + C_ - 1) / C_;
      if (nchunks_ == 0) nchunks_ = 1;
    }
    out_.resize(nchunks_);
    done_.reset(new std::atomic<int>[nchunks_]);
    sstate_.reset(new std::atomic<int>[nchunks_]);
    sbit_.reset(new std::atomic<uint64_t>[nchunks_]);
    for (size_t i = 0; i < nchunks_; ++i) { done_[i] = 0; sstate_[i] = 0; sbit_[i] = NONE; }
    for (int t = 0; t < T_; ++t) th_.emplace_back([this] { worker(); });
    return true;
  }

  // the next piece of text in file order; false at the end of the file or on error (err non-empty)
  bool next(Piece& pc, std::string& err) {
    for (;;) {
      if (!pending_.empty()) { pc = std::move(pending_.front()); pending_.pop_front(); return true; }
      if (finished_) return false;
      // (1) chain every decoded chunk that is next in line: window hand-over, marker replacement tasks
      for (;;) {
        if (chain_end_ || chain_ >= nchunks_) break;
        if (done_[chain_].load() < 1) break;
        ChunkOut& co = *out_[chain_];
        if (!co.err.empty()) { err = co.err; finished_ = true; return false; }
        const uint64_t c0 = cpu_ns();
        const bool ok = bgzf_ || chain_chunk(co, chain_, err);
        consumer_ns_ += cpu_ns() - c0;
        if (!ok) { finished_ = true; return false; }
        order_.push_back(chain_);
        const size_t nxt = bgzf_ ? chain_ + 1 : co.next;
        if (co.file_end || nxt >= nchunks_) chain_end_ = true;
        {
          std::lock_guard<std::mutex> lk(mu_);
          const size_t to = chain_end_ ? nchunks_ : nxt;
          for (size_t k = chain_ + 1; k < to && k < claim_; ++k) skipped_.push_back(k);
          if (to > chain_ + 1) skipped_total_ += to - chain_ - 1;   // (claimed or not: claim_ jumps over them below)
          chain_ = to;
          passed_ = chain_;
          if (claim_ < passed_) claim_ = passed_;   // chunks the chain went through are not decoded a second time
        }
        drop_skipped();
      }
      // (2) deliver the first chunk in line once its markers are replaced
      if (!order_.empty() && done_[order_.front()].load() == 2) {
        const size_t i = order_.front();
        order_.pop_front();
        std::unique_ptr<ChunkOut> co = std::move(out_[i]);
        if (!co->err.empty()) { err = co->err; finished_ = true; return false; }
        const uint64_t c0 = cpu_ns();
        const bool ok = deliver_chunk(*co, err);
        consumer_ns_ += cpu_ns() - c0;
        if (!ok) { finished_ = true; return false; }
        co.reset();
        { std::lock_guard<std::mutex> lk(mu_); ++delivered_count_; }
        cv_slot_.notify_all();
        continue;
      }
      if (order_.empty() && (chain_end_ || chain_ >= nchunks_)) {
        if (len_run_ != 0) { err = "truncated gzip file (the last member has no trailer)"; }
        finished_ = true;
        if (!err.empty()) return false;
        continue;
      }
      // (3) wait for the next event: the chunk to chain is decoded, or the chunk to deliver is finished
      {
        std::unique_lock<std::mutex> lk(mu_);
        cv_done_.wait(lk, [&] {
          const bool can_chain = !chain_end_ && chain_ < nchunks_ && done_[chain_].load() >= 1;
          const bool can_deliver = !order_.empty() && done_[order_.front()].load() == 2;
          return can_chain || can_deliver;
        });
      }
    }
  }

  void stop() {
    {
      std::lock_guard<std::mutex> lk(mu_);
      stop_ = true;
    }
    cv_slot_.notify_all();
    for (auto& t : th_) if (t.joinable()) t.join();
    th_.clear();
  }

  bool is_bgzf() const { return bgzf_; }
  // where the time went (thread CPU seconds): the workers' decode, the consumer's serial part
  double worker_cpu_s() const { return (double)worker_ns_.load() * 1e-9; }
  double consumer_cpu_s() const { return (double)consumer_ns_ * 1e-9; }
  double resolve_cpu_s() const { return (double)resolve_ns_.load() * 1e-9; }   // (part of worker_cpu_s)
  uint64_t marker_symbols() const { return n16_total_; }

 private:
  const uint8_t* d_;
  size_t len_;
  int T_;
  size_t C_;
  std::shared_ptr<BufPool> pool_;
  bool bgzf_ = false;
  uint64_t first_bit_ = 0;
  size_t nchunks_ = 0;
  std::vector<std::pair<size_t, size_t>> bg_runs_;
  std::vector<std::unique_ptr<ChunkOut>> out_;
  std::unique_ptr<std::atomic<int>[]> done_;     // 0 = not decoded, 1 = decoded, 2 = markers replaced (ready to deliver)
  std::unique_ptr<std::atomic<int>[]> sstate_;
  std::unique_ptr<std::atomic<uint64_t>[]> sbit_;
  std::vector<std::thread> th_;
  std::mutex mu_;
  std::condition_variable cv_done_, cv_slot_;
  size_t claim_ = 0, passed_ = 0, delivered_count_ = 0, skipped_total_ = 0;
  std::deque<size_t> resolve_q_;
  bool stop_ = false, finished_ = false;
  std::vector<size_t> skipped_;
  std::deque<Piece> pending_;
  // consumer state
  size_t chain_ = 0;
  bool chain_end_ = false;
  std::deque<size_t> order_;      // chained chunks not yet delivered
  uint8_t win_[WSIZE];            // the text before the next chunk to chain (at most WSIZE bytes of the current member)
  size_t win_n_ = 0;
  uint32_t crc_run_ = 0;          // CRC / length of the current member's text delivered so far
  uint64_t len_run_ = 0;
  std::atomic<uint64_t> worker_ns_{0}, resolve_ns_{0};
  uint64_t consumer_ns_ = 0, n16_total_ = 0;
  static uint64_t cpu_ns() {
    timespec ts;
    clock_gettime(CLOCK_THREAD_CPUTIME_ID, &ts);
    return (uint64_t)ts.tv_sec * 1000000000ull + (uint64_t)ts.tv_nsec;
  }

  void drop_skipped() {
    std::vector<size_t> s;
    { std::lock_guard<std::mutex> lk(mu_); s.swap(skipped_); }
    for (size_t k : s)
      if (done_[k].load()) out_[k].reset();   // (a chunk still running is dropped by its worker: it sees passed_)
  }

  void push_window(const uint8_t* p, size_t n) {
    if (n >= WSIZE) { memcpy(win_, p + n - WSIZE, WSIZE); win_n_ = WSIZE; return; }
    if (win_n_ + n > WSIZE) { const size_t drop = win_n_ + n - WSIZE; memmove(win_, win_ + drop, win_n_ - drop); win_n_ -= drop; }
    memcpy(win_ + win_n_, p, n);
    win_n_ += n;
  }

  static bool resolve_scalar(const uint16_t* s, size_t m, const uint8_t* win, size_t win_n, uint8_t* t) {
    for (size_t i = 0; i < m; ++i) {
      const uint16_t v = s[i];
      if (v & 0x8000u) {
        const size_t back = WSIZE - (v & 0x7fffu);   // window index WSIZE - 1 = the byte just before the chunk
        if (back > win_n) return false;
        t[i] = win[win_n - back];
      } else t[i] = (uint8_t)v;
    }
    return true;
  }
#if defined(__x86_64__)
  // 32 symbols at a time: groups without a marker (most of a FASTQ record's sequence and quality lines) are narrowed
  // with one pack, the others go through the scalar loop
  __attribute__((target("avx2"))) static bool resolve_avx2(const uint16_t* s, size_t m, const uint8_t* win, size_t win_n, uint8_t* t) {
    size_t i = 0;
    for (; i + 32 <= m; i += 32) {
      const __m256i a = _mm256_loadu_si256((const __m256i*)(s + i)), b = _mm256_loadu_si256((const __m256i*)(s + i + 16));
      // narrow all 32 (a marker saturates to 255), then put the window byte where a marker was: the cost follows the
      // number of markers, not the number of groups that hold one (in FASTQ every record's name carries a few)
      const __m256i p = _mm256_permute4x64_epi64(_mm256_packus_epi16(a, b), 0xD8);
      _mm256_storeu_si256((__m256i*)(t + i), p);
      uint32_t ma = (uint32_t)_mm256_movemask_epi8(a) & 0xAAAAAAAAu, mb = (uint32_t)_mm256_movemask_epi8(b) & 0xAAAAAAAAu;
      while (ma) {
        const int j = __builtin_ctz(ma) >> 1;
        ma &= ma - 1;
        const size_t back = WSIZE - (s[i + j] & 0x7fffu);
        if (back > win_n) return false;
        t[i + j] = win[win_n - back];
      }
      while (mb) {
        const int j = 16 + (__builtin_ctz(mb) >> 1);
        mb &= mb - 1;
        const size_t back = WSIZE - (s[i + j] & 0x7fffu);
        if (back > win_n) return false;
        t[i + j] = win[win_n - back];
      }
    }
    return resolve_scalar(s + i, m - i, win, win_n, t + i);
  }
#endif
  static bool resolve(const uint16_t* s, size_t m, const uint8_t* win, size_t win_n, uint8_t* t) {
#if defined(__x86_64__)
    static const bool have_avx2 = __builtin_cpu_supports("avx2");
    if (have_avx2) return resolve_avx2(s, m, win, win_n, t);
#endif
    return resolve_scalar(s, m, win, win_n, t);
  }

  // serial, cheap: the window after this chunk; the marker replacement itself becomes a task
  bool chain_chunk(ChunkOut& co, size_t idx, std::string& err) {
    const size_t m = co.m16;
    n16_total_ += m;
    if (m) {
      co.win_in.reset(new uint8_t[WSIZE]);
      memcpy(co.win_in.get(), win_, win_n_);
      co.win_in_n = win_n_;
    }
    if (!co.ends.empty()) {
      // a member started inside the chunk: the window is what followed the last member start (byte-mode text)
      win_n_ = 0;
      push_window(co.buf8 + HEAD + co.n8 - co.tail_len8, co.tail_len8);
    } else {
      if (co.n8 < WSIZE && m) {
        const size_t k = std::min<size_t>(m, WSIZE);
        uint8_t tmp[WSIZE];
        if (!resolve(co.s16 + m - k, k, co.win_in.get(), co.win_in_n, tmp)) { err = "corrupt gzip data (reference before the start of the member)"; return false; }
        // markers index the window before the chunk: correct for the tail only when looked up relative to the chunk
        push_window(tmp, k);
      }
      if (co.n8) push_window(co.buf8 + HEAD, co.n8);
    }
    if (m) {
      { std::lock_guard<std::mutex> lk(mu_); resolve_q_.push_back(idx); }
      cv_slot_.notify_all();
    } else {
      done_[idx].store(2);
    }
    return true;
  }

  bool member_end(const MemberEnd& me, std::string& err) {
    crc_run_ = (uint32_t)crc32_combine(crc_run_, me.crc8, (z_off_t)me.len8);
    len_run_ += me.len8;
    if (crc_run_ != me.crc_stored || (uint32_t)len_run_ != me.isize_stored) { err = "gzip CRC / length check failed (corrupt file)"; return false; }
    crc_run_ = 0; len_run_ = 0;
    return true;
  }

  // in file order: member checks, then the chunk's text becomes pieces
  bool deliver_chunk(ChunkOut& co, std::string& err) {
    if (bgzf_) {
      if (co.n8) pending_.push_back(make_piece(co.buf8, HEAD + co.cap8, co.n8));
      return true;
    }
    if (co.m16) {
      crc_run_ = (uint32_t)crc32_combine(crc_run_, co.crc16, (z_off_t)co.m16);
      len_run_ += co.m16;
      pending_.push_back(make_piece(co.text16, co.cap_text16, co.m16));
    }
    for (const MemberEnd& me : co.ends)
      if (!member_end(me, err)) return false;
    crc_run_ = (uint32_t)crc32_combine(crc_run_, co.tail_crc8, (z_off_t)co.tail_len8);
    len_run_ += co.tail_len8;
    if (co.n8) pending_.push_back(make_piece(co.buf8, HEAD + co.cap8, co.n8));
    return true;
  }

  // hands a chunk buffer over to the consumer; it returns to the pool with the last reference
  Piece make_piece(uint8_t*& buf, size_t cap_bytes, size_t len) {
    Piece p;
    uint8_t* b = buf;
    buf = nullptr;
    std::shared_ptr<BufPool> pool = pool_;
    p.keep = std::shared_ptr<void>(b, [pool, cap_bytes](void* q) { pool->put(q, cap_bytes); });
    p.data = b + HEAD; p.len = len;
    return p;
  }

  // the first block start of chunk j (searched once, by whoever asks first)
  uint64_t ensure_start(size_t j, Tables& scratch) {
    if (j >= nchunks_) return NONE;
    int exp = 0;
    if (sstate_[j].compare_exchange_strong(exp, 1)) {
      uint64_t s;
      if (j == 0) s = first_bit_;
      else s = find_block(d_, len_, (uint64_t)j * C_ * 8, std::min<uint64_t>((uint64_t)(j + 1) * C_, len_) * 8, scratch);
      sbit_[j].store(s);
      sstate_[j].store(2);
      return s;
    }
    while (sstate_[j].load() != 2) std::this_thread::yield();
    return sbit_[j].load();
  }

  void worker() {
    std::unique_ptr<Tables> tab(new Tables()), scratch(new Tables());
    for (;;) {
      size_t i = 0;
      bool is_resolve = false;
      {
        std::unique_lock<std::mutex> lk(mu_);
        cv_slot_.wait(lk, [&] {
          return stop_ || !resolve_q_.empty() || (claim_ < nchunks_ && claim_ < passed_ + (size_t)T_ * 2 + 2 && in_flight() < (size_t)T_ * 3 + 2);
        });
        if (stop_) return;
        if (!resolve_q_.empty()) { i = resolve_q_.front(); resolve_q_.pop_front(); is_resolve = true; }
        else i = claim_++;
      }
      const uint64_t c0 = cpu_ns();
      if (is_resolve) {
        ChunkOut& co = *out_[i];
        co.text16 = (uint8_t*)pool_->get(HEAD + co.m16, &co.cap_text16);
        if (!co.text16) co.err = "out of memory";
        else if (!resolve(co.s16, co.m16, co.win_in.get(), co.win_in_n, co.text16 + HEAD)) co.err = "corrupt gzip data (reference before the start of the member)";
        else co.crc16 = crc_of(co.text16 + HEAD, co.m16);
        pool_->put(co.s16, co.cap16 * 2); co.s16 = nullptr;
        co.win_in.reset();
        worker_ns_ += cpu_ns() - c0;
        resolve_ns_ += cpu_ns() - c0;
        { std::lock_guard<std::mutex> lk(mu_); done_[i].store(2); }
        cv_done_.notify_all();
        continue;
      }
      std::unique_ptr<ChunkOut> co(new ChunkOut());
      co->pool = pool_;
      if (bgzf_) inflate_bgzf(i, *co);
      else decode_chunk(i, *co, *tab, *scratch);
      worker_ns_ += cpu_ns() - c0;
      {
        std::lock_guard<std::mutex> lk(mu_);
        const bool drop = i < passed_;            // the chain went past this chunk while it ran
        if (!drop) out_[i] = std::move(co);
        done_[i].store(bgzf_ ? 2 : 1);
      }
      cv_done_.notify_all();
    }
  }
  // chunks claimed and not yet delivered or skipped (bounds the memory held); call with mu_ held
  size_t in_flight() const { return claim_ - std::min(claim_, delivered_count_ + skipped_total_); }

  void inflate_bgzf(size_t i, ChunkOut& co) {
    const size_t a = bg_runs_[i].first, b = bg_runs_[i].second;
    z_stream zs;
    memset(&zs, 0, sizeof zs);
    if (inflateInit2(&zs, -15) != Z_OK) { co.err = "zlib: inflateInit2 failed"; return; }
    size_t cap = (b - a) * 4 + 65536, n = 0, got = 0;
    uint8_t* out = (uint8_t*)pool_->get(HEAD + cap, &got);
    if (!out) { co.err = "out of memory"; inflateEnd(&zs); return; }
    cap = got - HEAD;
    size_t off = a;
    while (off < b) {
      uint32_t sz = 0;
      const size_t h = parse_gzip_header(d_ + off, d_ + len_, &sz);
      if (!h || !sz || off + sz > b || sz < h + 8) { co.err = "corrupt BGZF member"; break; }
      const uint8_t* tr = d_ + off + sz - 8;
      const uint32_t crc_st = tr[0] | (tr[1] << 8) | (tr[2] << 16) | ((uint32_t)tr[3] << 24);
      const uint32_t isz = tr[4] | (tr[5] << 8) | (tr[6] << 16) | ((uint32_t)tr[7] << 24);
      if (n + isz > cap) {
        while (n + isz > cap) cap *= 2;
        uint8_t* q = (uint8_t*)realloc(out, HEAD + cap);
        if (!q) { co.err = "out of memory"; break; }
        out = q;
      }
      inflateReset(&zs);
      zs.next_in = const_cast<Bytef*>(d_ + off + h); zs.avail_in = (uInt)(sz - h - 8);
      zs.next_out = out + HEAD + n; zs.avail_out = (uInt)isz;
      const int rc = inflate(&zs, Z_FINISH);
      if (rc != Z_STREAM_END || zs.avail_out != 0 || (uint32_t)crc32(0, out + HEAD + n, isz) != crc_st) { co.err = "corrupt BGZF member (inflate / CRC)"; break; }
      n += isz;
      off += sz;
    }
    inflateEnd(&zs);
    co.buf8 = out; co.n8 = n; co.cap8 = cap;
    co.next = i + 1;
    co.file_end = (i + 1 == nchunks_);
  }

  void decode_chunk(size_t i, ChunkOut& co, Tables& tab, Tables& scratch) {
    const uint64_t s = ensure_start(i, scratch);
    co.start_bit = s;
    co.next = i + 1;
    if (s == NONE) return;                 // nothing found here: the predecessor decodes through this range
    Decoder D;
    D.pool = pool_.get();
    D.br.init(d_, d_ + len_, s);
    D.markers = i != 0;
    if (D.markers) { if (!D.grow16((size_t)C_ * 5)) { co.err = D.err; return; } }
    else if (!D.grow8((size_t)C_ * 5)) { co.err = D.err; return; }
    size_t target = i + 1;                 // the chunk whose start we expect to hit
    uint64_t tbit = NONE;
    bool have_t = false;
    const uint64_t nominal_end = std::min<uint64_t>((uint64_t)(i + 1) * C_, len_) * 8;
    for (;;) {
      // a block boundary
      const uint64_t pos = D.br.bitpos();
      if (pos >= nominal_end) {
        bool stop_here = false;
        for (;;) {
          if (target >= nchunks_) break;                       // no chunk after: on to the end of the file
          if (!have_t) { tbit = ensure_start(target, scratch); have_t = true; }
          if (tbit == NONE || pos > tbit) { ++target; have_t = false; continue; }   // nothing there / a false positive
          if (pos == tbit) stop_here = true;
          break;
        }
        if (stop_here) { co.next = target; break; }
      }
      if (D.markers && D.m >= WSIZE && D.last_marker + WSIZE <= D.m) {
        if (!D.switch_to_bytes()) { co.err = D.err; break; }
      }
      if (D.br.cnt < 16) D.br.refill();
      const uint32_t hdr = D.br.get(3);
      const bool final_blk = hdr & 1;
      const uint32_t type = hdr >> 1;
      int rc = 0;
      if (type == 0) rc = D.stored();
      else if (type == 1) { const Tables& F = fixed_tables(); rc = D.markers ? D.codes<true>(F.lit, F.dist, F.pair) : D.codes<false>(F.lit, F.dist, F.pair); }
      else if (type == 2) {
        if (read_dynamic_header(D.br, tab, true) != 0) { D.err = "invalid dynamic block header"; rc = -1; }
        else rc = D.markers ? D.codes<true>(tab.lit, tab.dist, tab.pair) : D.codes<false>(tab.lit, tab.dist, tab.pair);
      } else { D.err = "invalid block type"; rc = -1; }
      if (rc != 0 || D.br.overrun) {
        co.err = "corrupt gzip data: " + (D.err.empty() ? std::string("unexpected end of the compressed data") : D.err);
        break;
      }
      if (!final_blk) continue;
      // end of a member: trailer, then the next member's header (or the end of the file)
      D.br.align_byte();
      const uint8_t* q = D.br.byte_ptr();
      if (d_ + len_ - q < 8) { co.err = "truncated gzip file (member trailer missing)"; break; }
      MemberEnd me;
      me.crc_stored = q[0] | (q[1] << 8) | (q[2] << 16) | ((uint32_t)q[3] << 24);
      me.isize_stored = q[4] | (q[5] << 8) | (q[6] << 16) | ((uint32_t)q[7] << 24);
      if (D.markers) { me.len8 = 0; me.crc8 = 0; }
      else { me.len8 = D.n - D.seg_start; me.crc8 = crc_of(D.out + HEAD + D.seg_start, me.len8); }
      co.ends.push_back(me);
      q += 8;
      // zero padding / trailing garbage after a member ends the file, as zlib's gzread treats it
      const size_t h = parse_gzip_header(q, d_ + len_, nullptr);
      if (D.markers) { D.markers = false; if (!D.grow8(1)) { co.err = D.err; break; } D.n = 0; }
      D.seg_start = D.n;
      if (!h) { co.file_end = true; co.next = nchunks_; break; }
      // a reference may not reach across the member start; distances are checked against n + valid_back, which is
      // (in wrapping arithmetic) the number of bytes of THIS member
      D.valid_back = (size_t)0 - D.n;
      D.br.init(d_, d_ + len_, (uint64_t)(q + h - d_) * 8);
    }
    if (co.err.empty() && !D.markers && D.out) {
      co.tail_len8 = D.n - D.seg_start;
      co.tail_crc8 = crc_of(D.out + HEAD + D.seg_start, co.tail_len8);
    }
    co.end_bit = D.br.bitpos();
    co.s16 = D.s16; co.m16 = D.m; co.cap16 = D.cap16;
    co.buf8 = D.out; co.n8 = D.n; co.cap8 = D.cap;
    D.s16 = nullptr; D.out = nullptr;
  }
};

}  // namespace pgz
}  // namespace sb
