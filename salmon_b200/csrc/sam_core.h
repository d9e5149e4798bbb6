// sam_core.h -- the per-record rules of the SAM output (DESIGN.md "SAM output").  Device code of the formatting kernels
// (sam.cu) and compiled for the host by the tests (tests/host_sam.cpp), so both write the same bytes.
//
// A fragment's alignments come from assign_read: transcript, read start `pos` of the first aligned mate (can be
// negative or run past the transcript end), `mate_pos`, flags (bit 0: first aligned mate forward, bit 1: mate 2
// forward, bits 2-3: mate status 0 pair / 1 mate 1 only / 2 mate 2 only), fragment length, and the per-mate DP scores
// of the SamSide output.  Every alignment of a pair gives two records, mate 1 first; a single-end read gives one.
#pragma once
#include <stdint.h>

#include "../../include/sb_detmath.h"

namespace sbsam {

struct Aln {
  uint32_t tid;
  int32_t pos, mate_pos;
  uint8_t flags;
  int32_t flen;
  int32_t score1, score2;
};

// One SAM line, before it is text.  rname / rnext are transcript ids ('=' when rnext equals rname).
struct Rec {
  uint32_t flag, mapq, nh;
  uint32_t tid;
  int32_t pos, pnext, tlen;          // 1-based POS / PNEXT
  uint32_t clip_l, match, clip_r;    // CIGAR (clip_l)S (match)M (clip_r)S; match == 0: '*'
  int32_t as;
  bool has_as, rnext_eq, rev;        // rev: SEQ reverse-complemented, QUAL reversed
};

SB_HD int32_t sam_pos1(int32_t p) { return (p < 0 ? 0 : p) + 1; }

// record `mate` (0 = mate 1, 1 = mate 2; always 0 for single-end reads) of alignment `idx` of a fragment with `nh`
// alignments; L = mapped read length, ref_len = indexed length of the transcript
SB_HD Rec sam_record(const Aln& a, uint32_t mate, uint32_t idx, uint32_t nh, bool paired, uint32_t L, uint32_t ref_len) {
  Rec r;
  const uint32_t status = (a.flags >> 2) & 3u;
  const bool fw_first = (a.flags & 1u) != 0, fw_mate = (a.flags & 2u) != 0;
  // which mates are aligned, where they start, which strand
  bool al[2] = {false, false}, rv[2] = {false, false};
  int32_t ps[2] = {0, 0};
  int32_t sc[2] = {a.score1, a.score2};
  if (!paired || status == 1) { al[0] = true; ps[0] = a.pos; rv[0] = !fw_first; }
  else if (status == 2) { al[1] = true; ps[1] = a.pos; rv[1] = !fw_first; }
  else { al[0] = al[1] = true; ps[0] = a.pos; rv[0] = !fw_first; ps[1] = a.mate_pos; rv[1] = !fw_mate; }
  const uint32_t o = 1u - mate;
  r.tid = a.tid;
  r.nh = nh;
  r.flag = idx ? 0x100u : 0u;
  r.tlen = 0;
  r.clip_l = r.match = r.clip_r = 0;
  r.has_as = al[mate];
  r.as = sc[mate];
  r.mapq = 255;
  if (al[mate]) {
    const int32_t p = ps[mate];
    r.pos = sam_pos1(p);
    r.rev = rv[mate];
    if (r.rev) r.flag |= 0x10u;
    // overhangs (rapmap's rule): bases before the transcript start or after its end are soft-clipped
    const int64_t lc = p < 0 ? -(int64_t)p : 0, end = (int64_t)p + (int64_t)L;
    r.clip_l = (uint32_t)(lc < (int64_t)L ? lc : (int64_t)L);
    const int64_t rc = end > (int64_t)ref_len ? end - (int64_t)ref_len : 0;
    r.clip_r = (uint32_t)(rc < (int64_t)(L - r.clip_l) ? rc : (int64_t)(L - r.clip_l));
    r.match = L - r.clip_l - r.clip_r;
  } else {   // the unaligned mate of an orphan: placed at its aligned mate
    r.flag |= 0x4u;
    r.pos = sam_pos1(ps[o]);
    r.rev = false;
  }
  if (!paired) {
    r.rnext_eq = false;
    r.pnext = 0;
    return r;
  }
  r.flag |= 0x1u | (mate ? 0x80u : 0x40u);
  r.rnext_eq = true;
  if (al[0] && al[1]) {
    r.flag |= 0x2u;
    if (rv[o]) r.flag |= 0x20u;
    r.pnext = sam_pos1(ps[o]);
    // positive on the leftmost mate (mate 1 on a tie)
    const bool left = ps[mate] < ps[o] || (ps[mate] == ps[o] && mate == 0);
    r.tlen = left ? a.flen : -a.flen;
  } else if (al[mate]) {
    r.flag |= 0x8u;
    r.pnext = r.pos;
  } else {
    if (rv[o]) r.flag |= 0x20u;
    r.pnext = r.pos;
  }
  return r;
}

SB_HD uint32_t ndig(uint32_t v) {
  uint32_t d = 1;
  while (v >= 10) { v /= 10; ++d; }
  return d;
}
SB_HD uint32_t sdig(int32_t v) { return v < 0 ? 1 + ndig((uint32_t)(-(int64_t)v)) : ndig((uint32_t)v); }
SB_HD uint32_t put_u(char* o, uint32_t v) {
  const uint32_t d = ndig(v);
  for (uint32_t i = d; i-- > 0;) { o[i] = (char)('0' + v % 10); v /= 10; }
  return d;
}
SB_HD uint32_t put_i(char* o, int32_t v) {
  if (v < 0) { o[0] = '-'; return 1 + put_u(o + 1, (uint32_t)(-(int64_t)v)); }
  return put_u(o, (uint32_t)v);
}
SB_HD uint32_t put_s(char* o, const char* s, uint32_t n) {
  for (uint32_t i = 0; i < n; ++i) o[i] = s[i];
  return n;
}

SB_HD uint32_t cigar_len(const Rec& r) {
  if (r.match == 0) return 1;
  return (r.clip_l ? ndig(r.clip_l) + 1 : 0) + ndig(r.match) + 1 + (r.clip_r ? ndig(r.clip_r) + 1 : 0);
}
// QNAME .. TLEN and the tab after it
SB_HD uint32_t head_len(const Rec& r, uint32_t name_len, uint32_t rname_len) {
  return name_len + 1 + ndig(r.flag) + 1 + rname_len + 1 + sdig(r.pos) + 1 + ndig(r.mapq) + 1 + cigar_len(r) + 1 +
         1 + 1 + sdig(r.pnext) + 1 + sdig(r.tlen) + 1;
}
SB_HD uint32_t head_write(char* o, const Rec& r, const char* name, uint32_t name_len, const char* rname, uint32_t rname_len) {
  uint32_t k = put_s(o, name, name_len);
  o[k++] = '\t'; k += put_u(o + k, r.flag);
  o[k++] = '\t'; k += put_s(o + k, rname, rname_len);
  o[k++] = '\t'; k += put_i(o + k, r.pos);
  o[k++] = '\t'; k += put_u(o + k, r.mapq);
  o[k++] = '\t';
  if (r.match == 0) o[k++] = '*';
  else {
    if (r.clip_l) { k += put_u(o + k, r.clip_l); o[k++] = 'S'; }
    k += put_u(o + k, r.match); o[k++] = 'M';
    if (r.clip_r) { k += put_u(o + k, r.clip_r); o[k++] = 'S'; }
  }
  o[k++] = '\t'; o[k++] = r.rnext_eq ? '=' : '*';
  o[k++] = '\t'; k += put_i(o + k, r.pnext);
  o[k++] = '\t'; k += put_i(o + k, r.tlen);
  o[k++] = '\t';
  return k;
}
// SEQ (L bases) '\t' QUAL (L characters, or '*') '\t': the body, written one character per index so that a warp can
// share it out; `i` in [0, body_len)
SB_HD uint32_t body_len(uint32_t L, bool qual) { return L + 1 + (qual ? L : 1) + 1; }
SB_HD char base_char(uint8_t b, bool ascii) {
  if (ascii) {
    const uint8_t u = (uint8_t)(b & 0xDF);
    return (u == 'A' || u == 'C' || u == 'G' || u == 'T') ? (char)u : (u == 'U' ? 'T' : 'N');
  }
  return b < 4 ? "ACGT"[b] : 'N';
}
SB_HD char comp_char(char c) { return c == 'A' ? 'T' : c == 'C' ? 'G' : c == 'G' ? 'C' : c == 'T' ? 'A' : 'N'; }
SB_HD char body_char(uint32_t i, uint32_t L, bool rev, const uint8_t* codes, const uint8_t* qual, bool ascii) {
  if (i < L) return rev ? comp_char(base_char(codes[L - 1 - i], ascii)) : base_char(codes[i], ascii);
  if (i == L) return '\t';
  if (!qual) return i == L + 1 ? '*' : '\t';
  if (i < 2 * L + 1) { const uint32_t q = i - L - 1; return (char)(rev ? qual[L - 1 - q] : qual[q]); }
  return '\t';
}
// NH:i:n [\tAS:i:s] \n
SB_HD uint32_t tail_len(const Rec& r) { return 5 + ndig(r.nh) + (r.has_as ? 6 + sdig(r.as) : 0) + 1; }
SB_HD uint32_t tail_write(char* o, const Rec& r) {
  uint32_t k = put_s(o, "NH:i:", 5);
  k += put_u(o + k, r.nh);
  if (r.has_as) { k += put_s(o + k, "\tAS:i:", 6); k += put_i(o + k, r.as); }
  o[k++] = '\n';
  return k;
}
SB_HD uint32_t rec_len(const Rec& r, uint32_t name_len, uint32_t rname_len, uint32_t L, bool qual) {
  return head_len(r, name_len, rname_len) + body_len(L, qual) + tail_len(r);
}

// aux_info/unmapped_names.txt type of a fragment (salmon::utils::str(MappingType), SalmonUtils.cpp:62-80), nullptr when
// the fragment is not listed (a concordant pair, a mapped single-end read)
SB_HD const char* unmapped_type(uint32_t n_out, bool decoy, uint8_t first_flags, bool paired) {
  if (decoy) return "d";
  if (n_out == 0) return "u";
  if (!paired) return nullptr;
  const uint32_t st = (first_flags >> 2) & 3u;
  return st == 0 ? nullptr : (st == 1 ? "m1" : "m2");
}
SB_HD uint32_t str_len(const char* s) {
  uint32_t n = 0;
  while (s[n]) ++n;
  return n;
}

}  // namespace sbsam
