// map_kernels.cuh -- Stage A hot kernels for sm_90a (warp-cooperative forms of MAPSPEC, map_core.h).
//
//   k_pack_reads   byte codes -> 2-bit packed reads + N masks (once per batch; both later kernels read 48 B
//                  per mate instead of L bytes)
//   k_seed_chain_w one WARP per read pair.  Lanes = seed positions: the hash probes and the posting reads of
//                  a mate are all in flight together (memory-level parallelism instead of a serial per-thread
//                  walk); seeds are expanded into a per-warp shared-memory key array by a warp prefix sum,
//                  bitonic-sorted there, chained by a segmented warp scan (coverage bit masks OR-ed along each
//                  chain), filtered, paired, and the DP task list is written with one atomic per read.
//   k_dp_classify  one warp per mate alignment.  Lanes = band diagonals evaluate the 2*band+1 ungapped alignments
//                  by XOR/popcount on 2-bit words; when the best of them is within (go+ge) of a perfect score no
//                  gapped path can beat it.  The rest is queued for
//   k_dp_pair      the banded affine DP (same recurrences as dp_score_serial), two alignments per warp, two band
//                  cells per lane, read and reference window in registers (no memory access in the row loop), or
//   k_dp_general   (band leaves the transcript, or an N is involved: rare).
//
// All three produce exactly what the serial forms in map_core.h produce (tests/test_map_gpu.py compares the
// CUDA path with the independent oracle bit for bit).
#pragma once
#include "map_core.h"

namespace sbmap {

constexpr int SEED_WARPS = 8;        // warps per block of k_seed_chain_w
constexpr int SK = 512;              // seed keys per warp held in shared memory (more: global scratch)
constexpr uint32_t MAX_LOOKUPS = 64; // seed positions per mate handled by the warp kernel (2 rounds of 32)
constexpr uint32_t MAX_READ_OCC = 1000;   // largest max_read_occ (--maxReadOcc; the value --mimicBT2 sets)

struct PackedReads {
  uint64_t* bits;    // [(2*n) * wpr]  base j of a mate at bits 2*(j&31) of word j>>5 (N stored as 0)
  uint64_t* nmask;   // [(2*n) * mpr]  bit j set: base j is N
  uint32_t wpr, mpr; // words per mate: ceil(Lcap/32)+1 (one zero guard word), ceil(Lcap/64)+1
};

// reverse the order of the 32 two-bit groups of a word
__device__ __forceinline__ uint64_t brev2(uint64_t x) {
  const uint64_t y = __brevll(x);
  return ((y >> 1) & 0x5555555555555555ull) | ((y & 0x5555555555555555ull) << 1);
}
// 64-bit window starting `sh` bits into lo (sh in 0..63), continuing into hi
__device__ __forceinline__ uint64_t funnel64(uint64_t lo, uint64_t hi, uint32_t sh) {
  return sh ? ((lo >> sh) | (hi << (64 - sh))) : lo;
}

// ---------------------------------------------------------------------------------------------
// k_pack_reads: one thread per (mate, 32-base word)
// ---------------------------------------------------------------------------------------------
// ascii != 0: the input bytes are sequence characters (A C G T, any case; everything else is N) as the reference's
// parser hands them over (klibpp::KSeq::seq), instead of base codes 0..4
__global__ void k_pack_reads(const uint8_t* __restrict__ left, const uint8_t* __restrict__ right, uint32_t n,
                             uint32_t L, PackedReads pr, int ascii) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t total = (uint64_t)2 * n * pr.wpr;
  if (t >= total) return;
  const uint32_t w = (uint32_t)(t % pr.wpr);
  const uint64_t m = t / pr.wpr;               // mate index: 2*r + mate
  const uint8_t* src = ((m & 1) ? right : left) + (m >> 1) * L;
  uint64_t bits = 0;
  uint32_t nm = 0;
  const uint32_t b0 = w * 32;
  for (uint32_t j = 0; j < 32; ++j) {
    const uint32_t q = b0 + j;
    if (q >= L) break;
    uint8_t c = src[q];
    if (ascii) {
      const uint8_t u = c & 0xDFu;      // upper case
      c = (u == 'A') ? 0 : (u == 'C') ? 1 : (u == 'G') ? 2 : (u == 'T') ? 3 : 4;
    }
    if (c > 3) nm |= 1u << j;
    else bits |= (uint64_t)c << (2 * j);
  }
  pr.bits[m * pr.wpr + w] = bits;
  // the N mask of word w is half of mask word w>>1: two threads of the same mate share a word
  if (w < 2 * pr.mpr) {
    uint32_t* nm32 = reinterpret_cast<uint32_t*>(pr.nmask + m * pr.mpr);
    nm32[w] = nm;
  }
}

// ---------------------------------------------------------------------------------------------
// k_seed_chain_w
// ---------------------------------------------------------------------------------------------
struct SeedOut {
  uint32_t* n_l; uint32_t* n_r;
  Cand* cand_l; Cand* cand_r;
  uint32_t* n_tasks; uint32_t* tasks;
  uint64_t* overflow_keys;   // [n_warps * MAXSEEDS]
  Counters* ctr;
};

// candidate packed like a seed key with the coverage in the qpos field
__device__ __forceinline__ uint64_t cand_word(uint64_t key, int32_t diag_c, uint32_t cov) {
  return (key & 0xffffffff80000000ull) | ((uint64_t)(uint32_t)(diag_c + (1 << 21)) << 9) | (uint64_t)cov;
}
__device__ __forceinline__ uint32_t cw_cov(uint64_t w) { return (uint32_t)(w & 0x1ffu); }

// (cov desc, tid, ori, diag_c) order of the oracle's cmp_cand_cov: does a beat b?
__device__ __forceinline__ bool cand_beats(uint64_t a, uint64_t b) {
  const uint32_t ca = cw_cov(a), cb = cw_cov(b);
  if (ca != cb) return ca > cb;
  return (a >> 9) < (b >> 9);
}

// general path of warp_mate_candidates: every seed becomes a key, bitonic sort of all of them
template <int RD>
__device__ __noinline__ void seeds_sort_all(const IndexView& ix, uint32_t span, const uint32_t (&off)[RD],
                                            const uint32_t (&cnt)[RD], const uint32_t (&meta)[RD],
                                            const uint32_t (&excl)[RD], const uint32_t (&tot)[RD], uint32_t T,
                                            uint64_t* keys, uint32_t lane) {
    uint32_t n2 = 32;
    while (n2 < T) n2 <<= 1;
    uint32_t carry = 0;
#pragma unroll
    for (int rd = 0; rd < RD; ++rd) {
      for (uint32_t it = 0; it < tot[rd]; it += 32) {
        const uint32_t item = it + lane;
        uint32_t lo = 0;
#pragma unroll
        for (int st = 16; st > 0; st >>= 1) {
          const uint32_t e = __shfl_sync(0xffffffffu, excl[rd], lo + st);
          if (e <= item) lo += st;
        }
        const uint32_t o_off = __shfl_sync(0xffffffffu, off[rd], lo);
        const uint32_t o_excl = __shfl_sync(0xffffffffu, excl[rd], lo);
        const uint32_t o_meta = __shfl_sync(0xffffffffu, meta[rd], lo);
        const uint32_t slot = carry + item;
        if (item < tot[rd] && slot < (uint32_t)MAXSEEDS) {
          const Posting po = ix.post[o_off + (item - o_excl)];
          const uint32_t pos_i = o_meta & 0xffffu;
          const uint32_t ori = (o_meta >> 16) ^ (po.tpos_rc >> 31);
          const int32_t qpos = ori ? (int32_t)(span - pos_i) : (int32_t)pos_i;
          keys[slot] = seed_key(po.tid, ori, (int32_t)(po.tpos_rc & 0x7fffffffu) - qpos, qpos);
        }
      }
      carry += tot[rd];
    }
    for (uint32_t i = T + lane; i < n2; i += 32) keys[i] = EMPTY_KEY;
    __syncwarp();
    for (uint32_t k = 2; k <= n2; k <<= 1)
      for (uint32_t j = k >> 1; j > 0; j >>= 1) {
        for (uint32_t t = lane; t < (n2 >> 1); t += 32) {
          const uint32_t i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
          const uint32_t l = i | j;
          const uint64_t a = keys[i], b = keys[l];
          const bool asc = (i & k) == 0;
          if ((a > b) == asc) { keys[i] = b; keys[l] = a; }
        }
        __syncwarp();
      }
}

// more than MAXCAND survivors (rare): keep the MAXCAND best by (coverage desc, tid, ori, diag)
__device__ __noinline__ void cands_top(const uint64_t* keys, uint32_t N, double thr, uint64_t* cands, uint32_t lane) {
    // rare: keep the MAXCAND best by (coverage desc, tid, ori, diag); rank by counting who beats whom
    uint32_t out = 0;
    for (uint32_t base = 0; base < N; base += 32) {
      const uint32_t i = base + lane;
      const uint64_t w = (i < N) ? keys[i] : EMPTY_KEY;
      const bool surv = (w != EMPTY_KEY) && ((double)cw_cov(w) >= thr);
      uint32_t beaten_by = 0;
      for (uint32_t q = 0; q < N; ++q) {
        const uint64_t x = keys[q];
        if (x != EMPTY_KEY && (double)cw_cov(x) >= thr && surv && cand_beats(x, w)) ++beaten_by;
      }
      const bool keep = surv && beaten_by < (uint32_t)MAXCAND;
      const uint32_t bal = __ballot_sync(0xffffffffu, keep);
      const uint32_t rank = out + (uint32_t)__popc(bal & ((1u << lane) - 1));
      if (keep) cands[rank] = w;
      out += (uint32_t)__popc(bal);
    }

}

constexpr uint32_t HS = 128;         // slots of the per-warp diagonal table (hash mode)
template <int CW> struct SeedRegion { static constexpr uint32_t WORDS = HS + HS * CW + HS; };   // keys | masks | dense
static_assert(SeedRegion<2>::WORDS == (uint32_t)SK, "sort mode reuses the table region");

// Candidates of one mate.  Seeds with the same (transcript, orientation, diagonal) only differ in the read bases
// they cover, and a read's seeds fall on a handful of diagonals (one per isoform), so the seeds are first merged
// per diagonal in a small shared-memory hash table (coverage masks OR-ed with shared atomics); only the distinct
// diagonals are sorted (in registers when there are <= 32) and chained.  If the table overflows (repeats), the
// general path sorts all seeds instead.  Both paths give what mate_candidates() (map_core.h) gives.
//   region: SeedRegion<CW>::WORDS words of shared memory;  gkeys: MAXSEEDS words of global scratch (T > SK)
template <int CW, int RD>   // coverage words: 2 for read_len <= 128, 4 for <= 256; lookup rounds of 32 positions
__device__ __forceinline__ uint32_t warp_mate_candidates(const IndexView& ix, const Params& p,
                                                         const uint64_t* __restrict__ rbits,   // shared: wpr words
                                                         const uint64_t* __restrict__ rnm,     // shared: mpr words
                                                         uint32_t L, uint64_t* region, uint64_t* gkeys,
                                                         uint64_t* cands /* shared, MAXCAND */, Counters& ctr,
                                                         uint32_t lane) {
  const uint32_t K = p.k;
  const uint64_t kmask = (1ull << (2 * K)) - 1;
  const uint32_t span = L - K;
  uint32_t npos = span / p.stride + 1;
  if (span % p.stride) ++npos;
  // ---- lookups: lane + 32*round = seed position index
  uint32_t off[RD], cnt[RD], meta[RD];   // meta: pos_i | read_rc << 16
  uint32_t n_valid = 0;
#pragma unroll
  for (int rd = 0; rd < RD; ++rd) {
    const uint32_t li = lane + 32u * rd;
    off[rd] = 0; cnt[rd] = 0; meta[rd] = 0;
    if (li < npos) {
      uint32_t pos_i = li * p.stride;
      if (pos_i > span) pos_i = span;
      const uint32_t wi = pos_i >> 5, sh = 2 * (pos_i & 31);
      const uint64_t fwle = funnel64(rbits[wi], rbits[wi + 1], sh) & kmask;
      const uint32_t mi = pos_i >> 6, msh = pos_i & 63;
      const uint64_t nwin = funnel64(rnm[mi], rnm[mi + 1], msh) & ((1ull << K) - 1);
      if (nwin == 0) {
        const uint64_t fw = brev2(fwle) >> (64 - 2 * K);
        const uint64_t rc = (~fwle) & kmask;
        const uint64_t canon = fw < rc ? fw : rc;
        ++n_valid;
        uint32_t o, c;
        if (index_lookup(ix, canon, o, c) && c <= p.max_occs_per_hit) {
          off[rd] = o; cnt[rd] = c;
          meta[rd] = pos_i | ((fw < rc ? 0u : 1u) << 16);
        }
      }
    }
  }
  // ---- slots: exclusive prefix over the lookups in position order
  uint32_t excl[RD], tot[RD];
#pragma unroll
  for (int rd = 0; rd < RD; ++rd) {
    uint32_t x = cnt[rd];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
      if ((int)lane >= o) x += y;
    }
    tot[rd] = __shfl_sync(0xffffffffu, x, 31);
    excl[rd] = x - cnt[rd];
  }
  uint32_t total = 0;
#pragma unroll
  for (int rd = 0; rd < RD; ++rd) total += tot[rd];
  const uint32_t T = total < (uint32_t)MAXSEEDS ? total : (uint32_t)MAXSEEDS;
  if (lane == 0) { ctr.postings += T; ctr.seeds += T; }
  ctr.lookups += n_valid;     // per lane; summed when the counters are flushed
  if (T == 0) return 0;

  uint64_t* tkeys = region;                 // [HS]
  uint64_t* tmask = region + HS;            // [HS * CW]
  uint64_t* dense = region + HS + HS * CW;  // [HS]
  uint64_t* keys = nullptr;                 // the sorted array the chain pass walks
  uint32_t N = 0;                           // its length
  bool hash_mode = true;
  // ---- hash mode: merge the seeds per diagonal
  for (uint32_t i = lane; i < HS; i += 32) tkeys[i] = EMPTY_KEY;
  for (uint32_t i = lane; i < HS * CW; i += 32) tmask[i] = 0ull;
  __syncwarp();
  {
    bool failed = false;
    uint32_t carry = 0;
#pragma unroll
    for (int rd = 0; rd < RD; ++rd) {
      for (uint32_t it = 0; it < tot[rd]; it += 32) {
        const uint32_t item = it + lane;
        uint32_t lo = 0;
#pragma unroll
        for (int st = 16; st > 0; st >>= 1) {
          const uint32_t e = __shfl_sync(0xffffffffu, excl[rd], lo + st);
          if (e <= item) lo += st;
        }
        const uint32_t o_off = __shfl_sync(0xffffffffu, off[rd], lo);
        const uint32_t o_excl = __shfl_sync(0xffffffffu, excl[rd], lo);
        const uint32_t o_meta = __shfl_sync(0xffffffffu, meta[rd], lo);
        const uint32_t slot = carry + item;
        if (item < tot[rd] && slot < (uint32_t)MAXSEEDS) {
          const Posting po = ix.post[o_off + (item - o_excl)];
          const uint32_t pos_i = o_meta & 0xffffu;
          const uint32_t ori = (o_meta >> 16) ^ (po.tpos_rc >> 31);
          const int32_t qpos = ori ? (int32_t)(span - pos_i) : (int32_t)pos_i;
          const uint64_t kd = seed_key(po.tid, ori, (int32_t)(po.tpos_rc & 0x7fffffffu) - qpos, 0);
          uint32_t h = (uint32_t)(((kd >> 9) * 0x9E3779B97F4A7C15ull) >> 57);
          bool done = false;
          for (uint32_t pr = 0; pr < 32 && !done; ++pr) {
            const unsigned long long old = atomicCAS((unsigned long long*)&tkeys[h], (unsigned long long)EMPTY_KEY,
                                                     (unsigned long long)kd);
            if (old == (unsigned long long)EMPTY_KEY || old == (unsigned long long)kd) {
#pragma unroll
              for (int w = 0; w < CW; ++w) {
                int32_t lo2 = qpos - 64 * w, hi2 = lo2 + (int32_t)K;
                lo2 = lo2 < 0 ? 0 : lo2;
                hi2 = hi2 > 64 ? 64 : hi2;
                if (lo2 < hi2) atomicOr((unsigned long long*)&tmask[h * CW + w], (unsigned long long)(((1ull << (hi2 - lo2)) - 1) << lo2));
              }
              done = true;
            } else {
              h = (h + 1) & (HS - 1);
            }
          }
          failed |= !done;
        }
      }
      carry += tot[rd];
    }
    __syncwarp();
    if (__any_sync(0xffffffffu, failed)) hash_mode = false;
  }
  if (hash_mode) {
    // ---- compact the table: dense[] = diagonal key | slot index (low bits, where qpos would be)
    uint32_t nd = 0;
#pragma unroll
    for (uint32_t s0 = 0; s0 < HS; s0 += 32) {
      const uint32_t sidx = s0 + lane;
      const uint64_t k = tkeys[sidx];
      const bool v = k != EMPTY_KEY;
      const uint32_t bal = __ballot_sync(0xffffffffu, v);
      if (v) dense[nd + (uint32_t)__popc(bal & ((1u << lane) - 1))] = k | (uint64_t)sidx;
      nd += (uint32_t)__popc(bal);
    }
    __syncwarp();
    N = nd;
    keys = dense;
    if (nd <= 32) {
      // one key per lane: bitonic network on shuffles
      uint64_t k = lane < nd ? dense[lane] : EMPTY_KEY;
#pragma unroll
      for (uint32_t kk = 2; kk <= 32; kk <<= 1)
#pragma unroll
        for (uint32_t j = kk >> 1; j > 0; j >>= 1) {
          const uint64_t o = __shfl_xor_sync(0xffffffffu, k, j);
          const bool keep_min = ((lane & j) == 0) == ((lane & kk) == 0);
          k = keep_min ? (k < o ? k : o) : (k > o ? k : o);
        }
      __syncwarp();
      dense[lane] = k;
      __syncwarp();
    } else {
      uint32_t n2 = 64;
      while (n2 < nd) n2 <<= 1;
      for (uint32_t i = nd + lane; i < n2; i += 32) dense[i] = EMPTY_KEY;
      __syncwarp();
      for (uint32_t k = 2; k <= n2; k <<= 1)
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
          for (uint32_t t = lane; t < (n2 >> 1); t += 32) {
            const uint32_t i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
            const uint32_t l = i | j;
            const uint64_t a = dense[i], b = dense[l];
            const bool asc = (i & k) == 0;
            if ((a > b) == asc) { dense[i] = b; dense[l] = a; }
          }
          __syncwarp();
        }
    }
  } else {
    // ---- general path (rare): all seeds as keys, bitonic sort -- kept out of line so that the common path stays
    //      small in the instruction cache
    keys = (T <= (uint32_t)SK) ? region : gkeys;
    N = T;
    seeds_sort_all<RD>(ix, span, off, cnt, meta, excl, tot, T, keys, lane);
  }
  // ---- chains: segmented scan over the sorted keys; the tail of every chain is replaced by its
  //      candidate word, every other slot by EMPTY
  uint32_t best = 0;
  uint64_t carry_key = EMPTY_KEY;
  uint64_t carry_m[CW];
  int32_t carry_dmin = 0;
#pragma unroll
  for (int w = 0; w < CW; ++w) carry_m[w] = 0;
  const int32_t gap = (int32_t)p.chain_gap;
  for (uint32_t base = 0; base < N; base += 32) {
    const uint32_t i = base + lane;
    const bool active = i < N;
    const uint64_t k = active ? keys[i] : EMPTY_KEY;
    uint64_t kprev = __shfl_up_sync(0xffffffffu, k, 1);
    if (lane == 0) kprev = carry_key;
    uint64_t knext = __shfl_down_sync(0xffffffffu, k, 1);
    if (lane == 31) knext = (i + 1 < N) ? keys[i + 1] : EMPTY_KEY;
    const int32_t dg = key_diag(k);
    const bool head = active && (i == 0 || (kprev >> 31) != (k >> 31) || dg - key_diag(kprev) > gap);
    const bool tail = active && (i + 1 >= N || (knext >> 31) != (k >> 31) || key_diag(knext) - dg > gap);
    uint64_t m[CW];
    if (hash_mode) {
      const uint32_t sidx = (uint32_t)(k & (HS - 1));
#pragma unroll
      for (int w = 0; w < CW; ++w) m[w] = active ? tmask[sidx * CW + w] : 0ull;
    } else {
      const int32_t q = key_qpos(k);
#pragma unroll
      for (int w = 0; w < CW; ++w) {
        int32_t lo = q - 64 * w, hi = lo + (int32_t)K;
        lo = lo < 0 ? 0 : lo;
        hi = hi > 64 ? 64 : hi;
        m[w] = (active && lo < hi) ? (((1ull << (hi - lo)) - 1) << lo) : 0ull;
      }
    }
    int32_t dmin = dg;
    uint32_t f = head ? 1u : 0u;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t pf = __shfl_up_sync(0xffffffffu, f, o);
      const int32_t pd = __shfl_up_sync(0xffffffffu, dmin, o);
      uint64_t pm[CW];
#pragma unroll
      for (int w = 0; w < CW; ++w) pm[w] = __shfl_up_sync(0xffffffffu, m[w], o);
      if ((int)lane >= o && !f) {
#pragma unroll
        for (int w = 0; w < CW; ++w) m[w] |= pm[w];
        dmin = pd;
        f = pf;
      }
    }
    if (!f) {   // the chain started in an earlier chunk
#pragma unroll
      for (int w = 0; w < CW; ++w) m[w] |= carry_m[w];
      dmin = carry_dmin;
    }
    carry_key = __shfl_sync(0xffffffffu, k, 31);
    carry_dmin = __shfl_sync(0xffffffffu, dmin, 31);
#pragma unroll
    for (int w = 0; w < CW; ++w) carry_m[w] = __shfl_sync(0xffffffffu, m[w], 31);
    uint32_t cov = 0;
#pragma unroll
    for (int w = 0; w < CW; ++w) cov += (uint32_t)__popcll(m[w]);
    if (tail && cov > best) best = cov;
    __syncwarp();
    if (active) keys[i] = tail ? cand_word(k, dmin + (dg - dmin) / 2, cov) : EMPTY_KEY;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const uint32_t y = __shfl_xor_sync(0xffffffffu, best, o);
    best = y > best ? y : best;
  }
  __syncwarp();
  // ---- survivors (coverage >= consensus_frac * best), in (tid, ori, diag) order
  const double thr = p.consensus_frac * (double)best;
  uint32_t nc = 0;
  for (uint32_t base = 0; base < N; base += 32) {
    const uint32_t i = base + lane;
    const uint64_t w = (i < N) ? keys[i] : EMPTY_KEY;
    const bool keep = (w != EMPTY_KEY) && ((double)cw_cov(w) >= thr);
    const uint32_t bal = __ballot_sync(0xffffffffu, keep);
    const uint32_t rank = nc + (uint32_t)__popc(bal & ((1u << lane) - 1));
    if (keep && rank < (uint32_t)MAXCAND) cands[rank] = w;
    nc += (uint32_t)__popc(bal);
  }
  if (nc > (uint32_t)MAXCAND) { cands_top(keys, N, thr, cands, lane); nc = (uint32_t)MAXCAND; }
  __syncwarp();
  return nc;
}

__device__ __forceinline__ uint32_t cwd_tid(uint64_t w) { return (uint32_t)(w >> 32); }
__device__ __forceinline__ uint32_t cwd_ori(uint64_t w) { return (uint32_t)(w >> 31) & 1u; }
__device__ __forceinline__ int32_t cwd_diag(uint64_t w) { return (int32_t)((w >> 9) & 0x3fffffu) - (1 << 21); }

template <int CW> struct SeedCfg { static constexpr int WARPS = (CW == 2) ? 8 : 6; };   // <= 48 KB static shared memory

template <int CW, int RD>
__global__ void __launch_bounds__(SeedCfg<CW>::WARPS * 32, 4)
k_seed_chain_w(IndexView ix, Params p, PackedReads pr, uint32_t n, uint32_t L, SeedOut o) {
  constexpr int WPB = SeedCfg<CW>::WARPS;
  __shared__ uint64_t s_keys[WPB][SeedRegion<CW>::WORDS];
  __shared__ uint64_t s_cand[WPB][2][MAXCAND];
  __shared__ uint64_t s_read[WPB][16];   // wpr (<= 9) + mpr (<= 5) words of the current mate
  const uint32_t lane = threadIdx.x & 31u, wib = threadIdx.x >> 5;
  const uint32_t warp = blockIdx.x * WPB + wib, nwarps = gridDim.x * WPB;
  uint64_t* gkeys = o.overflow_keys + (size_t)warp * MAXSEEDS;
  Counters ctr;
  ctr.lookups = ctr.postings = ctr.seeds = ctr.candidates = ctr.kept = ctr.label_entries = ctr.mapped = 0;
  ctr.lib_mask_sum[0] = ctr.lib_mask_sum[1] = ctr.lib_mask_sum[2] = ctr.lib_mask_sum[3] = 0;
  for (uint32_t r = warp; r < n; r += nwarps) {
    uint32_t ncand[2];
#pragma unroll 1
    for (int mate = 0; mate < 2; ++mate) {
      const uint64_t mi = (uint64_t)2 * r + mate;
      __syncwarp();
      if (lane < pr.wpr) s_read[wib][lane] = pr.bits[mi * pr.wpr + lane];
      else if (lane < pr.wpr + pr.mpr) s_read[wib][lane] = pr.nmask[mi * pr.mpr + (lane - pr.wpr)];
      __syncwarp();
      ncand[mate] = warp_mate_candidates<CW, RD>(ix, p, s_read[wib], s_read[wib] + pr.wpr, L, s_keys[wib], gkeys,
                                             s_cand[wib][mate], ctr, lane);
    }
    const uint32_t nl = ncand[0], nr = ncand[1];
    const uint64_t* cl = s_cand[wib][0];
    const uint64_t* cr = s_cand[wib][1];
    // ---- joint hits (IU) under the join policy of map_core.h::for_each_joint (the same five rules, lanes = left
    //      candidates): which candidates take part in a joint hit (they need a DP score), and how many joint hits
    __syncwarp();
    uint32_t* s_best = reinterpret_cast<uint32_t*>(s_keys[wib]);     // [64] best pair score per left candidate (scratch:
                                                                     // the seed keys are not needed any more)
    // (1) pre-merge masks
    bool kl[2] = {false, false}, kr[2] = {false, false};
#pragma unroll
    for (int rd = 0; rd < 2; ++rd) {
      const uint32_t a = lane + 32u * rd;
      if (a < nl) {
        uint32_t best = 0;
        for (uint32_t q = 0; q < nl; ++q) if (cwd_tid(cl[q]) == cwd_tid(cl[a])) best = max(best, cw_cov(cl[q]));
        kl[rd] = (double)cw_cov(cl[a]) >= p.pre_merge_thresh * (double)best;
      }
      if (a < nr) {
        uint32_t best = 0;
        for (uint32_t q = 0; q < nr; ++q) if (cwd_tid(cr[q]) == cwd_tid(cr[a])) best = max(best, cw_cov(cr[q]));
        kr[rd] = (double)cw_cov(cr[a]) >= p.pre_merge_thresh * (double)best;
      }
    }
    const unsigned long long keep_l = (unsigned long long)__ballot_sync(0xffffffffu, kl[0]) |
                                      ((unsigned long long)__ballot_sync(0xffffffffu, kl[1]) << 32);
    const unsigned long long keep_r = (unsigned long long)__ballot_sync(0xffffffffu, kr[0]) |
                                      ((unsigned long long)__ballot_sync(0xffffffffu, kr[1]) << 32);
    auto geometry = [&](uint64_t wa, uint64_t wb) -> bool {          // (2) a concordant pair?
      if (cwd_tid(wa) != cwd_tid(wb) || cwd_ori(wa) == cwd_ori(wb)) return false;
      const int32_t dfw = cwd_ori(wa) == 0 ? cwd_diag(wa) : cwd_diag(wb);
      const int32_t drv = cwd_ori(wa) == 0 ? cwd_diag(wb) : cwd_diag(wa);
      int32_t start = dfw, end = drv + (int32_t)L;
      if (drv < dfw) {
        if (!p.allow_dovetail) return false;
        start = drv; end = dfw + (int32_t)L;
      }
      const int32_t fl = end - start;
      return fl > 0 && fl <= (int32_t)p.max_frag_len;
    };
    // best pair score per left candidate, of the read
    uint32_t my_best[2] = {0, 0};
#pragma unroll
    for (int rd = 0; rd < 2; ++rd) {
      const uint32_t a = lane + 32u * rd;
      if (a < nl && ((keep_l >> a) & 1ull)) {
        const uint64_t wa = cl[a];
        for (uint32_t b = 0; b < nr; ++b)
          if (((keep_r >> b) & 1ull) && geometry(wa, cr[b])) my_best[rd] = max(my_best[rd], cw_cov(wa) + cw_cov(cr[b]));
      }
      if (a < 64u) s_best[a] = my_best[rd];
    }
    uint32_t best_all = max(my_best[0], my_best[1]);
#pragma unroll
    for (int sft = 16; sft > 0; sft >>= 1) best_all = max(best_all, __shfl_xor_sync(0xffffffffu, best_all, sft));
    __syncwarp();
    // (3) + (4): count the surviving pairs, mark their candidates
    uint32_t my_cnt = 0;
    unsigned long long my_used_r = 0ull;
    bool used_a[2] = {false, false};
#pragma unroll
    for (int rd = 0; rd < 2; ++rd) {
      const uint32_t a = lane + 32u * rd;
      if (a < nl && my_best[rd] > 0) {
        const uint64_t wa = cl[a];
        uint32_t best_t = 0;                                         // best pair score on this transcript
        for (uint32_t q = 0; q < nl; ++q) if (cwd_tid(cl[q]) == cwd_tid(wa)) best_t = max(best_t, s_best[q]);
        for (uint32_t b = 0; b < nr; ++b) {
          if (!((keep_r >> b) & 1ull) || !geometry(wa, cr[b])) continue;
          const double sc = (double)(cw_cov(wa) + cw_cov(cr[b]));
          if (sc < p.post_merge_thresh * (double)best_t || sc < p.consensus_frac * (double)best_all) continue;
          ++my_cnt;
          my_used_r |= 1ull << b;
          used_a[rd] = true;
        }
      }
    }
    unsigned long long used_l = (unsigned long long)__ballot_sync(0xffffffffu, used_a[0]) |
                                ((unsigned long long)__ballot_sync(0xffffffffu, used_a[1]) << 32);
    unsigned long long used_r = my_used_r;
    uint32_t nj = my_cnt;
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
      nj += __shfl_xor_sync(0xffffffffu, nj, s);
      used_r |= __shfl_xor_sync(0xffffffffu, used_r, s);
    }
    if (nj == 0 && p.allow_orphans) {   // (5) orphans above the orphan threshold
      uint32_t best_c = 0;
#pragma unroll
      for (int rd = 0; rd < 2; ++rd) {
        const uint32_t a = lane + 32u * rd;
        if (a < nl && ((keep_l >> a) & 1ull)) best_c = max(best_c, cw_cov(cl[a]));
        if (a < nr && ((keep_r >> a) & 1ull)) best_c = max(best_c, cw_cov(cr[a]));
      }
#pragma unroll
      for (int sft = 16; sft > 0; sft >>= 1) best_c = max(best_c, __shfl_xor_sync(0xffffffffu, best_c, sft));
      const double thr = (p.lib_type >= 3 ? 0.0 : p.orphan_thresh) * (double)best_c;
      bool ol[2], orr[2];
#pragma unroll
      for (int rd = 0; rd < 2; ++rd) {
        const uint32_t a = lane + 32u * rd;
        ol[rd] = a < nl && ((keep_l >> a) & 1ull) && (double)cw_cov(cl[a]) >= thr;
        orr[rd] = a < nr && ((keep_r >> a) & 1ull) && (double)cw_cov(cr[a]) >= thr;
      }
      used_l = (unsigned long long)__ballot_sync(0xffffffffu, ol[0]) | ((unsigned long long)__ballot_sync(0xffffffffu, ol[1]) << 32);
      used_r = (unsigned long long)__ballot_sync(0xffffffffu, orr[0]) | ((unsigned long long)__ballot_sync(0xffffffffu, orr[1]) << 32);
      nj = (uint32_t)(__popcll(used_l) + __popcll(used_r));
    }
    __syncwarp();      // s_best lives in the key scratch of the next read's seeds
    // ---- write the candidates and the DP tasks
    for (uint32_t a = lane; a < nl; a += 32) {
      Cand c; c.tid = cwd_tid(cl[a]); c.diag_c = cwd_diag(cl[a]); c.ori_cov = (cwd_ori(cl[a]) << 31) | cw_cov(cl[a]);
      o.cand_l[(size_t)r * MAXCAND + a] = c;
    }
    for (uint32_t a = lane; a < nr; a += 32) {
      Cand c; c.tid = cwd_tid(cr[a]); c.diag_c = cwd_diag(cr[a]); c.ori_cov = (cwd_ori(cr[a]) << 31) | cw_cov(cr[a]);
      o.cand_r[(size_t)r * MAXCAND + a] = c;
    }
    const bool unmapped = (nj == 0 || nj > p.max_read_occ);
    if (lane == 0) { o.n_l[r] = unmapped ? (nl | 0x80000000u) : nl; o.n_r[r] = nr; }
    if (!unmapped) {
      const uint32_t cl_n = (uint32_t)__popcll(used_l), cnt = cl_n + (uint32_t)__popcll(used_r);
      uint32_t slot = 0;
      if (lane == 0) { slot = atomicAdd(o.n_tasks, cnt); ctr.candidates += cnt; }
      slot = __shfl_sync(0xffffffffu, slot, 0);
#pragma unroll
      for (int rd = 0; rd < 2; ++rd) {
        const uint32_t a = lane + 32u * rd;
        if ((used_l >> a) & 1ull) o.tasks[slot + (uint32_t)__popcll(used_l & ((1ull << a) - 1))] = (r << 7) | a;
        if ((used_r >> a) & 1ull) o.tasks[slot + cl_n + (uint32_t)__popcll(used_r & ((1ull << a) - 1))] = (r << 7) | 64u | a;
      }
    }
  }
  // flush counters: lookups are per lane, the rest live in lane 0
  unsigned long long lk = ctr.lookups;
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) lk += __shfl_xor_sync(0xffffffffu, lk, s);
  if (lane == 0) {
    if (lk) atomicAdd(&o.ctr->lookups, lk);
    if (ctr.postings) atomicAdd(&o.ctr->postings, ctr.postings);
    if (ctr.seeds) atomicAdd(&o.ctr->seeds, ctr.seeds);
    if (ctr.candidates) atomicAdd(&o.ctr->candidates, ctr.candidates);
  }
}

// ---------------------------------------------------------------------------------------------
// DP scoring: k_dp_classify -> { k_dp_pair , k_dp_general }
// ---------------------------------------------------------------------------------------------
struct DpIo {
  const uint32_t* n_tasks; const uint32_t* tasks;
  const Cand* cand_l; const Cand* cand_r;
  int32_t* score_l; int32_t* score_r;
  uint32_t* next_task;            // dynamic task counter of k_dp_classify
  uint32_t* list_n;               // [0] interior alignments, [1] edge alignments, [2] alignments with N
  uint32_t* list_int; uint32_t* list_edge; uint32_t* list_n_tasks;   // task words
  unsigned long long* n_full_dp;  // statistics: alignments that needed the banded DP
};

// byte-code form (transcripts with N, reads with N): lanes = band cells, one reference byte per row
__device__ __forceinline__ uint8_t base_code(uint8_t c, int ascii) {   // same mapping as k_pack_reads
  if (!ascii) return c;
  const uint8_t u = c & 0xDFu;
  return (u == 'A') ? 0 : (u == 'C') ? 1 : (u == 'G') ? 2 : (u == 'T') ? 3 : 4;
}
// MODE = Params::softclip (dp_score_serial): 1 lets a path start in the cell of column 0 and end in the cell of column
// tlen-1 at any row, 2 lets any live cell start (diagonal predecessor floored at 0) and end a path.
template <int MODE>
__device__ __forceinline__ int32_t dp_warp_bytes(const IndexView& ix, const Params& p, const uint8_t* read, uint32_t L,
                                                 const Cand& c, uint32_t lane, int ascii) {
  const int32_t B = (int32_t)p.band, W = 2 * B + 1;
  const uint32_t ori = c.ori_cov >> 31;
  const int64_t tlen = (int64_t)(ix.tx_off[c.tid + 1] - ix.tx_off[c.tid]);
  const uint8_t* ref = ix.codes + ix.tx_off[c.tid];
  const bool in_band = (int32_t)lane < W;
  int32_t H = in_band ? 0 : NEG_SCORE, E = NEG_SCORE;
  int32_t top = NEG_SCORE;     // modes 1 and 2: the lane's best end before the last row
  int64_t rpos = (int64_t)c.diag_c + ((int32_t)lane - B);
  uint8_t rbase = (rpos >= 0 && rpos < tlen) ? ref[rpos] : (uint8_t)255;
  for (uint32_t i = 0; i < L; ++i) {
    const uint8_t cc = base_code(ori ? read[L - 1 - i] : read[i], ascii);
    const uint8_t rb = ori ? (uint8_t)(cc > 3 ? 4 : 3 - cc) : cc;
    const bool valid = in_band && rbase != 255;
    const int32_t Hup = __shfl_down_sync(0xffffffffu, H, 1);
    const int32_t Eup = __shfl_down_sync(0xffffffffu, E, 1);
    int32_t m = NEG_SCORE, e = NEG_SCORE;
    if (valid) {
      int32_t hd = H;
      if (MODE == 2 || (MODE == 1 && rpos == 0)) hd = max(hd, 0);
      m = hd + ((rb < 4 && rb == rbase) ? p.ma : p.mp);
      if ((int32_t)lane + 1 < W) e = max(Hup - p.go - p.ge, Eup - p.ge);
      if (e < NEG_SCORE) e = NEG_SCORE;
    }
    const int32_t hp = valid ? max(m, e) : NEG_SCORE;
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
    if (MODE != 0 && valid && (MODE == 2 || rpos == tlen - 1)) top = max(top, h);
    H = h;
    E = valid ? e : NEG_SCORE;
    const uint8_t nb = __shfl_down_sync(0xffffffffu, rbase, 1);
    ++rpos;
    if ((int32_t)lane == W - 1) rbase = (rpos >= 0 && rpos < tlen) ? ref[rpos] : (uint8_t)255;
    else rbase = nb;
  }
  int32_t best = in_band ? H : NEG_SCORE;
  if (MODE != 0) best = max(best, top);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
  return best;
}

// the read as it aligns to the forward reference strand (reverse-complemented when ori = 1), bases beyond L zeroed
template <int NWR>
__device__ __forceinline__ void load_oriented_read(const PackedReads& pr, uint64_t mi, uint32_t L, uint32_t ori,
                                                   uint64_t (&rw)[NWR]) {
#pragma unroll
  for (int m = 0; m < NWR; ++m) rw[m] = ((uint32_t)m < pr.wpr) ? pr.bits[mi * pr.wpr + m] : 0ull;
  if (ori) {
    uint64_t t2[NWR + 1];
#pragma unroll
    for (int m = 0; m < NWR; ++m) t2[m] = brev2(~rw[NWR - 1 - m]);
    t2[NWR] = 0;
    const uint32_t drop = (uint32_t)NWR * 32u - L;          // bases to drop at the low end
    const uint32_t dw = drop >> 5, dsh = 2 * (drop & 31);
#pragma unroll
    for (int m = 0; m < NWR; ++m) {
      uint64_t lo = 0, hi = 0;
#pragma unroll
      for (int q = 0; q <= NWR; ++q) {
        if ((uint32_t)q == (uint32_t)m + dw) lo = t2[q];
        if ((uint32_t)q == (uint32_t)m + dw + 1) hi = t2[q];
      }
      rw[m] = funnel64(lo, hi, dsh);
    }
  }
#pragma unroll
  for (int m = 0; m < NWR; ++m) {
    const int32_t nb = (int32_t)L - 32 * m;
    if (nb <= 0) rw[m] = 0;
    else if (nb < 32) rw[m] &= (1ull << (2 * nb)) - 1;
  }
}
// reference window: bases diag_c - B ... (window index 0 ... 32*(NWR+1) - 1), ww[NWR+1] = 0
template <int NWR>
__device__ __forceinline__ void load_window(const IndexView& ix, int64_t tbase, int32_t diag_c, int32_t B,
                                            uint64_t (&ww)[NWR + 2]) {
  const int64_t g0 = tbase + (int64_t)diag_c - B + (int64_t)PACK_GUARD_BASES;
  const uint64_t* P = ix.packed + (g0 >> 5);
  const uint32_t gsh = 2 * (uint32_t)(g0 & 31);
  uint64_t prev = __ldg(P);
#pragma unroll
  for (int m = 0; m < NWR + 1; ++m) {
    const uint64_t nxt = __ldg(P + m + 1);
    ww[m] = funnel64(prev, nxt, gsh);
    prev = nxt;
  }
  ww[NWR + 1] = 0;
}

// k_dp_classify: one THREAD per mate alignment (32 independent alignments in flight per warp hide the chain of
// dependent loads: task -> candidate -> read words -> reference window).  Each thread evaluates the ungapped
// alignment on the candidate diagonal first (XOR + popcount on the 2-bit words; a perfect match ends here), then
// the other 2*band diagonals; when the best ungapped score is within (go+ge) of a perfect score no gapped path can
// beat it.  Otherwise the alignment goes to the interior list (whole band inside the transcript -> k_dp_pair) or the
// edge list; anything touching an N goes to the byte-code list.  List slots are reserved once per warp.
//
// Why the shortcut is exact, per scoring mode (MODE = Params::softclip):
//   Every path with a gap scores at most ma*L - go - ge = bound: a deletion costs go + ge with at most L bases matched,
//   an insertion costs go + ge and leaves a base unmatched, and clipped bases (modes 1, 2) add nothing.  So when the
//   best ungapped path of the band reaches the bound, it is the DP's score.
//   mode 0: the ungapped paths are the diagonals that lie inside the transcript; the others are dead.
//   mode 1: a diagonal that leaves the transcript is a valid path as well (its overhang is clipped), so only interior
//           alignments (whole band inside the transcript) may take the shortcut; those score as in mode 0, since no band
//           cell reaches column 0 after row 0 or column tlen-1 before the last row.  Mode 1 only changes the DP kernels'
//           edge and N paths.
//   mode 2: only interior alignments, and only a perfect diagonal settles the alignment: ma*L is the most any path can
//           score, while a full-length diagonal with a mismatch may be beaten by a clipped run of the same diagonal, so
//           the DP scores those.
//
// Gapless settlement (gapless = 1, decided per launch by the host, mode 0 only; DESIGN.md section 14): the best
// ungapped score u settles the alignment whatever it is, when G = ma*L - go - ge < s_min, where s_min is the lowest mate
// score that can still change an outcome.  A hit's score is the sum of its mates' scores and passes when it reaches
// minScoreFraction * ma * L per mate; no mate scores above ma*L.  So a mate of a passing pair scores at least
// s_min = (2*minScoreFraction - 1)*ma*L (its partner perfect), and a passing orphan, single-end read, rescue anchor or
// rescued mate at least minScoreFraction*ma*L >= s_min.  Let d = max(u, best gapped score) be the DP's score; the best
// gapped score is at most G.
//   - d >= s_min: then d > G, so d = u.
//   - d < s_min: then u <= d < s_min too, and every hit with this mate fails its threshold with either value (or is
//     invalid: u = NEG_SCORE when no diagonal fits inside the transcript), so it is INVALID_SCORE either way.
// Hit scores, hence the decoy maximum, the filters and the written alignments, are the same; the rescue anchors pass
// rescue_mate_passes with u exactly when with d; the per-mate scores SAM writes belong to passing hits, where u = d.
// The host compares in double exactly as assign_read and rescue_mate_passes do, at G (single mate) and G + ma*L (pair).
template <int NWR, int MODE>   // read words: 4 (read_len <= 128) or 8 (<= 256)
__global__ void __launch_bounds__(256, 3)
k_dp_classify(IndexView ix, Params p, PackedReads pr, uint32_t L, int fast_ok, int gapless, DpIo io) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t ntasks = *io.n_tasks;
  const uint32_t nthreads = gridDim.x * blockDim.x;
  const int32_t B = (int32_t)p.band, W = 2 * B + 1;
  const int32_t perfect = p.ma * (int32_t)L, bound = perfect - p.go - p.ge;
  const uint32_t rounds = (ntasks + nthreads - 1) / nthreads;
  for (uint32_t rd = 0; rd < rounds; ++rd) {
    const uint32_t t = rd * nthreads + blockIdx.x * blockDim.x + threadIdx.x;
    const bool have = t < ntasks;
    uint32_t task = 0;
    int dest = -1;               // -1 resolved / none, 0 interior, 1 edge, 2 N
    if (have) {
      task = io.tasks[t];
      const uint32_t r = task >> 7, mate = (task >> 6) & 1u, ci = task & 63u;
      const Cand c = mate ? io.cand_r[(size_t)r * MAXCAND + ci] : io.cand_l[(size_t)r * MAXCAND + ci];
      const uint64_t mi = (uint64_t)2 * r + mate;
      bool slow = ix.tx_has_n[c.tid] != 0;
      for (uint32_t w = 0; w < pr.mpr; ++w) slow |= pr.nmask[mi * pr.mpr + w] != 0;
      if (slow) dest = 2;
      else {
        const int64_t tbase = (int64_t)ix.tx_off[c.tid];
        const int64_t tlen = (int64_t)ix.tx_off[c.tid + 1] - tbase;
        const bool interior = ((int64_t)c.diag_c - B >= 0) && ((int64_t)c.diag_c + (int64_t)L + B <= tlen);
        const bool try_fast = fast_ok && (MODE == 0 || interior);
        int32_t best_u = NEG_SCORE;
        if (try_fast) {
          uint64_t rw[NWR];
          load_oriented_read<NWR>(pr, mi, L, c.ori_cov >> 31, rw);
          uint64_t ww[NWR + 2];
          load_window<NWR>(ix, tbase, c.diag_c, B, ww);
          // diagonal order: the candidate's own (j = B) first, then the rest
          for (int32_t jj = 0; jj < W; ++jj) {
            const int32_t j = (jj == 0) ? B : (jj <= B ? jj - 1 : jj);
            const int64_t s0 = (int64_t)c.diag_c + (j - B);
            if (s0 < 0 || s0 + (int64_t)L > tlen) continue;
            uint32_t mm = 0;
#pragma unroll
            for (int m = 0; m < NWR; ++m) {
              const uint64_t x = funnel64(ww[m], ww[m + 1], 2u * (uint32_t)j) ^ rw[m];
              uint64_t d = (x | (x >> 1)) & 0x5555555555555555ull;
              const int32_t nb = (int32_t)L - 32 * m;
              if (nb <= 0) d = 0;
              else if (nb < 32) d &= (1ull << (2 * nb)) - 1;
              mm += (uint32_t)__popcll(d);
            }
            const int32_t u = p.ma * (int32_t)(L - mm) + p.mp * (int32_t)mm;
            if (u > best_u) best_u = u;
            if (best_u == perfect) break;
          }
        }
        if (try_fast && (gapless || best_u >= (MODE == 2 ? perfect : bound))) {
          (mate ? io.score_r : io.score_l)[(size_t)r * MAXCAND + ci] = best_u;
        } else {
          dest = interior ? 0 : 1;
        }
      }
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const uint32_t bal = __ballot_sync(0xffffffffu, dest == d);
      if (bal) {
        uint32_t base = 0;
        const uint32_t leader = (uint32_t)__ffs(bal) - 1;
        if (lane == leader) base = atomicAdd(io.list_n + d, (uint32_t)__popc(bal));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (dest == d) {
          uint32_t* list = d == 0 ? io.list_int : (d == 1 ? io.list_edge : io.list_n_tasks);
          list[base + (uint32_t)__popc(bal & ((1u << lane) - 1))] = task;
        }
      }
    }
  }
}

// k_dp_pair: banded affine DP for interior alignments, TWO alignments per warp: a half-warp owns one alignment,
// lane hl owns band cells 2*hl and 2*hl+1.  The band has W = 2*band+1 cells; cells W..31 do not exist and are forced
// dead in every row (cell 2*band+1 in lane band, both cells in the lanes above; at band 15 only cell 31): starting them
// dead is not enough, F would carry live values rightward into them.  Same recurrences as dp_score_serial; read and
// reference window live in registers (2-bit), no memory access in the row loop.  Values derived from dead cells (E, F
// and the prefix scan) stay below -2^27 without re-clamping, which every consumer treats like NEG_SCORE (the hit is
// invalid), and never reach a live cell's maximum.
// MODE 2 (soft-clip): diagonal predecessors floored at 0 and the best cell of any row.  Interior alignments score the
// same in modes 0 and 1 (k_dp_classify), so mode 1 runs the MODE 0 instance.
template <int NWR, int MODE>
__global__ void __launch_bounds__(256, 3)
k_dp_pair(IndexView ix, Params p, PackedReads pr, uint32_t L, DpIo io) {
  static_assert(MODE == 0 || MODE == 2, "interior alignments: mode 1 scores as mode 0");
  const uint32_t lane = threadIdx.x & 31u, hl = lane & 15u, half = lane >> 4;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t n = io.list_n[0];
  const int32_t B = (int32_t)p.band;
  const int32_t goe = p.go + p.ge, ge = p.ge;
  const int32_t kge0 = (int32_t)(2 * hl) * ge, kge1 = kge0 + ge;
  const bool dead0 = (int32_t)hl > B, dead1 = (int32_t)hl >= B;   // cells 2hl, 2hl+1 lie outside the band (>= W)
  for (uint32_t t2 = warp * 2; t2 < n; t2 += nwarps * 2) {
    const uint32_t t = (t2 + half < n) ? t2 + half : t2;       // odd tail: both halves do the same alignment
    const uint32_t task = io.list_int[t];
    const uint32_t r = task >> 7, mate = (task >> 6) & 1u, ci = task & 63u;
    const Cand c = mate ? io.cand_r[(size_t)r * MAXCAND + ci] : io.cand_l[(size_t)r * MAXCAND + ci];
    const uint64_t mi = (uint64_t)2 * r + mate;
    uint64_t rw[NWR];
    load_oriented_read<NWR>(pr, mi, L, c.ori_cov >> 31, rw);
    uint64_t ww[NWR + 2];
    load_window<NWR>(ix, (int64_t)ix.tx_off[c.tid], c.diag_c, B, ww);
    int32_t H0 = dead0 ? NEG_SCORE : 0, H1 = dead1 ? NEG_SCORE : 0, E0 = NEG_SCORE, E1 = NEG_SCORE;
    int32_t top = NEG_SCORE;   // mode 2: the lane's best cell of any row
    // blocks of 16 rows: the lane's reference bases for rows r0 .. r0+15 are window indices r0 + 2hl (+1) ...
#pragma unroll
    for (int blk = 0; blk < 2 * NWR; ++blk) {
      const uint32_t r0 = 16u * blk;
      if (r0 >= L) break;
      const uint32_t rows = (L - r0 < 16u) ? (L - r0) : 16u;
      const int q = blk >> 1;
      const uint32_t off = 32u * (blk & 1) + 4u * hl;          // bit offset of window index r0 + 2hl inside ww[q]
      const uint64_t lo = (off >= 64u) ? ww[q + 1] : ww[q];
      const uint64_t hi = (off >= 64u) ? ww[q + 2] : ww[q + 1];
      const uint64_t st = funnel64(lo, hi, off & 63u);
      uint32_t rb0 = (uint32_t)(st & 3ull);
      uint32_t stream = (uint32_t)(st >> 2);                   // bases r0 + 2hl + 1 ... (16 of them)
      uint32_t cur = (uint32_t)(rw[q] >> (32 * (blk & 1)));    // read bases r0 ... r0 + 15
      for (uint32_t ii = 0; ii < rows; ++ii) {
        const uint32_t rb = cur & 3u; cur >>= 2;
        const uint32_t rb1 = stream & 3u; stream >>= 2;
        const int32_t s0 = (rb == rb0) ? p.ma : p.mp;
        const int32_t s1 = (rb == rb1) ? p.ma : p.mp;
        const int32_t Hn = __shfl_down_sync(0xffffffffu, H0, 1, 16);   // cell 2hl+2 of the previous row
        const int32_t En = __shfl_down_sync(0xffffffffu, E0, 1, 16);
        const int32_t e0 = max(H1 - goe, E1 - ge);
        int32_t e1 = max(Hn - goe, En - ge);
        int32_t hp0 = max((MODE == 2 ? max(H0, 0) : H0) + s0, e0);
        int32_t hp1 = max((MODE == 2 ? max(H1, 0) : H1) + s1, e1);
        if (dead1) { e1 = NEG_SCORE; hp1 = NEG_SCORE; }
        const int32_t x0 = hp0 + kge0, x1 = hp1 + kge1;
        int32_t inc = max(x0, x1);
#pragma unroll
        for (int o = 1; o < 16; o <<= 1) {
          const int32_t y = __shfl_up_sync(0xffffffffu, inc, o, 16);
          if ((int)hl >= o) inc = max(inc, y);
        }
        int32_t exc = __shfl_up_sync(0xffffffffu, inc, 1, 16);
        if (hl == 0) exc = NEG_SCORE;
        const int32_t f0 = exc - p.go - kge0;
        const int32_t f1 = max(exc, x0) - p.go - kge1;
        H0 = dead0 ? NEG_SCORE : max(hp0, f0);
        H1 = dead1 ? NEG_SCORE : max(hp1, f1);
        E0 = dead0 ? NEG_SCORE : e0; E1 = e1;
        rb0 = rb1;
        if (MODE == 2) top = max(top, max(H0, H1));
      }
    }
    int32_t best = max(H0, H1);
    if (MODE == 2) best = max(best, top);
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o, 16));
    if (best < -(1 << 27)) best = NEG_SCORE;
    if (hl == 0 && t2 + half < n) (mate ? io.score_r : io.score_l)[(size_t)r * MAXCAND + ci] = best;
  }
}

// k_dp_general: the rare rest -- alignments whose band leaves the transcript (register form with per-cell validity)
// and alignments touching an N (byte form).  One warp per alignment, lanes = band cells.  MODE as in dp_warp_bytes.
template <int NWR, int MODE>
__global__ void __launch_bounds__(256, 3)
k_dp_general(IndexView ix, Params p, PackedReads pr, const uint8_t* __restrict__ left,
             const uint8_t* __restrict__ right, uint32_t L, int ascii, DpIo io) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t n_edge = io.list_n[1], n_n = io.list_n[2];
  const int32_t B = (int32_t)p.band, W = 2 * B + 1;
  if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(io.n_full_dp, (unsigned long long)io.list_n[0] + n_edge + n_n);
  for (uint32_t t = warp; t < n_edge + n_n; t += nwarps) {
    const bool bytes = t >= n_edge;
    const uint32_t task = bytes ? io.list_n_tasks[t - n_edge] : io.list_edge[t];
    const uint32_t r = task >> 7, mate = (task >> 6) & 1u, ci = task & 63u;
    const Cand c = mate ? io.cand_r[(size_t)r * MAXCAND + ci] : io.cand_l[(size_t)r * MAXCAND + ci];
    int32_t* out = (mate ? io.score_r : io.score_l) + (size_t)r * MAXCAND + ci;
    if (bytes) {
      const int32_t s = dp_warp_bytes<MODE>(ix, p, (mate ? right : left) + (size_t)r * L, L, c, lane, ascii);
      if (lane == 0) *out = s;
      continue;
    }
    const uint64_t mi = (uint64_t)2 * r + mate;
    const int64_t tbase = (int64_t)ix.tx_off[c.tid];
    const int64_t tlen = (int64_t)ix.tx_off[c.tid + 1] - tbase;
    uint64_t rw[NWR];
    load_oriented_read<NWR>(pr, mi, L, c.ori_cov >> 31, rw);
    uint64_t ww[NWR + 2];
    load_window<NWR>(ix, tbase, c.diag_c, B, ww);
    const bool in_band = (int32_t)lane < W;
    int32_t H = in_band ? 0 : NEG_SCORE, E = NEG_SCORE;
    int32_t top = NEG_SCORE;   // modes 1 and 2: the lane's best end before the last row
    int64_t rpos = (int64_t)c.diag_c + ((int32_t)lane - B);
    uint32_t rbase = (rpos >= 0 && rpos < tlen) ? (uint32_t)((ww[0] >> (2 * lane)) & 3ull) : 255u;
    // stream of the bases entering at the last band lane: window index W, W+1, ...
    uint64_t rs[NWR + 1];
#pragma unroll
    for (int m = 0; m < NWR + 1; ++m) rs[m] = funnel64(ww[m], ww[m + 1], 2 * (uint32_t)W);
#pragma unroll
    for (int m = 0; m < NWR; ++m) {
      uint64_t cur = rw[m], curs = rs[m];
      const uint32_t i0 = 32u * m;
      if (i0 >= L) break;
      const uint32_t iend = (L - i0 < 32u) ? (L - i0) : 32u;
      for (uint32_t ii = 0; ii < iend; ++ii) {
        const uint32_t rb = (uint32_t)(cur & 3ull);
        cur >>= 2;
        const bool valid = in_band && rbase != 255u;
        const int32_t Hup = __shfl_down_sync(0xffffffffu, H, 1);
        const int32_t Eup = __shfl_down_sync(0xffffffffu, E, 1);
        int32_t mval = NEG_SCORE, e = NEG_SCORE;
        if (valid) {
          int32_t hd = H;
          if (MODE == 2 || (MODE == 1 && rpos == 0)) hd = max(hd, 0);
          mval = hd + ((rb == rbase) ? p.ma : p.mp);
          if ((int32_t)lane + 1 < W) e = max(Hup - p.go - p.ge, Eup - p.ge);
          if (e < NEG_SCORE) e = NEG_SCORE;
        }
        const int32_t hp = valid ? max(mval, e) : NEG_SCORE;
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
        if (MODE != 0 && valid && (MODE == 2 || rpos == tlen - 1)) top = max(top, h);
        H = h;
        E = valid ? e : NEG_SCORE;
        const uint32_t nb = __shfl_down_sync(0xffffffffu, rbase, 1);
        ++rpos;
        if ((int32_t)lane == W - 1) rbase = (rpos >= 0 && rpos < tlen) ? (uint32_t)(curs & 3ull) : 255u;
        else rbase = nb;
        curs >>= 2;
      }
    }
    int32_t best = in_band ? H : NEG_SCORE;
    if (MODE != 0) best = max(best, top);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
    if (lane == 0) *out = best;
  }
}

}  // namespace sbmap
