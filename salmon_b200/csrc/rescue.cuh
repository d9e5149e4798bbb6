// rescue.cuh -- orphan rescue (--recoverOrphans, DESIGN.md §11) on sm_90a.  Runs per chunk on the main stream after
// the DP kernels, so k_assign sees the rescued candidates, scores and pair lists:
//
//   k_rescue_select  one thread per read: the anchors of orphan-only reads (rescue_anchors) -> search tasks, one atomic
//                    per read so that a read's tasks are contiguous and in anchor order
//   k_rescue_search  one thread per task: Peq masks of the other mate (2-bit codes from the packed reads), the window
//                    streamed from the 2-bit packed reference 32 bases per load (byte codes on transcripts with N),
//                    bit-vector infix search with limit K (myers_infix)
//   k_rescue_score   one warp per task that found a place: the banded DP of the rescued mate (dp_warp_bytes, the
//                    recurrence of k_dp_general and dp_score_serial)
//   k_rescue_commit  one thread per read with anchors: rescue_commit appends the rescued candidates and writes the
//                    read's pair list, which k_assign<.., true> then uses instead of the join
#pragma once
#include "map_kernels.cuh"

namespace sbmap {

struct RescueBufs {
  uint32_t* n_tasks;             // [1]
  uint32_t* tasks;               // [CH * 2 * MAXCAND]  read << 8 | side << 7 | candidate
  uint32_t* first;               // [CH] first task of the read
  uint8_t* n_anchor;             // [CH] anchors (tasks) of the read
  int32_t* diag;                 // [tasks] diagonal of the place found
  int32_t* score;                // [tasks] DP score of the rescued mate; INVALID_SCORE: nothing within K
  uint16_t* pairs;               // [CH * 2 * MAXCAND] rescued pairs of the read: left | right << 8 (candidate indices)
  uint32_t* n_pairs;             // [CH]
  unsigned long long* ctr;       // [3] fragments rescued, searches, anchors without room
};

// Bit-vector search of one window [g0, g0 + n) of the concatenated reference (global base offsets).  has_n: the window's
// transcript has a non-ACGT base, so its 2-bit form is unusable and the byte codes are read instead.
template <uint32_t NW, class PatF>
__device__ __forceinline__ void rescue_search_window(PatF&& pat, uint32_t m, const uint64_t* __restrict__ packed,
                                                     const uint8_t* __restrict__ codes, bool has_n, uint64_t g0,
                                                     uint32_t n, int32_t K, int32_t& dist, int32_t& end) {
  if (has_n) {
    const uint8_t* ref = codes + g0;
    myers_infix<NW>(pat, m, n, [&](uint32_t j) { return ref[j]; }, K, dist, end);
    return;
  }
  uint64_t g = g0 + PACK_GUARD_BASES;
  uint64_t word = packed[g >> 5] >> (2 * (g & 31));
  myers_infix<NW>(pat, m, n, [&](uint32_t) {
    const uint8_t c = (uint8_t)(word & 3u);
    ++g;
    word = (g & 31) ? (word >> 2) : packed[g >> 5];
    return c;
  }, K, dist, end);
}

__global__ void k_rescue_select(Params p, uint32_t n, uint32_t L, const uint32_t* __restrict__ n_l,
                                const uint32_t* __restrict__ n_r, const Cand* __restrict__ cand_l,
                                const Cand* __restrict__ cand_r, const int32_t* __restrict__ score_l,
                                const int32_t* __restrict__ score_r, RescueBufs rb) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  rb.n_pairs[r] = 0;
  rb.n_anchor[r] = 0;
  const uint32_t nl = n_l[r];
  if (nl & 0x80000000u) return;
  const uint32_t nr = n_r[r];
  uint8_t side[2 * MAXCAND], ci[2 * MAXCAND];
  const size_t o = (size_t)r * MAXCAND;
  const uint32_t na = rescue_anchors(p, cand_l + o, nl, cand_r + o, nr, score_l + o, score_r + o, L, side, ci);
  if (!na) return;
  uint32_t t = atomicAdd(rb.n_tasks, na);
  rb.first[r] = t;
  rb.n_anchor[r] = (uint8_t)na;
  for (uint32_t a = 0; a < na; ++a) rb.tasks[t + a] = (r << 8) | ((uint32_t)side[a] << 7) | ci[a];
  atomicAdd(&rb.ctr[1], (unsigned long long)na);
}

template <uint32_t NW>
__global__ void k_rescue_search(IndexView ix, Params p, PackedReads pr, uint32_t L, const Cand* __restrict__ cand_l,
                                const Cand* __restrict__ cand_r, RescueBufs rb) {
  const uint32_t ntasks = *rb.n_tasks;
  const int32_t K = rescue_edit_limit(p, L);
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < ntasks; t += gridDim.x * blockDim.x) {
    const uint32_t task = rb.tasks[t];
    const uint32_t r = task >> 8, side = (task >> 7) & 1u, c = task & 127u;
    const Cand a = (side ? cand_r : cand_l)[(size_t)r * MAXCAND + c];
    const int64_t tlen = (int64_t)(ix.tx_off[a.tid + 1] - ix.tx_off[a.tid]);
    int64_t lo, hi;
    int32_t dist = -1, end = -1;
    if (rescue_window(p, a, L, tlen, lo, hi)) {
      // the other mate: 2-bit codes + N mask of k_pack_reads (mate index 2r + other side)
      const uint64_t m = 2 * (uint64_t)r + (side ^ 1u);
      const uint64_t* bits = pr.bits + m * pr.wpr;
      const uint64_t* nm = pr.nmask + m * pr.mpr;
      const bool rc = (a.ori_cov >> 31) == 0;
      auto pat = [&](uint32_t i) -> uint8_t {
        const uint32_t q = rc ? L - 1 - i : i;
        if ((nm[q >> 6] >> (q & 63)) & 1ull) return 4;
        const uint8_t b = (uint8_t)((bits[q >> 5] >> (2 * (q & 31))) & 3u);
        return rc ? (uint8_t)(3 - b) : b;
      };
      rescue_search_window<NW>(pat, L, ix.packed, ix.codes, ix.tx_has_n[a.tid] != 0, ix.tx_off[a.tid] + (uint64_t)lo,
                               (uint32_t)(hi - lo), K, dist, end);
    }
    rb.diag[t] = dist >= 0 ? (int32_t)(lo + end) - (int32_t)L + 1 : 0;
    rb.score[t] = dist >= 0 ? 0 : INVALID_SCORE;
  }
}

template <int MODE>   // Params::softclip
__global__ void k_rescue_score(IndexView ix, Params p, const uint8_t* __restrict__ left, const uint8_t* __restrict__ right,
                               uint32_t L, int ascii, const Cand* __restrict__ cand_l, const Cand* __restrict__ cand_r,
                               RescueBufs rb) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t ntasks = *rb.n_tasks;
  for (uint32_t t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < ntasks; t += (gridDim.x * blockDim.x) >> 5) {
    if (rb.score[t] == INVALID_SCORE) continue;
    const uint32_t task = rb.tasks[t];
    const uint32_t r = task >> 8, side = (task >> 7) & 1u, c = task & 127u;
    const Cand a = (side ? cand_r : cand_l)[(size_t)r * MAXCAND + c];
    const Cand res = rescue_cand(a, rb.diag[t]);
    const int32_t s = dp_warp_bytes<MODE>(ix, p, (side ? left : right) + (size_t)r * L, L, res, lane, ascii);
    if (lane == 0) rb.score[t] = s;
  }
}

__global__ void k_rescue_commit(Params p, uint32_t n, uint32_t L, uint32_t* __restrict__ n_l, uint32_t* __restrict__ n_r,
                                Cand* __restrict__ cand_l, Cand* __restrict__ cand_r, int32_t* __restrict__ score_l,
                                int32_t* __restrict__ score_r, RescueBufs rb) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const uint32_t na = rb.n_anchor[r];
  if (!na) return;
  uint8_t side[2 * MAXCAND], ci[2 * MAXCAND];
  const uint32_t t0 = rb.first[r];
  for (uint32_t a = 0; a < na; ++a) {
    const uint32_t task = rb.tasks[t0 + a];
    side[a] = (uint8_t)((task >> 7) & 1u); ci[a] = (uint8_t)(task & 127u);
  }
  const size_t o = (size_t)r * MAXCAND;
  uint32_t nl = n_l[r], nr = n_r[r], no_room = 0;
  Joint jp[2 * MAXCAND];
  const uint32_t np = rescue_commit(p, L, cand_l + o, nl, cand_r + o, nr, score_l + o, score_r + o, na, side, ci,
                                    rb.diag + t0, rb.score + t0, jp, no_room);
  for (uint32_t q = 0; q < np; ++q) rb.pairs[(size_t)r * 2 * MAXCAND + q] = (uint16_t)(jp[q].li | (jp[q].ri << 8));
  rb.n_pairs[r] = np;
  if (np) { n_l[r] = nl; n_r[r] = nr; atomicAdd(&rb.ctr[0], 1ull); }
  if (no_room) atomicAdd(&rb.ctr[2], (unsigned long long)no_room);
}

// the pair list of a rescued read as joint hits (k_assign)
__device__ __forceinline__ uint32_t rescued_joints(const Params& p, const RescueBufs& rb, uint32_t r, const Cand* lc,
                                                   const Cand* rc, uint32_t L, Joint* out) {
  const uint32_t np = rb.n_pairs[r];
  for (uint32_t q = 0; q < np; ++q) {
    const uint16_t w = rb.pairs[(size_t)r * 2 * MAXCAND + q];
    Joint j;
    j.li = w & 0xff; j.ri = w >> 8; j.tid = lc[j.li].tid; j.status = 0;
    pair_geometry(p, lc[j.li], rc[j.ri], L, j.frag_len);
    out[q] = j;
  }
  return np;
}

// parity tap: one thread per case, the search of k_rescue_search on windows laid out like the index's packed reference
template <uint32_t NW>
__global__ void k_rescue_tap(uint32_t n, const uint8_t* __restrict__ pats, const uint64_t* __restrict__ pat_off,
                             const uint64_t* __restrict__ packed, const uint8_t* __restrict__ codes,
                             const uint64_t* __restrict__ win_off, const uint8_t* __restrict__ win_has_n,
                             const int32_t* __restrict__ K, int32_t* __restrict__ dist, int32_t* __restrict__ end) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* P = pats + pat_off[i];
  const uint32_t m = (uint32_t)(pat_off[i + 1] - pat_off[i]);
  if ((m + 63) / 64 != NW && !(m == 0 && NW == 1)) return;   // another instance's case
  int32_t d = -1, e = -1;
  const uint32_t w = (uint32_t)(win_off[i + 1] - win_off[i]);
  if (w > 0 && m > 0)
    rescue_search_window<NW>([&](uint32_t q) { return P[q]; }, m, packed, codes, win_has_n[i] != 0, win_off[i], w, K[i], d, e);
  dist[i] = d; end[i] = e;
}

}  // namespace sbmap
