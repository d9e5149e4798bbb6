// tests/host_sam.cpp -- TEST INFRASTRUCTURE.  Host build of the SAM record rules (sam_core.h), the code the CUDA
// kernels run, so that tests can check them against an independent Python renderer.  Not part of the product library.
#include <stdint.h>
#include <string.h>

#include "../salmon_b200/csrc/sam_core.h"

// the records of one fragment, written by sam_core.h's rules the way the kernel writes them; returns the bytes (out
// may be NULL to size)
extern "C" uint64_t hs_render(const char* name, uint32_t name_len, uint32_t n_aln, const uint32_t* tid, const int32_t* pos,
                              const int32_t* mate_pos, const uint8_t* flags, const int32_t* flen, const int32_t* score1,
                              const int32_t* score2, int paired, uint32_t L, const uint8_t* left, const uint8_t* right,
                              const uint8_t* qual_left, const uint8_t* qual_right, const char* const* ref_names,
                              const uint32_t* ref_len, char* out) {
  using namespace sbsam;
  uint64_t k = 0;
  for (uint32_t a = 0; a < n_aln; ++a) {
    Aln x{tid[a], pos[a], mate_pos[a], flags[a], flen[a], score1[a], score2[a]};
    const char* rn = ref_names[x.tid];
    const uint32_t rl = str_len(rn);
    for (uint32_t m = 0; m < (paired ? 2u : 1u); ++m) {
      const Rec r = sam_record(x, m, a, n_aln, paired != 0, L, ref_len[x.tid]);
      const uint8_t* codes = m ? right : left;
      const uint8_t* q = m ? qual_right : qual_left;
      const uint32_t hl = head_len(r, name_len, rl), bl = body_len(L, q != nullptr), tl = tail_len(r);
      if (out) {
        head_write(out + k, r, name, name_len, rn, rl);
        for (uint32_t i = 0; i < bl; ++i) out[k + hl + i] = body_char(i, L, r.rev, codes, q, false);
        tail_write(out + k + hl + bl, r);
      }
      k += hl + bl + tl;
    }
  }
  return k;
}
