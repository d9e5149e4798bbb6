// sam_internal.h -- what the mapping context (map.cu) needs of the SAM formatter (sam.cu).
#pragma once
#include "common.cuh"
#include "map_core.h"

struct SamDev;   // the formatter's device buffers, owned by a mapping context with a sink attached

// device views of one batch's alignments: the ReadOut arrays of sb_map_batch (cap entries per read)
struct SamBatch {
  uint32_t n, L, cap;
  int paired, ascii;
  const uint32_t* tid;
  const int32_t* pos;
  const int32_t* mate_pos;
  const uint8_t* flags;
  const int32_t* flen;
};

int sam_dev_create(SamDev** out, sb_sam* s, uint32_t batch_cap, uint32_t read_len_cap, uint32_t cap);
void sam_dev_destroy(SamDev* d);
// base pointers of the side output; read r of the batch uses n_out + r, decoy + r, score1 / score2 + r * cap
sbmap::SamSide sam_dev_side(SamDev* d);
// formats the batch (after its k_assign launches on `st`) and hands the text to the sink's writer thread.  left /
// right: the batch's reads (host or device memory, n x L); names / name_off / qualities: host memory.
int sam_dev_format(SamDev* d, cudaStream_t st, const SamBatch& b, const uint8_t* left, const uint8_t* right,
                   const char* names, const uint64_t* name_off, const uint8_t* qual_left, const uint8_t* qual_right,
                   uint64_t window_bytes, float* format_ms);
