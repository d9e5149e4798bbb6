"""Records edlib's infix (HW) search -- the aligner salmon's --recoverOrphans uses (src/edlib.cpp, compiled unmodified
into oracle/_ref/libedlib_ref.so by oracle/build_ref.sh) -- for every search case of tests/rescue_ref.py:
  edlib_rescue.npz   dist (edit distance, -1 above K), end (endLocations[0], -1 without a hit), crc (of the case)
A read N (code 4) is passed as a symbol the target never holds, so edlib matches it to nothing; a reference N likewise.
usage: REF=<salmon source tree> bash oracle/build_ref.sh && python tests/golden/make_rescue_golden.py"""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]
from make_ref_golden import REF, EdlibAlignConfig, EdlibAlignResult  # noqa: E402


def main():
    import rescue_ref as R
    lib = C.CDLL(os.path.join(REF, "libedlib_ref.so"))
    align = getattr(lib, "_Z10edlibAlignPKciS0_i16EdlibAlignConfig")
    align.restype = EdlibAlignResult
    align.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int, EdlibAlignConfig]
    free = getattr(lib, "_Z20edlibFreeAlignResult16EdlibAlignResult")
    free.restype = None
    free.argtypes = [EdlibAlignResult]
    qmap = np.frombuffer(b"ACGTN", np.uint8)      # read N: 'N', never in a target that spells its N as 'X'
    tmap = np.frombuffer(b"ACGTX", np.uint8)
    dist, end, crc = [], [], []
    for pat, win, K in R.search_cases():
        q, t = qmap[pat].tobytes(), tmap[win].tobytes()
        r = align(q, len(q), t, len(t), EdlibAlignConfig(K, 2, 0))     # EDLIB_MODE_HW, EDLIB_TASK_DISTANCE
        d = r.editDistance
        e = r.endLocations[0] if (d >= 0 and r.numLocations > 0) else -1
        free(r)
        dist.append(d); end.append(e if d >= 0 else -1); crc.append(R.case_crc(pat, win, K))
    np.savez_compressed(os.path.join(HERE, "edlib_rescue.npz"), dist=np.array(dist, np.int32), end=np.array(end, np.int32),
                        crc=np.array(crc, np.uint32))
    print(f"{len(dist)} cases, {sum(d >= 0 for d in dist)} with a hit")


if __name__ == "__main__":
    main()
