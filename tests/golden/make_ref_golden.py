"""Records what the reference tree's own code returns for the cases of three tests, so that the tests compare against it
without the reference tree:
  edlib_hw.npz        edlib's infix (HW) edit distance for every call of tests/test_dp_vs_edlib.py (+ a CRC of its input)
  kseq_records.json   kseq++'s records for every file of tests/test_reader_vs_kseq.py (count + per-block digests)
  eigen_digamma.npz   Eigen's digamma on a fixed sample of arguments (tests/test_math_pinning.py)
usage: REF=<salmon source tree> bash oracle/build_ref.sh && python tests/golden/make_ref_golden.py"""
import ctypes as C
import json
import os
import sys
import tempfile
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
REF = os.path.join(ROOT, "oracle", "_ref")


class EdlibAlignConfig(C.Structure):
    _fields_ = [("k", C.c_int), ("mode", C.c_int), ("task", C.c_int)]


class EdlibAlignResult(C.Structure):
    _fields_ = [("editDistance", C.c_int), ("endLocations", C.POINTER(C.c_int)), ("startLocations", C.POINTER(C.c_int)),
                ("numLocations", C.c_int), ("alignment", C.POINTER(C.c_ubyte)), ("alignmentLength", C.c_int),
                ("alphabetLength", C.c_int)]


def edlib_golden():
    import test_dp_vs_edlib as T
    lib = C.CDLL(os.path.join(REF, "libedlib_ref.so"))
    align = getattr(lib, "_Z10edlibAlignPKciS0_i16EdlibAlignConfig")      # edlibAlign(const char*, int, const char*, int, EdlibAlignConfig)
    align.restype = EdlibAlignResult
    align.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int, EdlibAlignConfig]
    free = getattr(lib, "_Z20edlibFreeAlignResult16EdlibAlignResult")
    free.restype = None
    free.argtypes = [EdlibAlignResult]
    rec = {}

    def recording(name):
        d_l, crc_l = rec.setdefault(name, ([], []))

        def hw(query, target):
            r = align(query, len(query), target, len(target), EdlibAlignConfig(-1, 2, 0))     # k = -1, EDLIB_MODE_HW, TASK_DISTANCE
            d = r.editDistance
            free(r)
            d_l.append(d)
            crc_l.append(zlib.crc32(query + b"|" + target))
            return d
        hw.assert_all_used = lambda: None
        return hw
    T._edlib = recording
    T.test_unit_cost_dp_equals_edlib_infix_distance()
    T.test_default_scores_bound_by_edit_distance()
    T.test_product_serial_dp_equals_edlib_and_oracle()
    out = {}
    for name, (d_l, crc_l) in rec.items():
        out[name + "_d"] = np.array(d_l, np.int32)
        out[name + "_crc"] = np.array(crc_l, np.uint32)
    np.savez_compressed(os.path.join(HERE, "edlib_hw.npz"), **out)


def kseq_golden():
    import test_reader_vs_kseq as T
    lib = C.CDLL(os.path.join(REF, "libkseq_ref.so"))
    lib.ref_kseq_parse.restype = C.c_long

    def parse(path):
        tot = C.c_ulong(0)
        n = lib.ref_kseq_parse(os.fsencode(path), None, C.c_ulong(0), None, C.c_ulong(0), C.byref(tot))
        assert n >= 0
        seq = np.empty(max(tot.value, 1), np.uint8)
        lens = np.empty(max(n, 1), np.uint32)
        assert n == lib.ref_kseq_parse(os.fsencode(path), seq.ctypes.data_as(C.c_void_p), C.c_ulong(len(seq)),
                                       lens.ctypes.data_as(C.c_void_p), C.c_ulong(len(lens)), C.byref(tot))
        off = np.concatenate(([0], np.cumsum(lens[:n]))).astype(np.int64)
        return [T.ENC[seq[off[i]:off[i + 1]]] for i in range(n)]
    out = {}
    with tempfile.TemporaryDirectory() as d:
        for flavour in T.FLAVOURS:
            recs = parse(T.write_fastq(d, flavour))
            out[flavour] = {"n": len(recs), "blocks": T.digests(recs)}
        recs = parse(T.write_fasta(d))
        out["fasta"] = {"n": len(recs), "blocks": T.digests(recs)}
    json.dump(out, open(os.path.join(HERE, "kseq_records.json"), "w"), indent=0)


def digamma_golden():
    lib = C.CDLL(os.path.join(REF, "libeigen_digamma_ref.so"))
    rng = np.random.default_rng(11)
    x = np.concatenate([10.0 ** rng.uniform(-10, 9, 40000), np.linspace(0.01, 40.0, 20000), rng.uniform(1.3, 1.6, 5000)])
    x = np.ascontiguousarray(x[::8])
    ref = np.empty_like(x)
    lib.ref_eigen_digamma(C.c_ulong(len(x)), x.ctypes.data_as(C.c_void_p), ref.ctypes.data_as(C.c_void_p))
    np.savez_compressed(os.path.join(HERE, "eigen_digamma.npz"), x=x, digamma=ref)


if __name__ == "__main__":
    edlib_golden()
    kseq_golden()
    digamma_golden()
