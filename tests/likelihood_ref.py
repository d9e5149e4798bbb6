"""TEST INFRASTRUCTURE for salmon's fragment-likelihood options (--incompatPrior, --noSingleFragProb, --noFragLengthDist,
--noEffectiveLengthCorrection; DESIGN.md section 13): the independent restatement on top of the CPU oracle
(tests/oracle_likelihood.c) and a planted stranded workload."""
import ctypes as C
import os

import numpy as np

import rescue_ref as R

ROOT = R.ROOT
_P = C.c_void_p
KEYS = R.KEYS

_orc = None


class orc_lk_opts(C.Structure):
    _fields_ = [("incompat_prior", C.c_double), ("model_single_frag_prob", C.c_int32), ("use_frag_len_dist", C.c_int32),
                ("no_eff_len_correction", C.c_int32), ("reserved", C.c_int32)]


def opts(incompat_prior=0.0, no_single_frag_prob=0, no_frag_len_dist=0, no_eff_len_correction=0):
    """the options as the command line gives them"""
    return orc_lk_opts(float(incompat_prior), 0 if no_single_frag_prob else 1, 0 if no_frag_len_dist else 1,
                       1 if no_eff_len_correction else 0, 0)


def product_fields(o):
    """the sb_map_params fields of the same options"""
    return dict(incompat_prior=o.incompat_prior if o.incompat_prior >= 1e-100 else 0.0,
                no_single_frag_prob=int(not o.model_single_frag_prob), no_frag_len_dist=int(not o.use_frag_len_dist),
                no_eff_len_correction=int(o.no_eff_len_correction))


def oracle_lib():
    global _orc
    if _orc is None:
        lib = R._build(os.path.join(ROOT, "tests", "oracle_likelihood.c"), "liboraclelikelihood.so", False)
        lib.orc_set_math_mode(1)             # the fdlibm restatement, as tests/oracle_lib.py sets it
        lib.orc_index_build.restype = _P
        lib.orc_index_build.argtypes = [C.c_uint32, _P, _P, C.c_uint32]
        lib.orc_online_create.restype = _P
        lib.orc_online_create.argtypes = [_P, _P, C.c_uint64, C.c_uint32]
        lib.orc_online_state.argtypes = [_P, _P, _P, _P, _P]
        lib.orc_map_reads.argtypes = [_P, _P, _P, _P, C.c_uint32, C.c_uint32, C.c_uint64] + [_P] * 11
        lib.orc_lk_map_reads.argtypes = [_P, _P, _P, _P, _P, C.c_uint32, C.c_uint32, C.c_uint64] + [_P] * 12
        lib.orc_lk_online_batch.argtypes = [_P, _P, _P, _P, C.c_uint32, C.c_uint32] + [_P] * 12
        _orc = lib
    return _orc


class OracleIndex:
    def __init__(self, txps, k=31):
        lens = np.array([len(t) for t in txps], dtype=np.uint64)
        self.off = np.concatenate(([0], np.cumsum(lens))).astype(np.uint64)
        self.codes = np.ascontiguousarray(np.concatenate(txps).astype(np.uint8))
        self.n = len(txps)
        self.h = oracle_lib().orc_index_build(self.n, self.off.ctypes.data, self.codes.ctypes.data, k)


def oracle_map(oix, p, o, left, right, frag_counter=0):
    """stateless: orc_lk_map_reads; p: orc_map_params (tests/oracle_lib.py), o: orc_lk_opts"""
    import oracle_lib as O
    left = np.ascontiguousarray(left, dtype=np.uint8); right = np.ascontiguousarray(right, dtype=np.uint8)
    n, L = left.shape
    a = R._alloc(n, p.max_read_occ)
    ctr, nc = O.orc_map_counters(), np.zeros(1, np.uint64)
    oracle_lib().orc_lk_map_reads(oix.h, C.addressof(p), C.addressof(o), left.ctypes.data, right.ctypes.data, n, L,
                                  frag_counter, *[a[k].ctypes.data for k in KEYS], C.addressof(ctr), nc.ctypes.data)
    a["counters"] = ctr.asdict()
    a["counters"]["compatible"] = int(nc[0])
    return a


def oracle_map_unchanged(oix, p, left, right, frag_counter=0):
    """the oracle's own stateless path (oracle/map_oracle.c orc_map_reads), for the defaults"""
    import oracle_lib as O
    left = np.ascontiguousarray(left, dtype=np.uint8); right = np.ascontiguousarray(right, dtype=np.uint8)
    n, L = left.shape
    a = R._alloc(n, p.max_read_occ)
    ctr = O.orc_map_counters()
    oracle_lib().orc_map_reads(oix.h, C.addressof(p), left.ctypes.data, right.ctypes.data, n, L, frag_counter,
                               *[a[k].ctypes.data for k in KEYS], C.addressof(ctr))
    a["counters"] = ctr.asdict()
    return a


class OracleOnline:
    def __init__(self, oix, p, o, seed=42, mini_batch=5000):
        self.oix, self.p, self.o = oix, p, o
        self.h = oracle_lib().orc_online_create(oix.h, C.addressof(p), seed, mini_batch)

    def batch(self, left, right):
        import oracle_lib as O
        left = np.ascontiguousarray(left, dtype=np.uint8); right = np.ascontiguousarray(right, dtype=np.uint8)
        n, L = left.shape
        a = R._alloc(n, self.p.max_read_occ)
        ctr, nc = O.orc_map_counters(), np.zeros(1, np.uint64)
        oracle_lib().orc_lk_online_batch(self.h, C.addressof(self.o), left.ctypes.data, right.ctypes.data, n, L,
                                         *[a[k].ctypes.data for k in KEYS], C.addressof(ctr), nc.ctypes.data)
        a["counters"] = ctr.asdict()
        a["counters"]["compatible"] = int(nc[0])
        return a

    def state(self):
        M, nf = self.oix.n, self.p.max_frag_len + 1
        mass, hist, le, sc = np.zeros(M), np.zeros(nf), np.zeros(M), np.zeros(6, np.uint64)
        oracle_lib().orc_online_state(self.h, mass.ctypes.data, hist.ctypes.data, le.ctypes.data, sc.ctypes.data)
        return dict(mass=mass, hist=hist, log_eff=le, assigned=int(sc[0]), burned_in=int(sc[3]), min_val=int(sc[4]))


def same(a, o, cap):
    """per-read alignments and labels equal, bit for bit; returns the first differing field or None"""
    if not np.array_equal(a["n_aln"], o["n_aln"]):
        return "n_aln"
    m = np.arange(cap)[None, :] < a["n_aln"][:, None]
    for k in ("tid", "score", "pos", "mate_pos", "flags", "flen", "prob", "weight"):
        if not np.array_equal(a[k][m], o[k][m]):
            return k
    lm = np.arange(2 * cap)[None, :] < 2 * a["n_aln"][:, None]
    if not np.array_equal(a["label"][lm], o["label"][lm]):
        return "label"
    return None


def _rc(s):
    return (3 - s[::-1]).astype(np.uint8)


def stranded_workload(seed=5, n=3000, L=100, n_txps=40, antisense=0.3, single_end=False):
    """Transcripts of 600..2000 random bases, the last two of them decoys that copy stretches of the others; ISR
    (read 1 antisense, read 2 sense) fragments of about 250 bases, with planted cases:
      - antisense-only fragments (the mates swapped: ISF, incompatible with ISR), `antisense` of the reads;
      - fragments on a transcript that holds the same fragment twice, once per strand, so a compatible and an
        incompatible hit tie on one transcript (every 10th read);
      - an incompatible best hit above a compatible lower hit: a transcript pair where the compatible copy carries
        mismatches (every 13th read);
      - orphans: one mate replaced by random bases (every 9th read).
    single_end: read 1 only (SR-compatible unless antisense)."""
    rng = np.random.default_rng(seed)
    txps = [rng.integers(0, 4, int(rng.integers(600, 2000)), dtype=np.uint8) for _ in range(n_txps - 6)]
    # tie transcript: a 400-base stretch followed by its reverse complement
    s = rng.integers(0, 4, 400, dtype=np.uint8)
    txps.append(np.concatenate([s, rng.integers(0, 4, 50, dtype=np.uint8), _rc(s)]))
    # a compatible copy with mismatches and an exact antisense copy (two transcripts)
    u = rng.integers(0, 4, 500, dtype=np.uint8)
    mut = u.copy(); mut[np.arange(20, 500, 40)] ^= 1     # a mismatch every 40 bases: the seeds still hit
    txps.append(mut)
    txps.append(_rc(u))
    txps.append(rng.integers(0, 4, 900, dtype=np.uint8))
    # decoys (the suffix of the id space)
    txps.append(np.concatenate([txps[0][:300], rng.integers(0, 4, 300, dtype=np.uint8)]))
    txps.append(np.concatenate([rng.integers(0, 4, 200, dtype=np.uint8), txps[1][100:500]]))
    M = len(txps)
    first_decoy = M - 2
    left = np.zeros((n, L), np.uint8); right = np.zeros((n, L), np.uint8)
    for i in range(n):
        if i % 10 == 0:
            t = M - 6; fl = int(rng.integers(150, 250)); st = int(rng.integers(0, 400 - fl + 1)) if fl <= 400 else 0
        elif i % 13 == 0:
            t = -1; fl = int(rng.integers(200, 300)); st = int(rng.integers(0, 500 - fl + 1))
        else:
            t = int(rng.integers(0, first_decoy))
            T = len(txps[t])
            fl = int(np.clip(rng.normal(250, 25), L + 10, min(T, 400)))
            st = int(rng.integers(0, T - fl + 1))
        frag = u[st:st + fl] if t < 0 else txps[t][st:st + fl]
        r1, r2 = _rc(frag)[:L].copy(), frag[:L].copy()       # ISR: read 1 antisense, read 2 sense
        if i % 13 == 0:
            pass   # ISR with mismatches on the mutated copy of u, ISF and exact on the reverse complement of u
        elif rng.random() < antisense:
            r1, r2 = r2, r1                                  # antisense-only fragment
        if i % 9 == 0:
            (r1 if i % 2 else r2)[:] = rng.integers(0, 4, L, dtype=np.uint8)
        if rng.random() < 0.05:
            r1 = r1.copy(); r1[rng.integers(0, L, 3)] = rng.integers(0, 4, 3, dtype=np.uint8)
        left[i], right[i] = r1, r2
    if single_end:
        right[:] = 4
    return txps, first_decoy, left, right
