"""TEST INFRASTRUCTURE for orphan rescue (--recoverOrphans, DESIGN.md section 11): the search cases edlib's goldens are
recorded for, the host build of the product's rescue (tests/host_rescue.cpp), the independent restatement on top of the
CPU oracle (tests/oracle_rescue.c), and a synthetic workload with planted orphans."""
import ctypes as C
import os
import subprocess
import tempfile
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "edlib_rescue.npz")
LENGTHS = (31, 63, 64, 65, 100, 127, 128, 129, 150, 200, 256)
_P = C.c_void_p


def _mutate(rng, s, n_edits):
    s = list(s)
    for _ in range(n_edits):
        kind = int(rng.integers(0, 3))
        pos = int(rng.integers(0, max(1, len(s))))
        if kind == 0 and s:
            s[pos] = (s[pos] + int(rng.integers(1, 4))) % 4 if s[pos] < 4 else int(rng.integers(0, 4))
        elif kind == 1:
            s.insert(pos, int(rng.integers(0, 4)))
        elif s:
            del s[pos]
    return np.array(s, dtype=np.uint8)


def search_cases(seed=71):
    """(pattern, window, K) triples: every read length of LENGTHS, windows of 1..2000 bases, 0..K+3 planted edits,
    repeats (ties), no hit, N (code 4) in the read and in the window"""
    rng = np.random.default_rng(seed)
    out = []
    for L in LENGTHS:
        K = int(0.35 * 2 * L / 2)
        for t in range(24):
            kind = t % 6
            W = int(rng.integers(1, 2001)) if t % 4 == 0 else int(rng.integers(L + 50, 2001))
            win = rng.integers(0, 4, W, dtype=np.uint8)
            pat = rng.integers(0, 4, L, dtype=np.uint8)
            if kind in (0, 1, 2) and W >= L + 8:
                start = int(rng.integers(0, W - L - 4))
                ne = int(rng.integers(0, K + 4)) if kind == 1 else int(rng.integers(0, 6))
                pat = _mutate(rng, win[start:start + L], ne)[:L]
                if len(pat) < L:
                    pat = np.concatenate([pat, rng.integers(0, 4, L - len(pat), dtype=np.uint8)])
            elif kind == 3 and W >= 2 * L + 2:   # the same stretch twice: equal distances at two ends
                start = int(rng.integers(0, W - 2 * L - 1))
                win[start + L + 1:start + 2 * L + 1] = win[start:start + L]
                pat = _mutate(rng, win[start:start + L], int(rng.integers(0, 3)))[:L]
                if len(pat) < L:
                    pat = np.concatenate([pat, rng.integers(0, 4, L - len(pat), dtype=np.uint8)])
            if kind == 4:                        # N in the read and in the window
                pat = pat.copy(); pat[rng.integers(0, L, 1 + L // 40)] = 4
                win[rng.integers(0, W, 1 + W // 100)] = 4
            if kind == 5 and W >= L + 8:         # N only in the window, the read planted across it
                start = int(rng.integers(0, W - L - 4))
                pat = win[start:start + L].copy()
                win[start + L // 2] = 4
            out.append((np.ascontiguousarray(pat, dtype=np.uint8), np.ascontiguousarray(win, dtype=np.uint8), K))
    return out


def case_crc(pat, win, K):
    return zlib.crc32(bytes(pat) + b"|" + bytes(win) + b"|" + str(K).encode())


def golden():
    g = np.load(GOLDEN)
    cases = search_cases()
    assert len(cases) == len(g["dist"])
    for i, (p, w, k) in enumerate(cases):
        assert case_crc(p, w, k) == int(g["crc"][i]), ("golden case differs", i)
    return cases, g["dist"], g["end"]


def _build(src, so_name, cxx):
    d = tempfile.mkdtemp(prefix="sb_rescue_")
    so = os.path.join(d, so_name)
    if cxx:
        cmd = ["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"),
               "-o", so, src]
    else:
        cmd = ["/usr/bin/gcc", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fPIC", "-fopenmp", "-shared",
               "-I" + os.path.join(ROOT, "oracle"), "-o", so, src, os.path.join(ROOT, "oracle", "em_oracle.c"), "-lm"]
    subprocess.check_call(cmd)
    return C.CDLL(so)


_host = _orc = None


def host_lib():
    global _host
    if _host is None:
        _host = _build(os.path.join(ROOT, "tests", "host_rescue.cpp"), "libhostrescue.so", True)
        _host.hrs_edit_limit.restype = C.c_int32
    return _host


def oracle_lib():
    global _orc
    if _orc is None:
        lib = _build(os.path.join(ROOT, "tests", "oracle_rescue.c"), "liboraclerescue.so", False)
        lib.orc_set_math_mode(1)             # the fdlibm restatement, as tests/oracle_lib.py sets it
        lib.orc_index_build.restype = C.c_void_p
        lib.orc_index_build.argtypes = [C.c_uint32, _P, _P, C.c_uint32]
        lib.orc_online_create.restype = C.c_void_p
        lib.orc_online_create.argtypes = [_P, _P, C.c_uint64, C.c_uint32]
        lib.orc_online_state.argtypes = [_P, _P, _P, _P, _P]
        lib.orc_rescue_online_batch.argtypes = [_P, _P, _P, C.c_uint32, C.c_uint32] + [_P] * 12
        lib.orc_rescue_map_reads.argtypes = [_P, _P, _P, _P, C.c_uint32, C.c_uint32, C.c_uint64] + [_P] * 12
        _orc = lib
    return _orc


def host_myers(pat, win, K):
    d, e = C.c_int32(), C.c_int32()
    host_lib().hrs_myers(pat.ctypes.data_as(_P), C.c_uint32(len(pat)), win.ctypes.data_as(_P), C.c_uint32(len(win)),
                         C.c_int32(K), C.byref(d), C.byref(e))
    return d.value, e.value


def sellers(pat, win, K):
    d, e = C.c_int32(), C.c_int32()
    oracle_lib().orc_sellers_infix(pat.ctypes.data_as(_P), C.c_uint32(len(pat)), win.ctypes.data_as(_P),
                                   C.c_uint32(len(win)), C.c_int32(K), C.byref(d), C.byref(e))
    return d.value, e.value


def _alloc(n, cap):
    return dict(n_aln=np.zeros(n, np.uint32), tid=np.zeros((n, cap), np.uint32), score=np.zeros((n, cap), np.int32),
                prob=np.zeros((n, cap)), pos=np.zeros((n, cap), np.int32), mate_pos=np.zeros((n, cap), np.int32),
                flags=np.zeros((n, cap), np.uint8), flen=np.zeros((n, cap), np.int32),
                label=np.zeros((n, 2 * cap), np.uint32), weight=np.zeros((n, cap)))


KEYS = ("n_aln", "tid", "score", "prob", "pos", "mate_pos", "flags", "flen", "label", "weight")


class OracleIndex:
    def __init__(self, txps, k=31):
        lens = np.array([len(t) for t in txps], dtype=np.uint64)
        self.off = np.concatenate(([0], np.cumsum(lens))).astype(np.uint64)
        self.codes = np.ascontiguousarray(np.concatenate(txps).astype(np.uint8))
        self.n = len(txps)
        self.h = oracle_lib().orc_index_build(self.n, self.off.ctypes.data, self.codes.ctypes.data, k)


def oracle_map(oix, p, left, right, frag_counter=0):
    """stateless: orc_rescue_map_reads; p: orc_map_params (tests/oracle_lib.py)"""
    import oracle_lib as O
    n, L = left.shape
    a = _alloc(n, p.max_read_occ)
    ctr, c3 = O.orc_map_counters(), np.zeros(3, np.uint64)
    oracle_lib().orc_rescue_map_reads(oix.h, C.addressof(p), left.ctypes.data, right.ctypes.data, n, L, frag_counter,
                                      *[a[k].ctypes.data for k in KEYS], C.addressof(ctr), c3.ctypes.data)
    a["counters"] = ctr.asdict()
    a["rescue"] = [int(x) for x in c3]
    return a


class OracleOnline:
    def __init__(self, oix, p, seed=42, mini_batch=5000):
        self.oix, self.p = oix, p
        self.h = oracle_lib().orc_online_create(oix.h, C.addressof(p), seed, mini_batch)

    def batch(self, left, right):
        import oracle_lib as O
        n, L = left.shape
        a = _alloc(n, self.p.max_read_occ)
        ctr, c3 = O.orc_map_counters(), np.zeros(3, np.uint64)
        oracle_lib().orc_rescue_online_batch(self.h, left.ctypes.data, right.ctypes.data, n, L,
                                             *[a[k].ctypes.data for k in KEYS], C.addressof(ctr), c3.ctypes.data)
        a["counters"] = ctr.asdict()
        a["rescue"] = [int(x) for x in c3]
        return a

    def state(self):
        M, nf = self.oix.n, self.p.max_frag_len + 1
        mass, hist, le, sc = np.zeros(M), np.zeros(nf), np.zeros(M), np.zeros(6, np.uint64)
        oracle_lib().orc_online_state(self.h, mass.ctypes.data, hist.ctypes.data, le.ctypes.data, sc.ctypes.data)
        return dict(mass=mass, hist=hist, log_eff=le, assigned=int(sc[0]), min_val=int(sc[4]))


def host_map(index, params, left, right, frag_counter=0):
    """the product's per-read path with rescue, compiled for the host; index: _capi.Index, params: sb_map_params"""
    import hostmap_lib
    ha = index.host_arrays()
    n, L = left.shape
    fld = hostmap_lib.fld_tables(params)
    a = _alloc(n, params.max_read_occ)
    c3 = np.zeros(3, np.uint64)
    host_lib().hrs_map_reads(C.c_uint32(index.n_txps), C.c_uint32(index.k), _P(ha["tx_off"]), _P(ha["codes"]),
                             _P(ha["table"]), C.c_uint64(ha["table_capacity"]), _P(ha["postings"]), C.byref(params),
                             fld.ctypes.data_as(_P), left.ctypes.data_as(_P), right.ctypes.data_as(_P), C.c_uint32(n),
                             C.c_uint32(L), C.c_uint64(frag_counter), *[a[k].ctypes.data_as(_P) for k in KEYS],
                             c3.ctypes.data_as(_P))
    a["rescue"] = [int(x) for x in c3]
    return a


def kill_seeds(read, rng, k=31):
    """substitutions spaced so that no k-mer of the read survives (every window of k bases holds one)"""
    r = read.copy()
    L = len(r)
    step = k - 6
    for q in range(int(rng.integers(3, step - 3)), L, step):
        r[q] = (r[q] + int(rng.integers(1, 4))) % 4 if r[q] < 4 else 0
    return r


def planted_workload(seed=5, n_genes=60, n=3000, n_planted=400, L=100, with_n=True, indels=True):
    """ordinary pairs + planted orphans (one mate made unseedable), transcripts with N, anchors near transcript ends.
    Returns txps, left, right, truth (tid, pos, flen, planted mask)."""
    from salmon_b200.synth import revcomp, synth_reads, synth_txome
    rng = np.random.default_rng(seed)
    txps, _ = synth_txome(seed=seed, n_genes=n_genes)
    clean = txps
    left, right, truth = synth_reads(clean, seed=seed + 1, n=n, read_len=L)
    txps = [t.copy() for t in clean]
    if with_n:                               # the index holds the N; the reads were drawn from the clean sequence
        for t in rng.choice(len(txps), max(1, len(txps) // 10), replace=False):
            txps[t][rng.integers(0, len(txps[t]), 2)] = 4
    planted = np.zeros(n, bool)
    lens = np.array([len(t) for t in txps])
    ok = np.flatnonzero(lens >= 400)
    for i in range(n_planted):
        t = int(rng.choice(ok))
        fl = int(np.clip(round(rng.normal(250, 25)), L + 20, min(600, lens[t])))
        near_end = i % 5 == 0
        pos = 0 if (near_end and i % 2) else (int(lens[t] - fl) if near_end else int(rng.integers(0, lens[t] - fl + 1)))
        frag = clean[t][pos:pos + fl]
        a, b = frag[:L].copy(), revcomp(frag[-L:]).copy()
        if rng.random() < 0.5:
            a, b = b, a
        victim = b if i % 2 == 0 else a
        victim[:] = kill_seeds(victim, rng)
        if indels and i % 3 == 0:           # an indel inside the band on top
            q = int(rng.integers(10, L - 10))
            victim[:] = np.concatenate([victim[:q], victim[q + 1:], rng.integers(0, 4, 1, dtype=np.uint8)])
        j = int(rng.integers(0, n))
        left[j], right[j] = a, b
        truth["tid"][j], truth["pos"][j], truth["flen"][j] = t, pos, fl
        planted[j] = True
    truth["planted"] = planted
    return txps, np.ascontiguousarray(left), np.ascontiguousarray(right), truth
