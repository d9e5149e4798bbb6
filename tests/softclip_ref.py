"""TEST INFRASTRUCTURE for the scoring modes of the DP (--softclipOverhangs, --softclip; DESIGN.md section 12): the
independent restatement on top of the CPU oracle (tests/oracle_softclip.c), the product's serial DP compiled for the host,
a pure-Python banded Gotoh of the three modes, and synthetic workloads with adapter tails and transcript overhangs."""
import ctypes as C
import os

import numpy as np

import rescue_ref as R

ROOT = R.ROOT
_P = C.c_void_p
KEYS = R.KEYS
ADAPTER = np.array(["ACGT".index(c) for c in "AGATCGGAAGAGCACACGTCTGAACTCCAGTCAC"], dtype=np.uint8)   # TruSeq read 1

_orc = _host = None


def oracle_lib():
    global _orc
    if _orc is None:
        lib = R._build(os.path.join(ROOT, "tests", "oracle_softclip.c"), "liboraclesoftclip.so", False)
        lib.orc_set_math_mode(1)             # the fdlibm restatement, as tests/oracle_lib.py sets it
        lib.orc_index_build.restype = _P
        lib.orc_index_build.argtypes = [C.c_uint32, _P, _P, C.c_uint32]
        lib.orc_online_create.restype = _P
        lib.orc_online_create.argtypes = [_P, _P, C.c_uint64, C.c_uint32]
        lib.orc_online_state.argtypes = [_P, _P, _P, _P, _P]
        lib.orc_sc_dp_score.restype = C.c_int32
        lib.orc_sc_dp_score.argtypes = [_P, _P, _P, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int32, C.c_int, C.c_int]
        lib.orc_dp_score.restype = C.c_int32
        lib.orc_dp_score.argtypes = [_P, _P, _P, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int32]
        lib.orc_sc_edit_limit.restype = C.c_int32
        lib.orc_sc_edit_limit.argtypes = [_P, C.c_int, C.c_uint32]
        lib.orc_sc_map_reads.argtypes = [_P, _P, C.c_int, C.c_int, _P, _P, C.c_uint32, C.c_uint32, C.c_uint64] + [_P] * 12
        lib.orc_sc_online_batch.argtypes = [_P, C.c_int, C.c_int, _P, _P, C.c_uint32, C.c_uint32] + [_P] * 12
        _orc = lib
    return _orc


class OracleIndex:
    def __init__(self, txps, k=31):
        lens = np.array([len(t) for t in txps], dtype=np.uint64)
        self.off = np.concatenate(([0], np.cumsum(lens))).astype(np.uint64)
        self.codes = np.ascontiguousarray(np.concatenate(txps).astype(np.uint8))
        self.n = len(txps)
        self.h = oracle_lib().orc_index_build(self.n, self.off.ctypes.data, self.codes.ctypes.data, k)


def oracle_dp(oix, p, read, ori, tid, diag, mode, form=0):
    """orc_sc_dp_score; p: orc_map_params (tests/oracle_lib.py)"""
    read = np.ascontiguousarray(read, dtype=np.uint8)
    return oracle_lib().orc_sc_dp_score(oix.h, C.addressof(p), read.ctypes.data, len(read), ori, tid, diag, mode, form)


def oracle_dp_default(oix, p, read, ori, tid, diag):
    """the CPU oracle's own (end-to-end) DP, orc_dp_score"""
    read = np.ascontiguousarray(read, dtype=np.uint8)
    return oracle_lib().orc_dp_score(oix.h, C.addressof(p), read.ctypes.data, len(read), ori, tid, diag)


def oracle_map(oix, p, mode, rescue, left, right, frag_counter=0):
    """stateless: orc_sc_map_reads"""
    import oracle_lib as O
    n, L = left.shape
    a = R._alloc(n, p.max_read_occ)
    ctr, c3 = O.orc_map_counters(), np.zeros(3, np.uint64)
    oracle_lib().orc_sc_map_reads(oix.h, C.addressof(p), mode, rescue, left.ctypes.data, right.ctypes.data, n, L,
                                  frag_counter, *[a[k].ctypes.data for k in KEYS], C.addressof(ctr), c3.ctypes.data)
    a["counters"] = ctr.asdict()
    a["rescue"] = [int(x) for x in c3]
    return a


class OracleOnline:
    def __init__(self, oix, p, mode, rescue=0, seed=42, mini_batch=5000):
        self.oix, self.p, self.mode, self.rescue = oix, p, mode, rescue
        self.h = oracle_lib().orc_online_create(oix.h, C.addressof(p), seed, mini_batch)

    def batch(self, left, right):
        import oracle_lib as O
        left = np.ascontiguousarray(left, dtype=np.uint8); right = np.ascontiguousarray(right, dtype=np.uint8)
        n, L = left.shape
        a = R._alloc(n, self.p.max_read_occ)
        ctr, c3 = O.orc_map_counters(), np.zeros(3, np.uint64)
        oracle_lib().orc_sc_online_batch(self.h, self.mode, self.rescue, left.ctypes.data, right.ctypes.data, n, L,
                                         *[a[k].ctypes.data for k in KEYS], C.addressof(ctr), c3.ctypes.data)
        a["counters"] = ctr.asdict()
        a["rescue"] = [int(x) for x in c3]
        return a

    def state(self):
        M, nf = self.oix.n, self.p.max_frag_len + 1
        mass, hist, le, sc = np.zeros(M), np.zeros(nf), np.zeros(M), np.zeros(6, np.uint64)
        oracle_lib().orc_online_state(self.h, mass.ctypes.data, hist.ctypes.data, le.ctypes.data, sc.ctypes.data)
        return dict(mass=mass, hist=hist, log_eff=le, assigned=int(sc[0]), min_val=int(sc[4]))


def product_dp(oix, params, read, ori, tid, diag):
    """the product's serial DP (map_core.h dp_score_serial, host build) in the mode params.softclip"""
    global _host
    if _host is None:
        import hostmap_lib
        _host = hostmap_lib.build()
        _host.hmc_dp_score.restype = C.c_int32
    lib = _host
    read = np.ascontiguousarray(read, dtype=np.uint8)
    return lib.hmc_dp_score(_P(oix.off.ctypes.data), _P(oix.codes.ctypes.data), C.byref(params), _P(read.ctypes.data),
                            C.c_uint32(len(read)), C.c_uint32(ori), C.c_uint32(tid), C.c_int32(diag))


NEG = -(1 << 28)


def gotoh(ref, read, diag, band, ma, mp, go, ge, mode):
    """pure-Python banded affine DP of the oriented read against ref, the three modes (DESIGN.md section 12)"""
    W, tlen, L = 2 * band + 1, len(ref), len(read)
    H, E = [0] * W, [NEG] * W
    best = NEG
    for i in range(L):
        Hn, En = [NEG] * W, [NEG] * W
        hl = fp = NEG            # the left neighbour's H and F in this row
        for j in range(W):
            r = diag + i + j - band
            h = e = f = NEG
            if 0 <= r < tlen:    # cells outside the transcript are dead
                s = ma if (read[i] < 4 and read[i] == ref[r]) else mp
                d = H[j]
                if mode == 2 or (mode == 1 and r == 0):
                    d = max(d, 0)
                if j + 1 < W:
                    e = max(H[j + 1] - go - ge, E[j + 1] - ge)
                if j > 0:
                    f = max(hl - go - ge, fp - ge)
                h, e, f = max(d + s, e, f, NEG), max(e, NEG), max(f, NEG)
                if mode == 2 or (mode == 1 and r == tlen - 1):
                    best = max(best, h)
            Hn[j], En[j] = h, e
            hl, fp = h, f
        H, E = Hn, En
    return max([best] + H)


def oriented(read, ori):
    read = np.asarray(read, dtype=np.uint8)
    if not ori:
        return read
    r = read[::-1]
    return np.where(r > 3, 4, 3 - r).astype(np.uint8)


def dp_cases(seed, n, txps, max_len=256):
    """(read, ori, tid, diag) cases: 31..max_len bases, both strands, N in the read, reads hanging 1..40 bases over either
    transcript end (a third of them), planted substitutions and indels"""
    from salmon_b200.synth import revcomp
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        t = int(rng.integers(0, len(txps)))
        ref = txps[t]
        tl = len(ref)
        L = int(rng.integers(31, max_len + 1))
        kind = int(rng.integers(0, 3))
        if kind == 0:
            pos = -int(rng.integers(1, 41))
        elif kind == 1:
            pos = tl - L + int(rng.integers(1, 41))
        else:
            pos = int(rng.integers(0, max(1, tl - L + 1)))
        seg = np.array([ref[q] if 0 <= q < tl else int(rng.integers(0, 4)) for q in range(pos, pos + L)], dtype=np.uint8)
        for _e in range(int(rng.integers(0, 6))):
            q = int(rng.integers(0, L))
            c = int(rng.integers(0, 3))
            if c == 0:
                seg[q] = (seg[q] + int(rng.integers(1, 4))) % 4
            elif c == 1:
                seg = np.concatenate([seg[:q], rng.integers(0, 4, 1, dtype=np.uint8), seg[q:]])[:L]
            else:
                seg = np.concatenate([seg[:q], seg[q + 1:], rng.integers(0, 4, 1, dtype=np.uint8)])
        if rng.random() < 0.2:
            seg[rng.integers(0, L, 1 + L // 50)] = 4
        if rng.random() < 0.3:   # a junk tail
            c = int(rng.integers(1, 31))
            seg[L - c:] = rng.integers(0, 4, c, dtype=np.uint8)
        ori = int(rng.integers(0, 2))
        read = oriented(seg, ori)   # the reverse complement (N stays N) when ori = 1
        out.append((np.ascontiguousarray(read, dtype=np.uint8), ori, t, pos + int(rng.integers(-3, 4))))
    return out


def dp_txome(seed=1):
    """transcripts of 40..1500 bases, some with N"""
    rng = np.random.default_rng(seed)
    txps = [rng.integers(0, 4, int(rng.integers(40, 1500)), dtype=np.uint8) for _ in range(24)]
    for t in range(0, 24, 5):
        txps[t][rng.integers(0, len(txps[t]), 3)] = 4
    return txps


def with_adapters(left, right, rng, frac, lo=20, hi=30):
    """a fraction of the pairs read through into the adapter: the last lo..hi bases of both mates replaced by adapter
    sequence (random bases beyond the adapter's 34).  Returns copies and the mask of the pairs changed."""
    left, right = left.copy(), right.copy()
    n, L = left.shape
    sel = rng.random(n) < frac
    for r in np.flatnonzero(sel):
        for m in (left, right):
            c = int(rng.integers(lo, hi + 1))
            tail = np.concatenate([ADAPTER, rng.integers(0, 4, max(0, c - len(ADAPTER)), dtype=np.uint8)])[:c]
            m[r, L - c:] = tail
    return np.ascontiguousarray(left), np.ascontiguousarray(right), sel


def overhang_pairs(txps, rng, n, L=100, max_over=40):
    """pairs whose fragment hangs 1..max_over bases over a transcript end (the overhang is random sequence).  Returns
    left, right, tid, over (bases of the hanging mate outside the transcript)."""
    from salmon_b200.synth import revcomp
    lens = np.array([len(t) for t in txps])
    ok = np.flatnonzero(lens >= 400)
    left = np.zeros((n, L), np.uint8); right = np.zeros((n, L), np.uint8)
    tids = np.zeros(n, np.int64); over = np.zeros(n, np.int64)
    for i in range(n):
        t = int(rng.choice(ok)); ref = txps[t]; tl = len(ref)
        k = int(rng.integers(1, max_over + 1))
        fl = int(rng.integers(L + 20, 300))
        start = -k if i % 2 == 0 else tl - fl + k
        frag = np.array([ref[q] if 0 <= q < tl else int(rng.integers(0, 4)) for q in range(start, start + fl)], np.uint8)
        a, b = frag[:L].copy(), revcomp(frag[-L:]).copy()
        if rng.random() < 0.5:
            a, b = b, a
        left[i], right[i], tids[i], over[i] = a, b, t, k
    return np.ascontiguousarray(left), np.ascontiguousarray(right), tids, over


def workload(seed=21, n=3000, L=100, n_genes=60, frac_adapter=0.15, n_over=300, with_n=True):
    """ordinary pairs, pairs with adapter tails, pairs hanging over transcript ends, transcripts with N"""
    from salmon_b200.synth import synth_reads, synth_txome
    rng = np.random.default_rng(seed)
    txps, _ = synth_txome(seed=seed, n_genes=n_genes)
    left, right, _ = synth_reads(txps, seed=seed + 1, n=n, read_len=L)
    left, right, _ = with_adapters(left, right, rng, frac_adapter)
    ol, orr, _, _ = overhang_pairs(txps, rng, n_over, L=L)
    idx = rng.choice(n, n_over, replace=False)
    left[idx], right[idx] = ol, orr
    if with_n:
        txps = [t.copy() for t in txps]
        for t in rng.choice(len(txps), max(1, len(txps) // 10), replace=False):
            txps[t][rng.integers(0, len(txps[t]), 2)] = 4
    return txps, np.ascontiguousarray(left), np.ascontiguousarray(right)
