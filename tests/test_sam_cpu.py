"""SAM output, host side: the reader's names / qualities against a Python re-parse, and the shared record rules
(sam_core.h, compiled for the host) against the independent Python renderer in sam_ref.py."""
import ctypes as C
import gzip
import os
import subprocess
import tempfile

import numpy as np
import pytest

import sam_ref
from salmon_b200 import _capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CODE = {"A": 0, "C": 1, "G": 2, "T": 3}


def host_sam_lib():
    d = tempfile.mkdtemp(prefix="sb_host_sam_")
    so = os.path.join(d, "libhostsam.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared",
                           "-I" + os.path.join(ROOT, "include"), "-o", so, os.path.join(ROOT, "tests", "host_sam.cpp")])
    return C.CDLL(so)


def _records(rng, n, lens, crlf=False, comments=False, suffix=None):
    recs = []
    for i in range(n):
        L = int(rng.choice(lens))
        seq = "".join(rng.choice(list("ACGTNacgt"), L))
        qual = "".join(chr(33 + int(x)) for x in rng.integers(0, 41, L))
        name = f"read{i}_{rng.integers(1 << 30)}"
        hdr = name + (suffix or "") + (f" comment {i}\tx" if comments else "")
        recs.append((name, hdr, seq, qual))
    return recs


def _write(path, recs, crlf=False, fasta=False):
    nl = "\r\n" if crlf else "\n"
    txt = "".join((f">{h}{nl}{s}{nl}" if fasta else f"@{h}{nl}{s}{nl}+{nl}{q}{nl}") for _, h, s, q in recs)
    if path.endswith(".gz"):
        with gzip.open(path, "wt", newline="") as f:
            f.write(txt)
    else:
        with open(path, "w", newline="") as f:
            f.write(txt)


def _codes(s):
    return [CODE.get(c.upper(), 4) for c in s]


@pytest.mark.parametrize("gz", [False, True])
@pytest.mark.parametrize("crlf", [False, True])
@pytest.mark.parametrize("threads", [1, 8])
def test_reader_names_and_qualities(tmp_path, gz, crlf, threads):
    rng = np.random.default_rng(7 + gz + 2 * crlf + threads)
    n = 3000
    r1 = _records(rng, n, [60, 75], comments=True, suffix="/1")
    r2 = [(nm, nm + "/2", s, q) for (nm, _, s, q) in _records(rng, n, [60, 75])]
    ext = ".fq.gz" if gz else ".fq"
    p1, p2 = str(tmp_path / ("a" + ext)), str(tmp_path / ("b" + ext))
    _write(p1, r1, crlf=crlf)
    _write(p2, r2, crlf=crlf)
    got_names, got_q1, got_q2 = [], [], []
    with _capi.ReadFiles(p1, p2, n_threads=threads) as rf:
        while True:
            k, left, right, ll, lr, names, q1, q2 = rf.next_batch_meta(1024, 80, quals=True)
            if k == 0:
                break
            got_names += names
            got_q1 += [bytes(q1[i, :ll[i]]) for i in range(k)]
            got_q2 += [bytes(q2[i, :lr[i]]) for i in range(k)]
            for i in range(k):
                assert list(left[i, :ll[i]]) == _codes(r1[len(got_names) - k + i][2])
    assert got_names == [nm.encode() for nm, _, _, _ in r1]
    assert got_q1 == [q.encode() for _, _, _, q in r1]
    assert got_q2 == [q.encode() for _, _, _, q in r2]


def test_reader_names_single_end_fasta(tmp_path):
    rng = np.random.default_rng(3)
    recs = _records(rng, 500, [50], comments=True)
    p = str(tmp_path / "r.fa")
    _write(p, recs, fasta=True)
    with _capi.ReadFiles(p, None, n_threads=4) as rf:
        k, left, right, ll, lr, names, q1, q2 = rf.next_batch_meta(1000, 64, quals=True)
    assert k == 500 and right is None and q2 is None
    assert names == [nm.encode() for nm, _, _, _ in recs]
    assert all(bytes(q1[i, :50]) == b"I" * 50 for i in range(k))


@pytest.mark.parametrize("threads", [1, 8])
def test_bucketed_meta_keeps_names_with_rows(tmp_path, threads):
    """mixed lengths and too-short pairs through the bucketer: every delivered row carries its own name and qualities"""
    rng = np.random.default_rng(11)
    n = 6000
    r1 = _records(rng, n, [20, 50, 64, 64, 64, 90])
    r2 = [(nm, nm, s, q) for (nm, _, s, q) in _records(rng, n, [20, 50, 64, 64, 90])]
    p1, p2 = str(tmp_path / "a.fq.gz"), str(tmp_path / "b.fq.gz")
    _write(p1, r1)
    _write(p2, r2)
    by_name = {a[0].encode(): (a, b) for a, b in zip(r1, r2)}
    seen = []

    def fn(left, right, L, names, ql, qr):
        for i, nm in enumerate(names):
            (_, _, s1, q1), (_, _, s2, q2) = by_name[nm]
            assert list(left[i]) == _codes(s1[:L]) and list(right[i]) == _codes(s2[:L])
            assert bytes(ql[i]) == q1[:L].encode() and bytes(qr[i]) == q2[:L].encode()
            seen.append(nm)
        return 0
    with _capi.ReadFiles(p1, p2, n_threads=threads) as rf:
        st, dropped = rf.bucketed_meta(fn, min_len=31, batch=1000, max_read_len=96, threads=threads, quals=True)
    short = {nm.encode() for (nm, _, a, _), (_, _, b, _) in zip(r1, r2) if min(len(a), len(b)) < 31}
    assert set(dropped) == short and len(dropped) == st["n_too_short"]
    assert sorted(seen + dropped) == sorted(nm.encode() for nm, _, _, _ in r1)


def _render_host(lib, name, alns, left, right, ref_names, ref_lens, paired, ql=None, qr=None):
    a = np.array([x[:5] for x in alns], dtype=np.int64).reshape(-1, 5)
    tid = np.ascontiguousarray(a[:, 0], np.uint32); pos = np.ascontiguousarray(a[:, 1], np.int32)
    mpos = np.ascontiguousarray(a[:, 2], np.int32); fl = np.ascontiguousarray(a[:, 3], np.uint8)
    flen = np.ascontiguousarray(a[:, 4], np.int32)
    s1 = np.array([x[5] for x in alns], np.int32); s2 = np.array([x[6] for x in alns], np.int32)
    L = len(left)
    left = np.ascontiguousarray(left, np.uint8)
    right = np.ascontiguousarray(right if right is not None else left, np.uint8)
    rn = (C.c_char_p * len(ref_names))(*[x.encode() for x in ref_names])
    rl = np.ascontiguousarray(ref_lens, np.uint32)
    qlb = C.c_char_p(ql) if ql is not None else None
    qrb = C.c_char_p(qr) if qr is not None else None
    args = [name.encode(), len(name), len(alns)] + [x.ctypes.data for x in (tid, pos, mpos, fl, flen, s1, s2)] + \
           [int(paired), L, left.ctypes.data, right.ctypes.data, qlb, qrb, rn, rl.ctypes.data]
    lib.hs_render.restype = C.c_uint64
    P = C.c_void_p
    lib.hs_render.argtypes = [C.c_char_p, C.c_uint32, C.c_uint32] + [P] * 7 + [C.c_int, C.c_uint32, P, P, C.c_char_p,
                                                                             C.c_char_p, P, P, P]
    n = lib.hs_render(*args, None)
    buf = C.create_string_buffer(int(n))
    lib.hs_render(*args, buf)
    return buf.raw.decode().splitlines()


def test_record_rules_host_vs_python():
    lib = host_sam_lib()
    rng = np.random.default_rng(5)
    ref_names = ["txA", "txB_long_name", "decoy1"]
    ref_lens = [300, 1000, 5000]
    L = 50
    cases = [
        # (paired, alignments (tid, pos, mate_pos, flags, flen, score1, score2))
        (True, [(0, 10, 180, 0b01 | 0 << 2, 220, 100, 96)]),                      # concordant, mate 2 reverse
        (True, [(1, 300, 120, 0b10 | 0 << 2, 230, 88, 90)]),                      # mate 1 reverse, downstream
        (True, [(0, -7, 200, 0b01, 257, 80, 100), (1, 5, 160, 0b01, 205, 94, 92)]),   # left overhang, two hits
        (True, [(0, 270, 40, 0b10, 280, 70, 99)]),                                # right overhang (270 + 50 > 300)
        (True, [(0, -3, 260, 0b01, 313, 90, 70)]),
        (True, [(1, 44, 0, 0b01 | 1 << 2, 0, 99, 0)]),                             # mate-1 orphan, forward
        (True, [(1, 44, 0, 0b00 | 1 << 2, 0, 99, 0)]),                             # mate-1 orphan, reverse
        (True, [(0, 12, 0, 0b01 | 2 << 2, 0, 0, 77), (1, 900, 0, 0 | 2 << 2, 0, 0, 77)]),   # mate-2 orphans
        (True, [(2, 4000, 4100, 0b01, 150, 100, 100), (2, 10, 60, 0b01, 100, 100, 100)]),  # decoy alignments
        (False, [(0, 5, 0, 0b01 | 1 << 2, 0, 100, 0), (1, -2, 0, 0b00 | 1 << 2, 0, 96, 0)]),  # single-end
        (False, [(0, 280, 0, 0b00 | 1 << 2, 0, 60, 0)]),
    ]
    for qual in (False, True):
        for paired, alns in cases:
            left = rng.integers(0, 5, L).astype(np.uint8)
            right = rng.integers(0, 5, L).astype(np.uint8)
            ql = (33 + rng.integers(0, 41, L)).astype(np.uint8).tobytes() if qual else None
            qr = (33 + rng.integers(0, 41, L)).astype(np.uint8).tobytes() if qual else None
            want = sam_ref.render_fragment("frag/x", alns, left, right if paired else None, ref_names, ref_lens, paired,
                                           ql, qr if paired else None)
            got = _render_host(lib, "frag/x", alns, left, right if paired else None, ref_names, ref_lens, paired,
                               ql, qr if paired else None)
            assert got == want, (alns, got, want)
            hdr = "@HD\tVN:1.0\tSO:unknown\n@PG\tID:salmon\n"
            sam_ref.validate(hdr + "\n".join(got) + "\n")


def test_unmapped_types():
    assert sam_ref.unmapped_type(0, False, 0, True) == "u"
    assert sam_ref.unmapped_type(2, True, 0, True) == "d"
    assert sam_ref.unmapped_type(1, False, 1 << 2, True) == "m1"
    assert sam_ref.unmapped_type(1, False, 2 << 2, True) == "m2"
    assert sam_ref.unmapped_type(1, False, 0, True) is None
    assert sam_ref.unmapped_type(1, False, 1 << 2, False) is None
