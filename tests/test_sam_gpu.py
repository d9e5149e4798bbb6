"""SAM output on the GPU (`--writeMappings`, `--writeQualities`, `--writeUnmappedNames`): record for record against the
Python renderer of the rules applied to the host build of the mapping logic, a forced-small output window, the
sample data through the command line, and the native driver against the Python mirror."""
import ctypes as C
import gzip
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import oracle_lib as O
import sam_ref
from salmon_b200 import _capi, quant
from salmon_b200.synth import revcomp, synth_reads, synth_txome

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIX = os.path.join(ROOT, "tests", "golden", "sample_data")
ACGT = "ACGT"


def _oracle_sam_lib():
    """tests/oracle_sam.c: the SAM side output restated on top of the CPU oracle"""
    d = tempfile.mkdtemp(prefix="sb_oracle_sam_")
    so = os.path.join(d, "liboraclesam.so")
    subprocess.check_call(["/usr/bin/gcc", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fPIC", "-fopenmp", "-shared",
                           "-I" + os.path.join(ROOT, "oracle"), "-o", so, os.path.join(ROOT, "tests", "oracle_sam.c"),
                           os.path.join(ROOT, "oracle", "em_oracle.c"), "-lm"])
    lib = C.CDLL(so)
    lib.orc_index_build.restype = C.c_void_p
    lib.orc_index_build.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32]
    lib.orc_sam_side.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 10
    return lib


def _workload(seed=21):
    """transcripts (the last 6 are decoys), reads of two lengths with multi-mappers, orphans and overhanging reads"""
    txps, _ = synth_txome(seed=seed, n_genes=40)
    rng = np.random.default_rng(seed)
    batches = []
    for L, n in ((76, 1500), (60, 700)):
        left, right, _ = synth_reads(txps, seed=seed + L, n=n, read_len=L)
        k = n // 10
        right[:k] = rng.integers(0, 4, (k, L))                     # mate 1 only
        left[k:2 * k] = rng.integers(0, 4, (k, L))                 # mate 2 only
        for i in range(2 * k, 2 * k + 40):                        # reads hanging over a transcript's start
            t = txps[i % len(txps)]
            h = 3 + i % 9
            left[i] = np.concatenate([rng.integers(0, 4, h), t[:L - h]])
            right[i] = revcomp(t[150:150 + L])
        for i in range(2 * k + 40, 2 * k + 80):                   # ... and over its end
            t = txps[i % len(txps)]
            h = 3 + i % 9
            right[i] = revcomp(np.concatenate([t[len(t) - (L - h):], rng.integers(0, 4, h)]))
            left[i] = t[len(t) - 200:len(t) - 200 + L]
        names = [f"r{L}_{i}" for i in range(n)]
        batches.append((left, right, names))
    return txps, batches


def _expected(txps, batches, ref_names, first_decoy, paired=True, qualities=None):
    """oracle mapping (oracle_lib.map_reads) + its SAM side output (tests/oracle_sam.c) + the Python renderer
    -> (SAM records, unmapped lines)"""
    lib = _oracle_sam_lib()
    op = O.map_params(first_decoy=first_decoy, lib_type=0 if paired else 3)
    oix = O.MapIndex(txps)
    off, codes = O.pack_txome(txps)
    six = lib.orc_index_build(len(txps), off.ctypes.data, codes.ctypes.data, 31)
    cap = op.max_read_occ
    ref_lens = [len(t) for t in txps]
    recs, un = [], []
    for b, (left, right, names) in enumerate(batches):
        n, L = left.shape
        left = np.ascontiguousarray(left, np.uint8)
        right = np.ascontiguousarray(right if paired else np.full((n, L), 4, np.uint8), np.uint8)
        m = O.map_reads(oix, op, left, right, 0)
        o = {k: np.ascontiguousarray(m[k]) for k in ("tid", "pos", "mate_pos", "flags", "flen")}
        n_out = np.zeros(n, np.uint32); decoy = np.zeros(n, np.uint8)
        s1 = np.zeros((n, cap), np.int32); s2 = np.zeros((n, cap), np.int32)
        assert lib.orc_sam_side(six, C.addressof(op), left.ctypes.data, right.ctypes.data, n, L, m["n_aln"].ctypes.data,
                                *[o[k].ctypes.data for k in ("tid", "pos", "mate_pos", "flags", "flen")],
                                n_out.ctypes.data, decoy.ctypes.data, s1.ctypes.data, s2.ctypes.data) == 0
        for r in range(n):
            a = [(int(o["tid"][r, j]), int(o["pos"][r, j]), int(o["mate_pos"][r, j]), int(o["flags"][r, j]),
                  int(o["flen"][r, j]), int(s1[r, j]), int(s2[r, j])) for j in range(n_out[r])]
            q = qualities[b] if qualities else (None, None)
            recs += sam_ref.render_fragment(names[r], a, left[r], right[r] if paired else None, ref_names, ref_lens,
                                            paired, None if q[0] is None else q[0][r].tobytes(),
                                            None if (q[1] is None or not paired) else q[1][r].tobytes())
            t = sam_ref.unmapped_type(int(n_out[r]), bool(decoy[r]), int(o["flags"][r, 0]), paired)
            if t:
                un.append(f"{names[r]} {t}")
    return recs, un


def _check_semantics(frags, txps, paired):
    """field meanings from the SAM specification, independent of how the records were made: the aligned bases of a
    forward or reverse record lie on the reference where POS and CIGAR put them (mostly matching), TLEN spans the two
    mates' outer ends"""
    match = total = 0
    for f in frags:
        for r in f:
            flag = int(r[1])
            if flag & 0x4:
                continue
            t = txps[int(r[2][1:])]
            lc, mlen = re.match(r"(?:(\d+)S)?(\d+)M", r[5]).groups()
            lc, mlen = int(lc or 0), int(mlen)
            p0 = int(r[3]) - 1
            seq = r[9][lc:lc + mlen]
            ref = "".join("ACGTN"[c] for c in t[p0:p0 + mlen])
            match += sum(x == y for x, y in zip(seq, ref))
            total += mlen
    assert match > 0.9 * total


def _run_gpu(txps, mp, batches, tmp_path, window=None, qualities=None):
    idx = _capi.Index(txps)
    sam, unp = str(tmp_path / "out.sam"), str(tmp_path / "un.txt")
    mc = _capi.MapContext(idx, mp, batch_cap=2048, max_read_len=96)
    if window:
        mc.set_option("sam_window_bytes", window)
    sink = _capi.SamSink(idx, sam, unp, cmdline="test run", qualities=qualities is not None)
    mc.attach_sam(sink)
    for b, (left, right, names) in enumerate(batches):
        mc.map_batch_sam(left, right, names, qualities[b] if qualities else None)
    st = sink.stats()
    mc.attach_sam(None)
    sink.close()
    mc.close()
    return idx, open(sam).read(), open(unp).read(), st


@pytest.mark.parametrize("window", [None, 4096])
def test_gpu_sam_equals_oracle(tmp_path, window):
    txps, batches = _workload()
    mp = _capi.map_default_params()
    mp.first_decoy = len(txps) - 6
    rng = np.random.default_rng(4)
    quals = [((33 + rng.integers(0, 41, l.shape)).astype(np.uint8), (33 + rng.integers(0, 41, l.shape)).astype(np.uint8))
             for l, _, _ in batches]
    idx, text, un, st = _run_gpu(txps, mp, batches, tmp_path, window, quals)
    ref_names = [f"t{i}" for i in range(len(txps))]
    want, want_un = _expected(txps, batches, ref_names, mp.first_decoy, True, quals)
    lines = text.splitlines()
    hdr = [ln for ln in lines if ln.startswith("@")]
    assert hdr[0] == "@HD\tVN:1.0\tSO:unknown"
    assert hdr[1:-1] == [f"@SQ\tSN:t{i}\tLN:{len(t)}" for i, t in enumerate(txps)]
    assert hdr[-1].startswith("@PG\tID:salmon\tPN:salmon\tVN:") and hdr[-1].endswith("\tCL:test run")
    got = [ln for ln in lines if not ln.startswith("@")]
    assert got == want
    assert un.splitlines() == want_un
    frags = sam_ref.validate(text, len(txps))
    _check_semantics(frags, txps, True)
    flags = [int(r[1]) for f in frags for r in f]
    # the workload exercises what it is meant to
    assert any(f & 0x8 for f in flags) and any(f & 0x4 for f in flags) and any(f & 0x100 for f in flags)
    assert any("S" in r[5] and r[5].index("S") < r[5].index("M") for f in frags for r in f)
    assert any(r[5].endswith("S") for f in frags for r in f)
    dec = [f for f in frags if int(f[0][2][1:]) >= mp.first_decoy]
    assert dec and all(int(r[2][1:]) >= mp.first_decoy for f in dec for r in f)
    assert {"u", "m1", "m2", "d"} <= {ln.split()[1] for ln in un.splitlines()}
    # AS is each mate's own score: the two mates of a pair differ somewhere
    assert any(r1[12] != r2[12] for f in frags for r1, r2 in zip(f[0::2], f[1::2]) if len(r1) > 12 and len(r2) > 12)
    if window:
        assert st["windows"] > len(batches)


def test_gpu_sam_single_end(tmp_path):
    txps, batches = _workload(seed=8)
    mp = _capi.map_default_params(lib_type=3)
    mp.first_decoy = len(txps) - 6
    se = [(left, None, names) for left, _, names in batches]
    idx, text, un, _ = _run_gpu(txps, mp, se, tmp_path)
    want, want_un = _expected(txps, [(l, l, nm) for l, _, nm in se], [f"t{i}" for i in range(len(txps))], mp.first_decoy,
                              paired=False)
    got = [ln for ln in text.splitlines() if not ln.startswith("@")]
    assert got == want and un.splitlines() == want_un
    frags = sam_ref.validate(text, len(txps))
    _check_semantics(frags, txps, False)
    assert all(int(r[1]) & ~0x110 == 0 and r[6] == "*" and r[7] == "0" and r[8] == "0" for f in frags for r in f)
    assert any(int(r[1]) & 0x10 for f in frags for r in f) and any(int(r[1]) & 0x100 for f in frags for r in f)


def test_no_sink_no_extra_kernel():
    txps, batches = _workload()
    mp = _capi.map_default_params()
    idx = _capi.Index(txps)
    mc = _capi.MapContext(idx, mp, batch_cap=2048, max_read_len=96)
    left, right, _ = batches[0]
    a = mc.map_batch(left, right).gpu_launches
    b = mc.map_batch(left, right).gpu_launches
    mc.close()
    mc2 = _capi.MapContext(idx, mp, batch_cap=2048, max_read_len=96)
    sink = _capi.SamSink(idx, os.devnull, None)
    mc2.attach_sam(sink)
    c = mc2.map_batch(left, right).gpu_launches       # a plain batch on a context with a sink: no SAM work
    mc2.attach_sam(None)
    sink.close()
    mc2.close()
    assert a == c and b > a


def _sample_quant(tmp_path, extra, name):
    exe = os.path.join(os.path.dirname(_capi.LIB_PATH), "sb_salmon")
    idx = str(tmp_path / "idx")
    if not os.path.exists(idx):
        r = subprocess.run([exe, "index", "-t", os.path.join(FIX, "transcripts.fasta.gz"), "-i", idx], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    out = str(tmp_path / name)
    r = subprocess.run([exe, "quant", "-i", idx, "-l", "IU", "-1", os.path.join(FIX, "reads_1.fastq.gz"), "-2",
                        os.path.join(FIX, "reads_2.fastq.gz"), "-o", out, "--dumpEq", "--batch", "4096", "--maxReadLen", "64"]
                       + extra, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out, r


def test_sample_data_sam(tmp_path):
    base, _ = _sample_quant(tmp_path, [], "plain")
    sam = str(tmp_path / "m.sam")
    out, _ = _sample_quant(tmp_path, ["--writeMappings=" + sam, "--writeUnmappedNames", "--writeQualities"], "sam")
    for f in ("quant.sf", "aux_info/eq_classes.txt.gz"):
        a, b = open(os.path.join(base, f), "rb").read(), open(os.path.join(out, f), "rb").read()
        if f.endswith(".gz"):
            a, b = gzip.decompress(a), gzip.decompress(b)
        assert a == b, f
    text = open(sam).read()
    names = [ln[1:].split()[0] for ln in gzip.open(os.path.join(FIX, "transcripts.fasta.gz"), "rt") if ln.startswith(">")]
    frags = sam_ref.validate(text, 15)
    sq = [ln.split("\t") for ln in text.splitlines() if ln.startswith("@SQ")]
    assert [x[1][3:] for x in sq] == names
    un = {ln.split()[0] for ln in open(os.path.join(out, "aux_info", "unmapped_names.txt"))}
    by = {f[0][0]: f for f in frags}
    assert len(by) == len(frags)                     # one run of records per pair
    assert len(by) + len(un - set(by)) == 10000     # every pair has records or is listed as unmapped
    assert len(by) > 9500
    pos0 = pos1 = tlen_ok = uniq = 0
    for qn, recs in by.items():
        _, tx, pos, flen = qn.split(":")
        hit = [r for r in recs if r[2] == tx]
        assert hit, qn
        lm = [min(int(r[3]) for r in hit[k:k + 2]) for k in range(0, len(hit), 2)]   # leftmost POS per alignment
        pos0 += int(pos) + 1 in lm                   # (simulated positions 0-based)
        pos1 += int(pos) in lm                       # (or 1-based)
        if len(recs) == 2 and int(recs[0][1]) & 0x2:
            uniq += 1
            tlen_ok += abs(int(recs[0][8])) == int(flen)
    assert max(pos0, pos1) > 0.97 * len(by), (pos0, pos1, len(by))
    assert tlen_ok > 0.97 * uniq
    assert all(len(r[10]) == len(r[9]) for f in frags for r in f)
    # -z: the same SAM on standard output, and nothing else there (the command line in @PG differs)
    _, r = _sample_quant(tmp_path, ["-z", "--writeQualities"], "stdout")
    strip = lambda t: [ln for ln in t.splitlines() if not ln.startswith("@PG")]
    assert strip(r.stdout) == strip(text)
    sam_ref.validate(r.stdout, 15)


def test_native_and_python_mirror_write_the_same_sam(tmp_path):
    txps, _ = synth_txome(seed=5, n_genes=50)
    left, right, _ = synth_reads(txps, seed=6, n=6000, read_len=80)
    right[:300] = np.random.default_rng(1).integers(0, 4, (300, 80))
    p1, p2 = str(tmp_path / "r1.fq"), str(tmp_path / "r2.fq")
    for p, m in ((p1, left), (p2, right)):
        with open(p, "w") as f:
            for i, s in enumerate(m):
                f.write(f"@p{i} x\n{''.join(ACGT[c] for c in s)}\n+\n{'I' * len(s)}\n")
    idx = _capi.Index(txps)
    a, b = str(tmp_path / "native.sam"), str(tmp_path / "mirror.sam")
    _capi.quant_files_native(idx, [p1], [p2], str(tmp_path / "n"), batch=2048, max_read_len=96, threads=4,
                             write_mappings=a.encode(), write_qualities=1, write_unmapped_names=1, cmdline=b"cl", dump_eq=1)
    _capi.quant_files_native(idx, [p1], [p2], str(tmp_path / "plain"), batch=2048, max_read_len=96, threads=4, dump_eq=1)
    for f in ("quant.sf", "aux_info/eq_classes.txt.gz"):   # SAM output changes no other output
        x, y = open(str(tmp_path / "n" / f), "rb").read(), open(str(tmp_path / "plain" / f), "rb").read()
        assert (gzip.decompress(x) == gzip.decompress(y)) if f.endswith(".gz") else x == y, f
    quant.quant_files(idx, [p1], [p2], str(tmp_path / "m"), batch=2048, max_read_len=96, threads=4,
                      write_mappings=b, write_qualities=True, write_unmapped_names=True, cmdline="cl")
    assert open(a, "rb").read() == open(b, "rb").read()
    ua = open(str(tmp_path / "n" / "aux_info" / "unmapped_names.txt"), "rb").read()
    ub = open(str(tmp_path / "m" / "aux_info" / "unmapped_names.txt"), "rb").read()
    assert ua == ub and len(ua) > 0
    sam_ref.validate(open(a).read(), len(txps))


def test_sharded_run_refuses_sam(tmp_path):
    exe = os.path.join(os.path.dirname(_capi.LIB_PATH), "sb_salmon")
    r = subprocess.run([exe, "quant", "-i", "x", "-l", "IU", "-1", "a", "-2", "b", "-o", str(tmp_path / "o"), "--gpus", "2",
                        "--writeMappings"], capture_output=True, text=True)
    assert r.returncode != 0 and "one-GPU run only" in r.stderr
