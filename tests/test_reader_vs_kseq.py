"""The read-file parser of the product (sb_reads_*, csrc/ingest.cu + pgzip.h) against the parser the reference tree
vendors for the same job: klibpp's kseq++ (include/kseq++.hpp).  Same files -> the same records in the same order with
the same sequence lines, for plain / gzip / concatenated-gzip FASTQ with names and comments, qualities that begin with
'@' or '+', lower case and N, CRLF line ends, a missing final newline, and single-line FASTA.  What kseq++ returns for
each file is stored in tests/golden/kseq_records.json as a record count and one digest per block of records, recorded by
tests/golden/make_ref_golden.py from kseq++ compiled through oracle/ref_shims/kseq_parse.cpp."""
import gzip
import hashlib
import json
import os

import numpy as np

import pytest

from salmon_b200 import _capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "kseq_records.json")
BLOCK = 1000

ENC = np.full(256, 4, np.uint8)
for _c, _v in zip(b"ACGTacgtUu", [0, 1, 2, 3, 0, 1, 2, 3, 3, 3]):
    ENC[_c] = _v


def digests(records):
    """one digest per BLOCK records over their lengths and encoded sequences (codes 0..4)"""
    out = []
    for b in range(0, len(records), BLOCK):
        blk = records[b:b + BLOCK]
        h = hashlib.sha256(np.array([len(r) for r in blk], np.uint32).tobytes())
        for r in blk:
            h.update(np.ascontiguousarray(r, np.uint8).tobytes())
        out.append(h.hexdigest()[:16])
    return out


def _kseq(name):
    return json.load(open(GOLDEN))[name]


def _check(name, got):
    want = _kseq(name)
    assert len(got) == want["n"], (name, len(got), want["n"])
    bad = [i for i, (g, w) in enumerate(zip(digests(got), want["blocks"])) if g != w]
    assert not bad, (name, "records %d.. differ" % (bad[0] * BLOCK))


def _ours(path, threads, stride=320):
    got = []
    with _capi.ReadFiles(str(path), None, n_threads=threads) as rf:
        while True:
            k, left, _, ll, _ = rf.next_batch(30000, stride)
            if k == 0:
                break
            got += [left[i, :ll[i]].copy() for i in range(k)]
    return got


def _fastq(rng, n, crlf=False, final_newline=True):
    nl = b"\r\n" if crlf else b"\n"
    letters = np.frombuffer(b"ACGTNacgtn", dtype=np.uint8)
    quals = np.frombuffer(b"@+#,:FFFFFFIIII", dtype=np.uint8)
    recs = []
    for i in range(n):
        L = int(rng.integers(31, 301))
        s = letters[rng.integers(0, 4 if i % 5 else 10, L)].tobytes()
        q = quals[rng.integers(0, len(quals), L)].tobytes()
        name = b"@SRR77.%d" % i + (b" comment %d/1" % i if i % 3 else b"")
        recs.append(name + nl + s + nl + b"+" + (name[1:] if i % 7 == 0 else b"") + nl + q)
    return nl.join(recs) + (nl if final_newline else b"")


FLAVOURS = ["plain", "gzip", "multi", "crlf", "nofinal"]


def write_fastq(d, flavour):
    rng = np.random.default_rng({"plain": 1, "gzip": 2, "multi": 3, "crlf": 4, "nofinal": 5}[flavour])
    text = _fastq(rng, 60000, crlf=flavour == "crlf", final_newline=flavour != "nofinal")
    if flavour in ("plain", "crlf", "nofinal"):
        p = os.path.join(d, "r.fq")
        open(p, "wb").write(text)
    elif flavour == "gzip":
        p = os.path.join(d, "r.fq.gz")
        open(p, "wb").write(gzip.compress(text, 6))
    else:
        p = os.path.join(d, "r.fq.gz")
        step = len(text) // 4 + 1
        open(p, "wb").write(b"".join(gzip.compress(text[a:a + step], 5) for a in range(0, len(text), step)))
    return p


def write_fasta(d):
    rng = np.random.default_rng(9)
    letters = np.frombuffer(b"ACGTN", dtype=np.uint8)
    recs = []
    for i in range(20000):
        L = int(rng.integers(31, 301))
        recs.append(b">read%d some text\n" % i + letters[rng.integers(0, 5 if i % 9 == 0 else 4, L)].tobytes() + b"\n")
    p = os.path.join(d, "r.fa.gz")
    open(p, "wb").write(gzip.compress(b"".join(recs), 4))
    return p


@pytest.mark.parametrize("flavour", FLAVOURS)
def test_fastq_records_match_kseq(tmp_path, monkeypatch, flavour):
    monkeypatch.setenv("SB_READS_INFLATERS", "3")
    monkeypatch.setenv("SB_READS_SCANNERS", "3")
    p = write_fastq(str(tmp_path), flavour)
    assert _kseq(flavour)["n"] == 60000
    for threads in (1, 8):
        _check(flavour, _ours(p, threads))


def test_fasta_records_match_kseq(tmp_path):
    p = write_fasta(str(tmp_path))
    assert _kseq("fasta")["n"] == 20000
    _check("fasta", _ours(p, 8))
