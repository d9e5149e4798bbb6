"""Scoring modes of the DP (--softclipOverhangs = 1, --softclip = 2; DESIGN.md section 12) on the GPU: the batch path
against the independent restatement (tests/oracle_softclip.c) bit for bit -- per-read alignments, labels, online state
and the merged class table; the ungapped shortcut off; planted adapter tails and overhangs; orphan rescue; the drivers."""
import gzip
import os
import subprocess

import numpy as np
import pytest

import oracle_lib as O
import rescue_ref as R
import softclip_ref as S
from salmon_b200 import _capi, quant
from salmon_b200._capi import Index, MapContext, map_default_params
from test_map_gpu import check_classes

pytestmark = pytest.mark.gpu
FIX = os.path.join(S.ROOT, "tests", "golden", "sample_data")
ACGT = "ACGT"


def _check_batch(a, o, cap, what=None):
    assert np.array_equal(a["n_aln"], o["n_aln"]), what
    m = np.arange(cap)[None, :] < a["n_aln"][:, None]
    for k in ("tid", "score", "pos", "mate_pos", "flags", "flen", "prob", "weight"):
        assert np.array_equal(a[k][m], o[k][m]), (what, k)
    lm = np.arange(2 * cap)[None, :] < 2 * a["n_aln"][:, None]
    assert np.array_equal(a["label"][lm], o["label"][lm]), what


@pytest.mark.parametrize("mode,L,chunk,overlap", [(1, 100, 0, 1), (2, 100, 1024, 0), (1, 150, 1024, 1), (2, 150, 0, 0),
                                                  (2, 100, 0, 1)])
def test_batch_equals_oracle(mode, L, chunk, overlap):
    txps, left, right = S.workload(seed=31 + L, n=3000, L=L, n_over=300)
    over = dict(num_pre_burnin=1000, num_burnin=5000)
    p = map_default_params(softclip=mode, **over)
    ctx = MapContext(Index(txps), p, batch_cap=4096, max_read_len=L)
    ctx.set_option("overlap_assign", overlap)
    if chunk:
        ctx.set_option("chunk", chunk)
    oix = S.OracleIndex(txps)
    on = S.OracleOnline(oix, O.map_params(**over), mode, seed=p.seed, mini_batch=p.mini_batch)
    parts = []
    for b in range(2):   # the second batch runs with the online state the first left
        sl = slice(b * 1500, (b + 1) * 1500)
        st = ctx.map_batch(left[sl], right[sl])
        want = on.batch(left[sl], right[sl])
        _check_batch(ctx.last_alignments(), want, p.max_read_occ, (mode, L, b))
        assert st.mapped == want["counters"]["mapped"]
        s, w = ctx.online_state(), on.state()
        assert np.array_equal(s["mass"], w["mass"]) and np.array_equal(s["hist"], w["hist"])
        parts.append(want)
    merged = {k: np.concatenate([q[k] for q in parts]) for k in ("n_aln", "label", "weight")}
    check_classes(ctx.finish(), O.eq_aggregate(merged, p.max_read_occ, True), exact_weights=False)
    ctx.close()


@pytest.mark.parametrize("mode", [1, 2])
def test_single_end_and_fast_dp_off(mode):
    txps, left, right = S.workload(seed=41, n=2000, n_over=250)
    idx, oix = Index(txps), S.OracleIndex(txps)
    # the ungapped shortcut is exact: the same alignments with it off
    outs = []
    for fast in (1, 0):
        ctx = MapContext(idx, map_default_params(softclip=mode), batch_cap=2048, max_read_len=100)
        ctx.set_option("fast_dp", fast)
        st = ctx.map_batch(left, right)
        outs.append((ctx.last_alignments(), st.full_dp))
        ctx.close()
    _check_batch(outs[0][0], outs[1][0], 200, "fast_dp")
    assert outs[1][1] > outs[0][1]
    want = S.oracle_map(oix, O.map_params(), mode, 0, left, right)
    _check_batch(outs[0][0], want, 200, "paired")
    # single-end reads (the oracle sees an all-N second mate)
    se = dict(lib_type=3, pre_merge_thresh=1.0)
    ctx = MapContext(idx, map_default_params(softclip=mode, **se), batch_cap=2048, max_read_len=100)
    ctx.map_batch(left, None)
    want = S.oracle_map(oix, O.map_params(**se), mode, 0, left, np.full_like(right, 4))
    _check_batch(ctx.last_alignments(), want, 200, "single-end")
    ctx.close()


def test_planted_adapters_and_overhangs():
    from salmon_b200.synth import synth_reads, synth_txome
    rng = np.random.default_rng(6)
    txps, _ = synth_txome(seed=6, n_genes=200)
    left, right, truth = synth_reads(txps, seed=7, n=4000, read_len=100)
    al, ar, _ = S.with_adapters(left, right, rng, 1.0, 25, 25)
    idx = Index(txps)
    res = {}
    for mode in (0, 1, 2):
        ctx = MapContext(idx, map_default_params(softclip=mode), batch_cap=4096, max_read_len=100)
        ctx.map_batch(al, ar)
        a = ctx.last_alignments()
        hit = [r for r in range(len(al)) if any(a["tid"][r, q] == truth["tid"][r] for q in range(a["n_aln"][r]))]
        res[mode] = (float((a["n_aln"] > 0).mean()), len(hit) / len(al))
        ctx.close()
    assert res[2][1] >= 0.95 and res[0][0] < 0.05, res   # measured on an H100: 0.966 and 0.0085
    # overhangs: the hanging mate scores ma * (L - k) in mode 1
    ol, orr, tids, k = S.overhang_pairs(txps, rng, 600)
    ctx = MapContext(idx, map_default_params(softclip=1), batch_cap=1024, max_read_len=100)
    ctx.map_batch(ol, orr)
    a = ctx.last_alignments()
    exact = at_least = 0
    for r in range(len(ol)):
        s = [a["score"][r, q] for q in range(a["n_aln"][r]) if a["tid"][r, q] == tids[r] and (a["flags"][r, q] >> 2) == 0]
        want = 2 * (100 - k[r]) + 200   # the other mate is exact; random overhang bases may add a little through a gap
        exact += bool(s) and s[0] == want
        at_least += bool(s) and s[0] >= want
    assert exact >= 0.8 * len(ol) and at_least >= 0.95 * len(ol), (exact, at_least)
    ctx.close()


@pytest.mark.parametrize("lib_type", [0, 1, 2])
def test_rescue_in_mode2_equals_oracle(lib_type):
    txps, left, right, truth = R.planted_workload(seed=11, n=3000, n_planted=400)
    al, ar, _ = S.with_adapters(left, right, np.random.default_rng(2), 0.1)
    over = dict(lib_type=lib_type, num_pre_burnin=1000, num_burnin=5000)
    p = map_default_params(recover_orphans=1, softclip=2, **over)
    ctx = MapContext(Index(txps), p, batch_cap=4096, max_read_len=100)
    on = S.OracleOnline(S.OracleIndex(txps), O.map_params(**over), 2, rescue=1, seed=p.seed, mini_batch=p.mini_batch)
    for b in range(2):
        sl = slice(b * 1500, (b + 1) * 1500)
        st = ctx.map_batch(al[sl], ar[sl])
        want = on.batch(al[sl], ar[sl])
        _check_batch(ctx.last_alignments(), want, p.max_read_occ, (lib_type, b))
        assert [st.orphans_rescued, st.rescue_searches, st.rescue_no_room] == want["rescue"]
        if lib_type == 0:
            assert want["rescue"][0] > 0
    ctx.close()


def _write_fq(path, m):
    with open(path, "w") as f:
        for i, s in enumerate(m):
            f.write(f"@p{i}\n{''.join(ACGT[c] for c in s)}\n+\n{'I' * len(s)}\n")


def test_drivers_agree(tmp_path):
    from salmon_b200.synth import synth_reads, synth_txome
    txps, _ = synth_txome(seed=9, n_genes=80)
    left, right, _ = synth_reads(txps, seed=10, n=4000, read_len=100)
    al, ar, _ = S.with_adapters(left, right, np.random.default_rng(3), 0.3)
    p1, p2 = str(tmp_path / "r1.fq"), str(tmp_path / "r2.fq")
    _write_fq(p1, al); _write_fq(p2, ar)
    idx = Index(txps)
    _capi.quant_files_native(idx, [p1], [p2], str(tmp_path / "n"), map_params=map_default_params(softclip=2), batch=4096,
                             max_read_len=100, threads=4)
    quant.quant_files(idx, [p1], [p2], str(tmp_path / "m"), batch=4096, max_read_len=100, threads=4, softclip=2)
    quant.quant_files(idx, [p1], [p2], str(tmp_path / "z"), batch=4096, max_read_len=100, threads=4)
    a, b, z = (open(str(tmp_path / d / "quant.sf"), "rb").read() for d in ("n", "m", "z"))
    assert a == b and a != z


def _sb(args):
    exe = os.path.join(os.path.dirname(_capi.LIB_PATH), "sb_salmon")
    r = subprocess.run([exe] + args, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return r


def test_cli_sample_data(tmp_path):
    idx = str(tmp_path / "idx")
    _sb(["index", "-t", os.path.join(FIX, "transcripts.fasta.gz"), "-i", idx])
    outs = {}
    for name, extra in (("plain", []), ("ovh", ["--softclipOverhangs"]), ("clip", ["--softclip"]),
                        ("both", ["--softclip", "--softclipOverhangs"])):
        out = str(tmp_path / name)
        _sb(["quant", "-i", idx, "-l", "IU", "-1", os.path.join(FIX, "reads_1.fastq.gz"), "-2",
             os.path.join(FIX, "reads_2.fastq.gz"), "-o", out, "--dumpEq", "--batch", "4096", "--maxReadLen", "64"] + extra)
        outs[name] = [open(os.path.join(out, "quant.sf"), "rb").read(),
                      gzip.decompress(open(os.path.join(out, "aux_info", "eq_classes.txt.gz"), "rb").read())]
        assert os.path.exists(os.path.join(out, "cmd_info.json"))
    assert outs["both"] == outs["clip"]          # both flags: mode 2
    assert len(outs["ovh"][0].splitlines()) == len(outs["plain"][0].splitlines())
