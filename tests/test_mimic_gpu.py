"""The Bowtie2-mimicking presets (`--mimicBT2`, `--mimicStrictBT2`), `--minAlnProb` and `--maxReadOcc` up to 1000 on
the GPU (DESIGN.md section 14): the mapping path against the oracle bit for bit under both presets, gapless settlement
in k_dp_classify (which alignments still reach the banded DP), reads with more than 255 joint hits, and the drivers."""
import json
import os
import subprocess

import numpy as np
import pytest

import mimic_ref as MR
import oracle_lib as O
import rescue_ref as R
import softclip_ref as S
from salmon_b200 import _capi, quant
from salmon_b200._capi import Index, MapContext, map_default_params
from salmon_b200.synth import synth_txome
from test_map_gpu import bits, check_classes, check_state
from test_map_host import compare
from test_map_options_gpu import check, gpu_map

pytestmark = pytest.mark.gpu
FIX = os.path.join(R.ROOT, "tests", "golden", "sample_data")


def _workload(over, L, seed, n=1200):
    """mates on both sides of s_min, planted indels and pairs hanging over a transcript end (the edge list); no N"""
    rng = np.random.default_rng(seed)
    txps, _ = synth_txome(seed=seed, n_genes=40)
    left, right, _ = MR.around_s_min(txps, over, L, n, seed)
    k = n // 10
    ol, orr, _, _ = S.overhang_pairs(txps, rng, k, L=L)
    left[-k:], right[-k:] = ol, orr
    return txps, np.ascontiguousarray(left), np.ascontiguousarray(right)


@pytest.mark.parametrize("strict", [False, True])
@pytest.mark.parametrize("L", [75, 100, 150])
def test_presets_equal_oracle(oracle, strict, L):
    """paired-end reads, shortcut on and off, one chunk and several: alignments, labels and counters are the oracle's.
    With the shortcut on, gapless settlement leaves nothing for the banded DP where it applies (strict, L < 125: the
    interior and the edge alignments are settled, and this workload has no N); elsewhere the DP runs as before."""
    over = MR.preset_over(strict)
    txps, left, right = _workload(over, L, seed=300 + L + strict)
    ref = oracle.map_reads(oracle.MapIndex(txps), oracle.map_params(**over), left, right, 0)
    idx = Index(txps)
    settles = MR.gapless(over, L)
    assert settles == (strict and L < 125)
    for opts in (dict(fast_dp=1), dict(fast_dp=0), dict(fast_dp=1, chunk=300)):
        got, st = gpu_map(idx, left, right, opts, **over)
        check(got, st, ref, over["max_read_occ"], (strict, L, opts))
        if not opts["fast_dp"]:
            assert st.full_dp == st.candidates > 0
        elif settles:
            assert st.full_dp == 0 and st.candidates > 0
        else:
            assert 0 < st.full_dp < st.candidates
    # a mate with an N goes to the byte-code DP whatever the rule says
    left = left.copy()
    left[:40, 7] = 4
    ref = oracle.map_reads(oracle.MapIndex(txps), oracle.map_params(**over), left, right, 0)
    got, st = gpu_map(idx, left, right, dict(fast_dp=1), **over)
    check(got, st, ref, over["max_read_occ"], (strict, L, "N"))
    assert st.full_dp > 0


@pytest.mark.parametrize("strict", [False, True])
def test_presets_single_end(oracle, strict):
    over = MR.preset_over(strict, lib_type=3)
    txps, _ = synth_txome(seed=41, n_genes=40)
    left, _, _ = MR.around_s_min(txps, over, 100, 900, seed=42, paired=False)
    ref = oracle.map_reads(oracle.MapIndex(txps), oracle.map_params(**over), left, np.full_like(left, 4), 0)
    for fast in (1, 0):
        p = map_default_params(**over)
        ctx = MapContext(Index(txps), p, batch_cap=1024, max_read_len=100)
        ctx.set_option("fast_dp", fast)
        st = ctx.map_batch(left, None)
        compare(ctx.last_alignments(), ref, p.max_read_occ)
        assert st.mapped == ref["counters"]["mapped"] > 0
        if fast and strict:
            assert st.full_dp == 0
        ctx.close()


@pytest.mark.parametrize("strict", [False, True])
def test_presets_online_state_and_classes(oracle, strict):
    """three batches that cross numPreBurninFrags and numBurninFrags: online state bit-exact after each, then the
    class table"""
    over = MR.preset_over(strict)
    txps, left, right = _workload(over, 100, seed=50 + strict, n=1800)
    oix = oracle.MapIndex(txps)
    m0 = oracle.map_reads(oix, oracle.map_params(**over), left[:600], right[:600], 0)["counters"]["mapped"]
    reg = dict(num_pre_burnin=m0 // 2, num_burnin=m0 + m0 // 2)
    p = map_default_params(mini_batch=250, seed=7, **reg, **over)
    ctx = MapContext(Index(txps), p, batch_cap=600, max_read_len=100)
    on = oracle.Online(oix, oracle.map_params(**reg, **over), seed=7, mini_batch=250)
    parts = []
    for b in range(3):
        sl = slice(600 * b, 600 * (b + 1))
        ctx.map_batch(left[sl], right[sl])
        ref = on.batch(left[sl], right[sl])
        compare(ctx.last_alignments(), ref, p.max_read_occ)
        check_state(ctx.online_state(), on.state())
        parts.append(ref)
    res = ctx.finish()
    merged = {k: np.concatenate([q[k] for q in parts]) for k in ("n_aln", "label", "weight")}
    check_classes(res, oracle.eq_aggregate(merged, p.max_read_occ, True), exact_weights=False)
    fin = on.finish(res["off"], res["tids"], res["counts"])
    assert np.array_equal(bits(res["eff_len"]), bits(fin["eff_len"]))
    ctx.close()


@pytest.mark.parametrize("strict", [False, True])
@pytest.mark.parametrize("allow_orphans", [0, 1])
def test_presets_with_recover_orphans(strict, allow_orphans):
    """--recoverOrphans under the presets against the rescue restatement; the presets discard orphans, so nothing is
    rescued unless orphans are allowed again"""
    txps, left, right, _ = R.planted_workload(seed=61, n=3000, n_planted=400)
    over = dict(MR.preset_over(strict), allow_orphans=allow_orphans)
    p = map_default_params(recover_orphans=1, **over)
    ctx = MapContext(Index(txps), p, batch_cap=4096, max_read_len=100)
    st = ctx.map_batch(left, right)
    want = R.oracle_map(R.OracleIndex(txps), O.map_params(**over), left, right)
    compare(ctx.last_alignments(), want, p.max_read_occ)
    assert [st.orphans_rescued, st.rescue_searches, st.rescue_no_room] == want["rescue"]
    assert (st.orphans_rescued > 0) == bool(allow_orphans)
    ctx.close()


def test_more_than_255_joint_hits(oracle):
    """reads from a tandem repeat: unmapped at max_read_occ 255, mapped at 1000, the oracle's results both times, with
    one chunk and several"""
    txps = MR.tandem_txome(seed=3)
    left, right, rep = MR.tandem_reads(txps, seed=4, n=1000)
    idx, oix = Index(txps), oracle.MapIndex(txps)
    for cap, want in ((255, 0.0), (1000, 1.0)):
        ref = oracle.map_reads(oix, oracle.map_params(max_read_occ=cap), left, right, 0)
        for opts in (None, dict(chunk=256)):
            got, st = gpu_map(idx, left, right, opts, max_read_occ=cap)
            check(got, st, ref, cap, (cap, opts))
            assert (got["n_aln"][rep] > 0).mean() == want and (got["n_aln"][~rep] > 0).mean() > 0.95


def test_min_aln_prob(oracle):
    """--minAlnProb 0 keeps every mapping that passes the score filters, 0.5 drops those more than log(2) / scoreExp
    below the read's best; both are the oracle's"""
    txps, left, right = _workload(MR.preset_over(False), 100, seed=70)
    idx, oix = Index(txps), oracle.MapIndex(txps)
    kept = []
    for min_aln_prob in (0.0, 0.5):
        over = dict(min_aln_prob=min_aln_prob, score_exp=0.05)
        ref = oracle.map_reads(oix, oracle.map_params(**over), left, right, 0)
        got, st = gpu_map(idx, left, right, None, **over)
        check(got, st, ref, 200, over)
        kept.append(st.kept)
    assert kept[1] < kept[0]


@pytest.mark.parametrize("flag", ["--mimicBT2", "--mimicStrictBT2"])
def test_sample_data_drivers(tmp_path, flag):
    """sb_salmon quant with the flag equals the Python mirror with the same option, and meta_info.json reports the
    effective values"""
    exe = os.path.join(os.path.dirname(_capi.LIB_PATH), "sb_salmon")
    idx = str(tmp_path / "idx")
    subprocess.run([exe, "index", "-t", os.path.join(FIX, "transcripts.fasta.gz"), "-i", idx], check=True,
                   capture_output=True)
    out = str(tmp_path / "cli")
    r = subprocess.run([exe, "quant", "-i", idx, "-l", "IU", "-1", os.path.join(FIX, "reads_1.fastq.gz"), "-2",
                        os.path.join(FIX, "reads_2.fastq.gz"), "-o", out, "--batch", "4096", "--maxReadLen", "64",
                        "--softclipOverhangs", "--ma", "3", flag], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "increases maxReadOccs to 1000" in r.stderr and "Softclipping of overhangs is not allowed" in r.stderr
    strict = flag == "--mimicStrictBT2"
    quant.quant_files(idx + "/sb_index.bin", [os.path.join(FIX, "reads_1.fastq.gz")], [os.path.join(FIX, "reads_2.fastq.gz")],
                      str(tmp_path / "py"), batch=4096, max_read_len=64, threads=4, softclip=1,
                      map_params=map_default_params(ma=3), mimic_bt2=not strict, mimic_strict_bt2=strict)
    a, b = open(os.path.join(out, "quant.sf"), "rb").read(), open(str(tmp_path / "py" / "quant.sf"), "rb").read()
    assert a == b
    meta = json.load(open(os.path.join(out, "aux_info", "meta_info.json")))
    m = meta["sb_mapping_params"]
    assert (m["max_read_occ"], m["consensus_slack"], m["discard_orphans"], m["softclip_overhangs"]) == (1000, 0.5, True, False)
    assert (m["ma"], m["mp"], m["go"], m["ge"], m["min_score_fraction"]) == ((1, 0, 25, 25, 0.8) if strict else (2, -4, 5, 3, 0.65))
    assert json.load(open(os.path.join(out, "cmd_info.json")))[flag[2:]] == []
    assert meta["num_mapped"] > 0
