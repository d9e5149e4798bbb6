"""The Bowtie2-mimicking presets (`--mimicBT2`, `--mimicStrictBT2`), `--minAlnProb` and `--maxReadOcc` up to 1000
(DESIGN.md section 14) without a GPU: the preset function, the command line, the Python mirror's option handling, and
the host build of the per-read path (map_core.h) against the oracle under both presets."""
import json
import os
import subprocess

import numpy as np
import pytest

import mimic_ref as MR
from salmon_b200 import quant
from salmon_b200._capi import SalmonB200Error, map_default_params, map_mimic_bt2
from salmon_b200.synth import synth_txome
from test_map_host import run_both

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SB = os.path.join(ROOT, "salmon_b200", "sb_salmon")
FIX = os.path.join(ROOT, "tests", "golden", "sample_data")


@pytest.mark.parametrize("strict", [False, True])
@pytest.mark.parametrize("softclip,want_softclip", [(0, 0), (1, 0), (2, 2)])
def test_preset_values_override_the_user(strict, softclip, want_softclip):
    user = dict(max_read_occ=7, consensus_frac=0.9, allow_orphans=1, min_score_fraction=0.3, ma=5, mp=-1, go=1, ge=1,
                softclip=softclip, min_aln_prob=0.25, band=9, hard_filter=1)
    p = map_mimic_bt2(map_default_params(**user), strict=strict)
    want = dict(max_read_occ=1000, consensus_frac=0.5, allow_orphans=0, softclip=want_softclip)
    want.update(dict(min_score_fraction=0.8, ma=1, mp=0, go=25, ge=25) if strict else
                dict(min_score_fraction=0.3, ma=2, mp=-4, go=5, ge=3))
    for k, _ in p._fields_:
        assert getattr(p, k) == want.get(k, user.get(k, getattr(map_default_params(), k))), k
    # single-end reads are left orphans in this mapper: discardOrphansQuasi leaves them alone
    for lib_type, allow in ((1, 0), (2, 0), (6, 0), (3, 1), (4, 1), (5, 1), (7, 1)):
        assert map_mimic_bt2(map_default_params(lib_type=lib_type), strict=strict).allow_orphans == allow, lib_type


def test_gapless_rule_examples():
    """--mimicStrictBT2 at L = 100: G = 50 < s_min = 60; for pairs it holds below L = 125 (at 125 a mate at G makes a
    pair exactly at the threshold), for single-end reads (s_min = 0.8 L) below 250.  --mimicBT2 and the defaults never
    meet it."""
    st, bt2 = MR.preset_over(True), MR.preset_over(False)
    assert (st["ma"] * 100 - st["go"] - st["ge"], MR.s_min(st, 100)) == (50, pytest.approx(60))
    assert [L for L in range(31, 257) if MR.gapless(st, L)] == list(range(31, 125))
    assert [L for L in range(31, 257) if MR.gapless(st, L, paired=False)] == list(range(31, 250))
    defaults = {k: getattr(map_default_params(), k) for k in MR.PRESET_KEYS}
    for over in (bt2, defaults):
        assert not any(MR.gapless(over, L) or MR.gapless(over, L, paired=False) for L in range(31, 257))


def _cli(*args):
    return subprocess.run([SB, "quant", *args], capture_output=True, text=True, timeout=120)


@pytest.mark.parametrize("args,msg", [
    (["--mimicBT2", "--mimicStrictBT2"], "You passed both the --mimicBT2 and --mimicStrictBT2 parameters"),
    (["--minAlnProb", "-0.1"], "--minAlnProb takes a probability"),
    (["--minAlnProb", "abc"], "--minAlnProb takes a probability"),
    (["--minAlnProb", "1e-3x"], "--minAlnProb takes a probability"),
    (["--minAlnProb", "1.5"], "--minAlnProb takes a probability"),
])
def test_cli_refusals(tmp_path, args, msg):
    r = _cli("-i", str(tmp_path / "none"), "-l", "IU", "-1", "a.fq", "-2", "b.fq", "-o", str(tmp_path / "o"), *args)
    assert r.returncode != 0 and msg in r.stderr, r.stderr


def test_cli_refuses_max_read_occ_above_1000(tmp_path):
    """sb_map_create refuses it before it needs a device; 1000 gets past that check"""
    idx = tmp_path / "idx"
    subprocess.run([SB, "index", "-t", os.path.join(FIX, "transcripts.fasta.gz"), "-i", str(idx)], check=True,
                   capture_output=True, timeout=120)
    reads = ["-1", os.path.join(FIX, "reads_1.fastq.gz"), "-2", os.path.join(FIX, "reads_2.fastq.gz")]
    r = _cli("-i", str(idx), "-l", "IU", *reads, "-o", str(tmp_path / "o"), "--maxReadOcc", "1001")
    assert r.returncode != 0 and "max_read_occ 1001 is above the supported 1000" in r.stderr, r.stderr
    r = _cli("-i", str(idx), "-l", "IU", *reads, "-o", str(tmp_path / "o2"), "--maxReadOcc", "1000")
    assert "is above the supported" not in r.stderr, r.stderr
    with pytest.raises(SalmonB200Error, match="max_read_occ 1001 is above the supported 1000"):
        from salmon_b200._capi import Index, MapContext
        MapContext(Index(synth_txome(seed=1, n_genes=3)[0]), map_default_params(max_read_occ=1001))


@pytest.mark.parametrize("args", [["--mimicBT2"], ["--mimicStrictBT2", "--softclipOverhangs"],
                                  ["--mimicBT2", "--softclip"], ["--minAlnProb", "0"], ["--minAlnProb", "0.5"],
                                  ["--minAlnProb", "1"]])
def test_cli_accepts_and_records(tmp_path, args):
    """the options parse (the run then stops at the missing index, no device needed), salmon's info lines are printed and
    cmd_info.json records the options as given"""
    out = tmp_path / "o"
    r = _cli("-i", str(tmp_path / "none"), "-l", "IU", "-1", "a.fq", "-2", "b.fq", "-o", str(out), *args)
    assert "unknown option" not in r.stderr and "takes a probability" not in r.stderr, r.stderr
    assert "loading the index" in r.stderr, r.stderr
    info = json.load(open(out / "cmd_info.json"))
    for a in args:
        if a.startswith("--"):
            assert a[2:] in info
    if args[0] == "--minAlnProb":
        assert info["minAlnProb"] == args[1] and "[info]" not in r.stderr
        return
    strict = args[0] == "--mimicStrictBT2"
    assert "increases maxReadOccs to 1000." in r.stderr and "increases consensusSlack to 0.5." in r.stderr
    assert ("strict RSEM+Bowtie2-like parameters" in r.stderr) == strict
    assert ("Softclipping of overhangs is not allowed" in r.stderr) == ("--softclipOverhangs" in args), r.stderr


def test_python_mirror_options():
    mp = quant._mimic_options(map_default_params(ma=3, softclip=1), 0.5, True, False)
    assert (mp.min_aln_prob, mp.ma, mp.softclip, mp.max_read_occ) == (0.5, 2, 0, 1000)
    mp = quant._mimic_options(map_default_params(), None, False, False)
    assert (mp.min_aln_prob, mp.max_read_occ, mp.ma) == (1e-5, 200, 2)
    with pytest.raises(SalmonB200Error, match="mutually"):
        quant._mimic_options(map_default_params(), None, True, True)
    with pytest.raises(SalmonB200Error, match="minAlnProb"):
        quant._mimic_options(map_default_params(), 2.0, False, False)


@pytest.mark.parametrize("strict", [False, True])
@pytest.mark.parametrize("L", [75, 100, 150])
def test_host_path_equals_oracle_under_presets(oracle, strict, L):
    """paired-end and single-end reads with one mate on each side of s_min and planted indels: the host build of the
    per-read path (full DP) equals the oracle; planted mates at m0 - 1 mismatches map, most at m0 + 1 do not"""
    over = MR.preset_over(strict)
    txps, _ = synth_txome(seed=200 + L, n_genes=40)
    left, right, groups = MR.around_s_min(txps, over, L, 900, seed=L + strict)
    got, ref = run_both(oracle, txps, left, right, **over)
    mapped = ref["n_aln"] > 0
    m0, m2 = mapped[groups == 0].mean(), mapped[groups == 2].mean()
    assert m0 > 0.9 and m2 < m0 - 0.3, (m0, m2)      # (a gapped path can lift a mate past s_min under --mimicBT2)
    if strict:
        assert m2 < 0.2, m2
    se = MR.preset_over(strict, lib_type=3)
    left, _, _ = MR.around_s_min(txps, se, L, 600, seed=L + strict + 7, paired=False)
    got, ref = run_both(oracle, txps, left, np.full_like(left, 4), **se)
    assert ref["counters"]["mapped"] > 0.5 * len(left)


def test_host_path_tandem_repeats(oracle):
    """reads from a tandem repeat have more than 255 joint hits: unmapped at max_read_occ 255, mapped at 1000, the oracle's
    results both times"""
    txps = MR.tandem_txome(seed=3)
    left, right, rep = MR.tandem_reads(txps, seed=4, n=400)
    for cap, want in ((255, 0.0), (1000, 1.0)):
        got, _ = run_both(oracle, txps, left, right, max_read_occ=cap)
        assert (got["n_aln"][rep] > 0).mean() == want, cap
        assert (got["n_aln"][~rep] > 0).mean() > 0.95
