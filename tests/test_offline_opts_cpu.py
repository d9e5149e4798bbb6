"""salmon's offline-phase options (`--bootstrapReproject`, `--skipQuant`, `--meta`, `--alternativeInitMode`; DESIGN.md
section 15) without a GPU: the doBootstrap restatement against the unchanged oracle, the combined-weights formula of
`--skipQuant --dumpEqWeights`, the command line and the Python mirror's option handling."""
import json
import os
import subprocess

import numpy as np
import pytest

import bootstrap_ref as BR
from salmon_b200 import quant
from salmon_b200._capi import default_params, sb_em_params
from salmon_b200.synth import synth_eq

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SB = os.path.join(ROOT, "salmon_b200", "sb_salmon")


def boot_case(oracle, vbem, seed=31):
    eq, proj, eff, uniq = synth_eq(seed=seed, C=1500, M=400, total_count=40_000)
    nmapped = float(eq.counts.sum())
    cw, valid, valid_boot, prior, active = BR.boot_inputs(oracle, eq, proj, eff, uniq, default_params(use_vbem=vbem),
                                                          nmapped)
    return eq, cw, valid_boot, prior, active


@pytest.mark.parametrize("vbem", [1, 0])
def test_restatement_without_reprojection_is_the_oracle(oracle, vbem):
    eq, cw, valid_boot, prior, active = boot_case(oracle, vbem)
    p = default_params(use_vbem=vbem, min_iter=50, max_iter=10000)
    ref, samp_ref, rc = oracle.bootstrap(eq, cw, valid_boot, prior, active, p, 3, 0xBEEF)
    got, samp, rc2 = BR.bootstrap(oracle, eq, cw, valid_boot, prior, active, p, 3, 0xBEEF, reproject=False)
    assert rc == rc2 == 0
    assert np.array_equal(samp, samp_ref)
    assert np.array_equal(got, ref)                                   # bit for bit


@pytest.mark.parametrize("vbem", [1, 0])
def test_reprojection_is_one_update_on_the_original_counts(oracle, vbem):
    """the reprojected replicate is the replicate's converged alpha after one update against the original counts of the
    valid_boot classes: it moves every replicate, and it carries the mass of those classes less the few whose
    transcripts the replicate left at zero (a class the replicate did not draw can lose all its abundance, and the
    update then drops it)"""
    eq, cw, valid_boot, prior, active = boot_case(oracle, vbem)
    p = default_params(use_vbem=vbem, min_iter=50, max_iter=10000)
    off, _, _ = BR.bootstrap(oracle, eq, cw, valid_boot, prior, active, p, 3, 0xBEEF, reproject=False)
    on, _, rc = BR.bootstrap(oracle, eq, cw, valid_boot, prior, active, p, 3, 0xBEEF, reproject=True)
    assert rc == 0 and on.shape == off.shape
    total = float(eq.counts[valid_boot > 0].sum())
    for b in range(3):
        assert not np.array_equal(on[b], off[b])
        np.testing.assert_allclose(off[b].sum(), total, rtol=1e-9)
        assert 0.999 * total < on[b].sum() <= total * (1 + 1e-9)
    # the reprojection pulls the replicates toward the original counts: they agree with each other more than before
    assert np.std(on, axis=0).sum() < np.std(off, axis=0).sum()


def combined_ref(eq, eff_len, no_rich_eq):
    """MappingPipelineStages.cpp:112-162, serially in the reference's order"""
    out = np.zeros(eq.nnz)
    for c in range(eq.n_classes):
        b, e = int(eq.off[c]), int(eq.off[c + 1])
        wsum = 0.0
        for j in range(b, e):
            el = float(eff_len[eq.tids[j]])
            if el <= 1.0:
                el = 1.0
            w = 1.0 if no_rich_eq else float(eq.weights[j])
            wt = float(eq.counts[c]) * w * (1.0 / el)
            out[j] = wt
            wsum += wt
        wnorm = 1.0 / wsum
        for j in range(b, e):
            out[j] = out[j] * wnorm
    return out


@pytest.mark.parametrize("no_rich_eq", [False, True])
def test_combined_weights_formula(no_rich_eq):
    """the restatement against a vectorised form of the same formula, with effective lengths at and below 1 (clamped to
    1) and the transcript lengths of --noEffectiveLengthCorrection standing in for them"""
    eq, proj, eff, uniq = synth_eq(seed=5, C=300, M=80, total_count=5000)
    eff = eff.copy()
    eff[:10] = np.array([1.0, 0.5, 0.0, -3.0, 1e-9, 1.0000001, 2.0, 0.999, 1.0, 0.25])
    for lens in (eff, np.arange(1, eq.n_txps + 1, dtype=np.float64) * 37.0):
        got = combined_ref(eq, lens, no_rich_eq)
        el = np.maximum(lens, 1.0)[eq.tids]
        w = np.ones(eq.nnz) if no_rich_eq else eq.weights
        cls = np.repeat(np.arange(eq.n_classes), np.diff(eq.off).astype(np.int64))
        raw = eq.counts[cls].astype(np.float64) * w / el
        want = raw / np.bincount(cls, raw, minlength=eq.n_classes)[cls]
        np.testing.assert_allclose(got, want, rtol=1e-14)
        np.testing.assert_allclose(np.bincount(cls, got), 1.0, rtol=1e-13)
    # at effLen <= 1 every entry of a class weighs w * count: a class whose transcripts are all that short keeps w's ratios
    short = np.full(eq.n_txps, 0.5)
    got = combined_ref(eq, short, no_rich_eq)
    c = int(np.argmax(np.diff(eq.off)))
    b, e = int(eq.off[c]), int(eq.off[c + 1])
    want = np.full(e - b, 1.0 / (e - b)) if no_rich_eq else eq.weights[b:e] / eq.weights[b:e].sum()
    np.testing.assert_allclose(got[b:e], want, rtol=1e-14)


def test_python_mirror_options():
    ep = quant._em_options(default_params(use_vbem=1), meta=True)
    assert (ep.use_vbem, ep.init_uniform, ep.no_rich_eq, ep.alt_init, ep.bootstrap_reproject) == (0, 1, 1, 1, 0)
    ep = quant._em_options(default_params(), alternative_init_mode=True, bootstrap_reproject=True)
    assert (ep.use_vbem, ep.init_uniform, ep.no_rich_eq, ep.alt_init, ep.bootstrap_reproject) == (1, 0, 0, 1, 1)
    d = default_params()
    ep = quant._em_options(default_params())
    assert all(getattr(ep, k) == getattr(d, k) for k, _ in d._fields_)
    assert default_params().bootstrap_reproject == 0


def test_quant_files_hands_the_options_to_the_optimiser(monkeypatch):
    """quant.quant_files passes the EM parameters it was given, with the new options applied and nothing else changed,
    to the stage after mapping (mapping context and read files stubbed: no device needed)"""
    seen = []

    class Ctx:
        def __init__(self, *a, **k):
            pass

    class Files:
        def __init__(self, *a, **k):
            pass

        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False

        def bucketed(self, *a, **k):
            return {"n_observed": 0}

    class Index:
        n_txps = 3

        def meta(self):
            return {"first_decoy": 3}

    monkeypatch.setattr(quant, "MapContext", Ctx)
    monkeypatch.setattr(quant._capi, "ReadFiles", Files)
    monkeypatch.setattr(quant, "_quantify", lambda index, ctx, ep, *a, **k: seen.append((ep, k["skip_quant"])))
    d = default_params()
    quant.quant_files(Index(), "a.fq", "b.fq")
    quant.quant_files(Index(), "a.fq", "b.fq", meta=True, skip_quant=True)
    quant.quant_files(Index(), "a.fq", "b.fq", alternative_init_mode=True, bootstrap_reproject=True)
    (e0, s0), (e1, s1), (e2, s2) = seen
    assert all(getattr(e0, k) == getattr(d, k) for k, _ in d._fields_) and not s0
    assert (e1.use_vbem, e1.init_uniform, e1.no_rich_eq) == (0, 1, 1) and s1
    assert (e2.use_vbem, e2.init_uniform, e2.alt_init, e2.bootstrap_reproject) == (1, 0, 1, 1) and not s2


def _cli(*args):
    return subprocess.run([SB, "quant", *args], capture_output=True, text=True, timeout=120)


@pytest.mark.parametrize("args", [["--meta", "--useVBOpt"], ["--useVBOpt", "--meta"], ["--bootstrapReproject"],
                                  ["--alternativeInitMode"], ["--skipQuant", "--dumpEq", "--dumpEqWeights"],
                                  ["--skipQuant", "--numBootstraps", "4"]])
def test_cli_accepts_and_records(tmp_path, args):
    """the options parse (the run then stops at the missing index, no device needed); cmd_info.json records them as
    given; --meta says that it overrides --useVBOpt wherever that stands"""
    out = tmp_path / "o"
    r = _cli("-i", str(tmp_path / "none"), "-l", "IU", "-1", "a.fq", "-2", "b.fq", "-o", str(out), *args)
    assert "unknown option" not in r.stderr, r.stderr
    assert "loading the index" in r.stderr, r.stderr
    info = json.load(open(out / "cmd_info.json"))
    for a in args:
        if a.startswith("--"):
            assert info[a[2:]] == ([] if a != "--numBootstraps" else "4")
    assert ("--meta sets --useEM --initUniform --noRichEqClasses" in r.stderr) == ("--meta" in args), r.stderr


def test_cli_eqclasses_mode(tmp_path):
    """quant -e takes --bootstrapReproject, --meta and --alternativeInitMode, and refuses --skipQuant"""
    out = tmp_path / "o"
    r = _cli("-e", str(tmp_path / "none.txt"), "-o", str(out), "--bootstrapReproject", "--meta", "--alternativeInitMode")
    assert "unknown option" not in r.stderr and r.returncode != 0, r.stderr
    info = json.load(open(out / "cmd_info.json"))
    assert info["bootstrapReproject"] == info["meta"] == info["alternativeInitMode"] == []
    r = _cli("-e", str(tmp_path / "none.txt"), "-o", str(tmp_path / "o2"), "--skipQuant")
    assert r.returncode != 0 and "--skipQuant applies to mapping mode" in r.stderr, r.stderr


@pytest.mark.parametrize("args,msg", [(["--bootstrapReprojection"], "unknown option --bootstrapReprojection"),
                                      (["--metagenome"], "unknown option --metagenome"),
                                      (["--skipquant"], "unknown option --skipquant"),
                                      (["--geneMap", "g.tsv"], "outside the hot path"),
                                      (["--minAssignedFrags", "10"], "unknown option --minAssignedFrags")])
def test_cli_other_options_unchanged(tmp_path, args, msg):
    r = _cli("-i", str(tmp_path / "none"), "-l", "IU", "-1", "a.fq", "-2", "b.fq", "-o", str(tmp_path / "o"), *args)
    assert r.returncode != 0 and msg in r.stderr, r.stderr


def test_em_params_layout_unchanged():
    """bootstrap_reproject takes the place of the former reserved field: the layout is what it was"""
    import ctypes as C
    assert C.sizeof(sb_em_params) == 8 * 4 + 3 * 8 + 2 * 4
    assert sb_em_params.bootstrap_reproject.offset == 7 * 4 and sb_em_params.vb_prior.offset == 32
