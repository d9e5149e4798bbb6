"""salmon's offline-phase options on the GPU (DESIGN.md section 15): `--bootstrapReproject` in sb_bootstrap against the
doBootstrap restatement (tests/bootstrap_ref.py), `--skipQuant` through the native driver, `--meta` and
`--alternativeInitMode` through the command line, and the command line against the Python mirror."""
import gzip
import json
import os
import subprocess

import numpy as np
import pytest

import bootstrap_ref as BR
from salmon_b200 import EMContext, _capi, default_params, quant
from salmon_b200._capi import EqClasses
from salmon_b200.synth import synth_eq
from test_offline_opts_cpu import combined_ref

pytestmark = pytest.mark.gpu
FIX = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sample_data")
READS = ["-1", os.path.join(FIX, "reads_1.fastq.gz"), "-2", os.path.join(FIX, "reads_2.fastq.gz")]


def exe():
    return os.path.join(os.path.dirname(_capi.LIB_PATH), "sb_salmon")


def planted_table():
    """a synthetic table with distinct labels (per-class drawn counts are then well defined), single-transcript classes,
    and degenerate classes: every weight of a few multi-transcript classes is 0, so their combined weights are NaN and
    the optimiser (and with it the bootstrap) drops them"""
    eq, proj, eff, uniq = synth_eq(seed=12, C=6000, M=1500, total_count=150_000)
    seen, keep = set(), []
    for c in range(eq.n_classes):
        k = eq.tids[int(eq.off[c]):int(eq.off[c + 1])].tobytes()
        if k not in seen:
            seen.add(k); keep.append(c)
    keep = np.array(keep)
    sizes = np.diff(eq.off).astype(np.int64)[keep]
    off = np.concatenate(([0], np.cumsum(sizes)))
    idx = np.concatenate([np.arange(int(eq.off[c]), int(eq.off[c + 1])) for c in keep])
    w = eq.weights[idx].copy()
    multi = np.nonzero(sizes > 1)[0]
    for c in multi[::97][:8]:
        w[off[c]:off[c + 1]] = 0.0
    eq = EqClasses(eq.n_txps, off, eq.tids[idx], w, eq.counts[keep])
    assert (sizes == 1).sum() > 50 and len(multi) > 1000
    return eq, proj, eff, uniq


@pytest.fixture(scope="module")
def ctx():
    c = EMContext(0)
    yield c
    c.close()


@pytest.mark.parametrize("vbem", [1, 0])
def test_reprojection_equals_restatement(ctx, oracle, vbem):
    eq, proj, eff, uniq = planted_table()
    nmapped = float(eq.counts.sum())
    p_main = default_params(use_vbem=vbem)
    alpha, st, ok = ctx.optimize(eq, p_main, proj, eff, uniq)
    assert ok
    cw, valid, valid_boot, prior, active = BR.boot_inputs(oracle, eq, proj, eff, uniq, p_main, nmapped)
    assert (valid == 0).sum() >= 8                                       # the planted degenerate classes
    n_boot, seed = 4, 0x1234ABCD5678
    p_boot = default_params(use_vbem=vbem, min_iter=50, max_iter=10000)
    off_gpu, ok0 = ctx.bootstrap(p_boot, nmapped, n_boot, seed)
    p_boot.bootstrap_reproject = 1
    got, okb = ctx.bootstrap(p_boot, nmapped, n_boot, seed)
    counts_last = ctx.bootstrap_last_counts()
    ref, samp, rc = BR.bootstrap(oracle, eq, cw, valid_boot, prior, active, p_boot, n_boot, seed, reproject=True)
    assert ok0 and okb and rc == 0 and got.shape == ref.shape == (n_boot, eq.n_txps)
    assert np.array_equal(counts_last, samp[-1])                         # the draws are the oracle's
    np.testing.assert_allclose(got, ref, rtol=1e-9, atol=1e-9)
    # the update moved every replicate, and the switch-off run on the same draws is the plain bootstrap
    ref_off, _, _ = BR.bootstrap(oracle, eq, cw, valid_boot, prior, active, p_boot, n_boot, seed, reproject=False)
    np.testing.assert_allclose(off_gpu, ref_off, rtol=1e-9, atol=1e-9)
    assert all(np.max(np.abs(got[b] - off_gpu[b])) > 1e-3 for b in range(n_boot))


@pytest.mark.parametrize("vbem", [1, 0])
def test_switch_off_leaves_no_trace(ctx, vbem):
    """with bootstrap_reproject = 0 the replicates are bit for bit what they are on a context that never reprojected,
    and after a reprojecting bootstrap the context's own optimiser state still runs to the same alpha bit for bit (the
    original counts stayed as uploaded)"""
    eq, proj, eff, uniq = planted_table()
    nmapped = float(eq.counts.sum())
    p_main = default_params(use_vbem=vbem)
    p_boot = default_params(use_vbem=vbem, min_iter=50, max_iter=10000)
    fresh = EMContext(0)
    fresh.optimize(eq, p_main, proj, eff, uniq)
    want, _ = fresh.bootstrap(p_boot, nmapped, 3, 99)
    fresh.close()
    alpha, _, _ = ctx.optimize(eq, p_main, proj, eff, uniq)
    p_on = default_params(use_vbem=vbem, min_iter=50, max_iter=10000, bootstrap_reproject=1)
    ctx.bootstrap(p_on, nmapped, 3, 99)
    got, _ = ctx.bootstrap(p_boot, nmapped, 3, 99)
    assert np.array_equal(got, want)
    ctx.run()
    a2, _, ok = ctx.download()
    assert ok and np.array_equal(a2, alpha)


def _index(tmp_path):
    idx = str(tmp_path / "idx")
    subprocess.run([exe(), "index", "-t", os.path.join(FIX, "transcripts.fasta.gz"), "-i", idx], check=True,
                   capture_output=True)
    return idx


def _quant(tmp_path, name, idx, *args):
    out = str(tmp_path / name)
    r = subprocess.run([exe(), "quant", "-i", idx, "-l", "IU", *READS, "-o", out, "--batch", "4096", "--maxReadLen", "64",
                        *args], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out, r


def _boots(out, M):
    raw = gzip.open(os.path.join(out, "aux_info", "bootstrap", "bootstraps.gz"), "rb").read()
    return np.frombuffer(raw, dtype=np.float64).reshape(-1, M)


def test_cli_bootstrap_reproject(tmp_path):
    """`sb_salmon quant --numBootstraps 8 --bootstrapReproject` and `quant -e ... --bootstrapReproject` write the
    bootstraps.gz of quant.quant_files / quant.quant_eqclasses, and the replicates differ from the plain ones"""
    idx = _index(tmp_path)
    out, _ = _quant(tmp_path, "cli", idx, "--numBootstraps", "8", "--bootstrapReproject", "--dumpEq", "--dumpEqWeights")
    plain, _ = _quant(tmp_path, "plain", idx, "--numBootstraps", "8")
    py = quant.quant_files(idx + "/sb_index.bin", READS[1], READS[3], batch=4096, max_read_len=64, threads=4,
                           num_bootstraps=8, seed=42, bootstrap_reproject=True)
    M = len(py["alpha"])
    got = _boots(out, M)
    assert got.shape == (8, M) and np.array_equal(got, py["bootstraps"])
    assert not np.array_equal(got, _boots(plain, M))
    eqf = os.path.join(out, "aux_info", "eq_classes.txt.gz")
    r = subprocess.run([exe(), "quant", "-e", eqf, "-o", str(tmp_path / "e"), "--numBootstraps", "8",
                        "--bootstrapReproject", "--seed", "11"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    pye = quant.quant_eqclasses(eqf, num_bootstraps=8, seed=11, bootstrap_reproject=True)
    assert np.array_equal(_boots(str(tmp_path / "e"), M), pye["bootstraps"])
    pye_off = quant.quant_eqclasses(eqf, num_bootstraps=8, seed=11)
    assert not np.array_equal(pye["bootstraps"], pye_off["bootstraps"])


def test_cli_skip_quant(tmp_path):
    """--skipQuant --dumpEq --dumpEqWeights: no quant.sf and no samples; the classes and counts of a normal run; the
    combined weights of the restatement; lib_format_counts.json and flenDist.txt as a normal run writes them"""
    idx = _index(tmp_path)
    skip, _ = _quant(tmp_path, "skip", idx, "--skipQuant", "--dumpEq", "--dumpEqWeights", "--numBootstraps", "4")
    full, _ = _quant(tmp_path, "full", idx, "--dumpEq", "--dumpEqWeights")
    assert not os.path.exists(os.path.join(skip, "quant.sf")) and os.path.exists(os.path.join(full, "quant.sf"))
    assert not os.path.exists(os.path.join(skip, "aux_info", "bootstrap"))
    a = _capi.read_eq_classes(os.path.join(skip, "aux_info", "eq_classes.txt.gz"))
    b = _capi.read_eq_classes(os.path.join(full, "aux_info", "eq_classes.txt.gz"))
    assert a["has_weights"] and b["has_weights"] and a["names"] == b["names"]
    for k in ("off", "tids", "counts"):
        assert np.array_equal(a[k], b[k]), k
    assert not np.allclose(a["weights"], b["weights"], rtol=1e-3)     # combined weights, not the auxiliary ones
    for f in ("lib_format_counts.json", os.path.join("libParams", "flenDist.txt")):
        assert open(os.path.join(skip, f)).read() == open(os.path.join(full, f)).read(), f
    # the Python mirror computes the same weights on the device, equal to the restatement; the file holds them at %g
    py = quant.quant_files(idx + "/sb_index.bin", READS[1], READS[3], str(tmp_path / "py"), batch=4096, max_read_len=64,
                           threads=4, dump_eq=True, dump_eq_weights=True, skip_quant=True)
    assert py["alpha"] is None and not os.path.exists(str(tmp_path / "py" / "quant.sf"))
    cls = py["classes"]
    M = len(py["eff_len"])
    eq = EqClasses(M, cls["off"], cls["tids"], cls["weights"], cls["counts"])
    want = combined_ref(eq, py["eff_len"], no_rich_eq=False)
    np.testing.assert_allclose(py["combined_weights"], want, rtol=1e-15, atol=0)
    np.testing.assert_allclose(a["weights"], want, rtol=1e-5, atol=1e-300)
    # --noRichEqClasses and --noEffectiveLengthCorrection: w = 1 and the transcript lengths
    nr, _ = _quant(tmp_path, "nr", idx, "--skipQuant", "--dumpEqWeights", "--noRichEqClasses",
                   "--noEffectiveLengthCorrection")
    c = _capi.read_eq_classes(os.path.join(nr, "aux_info", "eq_classes.txt.gz"))
    lens = _capi.Index.load(idx + "/sb_index.bin").tx_lengths()[:M].astype(np.float64)
    np.testing.assert_allclose(c["weights"], combined_ref(eq, lens, no_rich_eq=True), rtol=1e-5, atol=1e-300)
    ec = EMContext(0)
    got = ec.combined_weights(eq, np.full(M, 0.5), no_rich_eq=False)  # every effective length at or below 1
    ec.close()
    assert np.array_equal(got, combined_ref(eq, np.full(M, 0.5), no_rich_eq=False))


def test_cli_meta(tmp_path):
    """--meta gives the quant.sf of --useEM --initUniform --noRichEqClasses bit for bit, also with --useVBOpt given, and
    meta_info.json reports the EM"""
    idx = _index(tmp_path)
    m, r = _quant(tmp_path, "meta", idx, "--useVBOpt", "--meta")
    e, _ = _quant(tmp_path, "em", idx, "--useEM", "--initUniform", "--noRichEqClasses")
    v, _ = _quant(tmp_path, "vb", idx)
    qa, qe, qv = (open(os.path.join(d, "quant.sf"), "rb").read() for d in (m, e, v))
    assert qa == qe and qa != qv
    assert json.load(open(os.path.join(m, "aux_info", "meta_info.json")))["opt_type"] == "em"
    assert json.load(open(os.path.join(m, "cmd_info.json")))["meta"] == []
    py = quant.quant_files(idx + "/sb_index.bin", READS[1], READS[3], str(tmp_path / "py"), batch=4096, max_read_len=64,
                           threads=4, meta=True, em_params=default_params(use_vbem=1))
    assert open(str(tmp_path / "py" / "quant.sf"), "rb").read() == qa


def test_cli_alternative_init_mode(tmp_path, oracle):
    """--alternativeInitMode through the command line is orc_em_optimize with alt_init = 1"""
    idx = _index(tmp_path)
    out, _ = _quant(tmp_path, "alt", idx, "--alternativeInitMode")
    py = quant.quant_files(idx + "/sb_index.bin", READS[1], READS[3], str(tmp_path / "py"), batch=4096, max_read_len=64,
                           threads=4, alternative_init_mode=True)
    assert open(os.path.join(out, "quant.sf"), "rb").read() == open(str(tmp_path / "py" / "quant.sf"), "rb").read()
    cls = py["classes"]
    eq = EqClasses(len(py["alpha"]), cls["off"], cls["tids"], cls["weights"], cls["counts"])
    ref, rst = oracle.em_optimize(eq, py["projected_counts"], py["eff_len"], py["unique_counts"],
                                  default_params(alt_init=1))
    np.testing.assert_allclose(py["alpha"], ref, rtol=1e-9, atol=1e-9)
    assert py["em_stats"].iters == rst.iters
    base, _ = oracle.em_optimize(eq, py["projected_counts"], py["eff_len"], py["unique_counts"], default_params())
    assert not np.array_equal(ref, base)
