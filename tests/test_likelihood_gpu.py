"""salmon's fragment-likelihood options (--incompatPrior, --noSingleFragProb, --noFragLengthDist,
--noEffectiveLengthCorrection; DESIGN.md section 13) on the GPU: k_assign against the independent restatement
(tests/oracle_likelihood.c) bit for bit -- per-read alignments, labels, weights, online state and counters -- for each
option alone and in combination, paired-end and single-end, one and several chunks; the defaults unchanged; the drivers
and the command line on a stranded sample."""
import json
import os
import subprocess

import numpy as np
import pytest

import likelihood_ref as LK
import oracle_lib as O
from salmon_b200 import _capi, quant
from salmon_b200._capi import Index, MapContext, map_default_params

pytestmark = pytest.mark.gpu
ACGT = "ACGT"

CASES = [
    dict(),
    dict(incompat_prior=1e-20),
    dict(incompat_prior=0.25),
    dict(no_single_frag_prob=1),
    dict(no_frag_len_dist=1, no_eff_len_correction=1),
    dict(no_eff_len_correction=1),
    dict(incompat_prior=1e-5, no_single_frag_prob=1, no_frag_len_dist=1, no_eff_len_correction=1),
]


@pytest.fixture(scope="module")
def work():
    txps, fd, left, right = LK.stranded_workload(seed=7, n=3600)
    return txps, fd, left, right, Index(txps), LK.OracleIndex(txps)


@pytest.mark.parametrize("single_end", [False, True])
@pytest.mark.parametrize("chunk", [0, 1024])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_k_assign_equals_restatement(work, case, chunk, single_end):
    txps, fd, left, right, idx, oix = work
    o = LK.opts(**CASES[case])
    base = dict(lib_type=5 if single_end else 2, first_decoy=fd, num_pre_burnin=600, num_burnin=1800)
    if single_end:
        base["pre_merge_thresh"] = 1.0
    p = map_default_params(**base, **LK.product_fields(o))
    ctx = MapContext(idx, p, batch_cap=4096, max_read_len=100)
    if chunk:
        ctx.set_option("chunk", chunk)
    on = LK.OracleOnline(oix, O.map_params(**base), o, seed=p.seed, mini_batch=p.mini_batch)
    r_all = np.full_like(right, 4) if single_end else right
    n_comp = 0
    for b in range(3):   # batches before the aux model, across and after burn-in
        sl = slice(b * 1200, (b + 1) * 1200)
        st = ctx.map_batch(left[sl], None if single_end else right[sl])
        want = on.batch(left[sl], r_all[sl])
        diff = LK.same(ctx.last_alignments(), want, p.max_read_occ)
        assert diff is None, (CASES[case], b, diff)
        for k in ("mapped", "kept", "label_entries", "compatible"):
            assert getattr(st, k) == want["counters"][k], (k, b)
        n_comp += st.compatible
        s, w = ctx.online_state(), on.state()
        assert np.array_equal(s["mass"], w["mass"]) and np.array_equal(s["hist"], w["hist"]), b
        assert np.array_equal(s["log_eff"], w["log_eff"]) and s["burned_in"] == w["burned_in"], b
    assert on.state()["burned_in"] == 1
    res = ctx.finish()
    assert res["counters"]["n_compatible"] == n_comp
    lens = np.diff(oix.off).astype(np.float64)
    if CASES[case].get("no_eff_len_correction"):
        assert np.array_equal(res["eff_len"], lens)
    else:
        assert not np.array_equal(res["eff_len"], lens)
    ctx.close()


def test_defaults_unchanged(work):
    """a prior below 1e-100 is the default; both equal the unchanged oracle, and the counters agree"""
    txps, fd, left, right, idx, oix = work
    outs = []
    for extra in (dict(), dict(incompat_prior=1e-101)):
        p = map_default_params(lib_type=2, first_decoy=fd, **extra)
        ctx = MapContext(idx, p, batch_cap=4096, max_read_len=100)
        st = ctx.map_batch(left, right)
        outs.append((ctx.last_alignments(), st.mapped, st.compatible, ctx.online_state()))
        ctx.close()
    assert LK.same(outs[0][0], outs[1][0], 200) is None
    assert outs[0][1] == outs[0][2] == outs[1][2]
    assert np.array_equal(outs[0][3]["mass"], outs[1][3]["mass"])
    want = LK.oracle_map_unchanged(oix, O.map_params(lib_type=2, first_decoy=fd), left, right)
    assert np.array_equal(outs[0][0]["n_aln"], want["n_aln"])


def test_create_refuses():
    idx = Index([np.random.default_rng(0).integers(0, 4, 500, dtype=np.uint8)])
    for bad in (dict(incompat_prior=-0.1), dict(incompat_prior=float("nan")), dict(incompat_prior=2.0),
                dict(no_frag_len_dist=1)):
        with pytest.raises(_capi.SalmonB200Error):
            MapContext(idx, map_default_params(**bad), batch_cap=1024, max_read_len=100)


def _write_fq(path, m):
    with open(path, "w") as f:
        for i, s in enumerate(m):
            f.write(f"@p{i}\n{''.join(ACGT[c] for c in s)}\n+\n{'I' * len(s)}\n")


def _sb(args):
    exe = os.path.join(os.path.dirname(_capi.LIB_PATH), "sb_salmon")
    r = subprocess.run([exe] + args, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return r


@pytest.fixture(scope="module")
def sample(tmp_path_factory):
    d = tmp_path_factory.mktemp("lk")
    txps, fd, left, right = LK.stranded_workload(seed=11, n=6000)
    idx = Index(txps)
    idx.set_meta(names=[f"tx{i}" for i in range(len(txps))], first_decoy=fd)
    os.makedirs(d / "idx")
    idx.save(str(d / "idx" / "sb_index.bin"))
    p1, p2 = str(d / "r1.fq"), str(d / "r2.fq")
    _write_fq(p1, left); _write_fq(p2, right)
    return d, idx, fd, left, right, p1, p2


def _cli(sample, name, *extra, lib="ISR"):
    d, idx, fd, left, right, p1, p2 = sample
    out = str(d / name)
    _sb(["quant", "-i", str(d / "idx"), "-l", lib, "-1", p1, "-2", p2, "-o", out, "--batch", "2048",
         "--maxReadLen", "100", "-p", "4"] + list(extra))
    return out


def _read(out, f):
    return open(os.path.join(out, f), "rb").read()


def test_drivers_write_the_same_quant_sf(sample):
    d, idx, fd, left, right, p1, p2 = sample
    opt = dict(incompat_prior=1e-20, no_single_frag_prob=True, no_frag_len_dist=True, no_eff_len_correction=True)
    cli = _cli(sample, "cli", "--incompatPrior", "1e-20", "--noSingleFragProb", "--noFragLengthDist",
               "--noEffectiveLengthCorrection")
    _capi.quant_files_native(idx, [p1], [p2], str(d / "nat"),
                             map_params=map_default_params(lib_type=2, **LK.product_fields(LK.opts(**opt))), batch=2048,
                             max_read_len=100, threads=4)
    quant.quant_files(idx, [p1], [p2], str(d / "py"), map_params=map_default_params(lib_type=2), batch=2048,
                      max_read_len=100, threads=4, **opt)
    a, b, c = _read(cli, "quant.sf"), _read(str(d / "nat"), "quant.sf"), _read(str(d / "py"), "quant.sf")
    assert a == b == c
    assert a != _read(_cli(sample, "plain"), "quant.sf")


def test_incompat_prior_keeps_antisense_fragments(sample):
    d, idx, fd, left, right, p1, p2 = sample
    zero, kept = _cli(sample, "p0"), _cli(sample, "p20", "--incompatPrior", "1e-20")
    lz = json.load(open(os.path.join(zero, "lib_format_counts.json")))
    lk = json.load(open(os.path.join(kept, "lib_format_counts.json")))
    assert lz["compatible_fragment_ratio"] == 1.0 and lz["num_compatible_fragments"] == lz["num_assigned_fragments"]
    assert lk["num_assigned_fragments"] > lz["num_assigned_fragments"] + 500
    assert lk["compatible_fragment_ratio"] < 1.0
    # the count the test computes: fragments with a kept ISR-compatible mapping, the same reads in the same batches
    ctx = MapContext(idx, map_default_params(lib_type=2, first_decoy=fd, incompat_prior=1e-20), batch_cap=2048,
                     max_read_len=100)
    n_comp = n_ass = 0
    for s in range(0, len(left), 2048):
        ctx.map_batch(left[s:s + 2048], right[s:s + 2048])
        a = ctx.last_alignments()
        fl = a["flags"]
        st, fw, mfw = (fl >> 2) & 3, fl & 1, (fl >> 1) & 1
        comp = np.where(st == 0, (fw == 0) & (mfw == 1), np.where(st == 1, fw == 0, fw == 1))
        m = np.arange(fl.shape[1])[None, :] < a["n_aln"][:, None]
        n_comp += int(np.sum(np.any(comp & m, axis=1)))
        n_ass += int(np.sum(a["n_aln"] > 0))
    ctx.close()
    assert lk["num_compatible_fragments"] == n_comp and lk["num_assigned_fragments"] == n_ass
    assert abs(lk["compatible_fragment_ratio"] - n_comp / n_ass) < 1e-6
    info = json.load(open(os.path.join(kept, "cmd_info.json")))
    assert info["incompatPrior"] == "1e-20"


def test_eff_len_and_fld_file(sample):
    plain = _cli(sample, "pl")
    nel = _cli(sample, "nel", "--noEffectiveLengthCorrection")
    nfl = _cli(sample, "nfl", "--noFragLengthDist", "--noEffectiveLengthCorrection")
    for out in (nel, nfl):
        rows = [ln.split("\t") for ln in _read(out, "quant.sf").decode().splitlines()[1:]]
        assert all(float(r[2]) == float(r[1]) for r in rows)
    rows = [ln.split("\t") for ln in _read(plain, "quant.sf").decode().splitlines()[1:]]
    assert any(float(r[2]) != float(r[1]) for r in rows)
    assert os.path.exists(os.path.join(plain, "libParams", "flenDist.txt"))
    assert os.path.exists(os.path.join(nel, "libParams", "flenDist.txt"))
    assert not os.path.exists(os.path.join(nfl, "libParams", "flenDist.txt"))


def test_auto_library_type_with_prior(tmp_path):
    """-l A: detected as ISR after 50 000 stranded fragments; the prior then keeps the antisense fragments of the
    batches that follow, so fewer fragments are compatible than assigned"""
    txps, fd, left, right = LK.stranded_workload(seed=13, n=80000, antisense=0.2)
    idx = Index(txps)
    idx.set_meta(names=[f"tx{i}" for i in range(len(txps))], first_decoy=fd)
    os.makedirs(tmp_path / "idx")
    idx.save(str(tmp_path / "idx" / "sb_index.bin"))
    p1, p2 = str(tmp_path / "r1.fq"), str(tmp_path / "r2.fq")
    _write_fq(p1, left); _write_fq(p2, right)
    res = {}
    for name, extra in (("a0", []), ("a20", ["--incompatPrior", "1e-20"])):
        out = str(tmp_path / name)
        r = _sb(["quant", "-i", str(tmp_path / "idx"), "-l", "A", "-1", p1, "-2", p2, "-o", out, "--batch", "16384",
                 "--maxReadLen", "100", "-p", "4"] + extra)
        assert "detected most likely library type as ISR" in r.stderr, r.stderr
        res[name] = json.load(open(os.path.join(out, "lib_format_counts.json")))
    assert res["a0"]["expected_format"] == res["a20"]["expected_format"] == "ISR"
    assert res["a0"]["compatible_fragment_ratio"] == 1.0
    assert res["a20"]["num_assigned_fragments"] > res["a0"]["num_assigned_fragments"]
    assert res["a20"]["num_compatible_fragments"] < res["a20"]["num_assigned_fragments"]
