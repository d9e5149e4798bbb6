"""The GPU posterior samplers draw for draw against the oracle, and against exact distributions.

The device and the oracle draw from the same Philox streams with the same Marsaglia-Tsang code, and the counts are
integers, so the Gibbs chains agree sample by sample: gamma draws differ only by libm ulps and FMA contraction, and a
category pick or a rejection decision flips only if a uniform lands within an ulp of a boundary (~1e-16 per draw).
The state a round leaves (sb_gibbs_last_state) is compared too: counts bit-exact, gamma draws at rtol 1e-12.  Values
below the normal range (shape < 1 draws reach 5e-324) carry fewer significant bits, hence the absolute floor TINY."""
import gzip
import os
import subprocess

import numpy as np
import pytest

from salmon_b200 import EMContext, _capi, default_params
from salmon_b200.synth import synth_eq
from sampler_ref import (GAMMA_SHAPES, category_probs, category_table, check_category_counts, gamma_checks,
                         gibbs_prior, singleton_table)

pytestmark = pytest.mark.gpu

PRIORS = [(1, 1, 1e-2), (1, 0, 1e-5), (0, 1, 1e-2)]   # VBEM per transcript / VBEM per nucleotide / EM
TINY = 1e-300


@pytest.fixture(scope="module")
def ctx():
    c = EMContext(0)
    yield c
    c.close()


def assert_mu_close(got, want, what=""):
    assert np.array_equal(got == 0, want == 0) or np.all(np.maximum(got, want)[(got == 0) != (want == 0)] < TINY), what
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=TINY, err_msg=what)


def assert_samples_close(got, want, what=""):
    """rtol 1e-10; atol 2e-8 lets a value next to the 1e-8 truncation be kept on one side and zeroed on the other"""
    assert got.shape == want.shape, what
    np.testing.assert_allclose(got, want, rtol=1e-10, atol=2e-8, err_msg=what)


# ------------------------------------------------------------------------------------------------ raw gamma draws
@pytest.fixture(scope="module")
def singletons():
    return singleton_table(GAMMA_SHAPES, 1 << 17, seed=17)


@pytest.mark.parametrize("prior", PRIORS)
def test_raw_gamma_draws_match_oracle_and_gamma_distribution(ctx, oracle, singletons, prior):
    """one round on a singleton-only table with init = shape - prior: the tap's mu is the raw gamma draw of
    Gamma(shape, 1/(0.1+effLen)), element for element equal to the oracle's, and per shape distributed as the gamma
    (zero atom, KS, mean and variance); the counts are the singletons' class counts"""
    eq, eff, shape = singletons
    M = eq.n_txps
    ctx.optimize(eq, default_params(min_iter=1, max_iter=1), eq.counts.astype(np.float64), eff,
                 eq.counts.astype(np.uint64))
    pa = gibbs_prior(eff, *prior)
    init = shape - pa
    ci = init + pa
    seed = 0xC0FFEE00 + prior[1]
    ctx.gibbs(init, *prior, n_samples=1, thinning=1, no_gamma_draw=0, num_mapped_frags=float(eq.counts.sum()), seed=seed)
    mu, cnt = ctx.gibbs_last_state()
    _, omu, ocnt = oracle.gibbs_ex(eq, np.ones(eq.n_classes), eff, init, *prior, 1, 1, 0, float(eq.counts.sum()), seed)
    assert np.array_equal(cnt, eq.counts.astype(np.float64)) and np.array_equal(ocnt, cnt)
    assert_mu_close(mu, omu, f"prior {prior}")
    n = 1 << 17
    for k, a in enumerate(GAMMA_SHAPES):
        s = slice(k * n, (k + 1) * n)
        gamma_checks(mu[s], ci[s], 1.0 / (0.1 + eff[s]), what=f"GPU shape {a} prior {prior}")
    # the shape < 1 draws really ran: an atom at 0 for shape 1e-3, none above
    assert (mu[:n] == 0).mean() > 0.4 and (mu[n:] > 0).all()
    assert M == len(GAMMA_SHAPES) * n


# ------------------------------------------------------------------------------------------------ chain parity
@pytest.fixture(scope="module")
def chain_table(ctx, oracle):
    eq, proj, eff, uniq = synth_eq(seed=41, C=3000, M=1200, total_count=30_000)
    p = default_params()
    alpha, _, ok = ctx.optimize(eq, p, proj, eff, uniq)
    _, _, _, valid = oracle.em_optimize(eq, proj, eff, uniq, default_params(min_iter=1, max_iter=1), want_combined=True)
    assert ok
    init = alpha.copy()
    rng = np.random.default_rng(4)
    init[rng.random(eq.n_txps) < 0.3] = 0.0                       # explicit zeros
    fr = rng.random(eq.n_txps) < 0.3
    init[fr] = rng.uniform(0.0, 0.9, size=int(fr.sum()))          # fractional values below 1
    return eq, (proj, eff, uniq), valid, init, float(eq.counts.sum())


@pytest.mark.parametrize("prior", PRIORS)
@pytest.mark.parametrize("thinning", [1, 16])
@pytest.mark.parametrize("n_samples", [1, 49, 50, 101, 200])
def test_gibbs_chain_parity_per_sample(ctx, oracle, chain_table, prior, thinning, n_samples):
    """every sample of the GPU chain against orc_gibbs_ex at rtol 1e-10, and the last round's state against the
    oracle's: n_samples 1/49 run one chain, 50 two, 101 four (a step that does not divide), 200 eight"""
    eq, txp, valid, init, nmapped = chain_table
    eff = txp[1]
    ctx.optimize(eq, default_params(), *txp)
    active = np.zeros(eq.n_txps, dtype=bool)
    active[eq.tids[np.repeat(valid > 0, np.diff(eq.off.astype(np.int64)))]] = True
    pa = gibbs_prior(eff, *prior)
    if pa.min() < 1.0:   # a prior below 1: round 0 draws gamma shapes < 1 (the boost branch)
        assert ((init + pa < 1.0) & active).sum() > 50
    seed = 1000 + 7 * n_samples + thinning
    got = ctx.gibbs(init, *prior, n_samples=n_samples, thinning=thinning, no_gamma_draw=0, num_mapped_frags=nmapped,
                    seed=seed)
    mu, cnt = ctx.gibbs_last_state()
    want, omu, ocnt = oracle.gibbs_ex(eq, valid, eff, init, *prior, n_samples, thinning, 0, nmapped, seed)
    assert_samples_close(got, want, f"prior {prior} thinning {thinning} n {n_samples}")
    assert np.array_equal(cnt, ocnt)
    assert_mu_close(mu, omu)
    assert cnt.sum() == eq.counts[valid > 0].sum()


# ------------------------------------------------------------------------------------------------ category draws
def test_category_draws_exact(ctx, oracle):
    """one no-gamma round on the hand-built table: counts bit-exact against the oracle, each class against its exact
    multinomial probabilities, zero-probability members never picked, the all-zero-weight class drawn with
    p ~ 1/effLen, and the counts sum to the fragments exactly.  --noRichEqClasses keeps the all-zero class valid (its
    combined weights are 1/effLen) while the draws use the raw weights."""
    eq, eff, init, kinds = category_table()
    p_em = default_params(no_rich_eq=1, min_iter=1, max_iter=1)
    ctx.optimize(eq, p_em, init, eff, np.zeros(eq.n_txps, dtype=np.uint64))
    _, _, _, valid = oracle.em_optimize(eq, init, eff, np.zeros(eq.n_txps, dtype=np.uint64), p_em, want_combined=True)
    assert valid.all()
    prior = (1, 1, 1e-2)
    nfr = float(eq.counts.sum())
    ctx.gibbs(init, *prior, n_samples=1, thinning=1, no_gamma_draw=1, num_mapped_frags=nfr, seed=2024)
    mu, cnt = ctx.gibbs_last_state()
    _, omu, ocnt = oracle.gibbs_ex(eq, valid, eff, init, *prior, 1, 1, 1, nfr, 2024)
    np.testing.assert_allclose(mu, omu, rtol=1e-15)
    assert np.array_equal(cnt, ocnt)
    check_category_counts(eq, kinds, category_probs(eq, eff, omu), cnt, what="GPU")
    assert cnt.sum() == eq.counts.sum()


# ------------------------------------------------------------------------------------------------ sample offsets
@pytest.mark.parametrize("offset,thinning", [(3, 4), (50, 2)])
def test_gibbs_sample_offset(ctx, oracle, chain_table, offset, thinning):
    """sample_offset k draws from rounds k*thinning on: the oracle's run with round0 = k*thinning"""
    eq, txp, valid, init, nmapped = chain_table
    eff = txp[1]
    ctx.optimize(eq, default_params(), *txp)
    ctx.set_option("sample_offset", offset)
    try:
        got = ctx.gibbs(init, 1, 0, 1e-5, n_samples=5, thinning=thinning, no_gamma_draw=0, num_mapped_frags=nmapped,
                        seed=31)
        mu, cnt = ctx.gibbs_last_state()
    finally:
        ctx.set_option("sample_offset", 0)
    want, omu, ocnt = oracle.gibbs_ex(eq, valid, eff, init, 1, 0, 1e-5, 5, thinning, 0, nmapped, 31,
                                      round0=offset * thinning)
    assert_samples_close(got, want)
    assert np.array_equal(cnt, ocnt)
    assert_mu_close(mu, omu)
    base = oracle.gibbs_ex(eq, valid, eff, init, 1, 0, 1e-5, 5, thinning, 0, nmapped, 31)[0]
    assert not np.allclose(got, base)


def test_bootstrap_sample_offset_draws_the_unsplit_replicates(ctx):
    """a bootstrap run with sample_offset lo and n = hi - lo draws replicates lo..hi-1 of the unsplit run, bit for bit"""
    eq, proj, eff, uniq = synth_eq(seed=43, C=4000, M=1000, total_count=60_000)
    ctx.optimize(eq, default_params(), proj, eff, uniq)
    pb = default_params(min_iter=50, max_iter=10000)
    nmapped = float(eq.counts.sum())
    lo, hi = 2, 5
    full, ok = ctx.bootstrap(pb, nmapped, hi, 0xB007)
    full_last = ctx.bootstrap_last_counts()
    ctx.set_option("sample_offset", lo)
    try:
        part, ok2 = ctx.bootstrap(pb, nmapped, hi - lo, 0xB007)
        part_last = ctx.bootstrap_last_counts()
    finally:
        ctx.set_option("sample_offset", 0)
    assert ok and ok2 and part.shape == (hi - lo, eq.n_txps)
    assert np.array_equal(part, full[lo:hi])
    assert np.array_equal(part_last, full_last)
    assert not np.array_equal(part[0], full[0])


# ------------------------------------------------------------------------------------------------ duplicate labels
@pytest.mark.parametrize("vbem", [1, 0])
def test_bootstrap_with_duplicate_labels(ctx, oracle, vbem):
    """synth_eq repeats labels (several classes on one transcript set): alphas match the oracle at 1e-9; per class, a
    multi-transcript class reports its own count and a single-transcript class reports the count all classes on its
    transcript drew together"""
    from test_sampling_gpu import boot_inputs
    eq, proj, eff, uniq = synth_eq(seed=12, C=6000, M=1500, total_count=150_000)
    sizes = np.diff(eq.off.astype(np.int64))
    single = sizes == 1
    first = eq.tids[eq.off[:-1].astype(np.int64)]
    assert len(np.unique(first[single])) < single.sum()        # duplicates exist
    nmapped = float(eq.counts.sum())
    p_main = default_params(use_vbem=vbem)
    ctx.optimize(eq, p_main, proj, eff, uniq)
    cw, valid, valid_boot, prior, active = boot_inputs(oracle, eq, proj, eff, uniq, p_main, nmapped)
    p_boot = default_params(use_vbem=vbem, min_iter=50, max_iter=10000)
    got, okb = ctx.bootstrap(p_boot, nmapped, 3, 0x77)
    last = ctx.bootstrap_last_counts()
    ref, samp, rc = oracle.bootstrap(eq, cw, valid_boot, prior, active, p_boot, 3, 0x77)
    assert okb and rc == 0
    np.testing.assert_allclose(got, ref, rtol=1e-9, atol=1e-9)
    o = samp[-1]
    multi = ~single
    assert np.array_equal(last[multi], o[multi])
    per_txp = np.bincount(first[single], weights=o[single].astype(np.float64), minlength=eq.n_txps)
    sv = single & (valid_boot > 0)
    assert np.array_equal(last[sv], per_txp[first[sv]].astype(np.uint64))
    assert (last[single & (valid_boot == 0)] == 0).all()


# ------------------------------------------------------------------------------------------------ scale
def test_gibbs_parity_at_scale(ctx, oracle):
    """C = 500 000, M = 250 000, ~5e6 fragments: grid-stride loops and cdf_search over 500k classes"""
    eq, proj, eff, uniq = synth_eq(seed=47, C=500_000, M=250_000, total_count=5_000_000)
    alpha, _, ok = ctx.optimize(eq, default_params(min_iter=20, max_iter=20), proj, eff, uniq)
    _, _, _, valid = oracle.em_optimize(eq, proj, eff, uniq, default_params(min_iter=1, max_iter=1), want_combined=True)
    nmapped = float(eq.counts.sum())
    got = ctx.gibbs(alpha, 1, 1, 1e-2, n_samples=2, thinning=2, no_gamma_draw=0, num_mapped_frags=nmapped, seed=5)
    mu, cnt = ctx.gibbs_last_state()
    want, omu, ocnt = oracle.gibbs_ex(eq, valid, eff, alpha, 1, 1, 1e-2, 2, 2, 0, nmapped, 5)
    assert_samples_close(got, want)
    assert np.array_equal(cnt, ocnt)
    assert_mu_close(mu, omu)


# ------------------------------------------------------------------------------------------------ command line
@pytest.mark.parametrize("flags", [[], ["--useEM"], ["--perNucleotidePrior"], ["--noGammaDraw"]])
def test_cli_gibbs_matches_oracle(tmp_path, oracle, flags):
    """`sb_salmon quant -e ... --numGibbsSamples 4 --thinningFactor 2 --seed 11`: bootstraps.gz against orc_gibbs with
    the settings each flag should pass to the sampler (a flag that does not reach sb_gibbs fails here)"""
    from salmon_b200.quant import quant_eqclasses
    eq0, proj, eff0, uniq = synth_eq(seed=16, C=5000, M=1200, total_count=100_000)
    path = str(tmp_path / "eq_classes.txt.gz")
    _capi.write_eq_classes(path, [f"t{i}" for i in range(eq0.n_txps)], eq0.off, eq0.tids, eq0.counts, eq0.weights)
    exe = os.path.join(os.path.dirname(_capi.LIB_PATH), "sb_salmon")
    r = subprocess.run([exe, "quant", "-e", path, "-o", str(tmp_path / "o"), "--numGibbsSamples", "4",
                        "--thinningFactor", "2", "--seed", "11"] + flags, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    use_vbem = 0 if "--useEM" in flags else 1
    per_txp = 0 if "--perNucleotidePrior" in flags else 1
    vb_prior = 1e-5 if "--perNucleotidePrior" in flags else 1e-2
    no_gamma = 1 if "--noGammaDraw" in flags else 0
    ep = default_params(use_vbem=use_vbem, per_txp_prior=per_txp, vb_prior=vb_prior)
    py = quant_eqclasses(path, em_params=ep)
    f = _capi.read_eq_classes(path)
    eq = _capi.EqClasses(f["n_txps"], f["off"], f["tids"], f["weights"], f["counts"])
    M = eq.n_txps
    ep_o = default_params(use_vbem=use_vbem, per_txp_prior=per_txp, vb_prior=vb_prior, eq_class_mode=1, init_uniform=1,
                          min_iter=1, max_iter=1)
    _, _, _, valid = oracle.em_optimize(eq, np.zeros(M), f["eff_len"], np.zeros(M, dtype=np.uint64), ep_o,
                                        want_combined=True)
    want = oracle.gibbs(eq, valid, f["eff_len"], py["alpha"], use_vbem, per_txp, vb_prior, 4, 2, no_gamma,
                        float(f["counts"].sum()), 11)
    raw = gzip.open(tmp_path / "o" / "aux_info" / "bootstrap" / "bootstraps.gz", "rb").read()
    got = np.frombuffer(raw, dtype=np.float64).reshape(4, M)
    assert_samples_close(got, want, f"flags {flags}")
