"""Exact distributions of the posterior samplers' draws, for the sampler tests (CPU and GPU).

gamma_checks: draws of the Gibbs sampler's gamma step against the gamma distribution (scipy.special.gammainc, the
regularised lower incomplete gamma function).  category_table / category_probs: a hand-built class table whose category
draws have known multinomial probabilities, with the edges of the draw: a 200-member class, a member of weight 0, a
class whose weights are all 0 (drawn with p ~ 1/effLen), classes of up to 10^6 fragments and singletons.
"""
import numpy as np
from scipy import special, stats

from salmon_b200._capi import EqClasses

DENORM_MIN = 4.9406564584124654e-324
# The draws are a fixed function of the seed, so each check below has one outcome; the thresholds are wide enough that
# a correct sampler passes at any seed (a false failure has probability ~1e-5 per check) and a shape or scale that is
# wrong by about 1 % fails at 2*10^5 draws.
KS_P_MIN = 1e-5
Z_MAX = 5.0
GAMMA_SHAPES = (1e-3, 0.05, 0.5, 0.999, 1.0, 1.5, 7.0, 1e3, 1e6)


def gamma_cdf(x, shape, scale):
    """P(X <= x) for X ~ Gamma(shape, scale), also where x / scale underflows: there the series' first term
    x^a / Gamma(a+1), whose relative error is O(x), is taken in log space."""
    x, shape, scale = np.broadcast_arrays(np.asarray(x, dtype=np.float64), np.asarray(shape, dtype=np.float64),
                                          np.asarray(scale, dtype=np.float64))
    tiny = x < 1e-300 * scale
    out = special.gammainc(shape, np.where(tiny, 1.0, x) / scale)
    with np.errstate(divide="ignore"):
        lt = shape[tiny] * (np.log(x[tiny]) - np.log(scale[tiny])) - special.gammaln(shape[tiny] + 1.0)
    out[tiny] = np.exp(lt)
    return out


def gamma_checks(x, shape, scale, what=""):
    """x[i] ~ Gamma(shape[i], scale[i]) (shape, scale broadcast).  Asserts:
    - the exact-zero fraction equals P(X < denorm_min) within 5 binomial standard errors (at shape 1e-3 about 47.5 %
      of draws underflow to 0);
    - a KS test of the probability-integral transform of the non-zero draws, conditioned on X >= denorm_min;
    - z-scores of the mean and the variance of x / scale against shape and shape (the gamma's two first moments)."""
    x = np.asarray(x, dtype=np.float64)
    shape = np.broadcast_to(np.asarray(shape, dtype=np.float64), x.shape)
    scale = np.broadcast_to(np.asarray(scale, dtype=np.float64), x.shape)
    n = x.size
    assert np.isfinite(x).all() and (x >= 0).all(), what
    p0 = gamma_cdf(DENORM_MIN, shape, scale)
    zeros = x == 0
    sd0 = np.sqrt(np.sum(p0 * (1 - p0)))
    e0 = p0.sum()
    if sd0 > 0:
        z0 = (zeros.sum() - e0) / sd0
        assert abs(z0) < Z_MAX, f"{what}: {zeros.sum()} zeros, expected {e0:.1f} +- {sd0:.1f}"
    else:
        assert zeros.sum() == 0, f"{what}: {zeros.sum()} zeros where P(0) = 0"
    nz = ~zeros
    u = (gamma_cdf(x[nz], shape[nz], scale[nz]) - p0[nz]) / (1 - p0[nz])
    ks = stats.kstest(u, "uniform")
    assert ks.pvalue > KS_P_MIN, f"{what}: KS p = {ks.pvalue:.3g} (D = {ks.statistic:.3g}, n = {nz.sum()})"
    y = x / scale
    a = shape
    zm = (y.mean() - a.mean()) / np.sqrt(a.sum() / n ** 2)
    var_hat = y.var()
    # Var(sample variance) ~ (mu4 - sigma^4) / n with mu4 = 3a^2 + 6a for Gamma(a, 1)
    zv = (var_hat - a.mean()) / np.sqrt(np.mean(2 * a ** 2 + 6 * a) / n)
    assert abs(zm) < Z_MAX, f"{what}: mean z = {zm:.2f}"
    assert abs(zv) < Z_MAX, f"{what}: variance z = {zv:.2f}"
    return dict(zeros=int(zeros.sum()), expected_zeros=float(e0), ks_p=float(ks.pvalue), z_mean=float(zm),
                z_var=float(zv))


def singleton_table(shapes, n_per, seed):
    """One single-transcript class per transcript, n_per transcripts per shape (transcript i has shape
    shapes[i // n_per]); effective lengths spread over 50..5000 so that the gamma scale 1/(0.1+effLen) varies.
    Returns (eq, eff_len, shape_of_txp)."""
    rng = np.random.default_rng(seed)
    M = len(shapes) * n_per
    eff = np.exp(rng.uniform(np.log(50.0), np.log(5000.0), size=M))
    counts = rng.integers(1, 20, size=M).astype(np.uint64)
    eq = EqClasses(M, np.arange(M + 1, dtype=np.uint64), np.arange(M, dtype=np.uint32), np.ones(M), counts)
    return eq, eff, np.repeat(np.asarray(shapes, dtype=np.float64), n_per)


def gibbs_prior(eff, use_vbem, per_txp_prior, vb_prior):
    """The per-transcript Gibbs prior (CollapsedGibbsSampler.cpp:296-315, :357-371), rounded as the samplers round it."""
    per_txp = per_txp_prior if use_vbem else 1
    prior = 1e-3
    if use_vbem:
        prior = max(1.0, vb_prior) if per_txp else max(1e-3, vb_prior)
    return np.full(eff.shape[0], prior) if per_txp else prior * np.maximum(eff, 1.0)


def category_table(seed=5):
    """A table of disjoint classes (no transcript is in two classes), so every transcript's drawn count is the count of
    its own class's draws.  Returns (eq, eff_len, init, kinds) with kinds[c] naming class c's edge."""
    rng = np.random.default_rng(seed)
    sizes, kinds, counts, weights = [], [], [], []

    def add(kind, w, count):
        sizes.append(len(w)); kinds.append(kind); counts.append(count); weights.append(np.asarray(w, dtype=np.float64))
    w = rng.exponential(1.0, size=200); w[[7, 123]] = 0.0
    add("wide", w / w.sum(), 400_000)                               # 200 members, two of them weight 0
    add("zero_weights", np.zeros(5), 100_000)                       # falls back to p ~ 1/effLen
    add("pair", [0.3, 0.7], 1_000_000)
    add("skewed", [1e-6, 0.5, 0.0, 0.499999], 250_000)
    for c in (1, 37, 12_345, 1_000_000):                             # singletons: added as integers
        add("single", [1.0], c)
    w = rng.exponential(1.0, size=12)
    add("small_count", w / w.sum(), 3)
    sizes = np.array(sizes)
    off = np.concatenate(([0], np.cumsum(sizes))).astype(np.uint64)
    M = int(off[-1])
    eq = EqClasses(M, off, np.arange(M, dtype=np.uint32), np.concatenate(weights), np.array(counts, dtype=np.uint64))
    eff = np.exp(rng.uniform(np.log(30.0), np.log(8000.0), size=M))
    init = rng.uniform(0.0, 50.0, size=M)
    init[rng.random(M) < 0.2] = 0.0
    return eq, eff, init, kinds


def category_probs(eq, eff, mu):
    """Exact category probabilities of every member under the sampler's rule (CollapsedGibbsSampler.cpp:188-260):
    p ~ 1000*mu*w, falling back to p ~ 1/effLen when the class's sum is <= denorm_min.  Returns p[nnz]."""
    p = np.zeros(eq.nnz)
    for c in range(eq.n_classes):
        b, e = int(eq.off[c]), int(eq.off[c + 1])
        t = eq.tids[b:e]
        q = (1000.0 * mu[t]) * eq.weights[b:e]
        if q.sum() <= DENORM_MIN:
            q = 1.0 / eff[t]
        p[b:e] = q / q.sum()
    return p


def check_category_counts(eq, kinds, p, cnt, what=""):
    """cnt[t]: draws per transcript after one round (disjoint classes).  Singletons hold their class count exactly,
    members of probability 0 hold nothing, every class holds exactly its count, and each multi-member class passes a
    chi-square test against its exact probabilities (cells with expectation < 5 are pooled)."""
    for c in range(eq.n_classes):
        b, e = int(eq.off[c]), int(eq.off[c + 1])
        t = eq.tids[b:e]
        n = int(eq.counts[c])
        got = cnt[t]
        assert np.array_equal(got, np.rint(got)), f"{what}: class {c} drew fractional counts"
        assert int(got.sum()) == n, f"{what}: class {c} ({kinds[c]}) drew {got.sum()} of {n}"
        if e - b == 1:
            continue
        pc = p[b:e]
        assert (got[pc == 0] == 0).all(), f"{what}: class {c} ({kinds[c]}) picked a member of probability 0"
        exp = n * pc
        big = exp >= 5
        obs_cells = list(got[big]) + ([got[~big & (pc > 0)].sum()] if (~big & (pc > 0)).any() else [])
        exp_cells = list(exp[big]) + ([exp[~big & (pc > 0)].sum()] if (~big & (pc > 0)).any() else [])
        if len(exp_cells) < 2:
            continue
        chi2 = float(np.sum((np.array(obs_cells) - np.array(exp_cells)) ** 2 / np.array(exp_cells)))
        pv = stats.chi2.sf(chi2, len(exp_cells) - 1)
        assert pv > KS_P_MIN, f"{what}: class {c} ({kinds[c]}): chi2 = {chi2:.1f} on {len(exp_cells) - 1} dof, p = {pv:.3g}"
