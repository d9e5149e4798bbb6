"""The oracle's posterior samplers against exact distributions (CPU only).

The GPU samplers are checked draw for draw against these same oracle entry points
(tests/test_sampler_exact_gpu.py), so what is pinned here -- the gamma draws against the gamma
distribution, the category draws against their multinomial probabilities -- carries over to the
device.  Seeds are fixed; thresholds are in tests/sampler_ref.py."""
import numpy as np
import pytest

from sampler_ref import (GAMMA_SHAPES, category_probs, category_table, check_category_counts, gamma_checks,
                         gibbs_prior, singleton_table)

N_DRAWS = 200_000


@pytest.mark.parametrize("shape", GAMMA_SHAPES)
@pytest.mark.parametrize("scale", [1.0 / (0.1 + 137.0), 3.5])
def test_oracle_gamma_draws_follow_the_gamma_distribution(oracle, shape, scale):
    seed = 0x5EED0000 + int(shape * 1000) % 9973
    x = oracle.gamma_draws(shape, scale, np.arange(N_DRAWS), 3, seed)
    r = gamma_checks(x, shape, scale, what=f"shape {shape} scale {scale}")
    if shape == 1e-3:   # the atom at 0: P(X < 4.9e-324) = 0.4753 at shape 1e-3
        assert 0.46 < r["zeros"] / N_DRAWS < 0.49
    else:
        assert r["zeros"] == 0


def test_gamma_draw_depends_on_index_round_and_key(oracle):
    """the counter streams: a draw is a function of (transcript, round, key) alone, and changes with each of them"""
    a = oracle.gamma_draws(0.5, 1.0, np.arange(64), 0, 1)
    assert np.array_equal(a, oracle.gamma_draws(0.5, 1.0, np.arange(64), 0, 1))
    for other in (oracle.gamma_draws(0.5, 1.0, np.arange(64), 1, 1), oracle.gamma_draws(0.5, 1.0, np.arange(64), 0, 2),
                  oracle.gamma_draws(0.5, 1.0, np.arange(64), 0, 1 << 32), oracle.gamma_draws(0.5, 1.0, np.arange(1, 65), 0, 1)):
        assert not np.any(a == other)


def test_gamma_draw_of_an_invalid_shape_is_nan(oracle):
    """a shape that is not a positive finite number (a negative count, a lost prior) gives NaN instead of a rejection
    loop that never accepts; the device draws the same way"""
    x = oracle.gamma_draws(np.array([0.0, -0.5, -3.0, np.inf, np.nan]), 1.0, np.arange(5), 0, 1)
    assert np.isnan(x).all()


@pytest.mark.parametrize("prior", [(1, 1, 1e-2), (1, 0, 1e-5), (0, 1, 1e-2)])
def test_gibbs_round_draws_the_gamma_of_count_plus_prior(oracle, prior):
    """one round of orc_gibbs_ex on a singleton table: mu is orc_gamma_draw(init + prior, 1/(0.1+effLen)) element for
    element, and the counts are the singletons' class counts"""
    eq, eff, shape = singleton_table((1e-3, 0.5, 7.0), 2000, seed=3)
    pa = gibbs_prior(eff, *prior)
    init = shape - pa
    _, mu, cnt = oracle.gibbs_ex(eq, np.ones(eq.n_classes), eff, init, *prior, 1, 1, 0, float(eq.counts.sum()), 77)
    want = oracle.gamma_draws(init + pa, 1.0 / (0.1 + eff), np.arange(eq.n_txps), 0, 77)
    assert np.array_equal(mu, want)
    assert np.array_equal(cnt, eq.counts.astype(np.float64))


def test_gibbs_ex_round0_and_state_outputs(oracle):
    """orc_gibbs is orc_gibbs_ex at round0 = 0; round0 moves the streams (a different round draws different values)"""
    from salmon_b200.synth import synth_eq
    eq, proj, eff, uniq = synth_eq(seed=31, C=600, M=200, total_count=6000)
    valid = np.ones(eq.n_classes, dtype=np.uint8)
    args = (eq, valid, eff, proj, 1, 1, 1e-2, 3, 2, 0, 6000.0, 9)
    s0 = oracle.gibbs(*args)
    s1, mu, cnt = oracle.gibbs_ex(*args, round0=0)
    assert np.array_equal(s0, s1)
    active = np.zeros(eq.n_txps, dtype=bool)
    active[eq.tids] = True
    assert cnt.sum() == eq.counts.sum() and (mu[active] > 0).all() and (mu[~active] == 0).all()
    s2, _, _ = oracle.gibbs_ex(*args, round0=6)
    assert not np.array_equal(s1, s2)


def test_oracle_category_draws_follow_exact_probabilities(oracle):
    """one no-gamma round of orc_gibbs_ex on the hand-built table: every class's draws against its exact multinomial
    probabilities (chi-square), members of weight 0 never picked, the all-zero class drawn with p ~ 1/effLen,
    singletons added as integers"""
    eq, eff, init, kinds = category_table()
    prior = (1, 1, 1e-2)
    mu_want = (init + gibbs_prior(eff, *prior)) / eff
    _, mu, cnt = oracle.gibbs_ex(eq, np.ones(eq.n_classes), eff, init, *prior, 1, 1, 1, float(eq.counts.sum()), 2024)
    assert np.array_equal(mu, mu_want)
    p = category_probs(eq, eff, mu)
    zc = kinds.index("zero_weights")
    b, e = int(eq.off[zc]), int(eq.off[zc + 1])
    np.testing.assert_allclose(p[b:e], (1 / eff[b:e]) / (1 / eff[b:e]).sum(), rtol=1e-14)
    check_category_counts(eq, kinds, p, cnt, what="oracle")
    assert cnt.sum() == eq.counts.sum()


def test_category_check_rejects_a_shifted_pick(oracle):
    """the chi-square check is sharp enough to see a pick that lands one member late"""
    eq, eff, init, kinds = category_table()
    prior = (1, 1, 1e-2)
    _, mu, cnt = oracle.gibbs_ex(eq, np.ones(eq.n_classes), eff, init, *prior, 1, 1, 1, float(eq.counts.sum()), 2024)
    p = category_probs(eq, eff, mu)
    shifted = cnt.copy()
    c = kinds.index("wide")
    b, e = int(eq.off[c]), int(eq.off[c + 1])
    shifted[b:e] = np.roll(cnt[b:e], 1)
    with pytest.raises(AssertionError):
        check_category_counts(eq, kinds, p, shifted)
