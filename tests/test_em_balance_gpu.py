"""GPU tests of the EM phases' long-row work queue (H100): each warp streams its slice range through its ring, then
takes long rows from the phase's work queue until it is empty.  Both variants give the oracle's alphas at 1e-9 and
the same bits, wherever a row is reduced.  The tuning options that were removed are refused, not silently ignored."""
import numpy as np
import pytest

from salmon_b200 import EMContext, SalmonB200Error, default_params
from salmon_b200.synth import synth_eq
from test_em_layout_gpu import local_labels, table

pytestmark = pytest.mark.gpu

ALPHA_RTOL = 1e-9
ALPHA_ATOL = 1e-9


@pytest.fixture(scope="module")
def ctx():
    c = EMContext(0)
    yield c
    c.close()


def reset(c):
    c.set_option("variant", 1); c.set_option("rebalance", 1); c.set_option("blocks_per_sm", 0)


def mixed_table():
    """Class rows of 2..13 entries (transcript rows of every length 1..13), a few class rows longer than 96, and
    transcript rows longer than 96 both below and above LWARP = 2048 (the warp and the block path)."""
    rng = np.random.default_rng(41)
    M = 12000
    labels = local_labels(rng, 16000, M, 2, 13)
    for _ in range(6):                                            # long class rows
        labels.append(np.sort(rng.choice(M, size=int(rng.integers(100, 300)), replace=False)))
    hubs = [(11, 2500), (5000, 700), (7000, 300), (9000, 120)]    # (transcript, classes it joins)
    for t, n in hubs:
        for i in rng.choice(16000, size=n, replace=False):
            if t not in labels[i]:
                labels[i] = np.sort(np.append(labels[i], t))
    return table(labels, M, seed=42)


@pytest.mark.parametrize("vbem", [1, 0])
def test_long_row_queue_both_variants(ctx, oracle, vbem):
    eq, proj, eff, uniq = mixed_table()
    lengths = np.bincount(eq.tids, minlength=eq.n_txps)
    assert set(range(1, 14)) <= set(lengths.tolist())
    assert lengths.max() > 2048 and ((lengths > 96) & (lengths <= 2048)).sum() >= 3
    p = default_params(use_vbem=vbem, min_iter=12, max_iter=12)
    ref, rst = oracle.em_optimize(eq, proj, eff, uniq, p)
    first = None
    try:
        for variant in (1, 0):
            ctx.set_option("variant", variant)
            alpha, st, ok = ctx.optimize(eq, p, proj, eff, uniq)
            assert ok and st.iters == 12
            assert ctx.info("long_rows_cm") > 0 and ctx.info("long_rows_tm") > 0
            np.testing.assert_allclose(alpha, ref, rtol=ALPHA_RTOL, atol=ALPHA_ATOL)
            if first is None:
                first = alpha
            assert np.array_equal(alpha.view(np.uint64), first.view(np.uint64)), variant
    finally:
        reset(ctx)


REMOVED_OPTIONS = ("tail_pct", "tail_tile_cols", "l2_keep_cm", "l2_keep_tm", "balance_long",
                   "config", "lmax", "lwarp", "overhead_p1", "overhead_p2", "rebalance_iters")
REMOVED_INFO = ("tail_tiles", "tail_cols", "home_cols")


def test_removed_tuning_keys_are_refused(ctx):
    """Tail tiles, L2 pinning, the long-row charge, the alternative kernel configurations and the layout knobs that
    became constants are gone: their option and info keys are errors, so a caller that still sets one learns that it
    has no effect."""
    eq, proj, eff, uniq = synth_eq(seed=1, C=20000, M=6000, total_count=400000)
    ctx.upload(eq, proj, eff, uniq)
    ctx.prepare(default_params(min_iter=2, max_iter=2))
    for key in REMOVED_OPTIONS:
        for value in (0, 25):
            with pytest.raises(SalmonB200Error, match=r"\(-1\): unknown option '%s'" % key):
                ctx.set_option(key, value)
    assert ctx.info("sell_cols_cm") > 0 and ctx.info("sell_cols_tm") > 0     # the context is prepared
    for key in REMOVED_INFO:
        for m in ("cm", "tm"):
            with pytest.raises(SalmonB200Error, match=r"\(-1\): unknown info key '%s_%s'" % (key, m)):
                ctx.info(key + "_" + m)
