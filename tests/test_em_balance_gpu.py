"""GPU tests of the work-conserving EM phases (H100): each warp's slice range is split into a home part, streamed
through the warp's ring, and tail tiles that any warp takes from the phase's work queue after the long rows.  A SELL
row is summed by one lane in label order on either path, so every share of tail tiles gives the oracle's alphas at
1e-9 and the same bits as the static ranges (tail_pct = 0)."""
import numpy as np
import pytest

from salmon_b200 import EMContext, default_params
from salmon_b200.synth import synth_eq
from test_em_layout_gpu import local_csr, local_labels, table, table_csr

pytestmark = pytest.mark.gpu

ALPHA_RTOL = 1e-9
ALPHA_ATOL = 1e-9
TAIL_PCTS = (0, 25, 50, 100)


@pytest.fixture(scope="module")
def ctx():
    c = EMContext(0)
    yield c
    c.close()


def reset(c):
    c.set_option("tail_pct", 0); c.set_option("config", 1); c.set_option("variant", 1)
    c.set_option("rebalance", 1); c.set_option("blocks_per_sm", 0)


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
def test_tail_tiles_every_configuration(ctx, oracle, vbem):
    eq, proj, eff, uniq = mixed_table()
    lengths = np.bincount(eq.tids, minlength=eq.n_txps)
    assert set(range(1, 14)) <= set(lengths.tolist())
    assert lengths.max() > 2048 and ((lengths > 96) & (lengths <= 2048)).sum() >= 3
    p = default_params(use_vbem=vbem, min_iter=12, max_iter=12)
    ref, rst = oracle.em_optimize(eq, proj, eff, uniq, p)
    first = None
    try:
        for tail in TAIL_PCTS:
            for cfg, variant in [(0, 1), (1, 1), (2, 1), (3, 1), (1, 0)]:
                ctx.set_option("tail_pct", tail); ctx.set_option("config", cfg); ctx.set_option("variant", variant)
                alpha, st, ok = ctx.optimize(eq, p, proj, eff, uniq)
                assert ok and st.iters == 12
                assert ctx.info("long_rows_cm") > 0 and ctx.info("long_rows_tm") > 0
                for m in ("cm", "tm"):
                    assert ctx.info("home_cols_" + m) + ctx.info("tail_cols_" + m) == ctx.info("sell_cols_" + m)
                    if tail == 0:
                        assert ctx.info("tail_tiles_" + m) == 0 and ctx.info("tail_cols_" + m) == 0
                    if tail == 100:
                        assert ctx.info("home_cols_" + m) == 0 and ctx.info("tail_tiles_" + m) > 0
                np.testing.assert_allclose(alpha, ref, rtol=ALPHA_RTOL, atol=ALPHA_ATOL)
                if first is None:
                    first = alpha
                assert np.array_equal(alpha.view(np.uint64), first.view(np.uint64)), (tail, cfg, variant)
    finally:
        reset(ctx)


@pytest.mark.parametrize("push_pass", [0, 1])
def test_tail_tiles_multi_gpu_kernel_loopback(oracle, push_pass):
    """k_em_persistent_mgpu (one GPU that is its own peer) takes tail tiles from the same queue, with both ways of
    delivering the partials to their owners."""
    eq, proj, eff, uniq = synth_eq(seed=5, C=40000, M=9000, total_count=900000)
    c = EMContext(0)
    try:
        c.peer_loopback(eq.n_txps)
        c.set_option("push_pass", push_pass)
        for vbem in (1, 0):
            p = default_params(use_vbem=vbem, min_iter=15, max_iter=15)
            ref, rst = oracle.em_optimize(eq, proj, eff, uniq, p)
            first = None
            for tail in TAIL_PCTS:
                c.set_option("tail_pct", tail)
                alpha, st, ok = c.optimize(eq, p, proj, eff, uniq)
                assert ok and st.iters == 15
                assert (c.info("tail_tiles_tm") > 0) == (tail > 0)
                np.testing.assert_allclose(alpha, ref, rtol=ALPHA_RTOL, atol=ALPHA_ATOL)
                if first is None:
                    first = alpha
                assert np.array_equal(alpha.view(np.uint64), first.view(np.uint64)), (vbem, tail)
    finally:
        c.close()


def test_all_slices_on_the_queue_one_block_per_sm(ctx, oracle):
    """tail_pct = 100: no warp streams a home range, every SELL slice is reduced from a tile; with one block per SM
    the fewest warps take the most tiles each."""
    rng = np.random.default_rng(51)
    M = 60000
    sizes, tids = local_csr(rng, 120000, M, 2, 13)
    eq, proj, eff, uniq = table_csr(sizes, tids, M, seed=52)
    p = default_params(min_iter=8, max_iter=8)
    ref, rst = oracle.em_optimize(eq, proj, eff, uniq, p)
    ctx.set_option("blocks_per_sm", 1)
    got = {}
    try:
        for tail in (0, 100):
            for variant in (1, 0):
                ctx.set_option("tail_pct", tail); ctx.set_option("variant", variant)
                alpha, st, ok = ctx.optimize(eq, p, proj, eff, uniq)
                assert ok and st.iters == 8
                np.testing.assert_allclose(alpha, ref, rtol=ALPHA_RTOL, atol=ALPHA_ATOL)
                got[(tail, variant)] = alpha
        assert ctx.info("home_cols_cm") == 0 and ctx.info("home_cols_tm") == 0
        assert ctx.info("tail_tiles_cm") >= ctx.info("warps") and ctx.info("tail_tiles_tm") >= ctx.info("warps")
    finally:
        reset(ctx)
    first = got[(0, 1)]
    for k, a in got.items():
        assert np.array_equal(a.view(np.uint64), first.view(np.uint64)), k


def test_tail_figures_of_the_bench_table(ctx):
    """The default (tail_pct = 0) keeps every slice in a home range; with a share of 25 % the bench table
    (synth_eq(seed=1)) has tail tiles in both layouts, and every SELL column is in exactly one home part or one tile."""
    eq, proj, eff, uniq = synth_eq(seed=1)
    ctx.upload(eq, proj, eff, uniq)
    ctx.prepare(default_params(min_iter=2, max_iter=2))
    for m in ("cm", "tm"):
        assert ctx.info("tail_tiles_" + m) == 0 and ctx.info("home_cols_" + m) == ctx.info("sell_cols_" + m)
    try:
        ctx.set_option("tail_pct", 25)
        ctx.prepare(default_params(min_iter=2, max_iter=2))
        for m in ("cm", "tm"):
            assert ctx.info("tail_tiles_" + m) > 0
            assert ctx.info("tail_cols_" + m) + ctx.info("home_cols_" + m) == ctx.info("sell_cols_" + m)
    finally:
        reset(ctx)
    with pytest.raises(Exception):
        ctx.set_option("tail_pct", 101)
