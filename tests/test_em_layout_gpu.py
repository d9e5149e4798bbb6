"""GPU tests of the SELL layout of the EM iteration (H100): exact slice widths (every row length and every
remainder mod 4, groups of 4 columns straddling ring chunks), 16-bit indices relative to a per-slice base, and the
long-row fallback of slices whose indices span more than 16 bits -- against the CPU oracle at 1e-9 and bit-identical
across both variants and both ways of cutting the warp ranges."""
import numpy as np
import pytest

from salmon_b200 import EMContext, default_params
from salmon_b200._capi import EqClasses

pytestmark = pytest.mark.gpu

ALPHA_RTOL = 1e-9
ALPHA_ATOL = 1e-9


@pytest.fixture(scope="module")
def ctx():
    c = EMContext(0)
    yield c
    c.close()


def table(labels, M, seed):
    """EqClasses + per-transcript inputs from a list of sorted label arrays"""
    return table_csr(np.array([len(l) for l in labels]), np.concatenate(labels), M, seed)


def table_csr(sizes, tids, M, seed):
    rng = np.random.default_rng(seed)
    off = np.concatenate(([0], np.cumsum(sizes)))
    tids = tids.astype(np.uint32)
    w = rng.random(len(tids)) + 0.05
    w /= np.repeat(np.add.reduceat(w, off[:-1]), sizes)
    counts = rng.integers(1, 200, size=len(sizes)).astype(np.uint64)
    eq = EqClasses(M, off, tids, w, counts)
    eff = rng.uniform(100, 3000, size=M)
    proj = np.bincount(tids, weights=np.repeat(counts.astype(float), sizes) * w, minlength=M)
    uniq = rng.integers(0, 3, size=M).astype(np.uint64)
    return eq, proj, eff, uniq


def local_labels(rng, C, M, lmin, lmax, window=40):
    """C classes of 2..13 (lmin..lmax) transcripts drawn from a window of neighbouring transcripts"""
    labels = []
    for _ in range(C):
        L = int(rng.integers(lmin, lmax + 1))
        start = int(rng.integers(0, M - window))
        labels.append(np.sort(start + rng.choice(window, size=L, replace=False)))
    return labels


def local_csr(rng, C, M, lmin, lmax, window=32):
    """local_labels for large C, vectorised: (sizes, tids)"""
    L = rng.integers(lmin, lmax + 1, size=C)
    start = rng.integers(0, M - window, size=C)
    offs = np.argsort(rng.random((C, window)), axis=1)[:, :lmax]          # distinct offsets in the window
    keep = np.arange(lmax)[None, :] < L[:, None]
    offs = np.sort(np.where(keep, offs, window), axis=1)                    # the chosen ones first, ascending
    return L, (start[:, None] + offs)[keep]


@pytest.mark.parametrize("group", [32, 1024])
def test_every_row_length_and_remainder(ctx, oracle, group):
    """Class rows of 2..13 entries, transcript rows of 1..~25.  With groups of 32 rows every slice mixes lengths (one
    slice = one bucketing group); with 1024 the slices are near-uniform, so every width residue mod 4 occurs as a slice
    of its own.  The persistent and the per-phase kernels, with both ways of cutting the warp ranges, give the oracle's
    alphas, and the same bits.  (At this size a warp's range is about one slice; the ring's wrap-around is
    test_ranges_wrap_the_ring's.)"""
    rng = np.random.default_rng(11)
    M = 12000
    eq, proj, eff, uniq = table(local_labels(rng, 16000, M, 2, 13), M, seed=12)
    lengths = np.bincount(eq.tids, minlength=M)
    assert set(range(1, 14)) <= set(lengths.tolist())        # transcript rows of every length 1..13
    p = default_params(min_iter=12, max_iter=12)
    ref, rst = oracle.em_optimize(eq, proj, eff, uniq, p)
    first = None
    ctx.set_option("sell_group_cm", group); ctx.set_option("sell_group_tm", group)
    try:
        for rebalance in (0, 3):
            for variant in (1, 0):
                ctx.set_option("rebalance", rebalance); ctx.set_option("variant", variant)
                alpha, st, ok = ctx.optimize(eq, p, proj, eff, uniq)
                assert ok and st.iters == 12
                assert ctx.info("fallback_rows_cm") == 0 and ctx.info("fallback_rows_tm") == 0
                np.testing.assert_allclose(alpha, ref, rtol=ALPHA_RTOL, atol=ALPHA_ATOL)
                if first is None:
                    first = alpha
                assert np.array_equal(alpha.view(np.uint64), first.view(np.uint64)), (variant, rebalance)
    finally:
        ctx.set_option("rebalance", 1); ctx.set_option("variant", 1)
        ctx.set_option("sell_group_cm", 1024); ctx.set_option("sell_group_tm", 1024)


@pytest.mark.parametrize("group", [32, 1024])
def test_ranges_wrap_the_ring(ctx, oracle, group):
    """Each warp's range spans several ring lengths, in both variants, in both layouts: 400 000 classes of 2..13 entries
    and one block per SM (the fewest warps).  So groups of 4 columns start at every offset mod 4 after slices of odd
    widths and straddle ring chunks, the ring (4 chunks of 8 columns) wraps, and chunks are handed back in the middle
    of slices and between them."""
    rng = np.random.default_rng(31)
    M = 200000
    sizes, tids = local_csr(rng, 400000, M, 2, 13)
    eq, proj, eff, uniq = table_csr(sizes, tids, M, seed=32)
    p = default_params(min_iter=6, max_iter=6)
    ref, rst = oracle.em_optimize(eq, proj, eff, uniq, p)
    first = None
    ctx.set_option("blocks_per_sm", 1)
    ctx.set_option("sell_group_cm", group); ctx.set_option("sell_group_tm", group)
    try:
        for rebalance in (0, 3):
            for variant in (1, 0):
                ctx.set_option("rebalance", rebalance); ctx.set_option("variant", variant)
                alpha, st, ok = ctx.optimize(eq, p, proj, eff, uniq)
                assert ok and st.iters == 6
                assert ctx.info("fallback_rows_cm") == 0 and ctx.info("fallback_rows_tm") == 0
                warps, ring = ctx.info("warps"), ctx.info("ring_cols")
                for m in ("cm", "tm"):     # columns per warp: at least two trips around the ring on average
                    assert ctx.info("sell_cols_" + m) >= 2 * ring * warps, (m, ctx.info("sell_cols_" + m), warps, ring)
                np.testing.assert_allclose(alpha, ref, rtol=ALPHA_RTOL, atol=ALPHA_ATOL)
                if first is None:
                    first = alpha
                assert np.array_equal(alpha.view(np.uint64), first.view(np.uint64)), (variant, rebalance)
    finally:
        ctx.set_option("blocks_per_sm", 0)
        ctx.set_option("rebalance", 1); ctx.set_option("variant", 1)
        ctx.set_option("sell_group_cm", 1024); ctx.set_option("sell_group_tm", 1024)


def test_wide_index_windows_fall_back(ctx, oracle):
    """Classes that pair transcripts 80 000 apart: their class-major slices span more than 16 bits of transcript rows,
    and the far transcript's transcript-major slice spans more than 16 bits of class ids.  Those rows take the
    long-row path (counted), and the results still match the oracle."""
    rng = np.random.default_rng(21)
    M = 100000
    labels = local_labels(rng, 120000, M, 2, 6)
    for a in rng.choice(M - 80000, size=64, replace=False):
        labels.append(np.array([a, a + 80000]))
    eq, proj, eff, uniq = table(labels, M, seed=22)
    for vbem in (1, 0):
        p = default_params(use_vbem=vbem, min_iter=10, max_iter=10)
        ref, rst = oracle.em_optimize(eq, proj, eff, uniq, p)
        for variant in (1, 0):
            ctx.set_option("variant", variant)
            try:
                alpha, st, ok = ctx.optimize(eq, p, proj, eff, uniq)
            finally:
                ctx.set_option("variant", 1)
            assert ok and st.iters == 10
            assert ctx.info("fallback_rows_cm") > 0 and ctx.info("fallback_rows_tm") > 0
            assert ctx.info("long_rows_cm") >= ctx.info("fallback_rows_cm")
            np.testing.assert_allclose(alpha, ref, rtol=ALPHA_RTOL, atol=ALPHA_ATOL)


def test_stream_figures_of_the_bench_table(ctx):
    """The bench table (synth_eq(seed=1)) needs no fallback, and the reported stream is the SELL columns at 10 bytes
    per entry plus the long rows' CSR at 12."""
    from salmon_b200.synth import synth_eq
    eq, proj, eff, uniq = synth_eq(seed=1)
    ctx.upload(eq, proj, eff, uniq)
    st = ctx.prepare(default_params(min_iter=2, max_iter=2))
    assert ctx.info("fallback_rows_cm") == 0 and ctx.info("fallback_rows_tm") == 0
    per = {m: ctx.info("sell_cols_" + m) * 320 + ctx.info("long_entries_" + m) * 12 for m in ("cm", "tm")}
    assert per["cm"] == ctx.info("stream_bytes_cm") and per["tm"] == ctx.info("stream_bytes_tm")
    assert ctx.info("stream_bytes") == per["cm"] + per["tm"]
    # every entry of a kept class is streamed once per layout: SELL entries (real + padding) or long-row entries
    for m in ("cm", "tm"):
        assert ctx.info("sell_cols_" + m) * 32 + ctx.info("long_entries_" + m) >= st.nnz_multi
    with pytest.raises(Exception):
        ctx.info("no_such_key")
