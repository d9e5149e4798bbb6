"""GPU parity tests (H100): the CUDA EM/VBEM path through the C ABI against the CPU
oracle on identical inputs.  Tolerances (BASELINE.md section 3):
  combinedWeights / validity flags : bit-exact
  alpha after k iterations          : 1e-9 relative (+1e-9 absolute floor)
  final TPM                         : 1e-4 relative on TPM > 1e-3
"""
import numpy as np
import pytest

from salmon_b200 import EMContext, default_params
from salmon_b200._capi import EqClasses
from salmon_b200.synth import synth_eq
from test_oracle import random_problem

pytestmark = pytest.mark.gpu

ALPHA_RTOL = 1e-9
ALPHA_ATOL = 1e-9


@pytest.fixture(scope="module")
def ctx():
    c = EMContext(0)
    yield c
    c.close()


def run_both(ctx, oracle, eq, proj, eff, uniq, variant=1, **kw):
    p = default_params(**kw)
    ctx.set_option("variant", variant)
    alpha, st, ok = ctx.optimize(eq, p, proj, eff, uniq)
    ref, rst = oracle.em_optimize(eq, proj, eff, uniq, p)
    return alpha, st, ok, ref, rst


def assert_alpha(alpha, ref):
    np.testing.assert_allclose(alpha, ref, rtol=ALPHA_RTOL, atol=ALPHA_ATOL)


@pytest.mark.parametrize("variant", [1, 0])
@pytest.mark.parametrize("k", [1, 2, 3, 10])
@pytest.mark.parametrize("vbem", [1, 0])
def test_per_iteration_parity(ctx, oracle, vbem, k, variant):
    eq, proj, eff, uniq = synth_eq(seed=2, C=20000, M=6000, total_count=500000)
    alpha, st, ok, ref, rst = run_both(ctx, oracle, eq, proj, eff, uniq, variant=variant,
                                       use_vbem=vbem, min_iter=k, max_iter=k)
    assert st.iters == rst.iters == k
    assert ok and rst.ok
    assert_alpha(alpha, ref)
    assert st.gpu_launches > 0


def test_combined_weights_and_validity_bit_exact(ctx, oracle):
    rng = np.random.default_rng(8)
    eq, proj, eff, uniq = random_problem(rng, C=3000, M=500, max_label=9, zero_frac=0.08)
    p = default_params(min_iter=1, max_iter=1)
    ctx.upload(eq, proj, eff, uniq)
    st = ctx.prepare(p)
    cw, valid = ctx.get_combined()
    _, rst, rcw, rvalid = oracle.em_optimize(eq, proj, eff, uniq, p, want_combined=True)
    assert np.array_equal(valid, rvalid)
    assert st.n_degenerate == rst.n_degenerate
    assert np.array_equal(cw.view(np.uint64), rcw.view(np.uint64))   # NaNs included


@pytest.mark.parametrize("kw", [
    dict(), dict(use_vbem=0), dict(per_txp_prior=0, vb_prior=1e-5), dict(init_uniform=1),
    dict(eq_class_mode=1, init_uniform=1), dict(no_rich_eq=1), dict(alt_init=1),
    dict(no_length_correction=1),
])
def test_option_matrix_full_run(ctx, oracle, kw):
    rng = np.random.default_rng(21)
    eq, proj, eff, uniq = random_problem(rng, C=4000, M=700, max_label=10, zero_frac=0.03)
    alpha, st, ok, ref, rst = run_both(ctx, oracle, eq, proj, eff, uniq, **kw)
    assert st.iters == rst.iters, (st.iters, rst.iters)
    assert bool(st.converged) == bool(rst.converged)
    assert st.n_degenerate == rst.n_degenerate
    assert_alpha(alpha, ref)
    assert abs(st.alpha_sum - rst.alpha_sum) <= 1e-9 * rst.alpha_sum
    assert abs(st.max_rel_diff - rst.max_rel_diff) <= 1e-6 * max(1e-3, abs(rst.max_rel_diff))


def test_final_tpm_within_1e4(ctx, oracle):
    eq, proj, eff, uniq = synth_eq(seed=4, C=60000, M=20000, total_count=2_000_000)
    alpha, st, ok, ref, rst = run_both(ctx, oracle, eq, proj, eff, uniq)   # run to convergence
    assert st.iters == rst.iters
    tpm = oracle.tpm(alpha, eff)
    rtpm = oracle.tpm(ref, eff)
    m = rtpm > 1e-3
    assert np.max(np.abs(tpm[m] - rtpm[m]) / rtpm[m]) < 1e-4
    assert_alpha(alpha, ref)


def test_edge_all_singletons(ctx, oracle):
    M = 50
    tids = np.arange(M, dtype=np.uint32)
    eq = EqClasses(M, np.arange(M + 1), tids, np.ones(M), np.arange(1, M + 1))
    proj = np.arange(1, M + 1, dtype=float)
    alpha, st, ok, ref, rst = run_both(ctx, oracle, eq, proj, np.full(M, 500.0),
                                       np.arange(1, M + 1).astype(np.uint64), min_iter=3, max_iter=3)
    assert st.n_multi_classes == 0
    assert_alpha(alpha, ref)
    for vb in (0,):
        alpha, st, ok, ref, rst = run_both(ctx, oracle, eq, proj, np.full(M, 500.0),
                                           np.arange(1, M + 1).astype(np.uint64), use_vbem=vb,
                                           min_iter=1, max_iter=1)
        assert_alpha(alpha, ref)   # EM first-iteration +1.0 quirk on inactive transcripts


def test_edge_long_rows(ctx, oracle):
    """A class wider than a tile (block path, class-major) and a transcript present in
    more classes than a tile holds (block path, transcript-major)."""
    rng = np.random.default_rng(3)
    M = 6000
    big = np.sort(rng.choice(M, size=5000, replace=False)).astype(np.uint32)   # > TILE + LMAX
    mid = np.sort(rng.choice(M, size=300, replace=False)).astype(np.uint32)    # LMAX < len < TILE
    labels = [big, mid]
    hub = 17
    for _ in range(4000):   # transcript `hub` sits in 4000 small classes
        other = rng.choice(M, size=rng.integers(1, 4), replace=False)
        labels.append(np.unique(np.concatenate(([hub], other))).astype(np.uint32))
    sizes = np.array([len(l) for l in labels])
    off = np.concatenate(([0], np.cumsum(sizes)))
    tids = np.concatenate(labels)
    w = rng.random(len(tids)) + 0.05
    w /= np.repeat(np.add.reduceat(w, off[:-1]), sizes)
    counts = rng.integers(1, 200, size=len(labels)).astype(np.uint64)
    eq = EqClasses(M, off, tids, w, counts)
    eff = rng.uniform(100, 3000, size=M)
    proj = np.bincount(tids, weights=np.repeat(counts.astype(float), sizes) * w, minlength=M)
    uniq = np.zeros(M, dtype=np.uint64)
    for vb in (1, 0):
        for variant in (1, 0):
            alpha, st, ok, ref, rst = run_both(ctx, oracle, eq, proj, eff, uniq, variant=variant,
                                               use_vbem=vb, min_iter=25, max_iter=25)
            assert_alpha(alpha, ref)


def test_edge_empty_and_tiny(ctx, oracle):
    # no classes at all: alpha collapses to 0 and the reference returns false
    eq = EqClasses(4, np.array([0]), np.array([], dtype=np.uint32), np.array([]), np.array([], dtype=np.uint64))
    p = default_params(min_iter=2, max_iter=2)
    alpha, st, ok = ctx.optimize(eq, p, np.ones(4), np.full(4, 100.0), np.zeros(4, dtype=np.uint64))
    ref, rst = oracle.em_optimize(eq, np.ones(4), np.full(4, 100.0), np.zeros(4, dtype=np.uint64), p)
    assert not ok and not rst.ok
    assert_alpha(alpha, ref)
    # a single two-transcript class
    eq = EqClasses(2, np.array([0, 2]), np.array([0, 1]), np.array([0.3, 0.7]), np.array([9]))
    alpha, st, ok, ref, rst = run_both(ctx, oracle, eq, np.array([4.0, 5.0]), np.array([200.0, 800.0]),
                                       np.zeros(2, dtype=np.uint64))
    assert st.iters == rst.iters
    assert_alpha(alpha, ref)


def test_full_size_properties(ctx, oracle):
    """BASELINE config 2 size (500k classes / 250k transcripts): size-independent
    properties + a short oracle comparison."""
    eq, proj, eff, uniq = synth_eq(seed=1)
    p = default_params(min_iter=60, max_iter=60)
    ctx.set_option("variant", 1)
    ctx.upload(eq, proj, eff, uniq)
    st0 = ctx.prepare(p)
    r1 = ctx.run()
    a1, s1, ok1 = ctx.download()
    r2 = ctx.run()
    a2, s2, ok2 = ctx.download()
    assert r1.iters == r2.iters == 60
    # bit-reproducible run to run (fixed summation order, no atomics on the data path)
    assert np.array_equal(a1.view(np.uint64), a2.view(np.uint64))
    # every valid class hands out exactly its count
    assert st0.n_degenerate == 0
    tot = float(eq.counts.sum())
    assert abs(s1 - tot) / tot < 1e-10
    assert (a1 >= 0).all()
    # variant 0 (one launch per phase) computes the same numbers
    ctx.set_option("variant", 0)
    ctx.run()
    a3, _, _ = ctx.download()
    ctx.set_option("variant", 1)
    assert np.array_equal(a1.view(np.uint64), a3.view(np.uint64))
    # oracle on the same 60 iterations
    ref, rst = oracle.em_optimize(eq, proj, eff, uniq, p)
    np.testing.assert_allclose(a1, ref, rtol=ALPHA_RTOL, atol=ALPHA_ATOL)
    # fixed point: at convergence one more step changes alpha by <= tol where alpha > cutoff
    pc = default_params()
    alpha, stc, ok = ctx.optimize(eq, pc, proj, eff, uniq)
    assert stc.converged == 1 and stc.max_rel_diff <= 0.01


@pytest.mark.parametrize("push_pass", [0, 1])
@pytest.mark.parametrize("vbem", [1, 0])
def test_fused_multi_gpu_kernel_loopback(oracle, vbem, push_pass):
    """k_em_persistent_mgpu on ONE GPU that is its own peer: pushes to the owner's recv rows, owner update, theta
    broadcast, exchange barriers, final alpha all-gather -- against the oracle (the 2-GPU run is scripts/check_multigpu.py)."""
    eq, proj, eff, uniq = synth_eq(seed=5, C=40000, M=9000, total_count=900000)
    c = EMContext(0)
    try:
        c.peer_loopback(eq.n_txps)
        c.set_option("push_pass", push_pass)    # both ways of getting the partials to their owners
        for k in (1, 2, 25):
            p = default_params(use_vbem=vbem, min_iter=k, max_iter=k)
            alpha, st, ok = c.optimize(eq, p, proj, eff, uniq)
            ref, rst = oracle.em_optimize(eq, proj, eff, uniq, p)
            assert ok and st.iters == rst.iters == k
            assert_alpha(alpha, ref)
            assert abs(st.max_rel_diff - rst.max_rel_diff) <= 1e-9 * max(1.0, abs(rst.max_rel_diff))

        # convergence decision taken inside the kernel from the exchanged maxima
        p = default_params(use_vbem=vbem, min_iter=10, max_iter=400)
        alpha, st, ok = c.optimize(eq, p, proj, eff, uniq)
        ref, rst = oracle.em_optimize(eq, proj, eff, uniq, p)
        assert st.iters == rst.iters and st.converged == rst.converged
        assert_alpha(alpha, ref)
    finally:
        c.close()


@pytest.mark.parametrize("rebalance", [0, 3])
def test_rebalanced_ranges_match_oracle(ctx, oracle, rebalance):
    """the column-count cut of the warp ranges and three rounds of the measured re-cut give the oracle's alphas
    (a row's sum is computed by one lane in label order wherever the row lands)"""
    eq, proj, eff, uniq = synth_eq(seed=6, C=60000, M=15000, total_count=2_000_000)
    p = default_params(min_iter=12, max_iter=12)
    ctx.set_option("variant", 1); ctx.set_option("rebalance", rebalance)
    try:
        alpha, st, ok = ctx.optimize(eq, p, proj, eff, uniq)
    finally:
        ctx.set_option("rebalance", 1)
    ref, rst = oracle.em_optimize(eq, proj, eff, uniq, p)
    assert ok and st.iters == 12
    assert_alpha(alpha, ref)
