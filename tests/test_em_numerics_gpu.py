"""The EM / VBEM kernels at their numeric edges, against a 40-digit restatement of the reference (tests/em_hp_ref.py) and
against the oracle, and the fixed-point sum of (alpha' + prior) on tables large enough to need a smaller unit.

Small hand-made tables put transcripts and classes clearly on both sides of every double-precision decision of the
reference: alpha + prior around digammaMin = 1e-10 and around the branch of the fused digamma at 10, alphas from 1e-9
to 1e12 in one class, start denominators of 1e-310 (skipped) and 1e-300 (kept), transcripts that cross
ALPHA_CHECK_CUTOFF between iterations, and final alphas on both sides of the 1e-8 cut.  The restatement reports how far
each decision's operand was from its threshold, and the tables are checked to keep that margin, so a double-precision
run must take the same branches: iteration counts, convergence, the classes skipped at the start and the zero alphas
must be equal, and the alphas agree to 1e-12 (classes skipped inside the loop show in the alphas of their members).
"""
import math
import os
import subprocess

import numpy as np
import pytest

import em_hp_ref as H
from salmon_b200 import EMContext, default_params
from salmon_b200._capi import EqClasses, SalmonB200Error, write_eq_classes
from salmon_b200.synth import synth_eq

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HP_RTOL = 1e-12
MARGIN = 1e-6           # smallest relative distance of any decision from its threshold in the hand-made tables
EFF_TINY = 1e-30        # effective length of the steered transcripts: alt_init's start term is then negligible


@pytest.fixture(scope="module")
def ctx():
    c = EMContext(0)
    yield c
    c.close()


class Table:
    """a hand-made table: transcripts with a projected count (their start alpha, steered through alt_init and
    num_required_frags = 1: alpha0 = 0.999 * projected + 1e-6 * (unique + 0.5) * eff_len) and classes"""

    def __init__(self):
        self.proj, self.eff, self.classes = [], [], []

    def txp(self, projected, eff=EFF_TINY):
        self.proj.append(float(projected)); self.eff.append(float(eff))
        return len(self.proj) - 1

    def cls(self, tids, count, weights=None):
        self.classes.append((list(tids), list(weights or [1.0] * len(tids)), int(count)))
        return len(self.classes) - 1

    def eq(self):
        sizes = [len(t) for t, _, _ in self.classes]
        off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)
        tids = np.concatenate([t for t, _, _ in self.classes]).astype(np.uint32)
        w = np.concatenate([ws for _, ws, _ in self.classes]).astype(np.float64)
        counts = np.array([c for _, _, c in self.classes], dtype=np.uint64)
        M = len(self.proj)
        return EqClasses(M, off, tids, w, counts), np.array(self.proj), np.array(self.eff), np.zeros(M, np.uint64)


def ap_target(ap, prior):
    """the projected count that starts a transcript at alpha + prior = ap"""
    return (ap - prior) / 0.999


def edge_table():
    """VBEM prior 1e-11 per transcript, so that alpha + prior can sit at digammaMin"""
    prior = 1e-11
    T = Table()
    host = T.txp(1000.0)
    T.cls([host], 1000)
    dmin = [T.txp(ap_target(1e-10 * (1 + s), prior)) for s in (-1e-3, 1e-3, -1e-2, 1e-2)]
    T.cls(dmin + [host], 50)
    ten = [T.txp(ap_target(10.0 * (1 + s), prior)) for s in (-1e-7, 1e-7, -1e-3, 1e-3)]
    T.cls(ten + [host], 40)
    wide = [T.txp(10.0 ** k) for k in range(-9, 13)]          # 1e-9 .. 1e12 in one class
    T.cls(wide, 1300)
    T.cls([wide[-1]], 10 ** 12)
    # start denominators: alpha0 = 1e-6 * 0.5 * eff_len with projected 0
    d310 = [T.txp(0.0, eff=2e-304), T.txp(0.0, eff=2e-304)]
    T.cls(d310, 7)                                            # 1e-310 <= DBL_MIN: skipped
    d300 = [T.txp(0.0, eff=2e-294), T.txp(0.0, eff=2e-294)]
    T.cls(d300, 7)                                            # 1e-300: kept
    # decaying shares of a class with the host: they cross ALPHA_CHECK_CUTOFF after a few iterations
    for p, c in ((0.05, 500), (0.02, 300), (0.5, 700), (3.0, 900)):
        T.cls([T.txp(p), host], c)
    return T, dict(vb_prior=prior)


def cut_table(w_host):
    """default prior; two probes whose final alphas are steered (w_host) to either side of the 1e-8 cut"""
    T = Table()
    host = T.txp(1e6)
    T.cls([host], 10 ** 6)
    probes = [T.txp(1e-3), T.txp(1e-3)]
    for b, w in zip(probes, w_host):
        T.cls([host, b], 100, [w, 1.0])
    for p, c in ((0.05, 5000), (0.3, 20000)):
        T.cls([T.txp(p), host], c)
    return T, probes


PARAMS = dict(alt_init=1, num_required_frags=1.0)


def hp_run(T, vbem, min_iter, max_iter, **kw):
    eq, proj, eff, uniq = T.eq()
    return H.optimize(T.classes, eq.n_txps, proj, eff, uniq, use_vbem=vbem, alt_init=True, num_required_frags=1.0,
                      min_iter=min_iter, max_iter=max_iter, **kw)


def steer_cut(vbem, min_iter, max_iter):
    """host weights that put the two probes at 1e-8 * (1 -/+ 5e-4) after the run (secant in log-log, on the
    restatement); None where the first plain-EM iteration's 1.0 keeps every alpha above the cut"""
    if not vbem and max_iter == 1:
        return None
    targets = [1e-8 * (1 - 5e-4), 1e-8 * (1 + 5e-4)]
    lw = [[0.0, -3.0], [0.0, -3.0]]
    la = [[None, None], [None, None]]
    for k in range(2):
        r = hp_run(cut_table([10.0 ** lw[0][k], 10.0 ** lw[1][k]])[0], vbem, min_iter, max_iter)
        for j in range(2):
            la[j][k] = math.log10(r["precut"][1 + j])
    for _ in range(8):
        nxt = []
        for j in range(2):
            (w0, w1), (a0, a1) = lw[j][-2:], la[j][-2:]
            nxt.append(w1 + (math.log10(targets[j]) - a1) * (w1 - w0) / (a1 - a0))
        r = hp_run(cut_table([10.0 ** nxt[0], 10.0 ** nxt[1]])[0], vbem, min_iter, max_iter)
        for j in range(2):
            lw[j].append(nxt[j]); la[j].append(math.log10(r["precut"][1 + j]))
        if all(abs(la[j][-1] - math.log10(targets[j])) < 1e-6 for j in range(2)):
            return [10.0 ** nxt[0], 10.0 ** nxt[1]]
    raise AssertionError("the cut probes did not settle")


def run_gpu(ctx, T, variant, vbem, min_iter, max_iter, **kw):
    eq, proj, eff, uniq = T.eq()
    p = default_params(use_vbem=int(vbem), min_iter=min_iter, max_iter=max_iter, **PARAMS, **kw)
    ctx.set_option("variant", variant)
    alpha, st, ok = ctx.optimize(eq, p, proj, eff, uniq)
    _, valid = ctx.get_combined()
    return alpha, st, valid, (eq, proj, eff, uniq, p)


def check_against_hp(oracle, alpha, st, valid, args, hp):
    for name, m in hp["margins"].items():
        assert m > MARGIN, (name, m)                       # the table keeps every decision clear
    assert st.iters == hp["iters"] and bool(st.converged) == hp["converged"]
    assert valid.astype(bool).tolist() == hp["valid"]
    assert np.flatnonzero(alpha == 0.0).tolist() == hp["zero"]
    want = np.array(hp["alpha"])
    nz = want > 1e-8
    rel = np.abs(alpha[nz] - want[nz]) / want[nz]
    assert rel.max() <= HP_RTOL, (float(rel.max()), int(np.flatnonzero(nz)[np.argmax(rel)]))
    eq, proj, eff, uniq, p = args
    ref, rst = oracle.em_optimize(eq, proj, eff, uniq, p)
    assert rst.iters == st.iters
    np.testing.assert_allclose(alpha, ref, rtol=1e-9, atol=1e-9)


ITERS = [(1, 1), (2, 2), (5, 5), (30, 30), (2, 30)]   # fixed counts, and a run that stops on convergence


@pytest.mark.parametrize("vbem", [1, 0])
@pytest.mark.parametrize("min_iter,max_iter", ITERS)
def test_edge_table_vs_high_precision(ctx, oracle, vbem, min_iter, max_iter):
    T, kw = edge_table()
    hp = hp_run(T, vbem, min_iter, max_iter, **kw)
    # the table reaches what it is for
    if vbem:
        assert hp["margins"]["digamma_min"] < 2e-2
    assert hp["valid"][5] is False and hp["valid"][6] is True       # the 1e-310 / 1e-300 start denominators
    for variant in (1, 0):
        alpha, st, valid, args = run_gpu(ctx, T, variant, vbem, min_iter, max_iter, **kw)
        check_against_hp(oracle, alpha, st, valid, args, hp)


@pytest.mark.parametrize("vbem", [1, 0])
@pytest.mark.parametrize("min_iter,max_iter", ITERS)
def test_final_cut_vs_high_precision(ctx, oracle, vbem, min_iter, max_iter):
    w = steer_cut(vbem, min_iter, max_iter)
    T, probes = cut_table(w or [1.0, 1.0])
    hp = hp_run(T, vbem, min_iter, max_iter)
    if w is not None:
        assert probes[0] in hp["zero"] and probes[1] not in hp["zero"]
        assert 4e-4 < hp["margins"]["cut"] < 6e-4
    for variant in (1, 0):
        alpha, st, valid, args = run_gpu(ctx, T, variant, vbem, min_iter, max_iter)
        check_against_hp(oracle, alpha, st, valid, args, hp)
        if w is not None:
            assert alpha[probes[0]] == 0.0 and 1e-8 < alpha[probes[1]] < 1.001e-8


# ---- the fixed-point sum of (alpha' + prior) ------------------------------------------------------------------------
def large_tables():
    eq, proj, eff, uniq = synth_eq(seed=23, C=20000, M=4000, total_count=400000)
    vb = 1e15 / float(eff.sum())                     # per-nucleotide prior: sum of the priors ~ 1e15
    yield "prior_1e15", (eq, proj, eff, uniq), dict(per_txp_prior=0, vb_prior=vb)
    eq2, proj2, eff2, uniq2 = synth_eq(seed=24, C=20000, M=4000, total_count=int(2e13))
    assert float(eq2.counts.astype(np.float64).sum()) > 1.9e13
    yield "counts_2e13", (eq2, proj2, eff2, uniq2), {}


@pytest.mark.parametrize("case", ["prior_1e15", "counts_2e13"])
@pytest.mark.parametrize("vbem", [1, 0])
def test_large_sums_scale_down(ctx, oracle, case, vbem):
    """a sum of (alpha' + prior) beyond 2^43 no longer fits 2^-20 units in 64 bits: prepare picks a smaller unit, and
    the run still matches the oracle and repeats bit for bit"""
    name, (eq, proj, eff, uniq), kw = next(t for t in large_tables() if t[0] == case)
    p = default_params(use_vbem=vbem, min_iter=40, max_iter=40, **kw)
    ref, rst = oracle.em_optimize(eq, proj, eff, uniq, p)
    for variant in (1, 0):
        ctx.set_option("variant", variant)
        a1, st, ok = ctx.optimize(eq, p, proj, eff, uniq)
        s = ctx.info("sum_scale_log2")
        assert s < 20
        bound = 2.0 * (float(eq.counts.astype(np.float64).sum()) + eq.n_txps +
                       (kw["vb_prior"] * float(np.abs(eff).sum()) if "vb_prior" in kw else 1e-2 * eq.n_txps))
        assert bound * 2.0 ** s < 2.0 ** 62 <= bound * 2.0 ** (s + 1)
        a2, st2, _ = ctx.optimize(eq, p, proj, eff, uniq)
        assert st.iters == st2.iters == rst.iters == 40
        assert np.array_equal(a1.view(np.uint64), a2.view(np.uint64))
        np.testing.assert_allclose(a1, ref, rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("vbem", [1, 0])
def test_default_scale_keeps_alphas_bit_for_bit(ctx, vbem):
    """at ordinary sizes the unit stays 2^-20 and the alphas are the bits the build before the scale choice gave
    (tests/golden/em_alpha_synth21.npz, saved from that build on an H100)"""
    g = np.load(os.path.join(ROOT, "tests", "golden", "em_alpha_synth21.npz"))
    eq, proj, eff, uniq = synth_eq(seed=21, C=20000, M=4000, total_count=500000)
    p = default_params() if vbem else default_params(use_vbem=0)
    key = "vbem" if vbem else "em"
    for variant in (1, 0):
        ctx.set_option("variant", variant)
        alpha, st, ok = ctx.optimize(eq, p, proj, eff, uniq)
        assert ctx.info("sum_scale_log2") == 20
        assert [st.iters, st.converged] == g[key + "_iters"].tolist()
        assert np.array_equal(alpha.view(np.uint64), g[key].view(np.uint64))


@pytest.mark.parametrize("bad", [-1.0, -1e-300, float("nan"), float("inf")])
def test_vb_prior_refused(ctx, bad):
    eq, proj, eff, uniq = synth_eq(seed=3, C=200, M=50, total_count=2000)
    ctx.upload(eq, proj, eff, uniq)
    with pytest.raises(SalmonB200Error, match="must be a finite number >= 0"):
        ctx.prepare(default_params(vb_prior=bad))
    ctx.prepare(default_params(vb_prior=0.0))       # zero is a prior


def test_cli_refuses_negative_vb_prior(tmp_path):
    eq, proj, eff, uniq = synth_eq(seed=3, C=200, M=50, total_count=2000)
    path = tmp_path / "eq_classes.txt"
    write_eq_classes(path, [f"t{i}" for i in range(eq.n_txps)], eq.off, eq.tids, eq.counts, eq.weights)
    exe = os.path.join(ROOT, "salmon_b200", "sb_salmon")
    r = subprocess.run([exe, "quant", "-e", str(path), "-o", str(tmp_path / "out"), "--vbPrior", "-1"],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode != 0
    assert "the VB prior (--vbPrior) must be a finite number >= 0, not -1" in r.stderr, r.stderr
