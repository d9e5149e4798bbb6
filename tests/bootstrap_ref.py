"""Restatement of salmon's doBootstrap with `--bootstrapReproject` (src/inference/CollapsedEMOptimizer.cpp:398-552,
reprojection :495-505) on top of the oracle: the replicates' class counts are the oracle's Philox draws (orc_bootstrap),
every update is the oracle's serial EMUpdate_ / VBEMUpdate_ (orc_em_step_serial), and the loop, the reprojection and
the truncation are restated here.

With reproject=False this is orc_bootstrap itself, bit for bit.  With reproject=True each replicate's converged alpha
takes one more update against the ORIGINAL counts of the classes the replicates resample (origCounts over txpGroups:
the valid_boot classes), and that update's output is what is truncated and written.  (salmon's own code writes the
update into alphasPrime and then truncates and writes alphas, which the update did not touch; the option's help text
-- "reproject those parameters onto the original equivalence class counts" -- is what this build implements.)

The reprojection drops a class whose denominator is at most DBL_MIN times the largest count of a multi-transcript class
(salmon's degenerate-class rule, denom <= minEQClassWeight, scaled so that count / denom stays finite).  It starts from
alphas the replicate drove to zero or to subnormal values in the classes it did not draw, whose original counts are
positive: with salmon's guards count / denom overflows there and the replicate would carry infinities (or 0 * inf =
NaN).  The restatement's reprojection step is therefore the update written out here (_update) with that guard; the
loop keeps the oracle's step."""
from types import SimpleNamespace

import numpy as np


def boot_inputs(oracle, eq, proj, eff, uniq, p_main, nmapped):
    """valid flags, combined weights, priors and active transcripts exactly as gatherBootstraps sees them
    (:582-621): the optimiser's combined weights and validity, then markDegenerateClasses with the uniform start"""
    _, _, cw, valid = oracle.em_optimize(eq, proj, eff, uniq, p_main, want_combined=True)
    M = eq.n_txps
    active = np.zeros(M, dtype=np.uint8)
    active[eq.tids] = 1
    unif = (1.0 / active.sum()) * nmapped
    sizes = (eq.off[1:] - eq.off[:-1]).astype(np.int64)
    v = np.where(active[eq.tids] > 0, unif, 0.0) * cw
    v[np.isnan(v)] = 0.0
    denom = np.add.reduceat(v, eq.off[:-1].astype(np.int64)) if eq.nnz else np.zeros(eq.n_classes)
    denom[sizes == 0] = 0.0
    valid_boot = (valid.astype(bool) & (denom > np.finfo(float).tiny)).astype(np.uint8)
    prior = np.full(M, p_main.vb_prior) if p_main.per_txp_prior else p_main.vb_prior * eff
    return cw, valid, valid_boot, prior, active


def _step(oracle, eq, counts, cw, valid, prior, alpha, vbem):
    tab = SimpleNamespace(n_classes=eq.n_classes, n_txps=eq.n_txps, off=eq.off, tids=eq.tids,
                          counts=np.ascontiguousarray(counts, dtype=np.uint64))
    out, _ = oracle.em_step(tab, cw, valid, prior, alpha, vbem, serial=True)
    return out


def _update(oracle, eq, counts, cw, valid, prior, alpha, vbem, guard):
    """EMUpdate_ (EMUtils.cpp:7-53) / VBEMUpdate_ (CollapsedEMOptimizer.cpp:104-171) over the valid classes, a class
    kept only when its denominator is above `guard`; an entry adds to its transcript only where its theta * w > 0"""
    sizes = np.diff(eq.off).astype(np.int64)
    cls = np.repeat(np.arange(eq.n_classes), sizes)
    keep = (valid[cls] > 0)
    out = np.zeros(eq.n_txps)
    single = keep & (sizes[cls] == 1)
    np.add.at(out, eq.tids[single], counts[cls[single]].astype(np.float64))
    theta = alpha
    if vbem:
        ap = alpha + prior
        log_norm = oracle.digamma(float(np.sum(ap)))
        dg = np.array([oracle.digamma(float(x)) for x in ap])
        theta = np.where(ap > 1e-10, np.exp(dg - log_norm), 0.0)
    multi = keep & (sizes[cls] > 1)
    v = theta[eq.tids] * cw
    v = np.where(multi & (v > 0.0), v, 0.0)
    denom = np.bincount(cls, v, minlength=eq.n_classes)
    inv = np.where(denom > guard, counts.astype(np.float64) / np.where(denom > guard, denom, 1.0), 0.0)
    np.add.at(out, eq.tids, v * inv[cls])
    return out


def reproject_guard(eq, counts, valid):
    """DBL_MIN times the largest count of a valid multi-transcript class"""
    multi = (np.diff(eq.off) > 1) & (valid > 0)
    return np.finfo(float).tiny * max(1, int(counts[multi].max()) if multi.any() else 1)


def _converge_swap(alpha, alpha_prime, tol):
    """:478-492: converged unless some alpha' above alphaCheckCutoff moved by more than tol (relative)"""
    sel = alpha_prime > 1e-2
    rel = np.abs(alpha[sel] - alpha_prime[sel]) / alpha_prime[sel]
    return not bool(np.any(rel > tol))


def bootstrap(oracle, eq, cw, valid_boot, prior, active, p, n_boot, seed, reproject):
    """-> (alphas [n_boot, M], the replicates' class counts [n_boot, C], rc); rc = 1 where doBootstrap returns false"""
    _, samp, rc = oracle.bootstrap(eq, cw, valid_boot, prior, active, p, n_boot, seed)
    assert rc == 0
    M = eq.n_txps
    total = float(eq.counts[valid_boot > 0].sum())                # totalCount passed as totalNumFrags (:681)
    unif = (1.0 / float(active.sum())) * total                    # uniformTxpWeight * totalNumFrags (:450-453)
    orig = np.where(valid_boot > 0, eq.counts, 0).astype(np.uint64)
    out = np.zeros((n_boot, M))
    for b in range(n_boot):
        alpha = np.where(active > 0, unif, 0.0)
        it, converged = 0, False
        while it < p.min_iter or (it < p.max_iter and not converged):   # :467
            ap = _step(oracle, eq, samp[b], cw, valid_boot, prior, alpha, p.use_vbem)
            converged = _converge_swap(alpha, ap, p.tol)
            alpha = ap
            it += 1
        if reproject:                                                   # :495-505
            alpha = _update(oracle, eq, orig, cw, valid_boot, prior, alpha, p.use_vbem,
                            reproject_guard(eq, orig, valid_boot))
        alpha = np.where(alpha <= 1e-8, 0.0, alpha)                     # :507-519
        if alpha.sum() < np.finfo(float).tiny:
            return out[:b], samp[:b], 1
        out[b] = alpha
    return out, samp, 0
