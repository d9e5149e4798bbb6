"""py_ref.optimize (CollapsedEMOptimizer::optimize) restated in mpmath at 40 digits, for small hand-made tables at the
EM's numeric edges.  Every value is carried in high precision from the exact double inputs, but the reference's
double-precision DECISIONS stay decisions, taken at the same thresholds:
  theta = 0 unless alpha + prior > 1e-10 (digammaMin)       denominators <= DBL_MIN skip the class
  alpha' > 1e-2 enters the convergence test (ALPHA_CHECK_CUTOFF)    final alphas <= 1e-8 are cut to 0
Each decision also records how far its operand was from the threshold (relative), so a test can check that a table
puts its transcripts and classes clearly on one side: then the double-precision run must take the same branches.
"""
import sys

import mpmath

DBL_MIN = sys.float_info.min
DPS = 40


class Margins:
    """smallest relative distance of a decision's operand from its threshold (operands at 0 are not near)"""

    def __init__(self):
        self.m = {}

    def see(self, name, value, thr):
        if value == 0 or thr == 0:
            return
        d = abs(value - thr) / abs(thr)
        if name not in self.m or d < self.m[name]:
            self.m[name] = float(d)


def optimize(classes, M, projected, eff_len, unique, *, use_vbem=True, per_txp_prior=True, alt_init=False,
             vb_prior=1e-2, tol=0.01, num_required_frags=5e7, min_iter=100, max_iter=10000):
    """classes: list of (tids, weights, count).  Returns a dict: alpha (floats, after the final cut), precut (mpf, the
    alphas before it), iters, converged,
    valid (per class: kept at the start), skipped (per iteration: classes whose denominator was <= DBL_MIN),
    zero (transcripts cut to 0), margins (Margins.m)."""
    mpmath.mp.dps = DPS
    f = mpmath.mpf
    mg = Margins()
    eff = [f(float(x)) for x in eff_len]
    alphas = [f(float(x)) for x in projected]
    total_weight = sum(alphas, f(0))
    prior = [f(vb_prior) if per_txp_prior else f(vb_prior) * eff[i] for i in range(M)]
    uni_init = [(f(int(unique[i])) + f(0.5)) * f(1e-3) * eff[i] for i in range(M)]
    uniform_prior = total_weight / M
    frac = min(f(0.999), total_weight / f(num_required_frags))
    for i in range(M):
        uni = uni_init[i] if alt_init else uniform_prior
        alphas[i] = alphas[i] * frac + uni * (1 - frac)
    alphas_prime = [f(1)] * M                                     # the first plain-EM iteration starts at 1.0
    comb = []
    for tids, ws, count in classes:
        cw = []
        for t, w in zip(tids, ws):
            el = eff[t] if eff[t] > 1 else f(1)
            cw.append(f(count) * f(float(w)) / el)
        s = sum(cw, f(0))
        comb.append([x / s for x in cw])
    valid = []
    for (tids, _, _), cw in zip(classes, comb):
        d = sum((alphas[t] * a for t, a in zip(tids, cw)), f(0))
        mg.see("denom", d, DBL_MIN)
        valid.append(bool(d > DBL_MIN))
    it, converged, skipped = 0, False, []
    while it < min_iter or (it < max_iter and not converged):
        if use_vbem:
            log_norm = mpmath.digamma(sum((alphas[i] + prior[i] for i in range(M)), f(0)))
            theta = []
            for i in range(M):
                ap = alphas[i] + prior[i]
                mg.see("digamma_min", ap, 1e-10)
                theta.append(mpmath.exp(mpmath.digamma(ap) - log_norm) if ap > 1e-10 else f(0))
                alphas_prime[i] = f(0)
        else:
            theta = alphas
        sk = []
        for c, ((tids, _, count), cw, ok) in enumerate(zip(classes, comb, valid)):
            if not ok:
                continue
            if len(tids) > 1:
                denom = sum((theta[t] * a for t, a in zip(tids, cw) if theta[t] > 0), f(0))
                mg.see("denom", denom, DBL_MIN)
                if denom <= DBL_MIN:
                    sk.append(c)
                    continue
                for t, a in zip(tids, cw):
                    if theta[t] > 0:
                        alphas_prime[t] += theta[t] * a * f(count) / denom
            else:
                alphas_prime[tids[0]] += f(count)
        skipped.append(sk)
        converged = True
        for i in range(M):
            mg.see("alpha_check", alphas_prime[i], 1e-2)
            if alphas_prime[i] > 1e-2:
                rel = abs(alphas[i] - alphas_prime[i]) / alphas_prime[i]
                mg.see("tol", rel, tol)
                if rel > tol:
                    converged = False
            alphas[i] = alphas_prime[i]
            alphas_prime[i] = f(0)
        it += 1
    precut = list(alphas)
    zero = []
    for i in range(M):
        mg.see("cut", alphas[i], 1e-8)
        if alphas[i] <= 1e-8:
            alphas[i] = f(0)
            zero.append(i)
    return dict(alpha=[float(a) for a in alphas], precut=precut, iters=it, converged=converged, valid=valid,
                skipped=skipped, zero=zero, margins=mg.m)
