"""High-precision and double-precision restatements of the last step of mapping, written from salmon's sources:

  * the transcript clusters: ClusterForest::mergeClusters (include/salmon/internal/quant/ClusterForest.hpp) unions the
    transcripts of every fragment; with several ranks the global partition is the union of the per-rank partitions,
    each given as an array of cluster roots (the smallest member of each cluster);
  * normalizeAlphas (src/util/SalmonUtils.cpp:461-529): a cluster's projected counts are
    exp(mass_t - logSum_cluster mass + log numHits), then TranscriptCluster::projectToPolytope
    (include/salmon/internal/quant/TranscriptCluster.hpp:46-101) when one of them leaves [unique, total];
  * correctionFactorsFromMass and computeSmoothedEffectiveLengths (src/util/DistributionUtils.cpp:9-56) on the pmf
    of ReadExperiment::updateTranscriptLengthsAtomic (include/salmon/internal/quant/ReadExperiment.inl:61-94).

Log masses use salmon's LOG_0 = +inf for "no mass".  The *_exact forms evaluate in mpmath at 50 significant digits
from the double inputs; the *_double forms take the same steps in double, in salmon's (and the kernels') order."""
import math

import mpmath
import numpy as np

from py_ref_map import LOG_0, log_add, project_to_polytope

DPS = 50


def _find(parent, x):
    while parent[x] != x:
        parent[x] = parent[parent[x]]
        x = parent[x]
    return x


def _union(parent, a, b):
    a, b = _find(parent, a), _find(parent, b)
    if a != b:                      # the larger root goes under the smaller: a root is its cluster's smallest member
        parent[max(a, b)] = min(a, b)


def class_roots(M, classes):
    """cluster roots of the transcripts that share a class.  classes: iterable of transcript-id sequences."""
    parent = list(range(M))
    for tids in classes:
        t0 = int(tids[0])
        for t in tids[1:]:
            _union(parent, t0, int(t))
    return np.array([_find(parent, t) for t in range(M)], dtype=np.uint32)


def clusters_from_roots(M, roots_all):
    """the union of the partitions given by the rows of roots_all ([R, M]): returns each transcript's cluster root,
    the smallest member of its cluster."""
    parent = list(range(M))
    for row in np.asarray(roots_all).reshape(-1, M):
        for t, r in enumerate(row.tolist()):
            if r != t:
                _union(parent, t, r)
    return np.array([_find(parent, t) for t in range(M)], dtype=np.uint32)


def members(root):
    """{root: ascending member ids}"""
    order = np.argsort(root, kind="stable")
    rs = root[order]
    cut = np.flatnonzero(np.diff(rs)) + 1
    return {int(g[0]): order[s:e] for g, s, e in zip(np.split(rs, cut), np.r_[0, cut], np.r_[cut, len(rs)])}


def class_stats(M, classes_with_counts):
    """per-transcript (hits, unique, total): a class's count goes to the hits of its first transcript
    (updateCluster), to the unique count of its only transcript, and to the total count of each transcript."""
    hits = np.zeros(M, dtype=np.uint64)
    uniq = np.zeros(M, dtype=np.uint64)
    total = np.zeros(M, dtype=np.uint64)
    for tids, cnt in classes_with_counts:
        hits[tids[0]] += cnt
        if len(tids) == 1:
            uniq[tids[0]] += cnt
        total[np.asarray(tids, dtype=np.int64)] += cnt
    return hits, uniq, total


def project_double(log_mass, hits, uniq, total, root):
    """normalizeAlphas in double: members of a cluster in ascending id, the cluster mass by sequential logAdd, the
    polytope projection of py_ref_map.  Returns (projected counts, {root: rounds of the projection loop})."""
    log_mass = [float(x) for x in log_mass]
    uq = [int(x) for x in uniq]
    tt = [int(x) for x in total]
    proj = [0.0] * len(log_mass)
    for r, mem in members(np.asarray(root)).items():
        mem = mem.tolist()
        h = sum(int(hits[t]) for t in mem)
        lcm = LOG_0
        for t in mem:
            lcm = log_add(lcm, log_mass[t])
        if lcm == LOG_0:
            continue
        lcc = math.log(float(h)) if h > 0 else -math.inf
        needs = False
        for t in mem:
            if log_mass[t] != LOG_0:
                proj[t] = math.exp(log_mass[t] - lcm + lcc)
                needs |= proj[t] > tt[t] or proj[t] < uq[t]
        if len(mem) > 1 and needs:
            project_to_polytope(mem, proj, uq, tt, float(h))
    return np.array(proj)


def project_exact(log_mass, hits, root):
    """the unconstrained projection exp(m_t - log sum_cluster exp(m) + log hits_cluster), in mpmath at 50 digits"""
    out = np.zeros(len(log_mass))
    with mpmath.workdps(DPS):
        for r, mem in members(np.asarray(root)).items():
            h = sum(int(hits[t]) for t in mem)
            fin = [int(t) for t in mem if log_mass[t] != LOG_0]
            if not fin or h == 0:
                continue
            ms = {t: mpmath.mpf(float(log_mass[t])) for t in fin}
            mx = max(ms.values())
            lcm = mx + mpmath.log(mpmath.fsum(mpmath.exp(m - mx) for m in ms.values()))
            lh = mpmath.log(h)
            for t in fin:
                out[t] = float(mpmath.exp(ms[t] - lcm + lh))
    return out


def _min_v(fld_min, nf):
    return 1 if fld_min == nf - 1 else int(fld_min)


def eff_len_exact(hist, tot, fld_min, lengths, nf, raw=False):
    """correctionFactorsFromMass + computeSmoothedEffectiveLengths in mpmath.  hist: the log FLD histogram (nf bins),
    tot its log total, fld_min FragmentLengthDistribution's smallest observed length (nf-1 = none: the pmf then
    starts at 1).  raw=True also returns len - cf, before the effLen < 1 fallback."""
    minV, maxV = _min_v(fld_min, nf), nf - 1
    with mpmath.workdps(DPS):
        lp = [mpmath.mpf(float(hist[i])) - mpmath.mpf(float(tot)) for i in range(nf)]
        if minV <= maxV:
            mx = max(lp[minV:maxV + 1])
            s = mx + mpmath.log(mpmath.fsum(mpmath.exp(x - mx) for x in lp[minV:maxV + 1]))
        pmf = [mpmath.mpf(0)] * nf
        for i in range(minV, maxV):
            pmf[i] = 100 * mpmath.exp(lp[i] - s)
        cf = [mpmath.mpf(0)] * nf
        vals = mult = mpmath.mpf(0)
        mult += pmf[0]
        for i in range(1, nf):
            vals += pmf[i] * i
            mult += pmf[i]
            if mult > 0:
                cf[i] = vals / mult
        eff, rawv = [], []
        for L in lengths:
            L = int(L)
            d = L - cf[nf - 1 if L >= nf else L]
            rawv.append(float(d))
            eff.append(float(d) if d >= 1 else float(L))
    return (np.array(eff), np.array(rawv)) if raw else np.array(eff)


def eff_len_double(hist, tot, fld_min, lengths, nf):
    """the same steps in double, in the kernel's order (sequential logAdd, products rounded before the sums)"""
    minV, maxV = _min_v(fld_min, nf), nf - 1
    s = LOG_0
    for i in range(minV, maxV + 1):
        s = log_add(s, float(hist[i]) - float(tot))
    pmf = [0.0] * nf
    for i in range(minV, maxV):
        pmf[i] = 100.0 * math.exp((float(hist[i]) - float(tot)) - s)
    cf = [0.0] * nf
    vals, mult = 0.0, pmf[0]
    for i in range(1, nf):
        vals = pmf[i] * float(i) + vals
        mult = pmf[i] + mult
        cf[i] = vals / mult if mult > 0 else 0.0
    out = []
    for L in lengths:
        L = int(L)
        e = float(L) - cf[nf - 1 if L >= nf else L]
        out.append(e if e >= 1.0 else float(L))
    return np.array(out)
