"""The references of tests/project_ref.py against the CPU oracle's normalizeAlphas and effective lengths
(orc_online_finish) and against py_ref_map.normalize_alphas, on a small mapped workload that stays below burn-in
(the effective lengths then come from the final fragment-length distribution).  No GPU."""
import numpy as np
import pytest

from project_ref import (class_roots, class_stats, clusters_from_roots, eff_len_double, eff_len_exact, members,
                         project_double, project_exact)
from py_ref_map import normalize_alphas
from salmon_b200.synth import synth_reads, synth_txome


@pytest.fixture(scope="module")
def finished(oracle):
    txps, _ = synth_txome(seed=21, n_genes=80)
    left, right, _ = synth_reads(txps, seed=22, n=3000)
    p = oracle.map_params(num_pre_burnin=1000)
    on = oracle.Online(oracle.MapIndex(txps), p, seed=5, mini_batch=1000)
    parts = [on.batch(left[s], right[s]) for s in (slice(0, 1700), slice(1700, 3000))]
    merged = {k: np.concatenate([q[k] for q in parts]) for k in ("n_aln", "label", "weight")}
    e = oracle.eq_aggregate(merged, p.max_read_occ, True)
    st = on.state()
    assert st["burned_in"] == 0 and st["min_val"] < p.max_frag_len
    fin = on.finish(e["off"], e["tids"], e["counts"])
    off = e["off"].astype(np.int64)
    classes = [(e["tids"][off[c]:off[c + 1]].tolist(), int(e["counts"][c])) for c in range(len(e["counts"]))]
    lens = np.array([t.shape[0] for t in txps])
    return dict(M=len(txps), nf=p.max_frag_len + 1, st=st, fin=fin, classes=classes, lens=lens)


def test_project_double_matches_oracle(finished):
    M, st, fin, classes = finished["M"], finished["st"], finished["fin"], finished["classes"]
    hits, uniq, total = class_stats(M, classes)
    assert np.array_equal(uniq, fin["unique_counts"]) and np.array_equal(total, fin["total_counts"])
    root = class_roots(M, [t for t, _ in classes])
    got = project_double(st["mass"], hits, uniq, total, root)
    np.testing.assert_allclose(got, fin["projected_counts"], rtol=1e-12, atol=1e-12)
    ref, _, _ = normalize_alphas(st["mass"], classes)
    np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-12)
    # clusters of several members; where no bound binds, the double result is the exact unconstrained projection
    mem = members(root)
    assert max(len(m) for m in mem.values()) >= 4
    ex = project_exact(st["mass"], hits, root)
    free = np.concatenate([m for m in mem.values()
                           if np.all((ex[m] <= total[m]) & (ex[m] >= uniq[m]) | ~np.isfinite(st["mass"][m]))])
    assert len(free) > M // 2
    np.testing.assert_allclose(got[free], ex[free], rtol=1e-12, atol=0)


def test_eff_len_exact_matches_oracle(finished):
    st, fin, lens, nf = finished["st"], finished["fin"], finished["lens"], finished["nf"]
    ex = eff_len_exact(st["hist"], st["tot"], st["min_val"], lens, nf)
    assert np.all(np.abs(ex - fin["eff_len"]) <= 1e-12 * lens)
    dbl = eff_len_double(st["hist"], st["tot"], st["min_val"], lens, nf)
    assert np.all(np.abs(dbl - fin["eff_len"]) <= 1e-12 * lens)
    assert np.any(fin["eff_len"] < lens)


def test_clusters_from_roots_is_the_union_of_rank_partitions(finished):
    """the classes split round-robin over R ranks: the union of the per-rank partitions is the partition of all
    classes, the one normalize_alphas and the oracle project over"""
    M, classes = finished["M"], finished["classes"]
    full = class_roots(M, [t for t, _ in classes])
    for R in (1, 2, 3, 8):
        rows = np.stack([class_roots(M, [t for t, _ in classes[r::R]]) for r in range(R)])
        assert np.array_equal(clusters_from_roots(M, rows), full)
        assert np.array_equal(clusters_from_roots(M, rows[::-1]), full)
    # roots are the smallest members
    for r, mem in members(full).items():
        assert r == mem[0]


def test_exact_references_on_hand_cases():
    inf = np.inf
    # one cluster {0, 1, 2} with masses spanning +-700 and a member without mass; a singleton; a cluster of no mass
    mass = np.array([700.0, -700.0, inf, 3.0, inf, inf])
    root = np.array([0, 0, 0, 3, 4, 4], dtype=np.uint32)
    hits = np.array([5, 0, 5, 7, 2, 0], dtype=np.uint64)
    ex = project_exact(mass, hits, root)
    assert ex[0] == 10.0 and ex[2] == 0.0 and ex[3] == 7.0 and ex[4] == ex[5] == 0.0
    assert ex[1] == 0.0                                   # 10 exp(-1400) is below the range of double
    dbl = project_double(mass, hits, np.zeros(6, np.uint64), np.full(6, 100, np.uint64), root)
    np.testing.assert_allclose(dbl, ex, rtol=1e-15, atol=0)
    # effective lengths: the prior alone with fld_min = nf-1 takes minV = 1; a single bin at 5 gives cf = 5 from 5 on
    nf = 11
    hist = np.full(nf, np.log(0.375e-10))
    hist[5] = 0.0
    tot = float(np.log(np.exp(hist).sum()))
    lens = np.array([1, 4, 5, 6, 9, 10, 11, 100])
    eff, raw = eff_len_exact(hist, tot, 3, lens, nf, raw=True)
    assert eff[2] == 5.0 and raw[2] < 1.0                # len - cf = 0 < 1: the transcript length
    assert raw[3] == pytest.approx(1.0, abs=1e-6) and raw[-1] == pytest.approx(95.0, abs=1e-6)
    np.testing.assert_allclose(eff_len_double(hist, tot, 3, lens, nf), eff, rtol=1e-13)
    assert np.array_equal(eff_len_exact(hist, tot, nf - 1, [1], nf), [1.0])
