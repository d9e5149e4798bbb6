"""normalizeAlphas and the effective lengths on the GPU (k_cls_accumulate, k_union_roots, k_cluster_project,
k_online_correction, k_online_eff_len in salmon_b200/csrc/map.cu) against the references of tests/project_ref.py.

The seam is MapContext.project_global (sb_map_project_global): it takes the statistics of normalizeAlphas from the
host -- masses, counts, the fragment-length histogram and one cluster-root array per rank -- so the tests inject
cluster shapes, masses and bounds that synthetic reads never produce.  The last tests run the same kernels on
mapped reads: one context, and three contexts on one GPU whose partials are reduced by salmon_b200.dist."""
import math
import os

import numpy as np
import pytest

from project_ref import (class_roots, class_stats, clusters_from_roots, eff_len_exact, members, project_double,
                         project_exact)
from py_ref_map import LOG_EPSILON, fld_prior_tables
from salmon_b200._capi import Index, MapContext, map_default_params
from salmon_b200.synth import revcomp, synth_reads, synth_txome

pytestmark = pytest.mark.gpu

NF = 1001                                  # max_frag_len 1000 (the default)
M_SEAM = 70_000


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def random_txps(lengths, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 4, size=int(L), dtype=np.uint8) for L in lengths]


def global_stats(mass, hits, uniq, total, hist, tot, fld_min):
    """the dict MapContext.project_global takes (what salmon_b200.dist.reduce_partials returns)"""
    return dict(mass=np.asarray(mass, np.float64), fld_hist=np.asarray(hist, np.float64), fld_tot=float(tot),
                fld_prior_hist=np.asarray(hist, np.float64), fld_prior_tot=float(tot), fld_min=int(fld_min),
                unique_counts=np.asarray(uniq, np.uint64), total_counts=np.asarray(total, np.uint64),
                cluster_hits=np.asarray(hits, np.uint64), assigned=int(np.sum(hits)), compatible=0)


def prior_hist():
    pmf, _ = fld_prior_tables(250.0, 25.0, NF - 1)
    pmf = np.array(pmf)
    return pmf, float(np.log(np.exp(pmf).sum()))


# ---------------------------------------------------------------- injected clusters, masses and polytope bounds
MASS_KINDS = ("random", "inf_members", "span700", "equal", "dominant")


def _masses(rng, kind, n):
    if kind == "random":
        return rng.normal(0.0, 2.0, n) + rng.uniform(-50, 50)
    if kind == "inf_members":
        m = rng.normal(0.0, 2.0, n)
        m[rng.random(n) < 0.25] = np.inf
        m[rng.integers(0, n)] = 1.5
        return m
    if kind == "all_inf":
        return np.full(n, np.inf)
    if kind == "span700":                  # exp of the unshifted masses overflows and underflows
        m = rng.uniform(-700.0, 700.0, n)
        m[rng.permutation(n)[:2]] = (-700.0, 700.0)
        return m
    if kind == "equal":
        return np.full(n, 3.7)
    if kind == "dominant":
        m = rng.normal(0.0, 1.0, n)
        m[rng.integers(0, n)] += 40.0
        return m
    if kind == "flat":
        return rng.normal(0.0, 0.3, n)
    raise ValueError(kind)


def _shares(m, H):
    f = np.isfinite(m)
    s = np.zeros(len(m))
    if f.any():
        x = m[f] - m[f].max()
        s[f] = np.exp(x - np.log(np.exp(x).sum())) * H
    return s


def _cascade(rng, n, H, a=0.5):
    """shares and upper bounds of a cluster whose projection binds one more member per round: member k holds a
    fraction a of the mass the earlier members left, and its total lies between its values of rounds k and k+1"""
    sh, rem = [], 1.0
    while rem * H >= 50 and len(sh) < n - 1:
        sh.append(rem * a)
        rem -= rem * a
    K = len(sh)
    sh = np.array(sh + [rem / (n - K)] * (n - K)) * H
    total = np.full(n, 10 * H, dtype=np.int64)
    vals, bound = sh.copy(), np.zeros(n, bool)
    for k in range(K):
        lo = int(math.floor(0.7 * vals[k])) if k == 0 else int(math.ceil(prev[k] + 1e-6))
        if lo >= vals[k] - 1e-6:
            K = k
            break
        total[k] = lo
        vals[k] = lo
        bound[k] = True
        prev = vals.copy()
        vals[~bound] *= (H - vals[bound].sum()) / vals[~bound].sum()
    perm = rng.permutation(n)             # the binding members sit on arbitrary lanes
    return np.log(sh)[perm], total[perm], K


def _bounds(rng, kind, s, finite):
    """(unique, total) counts around the shares s: 'free' keeps every member inside, the others make some bind"""
    n = len(s)
    gen = kind != "free"
    uniq = np.floor(s * rng.uniform(0.0, 0.3 if gen else 0.9, n)).astype(np.int64)
    total = (np.ceil(s * rng.uniform(2.0 if gen else 1.1, 4.0 if gen else 3.0, n)) + 1).astype(np.int64)
    total[~finite] = rng.integers(0, 5, int((~finite).sum()))
    uniq = np.minimum(uniq, total)
    big = np.flatnonzero(s >= 5) if (s >= 5).any() else np.array([int(np.argmax(s))])
    if kind in ("upper", "both"):
        sel = rng.choice(big, size=max(1, len(big) // (5 if kind == "upper" else 7)), replace=False)
        total[sel] = np.floor(0.5 * s[sel])
        uniq[sel] = np.minimum(uniq[sel], total[sel])
    if kind in ("lower", "both"):
        pool = np.setdiff1d(np.arange(n), sel) if kind == "both" else np.arange(n)
        sel2 = rng.choice(pool, size=max(1, n // (5 if kind == "lower" else 7)), replace=False)
        uniq[sel2] = np.ceil(1.5 * s[sel2]) + 1
        total[sel2] = np.maximum(total[sel2], uniq[sel2] + 3)
    if kind == "all_bind":                 # the first round clamps every member: the unbound sum is 0
        order = np.argsort(s)
        lo_half, hi_half = order[: n // 2], order[n // 2:]
        total[hi_half] = np.floor(0.6 * s[hi_half])
        uniq[hi_half] = np.minimum(uniq[hi_half], total[hi_half])
        uniq[lo_half] = np.ceil(1.4 * s[lo_half]) + 1
        total[lo_half] = uniq[lo_half] + 10 * np.ceil(s[lo_half]) + 10
    return uniq, total


def seam_scenario(seed=2024):
    """M_SEAM transcripts in clusters of chosen shapes, with ids scattered over the index.  Returns the per-
    transcript statistics, the clusters (member ids, kind) and the link structure (edges, shape) of each cluster."""
    rng = np.random.default_rng(seed)
    plan = []
    for size in (31, 32, 33, 63, 64, 65, 1000):
        plan += [(size, mk, "free", "tree") for mk in MASS_KINDS]
        plan += [(size, "random", bk, "tree") for bk in ("upper", "lower", "both")]
        plan += [(size, "inf_members", "both", "tree"), (size, "flat", "all_bind", "tree"),
                 (size, "equal", "all_bind", "tree")]
    plan += [(64, "span700", "both", "tree"), (1000, "span700", "lower", "tree")]
    plan += [(100, "cascade", "cascade", "tree"), (130, "cascade", "cascade", "tree")]
    plan += [(50_000, "inf_members", "free", "tree"), (200, "random", "both", "star"), (300, "random", "free", "chain"),
             (257, "random", "upper", "chain"), (40, "random", "free", "star")]
    plan += [(5, "all_inf", "free", "tree")] * 3
    plan += [(2, "random", "free" if i % 3 else "upper", "tree") for i in range(1000)]
    used = sum(p[0] for p in plan)
    plan += [(1, "random", "free", "tree")] * (M_SEAM - used)
    ids = rng.permutation(M_SEAM)
    mass = np.full(M_SEAM, np.inf)
    hits = np.zeros(M_SEAM, np.uint64); uniq = np.zeros(M_SEAM, np.uint64); total = np.zeros(M_SEAM, np.uint64)
    clusters, pos = [], 0
    for size, mk, bk, shape in plan:
        mem = np.sort(ids[pos:pos + size]); pos += size
        H = int(rng.integers(10 * size + 10, 20 * size + 10)) if size < 50_000 else 900_000
        if bk == "cascade":
            H = 100_000
            m, tt, K = _cascade(rng, size, H)
            assert K >= 9
            uq = np.zeros(size, np.int64)
        else:
            if bk == "all_bind":
                H = 50 * size
            m = _masses(rng, mk, size)
            s = _shares(m, H)
            uq, tt = _bounds(rng, bk, s, np.isfinite(m))
            if tt.sum() < H:                 # a member inside its upper bound takes the missing total
                j = int(np.argmax(np.where(tt >= s, s, -1.0)))
                tt[j] += H - tt.sum() + 2
            while uq.sum() > H:              # and the members raised most above their share drop their unique count
                uq[int(np.argmax(uq - s))] = 0
            if size > 1 and bk != "free":    # real data: sum unique <= hits <= sum total
                assert uq.sum() <= H <= tt.sum(), (size, mk, bk)
            if size == 1:
                uq[:], tt[:] = (H, H) if rng.random() < 0.5 else (0, H + 3)
        mass[mem] = m
        hits[mem] = rng.multinomial(H, np.full(size, 1.0 / size)).astype(np.uint64)
        uniq[mem] = uq
        total[mem] = np.maximum(tt, uq)
        clusters.append(dict(mem=mem, mass_kind=mk, bound_kind=bk, shape=shape, H=H))
    return dict(mass=mass, hits=hits, uniq=uniq, total=total, clusters=clusters)


def rank_roots(sc, R, seed):
    """one cluster-root array per rank: the links of every cluster are spread over the ranks; a chain is connected
    only through all R arrays together (rank r links member t to t-1 for t = r mod R)"""
    rng = np.random.default_rng(seed)
    edges = [[] for _ in range(R)]
    for c in sc["clusters"]:
        mem = rng.permutation(c["mem"])
        n = len(mem)
        if n == 1:
            continue
        if c["shape"] == "chain":
            for t in range(1, n):
                edges[t % R].append((mem[t], mem[t - 1]))
        elif c["shape"] == "star":
            for t in range(1, n):
                edges[int(rng.integers(0, R))].append((mem[0], mem[t]))
        else:                                           # a random tree
            par = (rng.random(n - 1) * np.arange(1, n)).astype(np.int64)
            for t in range(1, n):
                edges[int(rng.integers(0, R))].append((mem[par[t - 1]], mem[t]))
    return np.stack([class_roots(M_SEAM, e) for e in edges])


@pytest.fixture(scope="module")
def seam():
    sc = seam_scenario()
    root = np.zeros(M_SEAM, np.uint32)
    for c in sc["clusters"]:
        root[c["mem"]] = c["mem"][0]
    sc["root"] = root
    sc["exact"] = project_exact(sc["mass"], sc["hits"], root)
    sc["double"] = project_double(sc["mass"], sc["hits"], sc["uniq"], sc["total"], root)
    idx = Index(random_txps([40] * M_SEAM, seed=77))
    ctx = MapContext(idx, map_default_params(), batch_cap=256, max_read_len=100)
    hist, tot = prior_hist()
    sc["g"] = global_stats(sc["mass"], sc["hits"], sc["uniq"], sc["total"], hist, tot, 200)
    yield sc, ctx
    ctx.close()
    idx.close()


def check_projection(sc, got):
    """free clusters against the exact projection, bound ones against the double reference"""
    ex, dbl, uq, tt = sc["exact"], sc["double"], sc["uniq"].astype(np.float64), sc["total"].astype(np.float64)
    n_bound = n_free = 0
    for c in sc["clusters"]:
        mem = c["mem"]
        g = got[mem]
        if c["mass_kind"] == "all_inf":                    # hits but no mass: exactly 0
            assert np.all(g == 0.0)
            continue
        if c["bound_kind"] == "free":
            assert np.all((ex[mem] >= uq[mem]) & (ex[mem] <= tt[mem]))
            rtol = 1e-12 if len(mem) <= 1024 else 1e-11
            np.testing.assert_allclose(g, ex[mem], rtol=rtol, atol=1e-300, err_msg=str(c["mass_kind"]))
            n_free += 1
            continue
        d = dbl[mem]
        at_u, at_t = d == uq[mem], d == tt[mem]
        assert (at_u | at_t).any()
        np.testing.assert_allclose(g, d, rtol=1e-10, atol=1e-290, err_msg=f"{c['bound_kind']} {len(mem)}")
        # members away from their bounds stay away: the bound set is not decided by rounding
        free = ~(at_u | at_t) & np.isfinite(sc["mass"][mem])
        assert np.all(np.minimum(np.abs(d[free] - uq[mem][free]), np.abs(d[free] - tt[mem][free])) > 1e-6 * d[free])
        assert np.array_equal(g == uq[mem], at_u) and np.array_equal(g == tt[mem], at_t), c["bound_kind"]
        assert abs(math.fsum(g) - c["H"]) <= 1e-12 * c["H"]
        n_bound += 1
    assert n_bound >= 30 and n_free >= 40


@pytest.mark.parametrize("R", [1, 2, 3, 8])
def test_projection_injected_clusters(seam, R):
    sc, ctx = seam
    roots_all = rank_roots(sc, R, seed=R)
    if R > 1:                       # the chains are split: no single rank array holds a whole chain
        chain = next(c for c in sc["clusters"] if c["shape"] == "chain")["mem"]
        assert all(len(set(roots_all[r][chain].tolist())) > 1 for r in range(R))
    assert np.array_equal(clusters_from_roots(M_SEAM, roots_all), sc["root"])
    res = ctx.project_global(sc["g"], roots_all)
    assert np.array_equal(res["unique_counts"], sc["uniq"]) and np.array_equal(res["total_counts"], sc["total"])
    check_projection(sc, res["projected_counts"])
    again = ctx.project_global(sc["g"], roots_all)
    assert np.array_equal(bits(again["projected_counts"]), bits(res["projected_counts"]))
    perm = ctx.project_global(sc["g"], roots_all[np.random.default_rng(R).permutation(R)[::-1]])
    assert np.array_equal(bits(perm["projected_counts"]), bits(res["projected_counts"]))
    assert np.array_equal(bits(perm["eff_len"]), bits(res["eff_len"]))


def test_projection_reference_sanity(seam):
    """the scenario does what it is meant to: the cascades need many rounds, the all-bind clusters bind every member
    in the first round, and large clusters carry bounds of several lanes"""
    sc, _ = seam
    uq, tt = sc["uniq"].astype(np.float64), sc["total"].astype(np.float64)
    for c in sc["clusters"]:
        mem = c["mem"]
        if c["bound_kind"] == "all_bind":
            s = _shares(sc["mass"][mem], c["H"])
            assert np.all((s > tt[mem]) | (s < uq[mem]))
        if c["bound_kind"] in ("upper", "lower", "both") and len(mem) > 32:
            d = sc["double"][mem]
            lanes = np.flatnonzero((d == uq[mem]) | (d == tt[mem])) % 32
            assert len(set(lanes.tolist())) > 1


# ---------------------------------------------------------------- effective lengths
EFF_LENS = np.array(list(range(1, 1100)) + [10_000], dtype=np.int64)


@pytest.fixture(scope="module")
def eff_ctx():
    idx = Index(random_txps(EFF_LENS, seed=78))
    ctx = MapContext(idx, map_default_params(), batch_cap=256, max_read_len=100)
    ctx_raw = MapContext(idx, map_default_params(no_eff_len_correction=1), batch_cap=256, max_read_len=100)
    yield ctx, ctx_raw
    ctx.close(); ctx_raw.close(); idx.close()


def histograms():
    prior, ptot = prior_hist()
    out = [("prior alone, minV = 1", prior, ptot, NF - 1)]
    single = np.full(NF, LOG_EPSILON - 50.0)
    single[300] = 0.0
    out.append(("single bin", single, float(np.log(np.exp(single).sum())), 300))
    rng = np.random.default_rng(5)
    obs = np.bincount(np.clip(np.round(rng.normal(260, 35, 20000)), 0, NF - 1).astype(int), minlength=NF).astype(float)
    real = np.log(np.exp(prior) + obs * 3.1)
    rtot = float(np.log(np.exp(real).sum()))
    out.append(("realistic", real, rtot, int(np.flatnonzero(obs)[0])))
    out.append(("realistic, fld_min 0", real, rtot, 0))
    out.append(("realistic, fld_min nf-2", real, rtot, NF - 2))
    tail = real.copy()
    tail[600:] = LOG_EPSILON
    out.append(("tail at LOG_EPSILON", tail, float(np.log(np.exp(tail).sum())), int(np.flatnonzero(obs)[0])))
    out.append(("shifted +40", real + 40.0, rtot + 40.0, int(np.flatnonzero(obs)[0])))
    out.append(("prior alone shifted +40", prior + 40.0, ptot + 40.0, NF - 1))
    return out


@pytest.mark.parametrize("case", range(8))
def test_effective_lengths(eff_ctx, case):
    ctx, ctx_raw = eff_ctx
    name, hist, tot, fld_min = histograms()[case]
    M = len(EFF_LENS)
    g = global_stats(np.full(M, np.inf), np.zeros(M), np.zeros(M), np.zeros(M), hist, tot, fld_min)
    got = ctx.project_global(g, np.arange(M, dtype=np.uint32)[None])["eff_len"]
    ex, raw = eff_len_exact(hist, tot, fld_min, EFF_LENS, NF, raw=True)
    L = EFF_LENS.astype(np.float64)
    # where the exact len - cf is within 1e-9 of 1.0, rounding decides the effLen < 1 branch: accept either
    near = np.abs(raw - 1.0) <= 1e-9
    ok = np.abs(got - ex) <= 1e-12 * L
    ok[near] |= (got[near] == L[near]) | (np.abs(got[near] - raw[near]) <= 1e-12 * L[near])
    assert ok.all(), (name, EFF_LENS[~ok][:10], got[~ok][:10], ex[~ok][:10])
    assert np.any(got < L) and np.any(got == L), name        # both branches of effLen < 1 are taken
    raw_res = ctx_raw.project_global(g, np.arange(M, dtype=np.uint32)[None])
    assert np.array_equal(raw_res["eff_len"], L)


# ---------------------------------------------------------------- mapped reads: a chain transcriptome
def chain_reads(seq, n, rng, L=100, sub=0.003):
    G = len(seq)
    fl = np.clip(np.round(rng.normal(250, 25, n)), 120, 400).astype(np.int64)
    pos = (rng.random(n) * (G - fl + 1)).astype(np.int64)
    left = np.stack([seq[p:p + L] for p in pos])
    right = np.stack([revcomp(seq[p + f - L:p + f]) for p, f in zip(pos, fl)])
    swap = rng.random(n) < 0.5
    left[swap], right[swap] = right[swap].copy(), left[swap].copy()
    for a in (left, right):
        m = rng.random(a.shape) < sub
        a[m] = (a[m] + rng.integers(1, 4, int(m.sum()))) % 4
    return left.astype(np.uint8), right.astype(np.uint8)


@pytest.fixture(scope="module")
def chain(oracle):
    """3000 windows of 500 bases at a stride of 150 of one sequence (neighbours share 350 bases), plus isolated
    genes; reads from the whole sequence link the windows into one cluster"""
    rng = np.random.default_rng(31)
    n_win, width, stride = 3000, 500, 150
    seq = rng.integers(0, 4, size=stride * (n_win - 1) + width, dtype=np.uint8)
    txps = [seq[i * stride:i * stride + width].copy() for i in range(n_win)]
    genes = [rng.integers(0, 4, size=900, dtype=np.uint8) for _ in range(6)]
    txps += genes
    l1, r1 = chain_reads(seq, 36_000, rng)
    parts = [chain_reads(gs, 400, rng) for gs in genes]
    left = np.concatenate([l1] + [p[0] for p in parts]); right = np.concatenate([r1] + [p[1] for p in parts])
    perm = rng.permutation(len(left))
    left, right = left[perm], right[perm]
    batches = [slice(0, 20_000), slice(20_000, len(left))]
    p = map_default_params()
    idx = Index(txps)
    on = oracle.Online(oracle.MapIndex(txps), oracle.map_params(), seed=42, mini_batch=5000)
    ctx = MapContext(idx, p, batch_cap=20_000, max_read_len=100)
    for s in batches:
        ctx.map_batch(left[s], right[s])
        on.batch(left[s], right[s])
    res = ctx.finish()
    part = ctx.partial()
    fin = on.finish(res["off"], res["tids"], res["counts"])
    yield dict(txps=txps, idx=idx, ctx=ctx, res=res, part=part, fin=fin, left=left, right=right, batches=batches,
               lens=np.array([len(t) for t in txps]))
    ctx.close()


def result_classes(res):
    off = res["off"].astype(np.int64)
    return [(res["tids"][off[c]:off[c + 1]].tolist(), int(res["counts"][c])) for c in range(len(res["counts"]))]


def check_free_exact(root, mass, hits, uniq, total, got):
    ex = project_exact(mass, hits, root)
    n = 0
    for r, mem in members(root).items():
        if np.all((ex[mem] >= uniq[mem]) & (ex[mem] <= total[mem])) and np.any(ex[mem] > 0):
            np.testing.assert_allclose(got[mem], ex[mem], rtol=1e-12 if len(mem) <= 1024 else 1e-11, atol=1e-300)
            n += 1
    return n


def test_chain_clusters_on_mapped_reads(chain):
    """k_cls_accumulate under contention: thousands of classes hook into one cluster"""
    res, part, fin = chain["res"], chain["part"], chain["fin"]
    M = len(chain["txps"])
    classes = result_classes(res)
    root = class_roots(M, [t for t, _ in classes])
    assert np.array_equal(part["cluster_root"], root)
    assert max(len(m) for m in members(root).values()) >= 2900
    hits, uniq, total = class_stats(M, classes)
    assert np.array_equal(part["cluster_hits"], hits)
    assert np.array_equal(part["unique_counts"], uniq) and np.array_equal(res["unique_counts"], uniq)
    assert np.array_equal(part["total_counts"], total) and np.array_equal(res["total_counts"], total)
    assert np.array_equal(uniq, fin["unique_counts"]) and np.array_equal(total, fin["total_counts"])
    np.testing.assert_allclose(res["projected_counts"], fin["projected_counts"], rtol=1e-9, atol=1e-9)
    assert check_free_exact(root, part["mass"], hits, uniq, total, res["projected_counts"]) >= 1
    assert np.array_equal(bits(res["eff_len"]), bits(fin["eff_len"]))


def test_single_rank_identity(chain):
    """a context that has not burned in: projecting its own partial gives finish()'s bits"""
    res, part = chain["res"], chain["part"]
    got = chain["ctx"].project_global(part, part["cluster_root"][None])
    assert np.array_equal(bits(got["projected_counts"]), bits(res["projected_counts"]))
    assert np.array_equal(bits(got["eff_len"]), bits(res["eff_len"]))
    assert np.array_equal(got["unique_counts"], res["unique_counts"])


def test_single_rank_after_burn_in():
    """after burn-in project_global recomputes the effective lengths from the final fragment-length distribution
    (the multi-rank behaviour) where finish() keeps those of burn-in; the projected counts are unchanged"""
    txps, _ = synth_txome(seed=8, n_genes=60)
    left, right, _ = synth_reads(txps, seed=9, n=6000)
    p = map_default_params(num_pre_burnin=1000, num_burnin=2500)
    idx = Index(txps)
    ctx = MapContext(idx, p, batch_cap=3000, max_read_len=100)
    for s in (slice(0, 3000), slice(3000, 6000)):
        ctx.map_batch(left[s], right[s])
    res = ctx.finish()
    part = ctx.partial()
    assert ctx.online_state()["burned_in"] == 1
    got = ctx.project_global(part, part["cluster_root"][None])
    assert np.array_equal(bits(got["projected_counts"]), bits(res["projected_counts"]))
    lens = np.array([len(t) for t in txps])
    ex = eff_len_exact(part["fld_hist"], part["fld_tot"], part["fld_min"], lens, NF)
    assert np.all(np.abs(got["eff_len"] - ex) <= 1e-12 * lens)
    # the distribution stops changing at burn-in (fragment lengths are only sampled before it), so on one rank
    # the recomputed lengths are finish()'s
    assert np.array_equal(bits(got["eff_len"]), bits(res["eff_len"]))
    ctx.close()


def _reduce_worker(rank, world, port, part, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    from salmon_b200.dist import reduce_partials
    dist.init_process_group("gloo", rank=rank, world_size=world)
    g, roots = reduce_partials(part, dist, "cpu")
    q.put((rank, g, roots))
    dist.destroy_process_group()


def reduce_in_gloo(parts):
    import torch.multiprocessing as mp
    world = len(parts)
    mpc = mp.get_context("spawn")
    q = mpc.Queue()
    port = 33500 + (os.getpid() % 2000)
    procs = [mpc.Process(target=_reduce_worker, args=(r, world, port, parts[r], q)) for r in range(world)]
    for p in procs:
        p.start()
    got =[q.get(timeout=300) for _ in range(world)]
    for p in procs:
        p.join(60)
    got.sort(key=lambda x: x[0])
    return [(g, roots) for _, g, roots in got]


def test_three_ranks_on_one_gpu(chain):
    """one read set's batches round-robin over three contexts (the third gets none), the partials reduced by
    salmon_b200.dist in gloo workers, then project_global on every context"""
    txps, left, right, batches = chain["txps"], chain["left"], chain["right"], chain["batches"]
    M, R = len(txps), 3
    ctxs = [MapContext(chain["idx"], map_default_params(), batch_cap=20_000, max_read_len=100) for _ in range(R)]
    for b, s in enumerate(batches):
        ctxs[b % R].map_batch(left[s], right[s])
    results = [c.finish() for c in ctxs]
    parts = [c.partial() for c in ctxs]
    reduced = reduce_in_gloo(parts)
    g, roots_all = reduced[0]
    for g2, r2 in reduced[1:]:
        assert np.array_equal(r2, roots_all) and np.array_equal(bits(g2["mass"]), bits(g["mass"]))
    outs = [c.project_global(g, roots_all) for c in ctxs]
    for o in outs[1:]:
        for k in ("projected_counts", "eff_len"):
            assert np.array_equal(bits(o[k]), bits(outs[0][k])), k
        assert np.array_equal(o["unique_counts"], outs[0]["unique_counts"])
    got = outs[0]
    classes = sum((result_classes(r) for r in results), [])
    root = class_roots(M, [t for t, _ in classes])
    assert np.array_equal(clusters_from_roots(M, roots_all), root)
    assert max(len(m) for m in members(root).values()) >= 2900
    hits, uniq, total = class_stats(M, classes)
    assert np.array_equal(g["cluster_hits"], hits)
    assert np.array_equal(got["unique_counts"], uniq) and np.array_equal(got["total_counts"], total)
    dbl = project_double(g["mass"], hits, uniq, total, root)
    np.testing.assert_allclose(got["projected_counts"], dbl, rtol=1e-10, atol=1e-12)
    assert check_free_exact(root, g["mass"], hits, uniq, total, got["projected_counts"]) >= 1
    lens = chain["lens"]
    ex = eff_len_exact(g["fld_hist"], g["fld_tot"], g["fld_min"], lens, NF)
    assert np.all(np.abs(got["eff_len"] - ex) <= 1e-12 * lens)
    for c in ctxs:
        c.close()
