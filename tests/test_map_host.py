"""CPU tests of Stage A: the product's per-read logic (map_core.h compiled for the host) against the
independent oracle -- bit-exact alignments, scores, probabilities, labels and weights."""
import numpy as np
import pytest

from salmon_b200._capi import Index, map_default_params
from salmon_b200.synth import synth_reads, synth_txome


def compare(a, b, cap, binned=True):
    """binned=False (range_bins 0): a label is its n_aln transcripts, the bin slots after them are not written"""
    assert np.array_equal(a["n_aln"], b["n_aln"])
    n = a["n_aln"].shape[0]
    m = np.arange(cap)[None, :] < a["n_aln"][:, None]
    for k in ("tid", "score", "pos", "mate_pos", "flags", "flen"):
        assert np.array_equal(a[k][m], b[k][m]), k
    assert np.array_equal(a["prob"][m].view(np.uint64), b["prob"][m].view(np.uint64))
    assert np.array_equal(a["weight"][m].view(np.uint64), b["weight"][m].view(np.uint64))
    m2 = np.arange(2 * cap)[None, :] < (2 if binned else 1) * a["n_aln"][:, None]
    assert np.array_equal(a["label"][m2], b["label"][m2])


def run_both(oracle, txps, left, right, frag_counter=0, **over):
    import hostmap_lib
    idx = Index(txps, k=over.get("k", 31))
    p = map_default_params(**over)
    got = hostmap_lib.map_reads(idx, p, left, right, frag_counter)
    oix = oracle.MapIndex(txps, k=over.get("k", 31))
    ref = oracle.map_reads(oix, oracle.map_params(**over), left, right, frag_counter)
    assert idx.info()["n_kmers"] == oix.n_kmers
    compare(got, ref, p.max_read_occ)
    for k in ("lookups", "postings", "seeds", "kept", "label_entries", "mapped"):
        assert got["counters"][k] == ref["counters"][k], k
    return got, ref


@pytest.mark.parametrize("frag_counter", [0, 6000, 6_000_000])
def test_host_logic_matches_oracle(oracle, frag_counter):
    txps, _ = synth_txome(seed=3, n_genes=150)
    left, right, truth = synth_reads(txps, seed=5, n=1500, indel_rate=0.002)
    got, ref = run_both(oracle, txps, left, right, frag_counter)
    na = got["n_aln"]
    ok = sum(1 for i in range(len(na)) if truth["tid"][i] >= 0 and truth["tid"][i] in got["tid"][i, :na[i]])
    assert ok >= 0.97 * (truth["tid"] >= 0).sum()
    assert ((truth["tid"] < 0) & (na > 0)).sum() == 0


def test_repeats_ns_short_transcripts_and_caps(oracle):
    rng = np.random.default_rng(9)
    unit = rng.integers(0, 4, size=400, dtype=np.uint8)
    txps = [unit.copy() for _ in range(90)]                 # 90 identical transcripts: > MAXCAND candidates
    txps += [np.concatenate([unit[:200], rng.integers(0, 4, size=150, dtype=np.uint8)]) for _ in range(130)]  # > maxReadOcc
    txps += [rng.integers(0, 4, size=20, dtype=np.uint8)]    # shorter than k
    withn = rng.integers(0, 4, size=500, dtype=np.uint8); withn[100:103] = 4
    txps += [withn]
    left, right, _ = synth_reads(txps, seed=2, n=400, read_len=75, frag_mean=180, frag_sd=15, random_frac=0.1)
    left[5, 10] = 4; right[7, 60] = 4                        # N in reads
    run_both(oracle, txps, left, right)
    run_both(oracle, txps, left, right, max_read_occ=50, max_occs_per_hit=64, stride=3, range_bins=0)


def test_decoys_and_hard_filter(oracle):
    txps, _ = synth_txome(seed=8, n_genes=60)
    n_real = len(txps) - 20
    left, right, _ = synth_reads(txps, seed=1, n=600)
    run_both(oracle, txps, left, right, first_decoy=n_real)
    run_both(oracle, txps, left, right, hard_filter=1)
    run_both(oracle, txps, left, right, first_decoy=n_real, decoy_threshold=0.9, min_score_fraction=0.8)


def test_detmath_close_to_libm():
    import ctypes as C, math, os, subprocess, tempfile
    src = r'''
    #include "sb_detmath.h"
    double e(double x) { return sbm_det_exp(x); }
    double l(double x) { return sbm_det_log(x); }
    '''
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        so = os.path.join(d, "t.so")
        subprocess.check_call(["/usr/bin/gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(root, "include"),
                               "-o", so, os.path.join(d, "t.c")])
        lib = C.CDLL(so)
        lib.e.restype = lib.l.restype = C.c_double
        lib.e.argtypes = lib.l.argtypes = [C.c_double]
        rng = np.random.default_rng(0)
        for x in rng.uniform(-700, 700, size=20000):
            assert abs(lib.e(x) - math.exp(x)) <= 2.3e-16 * math.exp(x)
        for x in np.exp(rng.uniform(-700, 700, size=20000)):
            assert abs(lib.l(x) - math.log(x)) <= 2.3e-16 * max(abs(math.log(x)), 1e-300) + 1e-320
        assert lib.e(0.0) == 1.0 and lib.l(1.0) == 0.0 and lib.e(-lib.l(2.0)) == 0.5


def test_decoys_host_logic_matches_oracle(oracle):
    """Decoy-aware mapping (BASELINE configs[3]; updateRefMappings / filterAndCollectAlignments with firstDecoyIndex,
    SalmonMappingUtils.hpp:225-405): decoy sequences that carry the transcripts' exons plus flanking sequence come last;
    no alignment to a decoy is ever reported, and a fragment that maps better to a decoy than to any transcript is
    dropped.  Host logic bit-exact against the oracle."""
    rng = np.random.default_rng(17)
    txps, _ = synth_txome(seed=8, n_genes=40)
    M = len(txps)
    # "genome" decoys: a few transcripts embedded in random flanks, and intron-like pieces that only exist in the decoy
    decoys = []
    for g in range(6):
        parts = [rng.integers(0, 4, size=300, dtype=np.uint8)]
        for t in rng.choice(M, size=5, replace=False):
            parts += [txps[t], rng.integers(0, 4, size=200, dtype=np.uint8)]
        decoys.append(np.concatenate(parts))
    allseq = txps + decoys
    l1, r1, _ = synth_reads(txps, seed=18, n=2000)
    l2, r2, _ = synth_reads(decoys, seed=19, n=1000, expressed_frac=1.0)      # fragments that come from the decoys
    left, right = np.concatenate([l1, l2]), np.concatenate([r1, r2])
    got, ref = run_both(oracle, allseq, left, right, first_decoy=M)
    na = got["n_aln"]
    sel = np.arange(got["tid"].shape[1])[None, :] < na[:, None]
    assert (got["tid"][sel] < M).all()                                   # decoys are never reported
    # decoy fragments: those lying in decoy-only sequence are dropped, those inside an embedded transcript map to it
    assert (na[2000:] == 0).sum() > 100 and (na[2000:] > 0).sum() > 100
    assert (na[:2000] > 0).mean() > 0.9
    # and without the decoy boundary the same reads do get decoy alignments
    got2, _ = run_both(oracle, allseq, left, right)
    assert (got2["tid"][np.arange(got2["tid"].shape[1])[None, :] < got2["n_aln"][:, None]] >= M).any()
    assert got2["counters"]["mapped"] > got["counters"]["mapped"]


# indel lengths planted in mates: each band of the sweeps (0, 1, 2, 3, 7, 8, 14, 15) has a gap just inside and one just
# outside its reach, and the longest ones lie beyond every band
INDEL_LENS = (1, 2, 3, 5, 8, 9, 12, 15, 16, 20, 24)
BANDS = (0, 1, 2, 3, 7, 8, 14, 15)
# (ma, mp, go, ge): the default, and sets where m * (ma - mp) = go + ge has an integer solution m (1, 2, 1 mismatches
# for the 2nd to 4th), i.e. an ungapped alignment with m mismatches lands exactly on the ungapped shortcut's bound
SCORES = ((2, -4, 6, 2), (1, -1, 1, 1), (2, -2, 6, 2), (3, -3, 4, 2), (2, -4, 0, 1))
_COMP5 = np.array([3, 2, 1, 0, 4], dtype=np.uint8)


def tie_mismatches(ma, mp, go, ge):
    """m with m * (ma - mp) == go + ge, or None"""
    return (go + ge) // (ma - mp) if (go + ge) % (ma - mp) == 0 else None


def plant_mate(src, L, rng, d=0, m=0):
    """an L-base mate read from src (its source on the mate's own strand, continuing at least d bases past the mate's
    end): with d > 0 one deletion or insertion of d bases at a random position or within 5 bases of either end; with
    m > 0 exactly m substitutions at distinct positions; else the plain bases"""
    src = np.asarray(src, dtype=np.uint8)
    if d:
        w = int(rng.integers(3))
        p = int(rng.integers(1, L)) if w == 0 else (int(rng.integers(1, 6)) if w == 1 else L - int(rng.integers(1, 6)))
        if rng.random() < 0.5:       # deletion: the mate skips d reference bases
            out = np.concatenate([src[:p], src[p + d:L + d]])
        else:                        # insertion of d random bases
            out = np.concatenate([src[:p], rng.integers(0, 4, d, dtype=np.uint8), src[p:max(p, L - d)]])[:L]
    else:
        out = src[:L].copy()
    if m:
        q = rng.choice(L, m, replace=False)
        out[q] = (out[q] + rng.integers(1, 4, m, dtype=np.uint8)) % 4
    assert out.shape[0] == L
    return out.astype(np.uint8)


def planted_pairs(txps, rng, n, L, frag_mean, frag_sd=20.0, indel_frac=0.4, subs=(), sub_frac=0.0):
    """n IU pairs from the transcripts of at least L + 48 bases; each mate independently carries one indel (length from
    INDEL_LENS) with probability indel_frac, else exactly m substitutions (m from subs) with probability sub_frac"""
    D = max(INDEL_LENS)
    ok = np.flatnonzero(np.array([len(t) for t in txps]) >= L + 2 * D)
    if len(ok) == 0:
        raise ValueError("no transcript long enough")
    left = np.zeros((n, L), np.uint8)
    right = np.zeros((n, L), np.uint8)
    for i in range(n):
        t = txps[int(rng.choice(ok))]
        tl = len(t)
        fl = int(np.clip(round(rng.normal(frag_mean, frag_sd)), L, tl - 2 * D))
        pos = int(rng.integers(D, tl - D - fl + 1))
        mates = []
        for src in (t[pos:pos + L + D], _COMP5[t[pos + fl - L - D:pos + fl][::-1]]):
            u = rng.random()
            d = int(rng.choice(INDEL_LENS)) if u < indel_frac else 0
            m = int(rng.choice(subs)) if (subs and indel_frac <= u < indel_frac + sub_frac) else 0
            mates.append(plant_mate(src, L, rng, d, m))
        if rng.random() < 0.5:
            mates.reverse()
        left[i], right[i] = mates
    return left, right


def fuzz_trials(master_seed, n_trials, read_lens=(35, 50, 75, 100, 125, 150, 200, 256)):
    """Randomised mapping trials: adversarial transcriptomes (shared blocks, homopolymers, N, short references), error
    rates up to 5 % / 2 % one-base indels, planted indels of up to 24 bases, and random settings of stride, maxReadOcc,
    maxOccsPerHit, range bins, hard filter, minScoreFraction, consensus fraction, k, band, scores, first decoy,
    fragLenDistMax and the fragment counter.  Yields dict(txps, left, right, L, over, frag_counter); the stride keeps
    (L - k) / stride + 2 within the 64 seed positions a GPU context takes."""
    rng = np.random.default_rng(master_seed)
    for trial in range(n_trials):
        seed = int(rng.integers(1, 1 << 30))
        if trial % 4 == 0:
            txps, _ = synth_txome(seed=seed, n_genes=int(rng.integers(5, 40)))
        else:
            r = np.random.default_rng(seed)
            unit = r.integers(0, 4, size=int(r.integers(60, 300)), dtype=np.uint8)
            txps = []
            for _ in range(int(r.integers(3, 40))):
                parts = []
                for _ in range(int(r.integers(1, 5))):
                    c = r.random()
                    if c < 0.4:
                        parts.append(unit[: int(r.integers(31, len(unit) + 1))])
                    elif c < 0.5:
                        parts.append(np.full(int(r.integers(5, 60)), int(r.integers(0, 4)), dtype=np.uint8))
                    else:
                        parts.append(r.integers(0, 4, size=int(r.integers(10, 400)), dtype=np.uint8))
                t = np.concatenate(parts)
                if r.random() < 0.2:
                    t[int(r.integers(0, len(t)))] = 4
                txps.append(t)
        L = int(rng.choice(read_lens))
        if max(len(t) for t in txps) < max(150, L + 60):
            txps.append(np.random.default_rng(seed + 2).integers(0, 4, size=max(400, 2 * L + 60), dtype=np.uint8))
        fm = float(rng.choice([max(L + 20, 120), max(250, L + 40)]))
        try:
            left, right, _ = synth_reads(txps, seed=seed + 1, n=int(rng.integers(50, 300)), read_len=L, frag_mean=fm,
                                         frag_sd=float(rng.choice([5, 25])), sub_rate=float(rng.choice([0.0, 0.01, 0.05])),
                                         indel_rate=float(rng.choice([0.0, 0.003, 0.02])), random_frac=0.1)
        except Exception:  # noqa: BLE001  (the simulator refuses transcriptomes shorter than its fragments)
            continue
        if rng.random() < 0.5:    # a third of the pairs replaced by pairs with planted multi-base indels
            sel = rng.choice(left.shape[0], left.shape[0] // 3, replace=False)
            try:
                left[sel], right[sel] = planted_pairs(txps, np.random.default_rng(seed + 3), len(sel), L, fm,
                                                      indel_frac=0.7)
            except ValueError:
                pass
        if rng.random() < 0.3:
            left[rng.integers(0, left.shape[0]), rng.integers(0, L)] = 4
        over = {}
        for key, p_use, choices in (("stride", 0.5, [1, 2, 3, 4, 7]), ("max_read_occ", 0.4, [1, 2, 5, 50]),
                                    ("max_occs_per_hit", 0.4, [1, 3, 16, 200]), ("range_bins", 0.4, [0, 1, 8]),
                                    ("hard_filter", 0.3, [1]), ("min_score_fraction", 0.3, [0.3, 0.8, 0.95]),
                                    ("consensus_frac", 0.3, [0.3, 0.9, 1.0]), ("k", 0.3, [15, 21, 25]),
                                    ("band", 0.4, list(BANDS)), ("max_frag_len", 0.3, [200, 400])):
            if rng.random() < p_use:
                v = rng.choice(choices)
                over[key] = float(v) if isinstance(choices[0], float) else int(v)
        if rng.random() < 0.3:
            over.update(zip(("ma", "mp", "go", "ge"), SCORES[int(rng.integers(len(SCORES)))]))
        if rng.random() < 0.2:
            over["first_decoy"] = max(1, len(txps) - int(rng.integers(1, 4)))
        k, stride = over.get("k", 31), over.get("stride", 4)
        while (L - k) // stride + 2 > 64:
            stride += 1
        if stride != over.get("stride", 4):
            over["stride"] = stride
        yield dict(txps=txps, left=left, right=right, L=L, over=over,
                   frag_counter=int(rng.choice([0, 0, 6000, 6_000_000])))


@pytest.mark.parametrize("master_seed", [1, 4])
def test_fuzz_host_logic_against_oracle(oracle, master_seed):
    """Randomised parity (fuzz_trials): the product's per-read logic stays bit-exact with the oracle, in all three
    regimes of the fragment counter."""
    done = 0
    for t in fuzz_trials(master_seed, 70):
        run_both(oracle, t["txps"], t["left"], t["right"], frag_counter=t["frag_counter"], **t["over"])
        done += 1
    assert done >= 40


JOIN_VARIANTS = [dict(), dict(allow_dovetail=1), dict(allow_orphans=0), dict(pre_merge_thresh=1.0, post_merge_thresh=1.0, orphan_thresh=1.0),
                 dict(pre_merge_thresh=0.0, post_merge_thresh=0.0, orphan_thresh=0.0, consensus_frac=0.3),
                 dict(post_merge_thresh=0.5, orphan_thresh=0.6, allow_dovetail=1)]


def join_reads(seed=71, n=6000):
    """reads that exercise the join policy: normal pairs, pairs whose mates dovetail (fragment shorter than a read), and
    pairs with one unmappable mate (orphans)"""
    txps, _ = synth_txome(seed=seed, n_genes=120)
    left, right, truth = synth_reads(txps, seed=seed + 1, n=n, indel_rate=0.001)
    rng = np.random.default_rng(seed + 2)
    L = left.shape[1]
    comp = np.array([3, 2, 1, 0, 4], dtype=np.uint8)
    for i in rng.choice(n, n // 6, replace=False):          # dovetail: the right mate starts upstream of the left mate
        t = txps[int(rng.integers(len(txps)))]
        if len(t) < L + 40:
            continue
        s = int(rng.integers(20, len(t) - L - 10))
        left[i] = t[s:s + L]
        right[i] = comp[t[s - 15:s - 15 + L][::-1]]
    for i in rng.choice(n, n // 8, replace=False):          # orphan: one mate is noise
        (left if rng.random() < 0.5 else right)[i] = rng.integers(0, 4, L).astype(np.uint8)
    return txps, left, right


@pytest.mark.parametrize("over", JOIN_VARIANTS)
def test_join_policy_knobs_host_logic_vs_oracle(oracle, over):
    """MAPSPEC step 4 with the knobs salmon exposes (preMerge / postMerge / orphan chain sub-thresholds, allowDovetail,
    discardOrphans; SalmonMappingUtils.hpp:208-220): the product's per-read logic against the oracle's independent
    restatement, plus what each knob must do."""
    txps, left, right = join_reads()
    got, ref = run_both(oracle, txps, left, right, **over)
    status = (got["flags"] >> 2) & 3
    valid = np.arange(got["flags"].shape[1])[None, :] < got["n_aln"][:, None]
    n_orphan_reads = int(((status != 0) & valid).any(axis=1).sum())
    if over.get("allow_orphans", 1) == 0:
        assert n_orphan_reads == 0
    else:
        assert n_orphan_reads > 100
    test_join_policy_knobs_host_logic_vs_oracle.mapped[tuple(sorted(over.items()))] = int((got["n_aln"] > 0).sum())


test_join_policy_knobs_host_logic_vs_oracle.mapped = {}


def test_join_policy_monotonicity(oracle):
    """dovetails only map as pairs when allowed; discarding orphans only loses reads; looser thresholds only add alignments"""
    txps, left, right = join_reads()
    oix = oracle.MapIndex(txps)
    run = lambda **o: oracle.map_reads(oix, oracle.map_params(**o), left, right, 0)
    base, dove, noorph = run(), run(allow_dovetail=1), run(allow_orphans=0)
    loose = run(pre_merge_thresh=0.0, post_merge_thresh=0.0, orphan_thresh=0.0)
    strict = run(pre_merge_thresh=1.0, post_merge_thresh=1.0, orphan_thresh=1.0)
    paired = lambda m: int((((m["flags"] >> 2) & 3) == 0)[np.arange(m["flags"].shape[1])[None, :] < m["n_aln"][:, None]].sum())
    assert paired(dove) > paired(base) + 300                 # the planted dovetails become concordant pairs
    assert (noorph["n_aln"] > 0).sum() < (base["n_aln"] > 0).sum() - 300
    assert int(loose["n_aln"].sum()) >= int(base["n_aln"].sum()) >= int(strict["n_aln"].sum())
    assert int(loose["n_aln"].sum()) > int(strict["n_aln"].sum())


LIB = dict(IU=0, ISF=1, ISR=2, U=3, SF=4, SR=5)


def stranded_reads(seed=81, n=5000, flip_frac=0.4):
    """pairs drawn as synth_reads draws them (the fragment's first mate is the left one, i.e. ISF-like when the fragment
    is on the forward strand) with a known fraction of pairs swapped (left <-> right), which flips their strandedness"""
    txps, _ = synth_txome(seed=seed, n_genes=100)
    left, right, truth = synth_reads(txps, seed=seed + 1, n=n)
    rng = np.random.default_rng(seed + 2)
    flip = rng.random(n) < flip_frac
    l2, r2 = left.copy(), right.copy()
    l2[flip], r2[flip] = right[flip], left[flip]
    return txps, l2, r2, flip


@pytest.mark.parametrize("lib", ["IU", "ISF", "ISR"])
def test_paired_library_types_host_logic_vs_oracle(oracle, lib):
    """expected library format (row a1): mappings incompatible with it are ignored (SalmonQuantify.cpp:1467-1521;
    salmon::utils::compatibleHit, SalmonUtils.cpp:193-298) -- product logic vs the oracle, and what the types mean"""
    txps, left, right, flip = stranded_reads()
    got, ref = run_both(oracle, txps, left, right, lib_type=LIB[lib])
    cap = got["flags"].shape[1]
    valid = np.arange(cap)[None, :] < got["n_aln"][:, None]
    st = (got["flags"] >> 2) & 3
    lfw = (got["flags"] & 1) == 1
    pair = valid & (st == 0)
    if lib == "ISF":
        assert lfw[pair].all()
    if lib == "ISR":
        assert (~lfw[pair]).all()
    test_paired_library_types_host_logic_vs_oracle.mapped[lib] = int((got["n_aln"] > 0).sum())
    m = test_paired_library_types_host_logic_vs_oracle.mapped
    if len(m) == 3:       # a stranded type keeps one orientation: together they cover what IU maps
        assert m["ISF"] < m["IU"] and m["ISR"] < m["IU"] and m["ISF"] + m["ISR"] >= m["IU"]


test_paired_library_types_host_logic_vs_oracle.mapped = {}


@pytest.mark.parametrize("lib", ["U", "SF", "SR"])
def test_single_end_library_types_host_logic_vs_oracle(oracle, lib):
    """single-end reads = pairs whose second mate is absent (all N): every mapping is a left orphan; SF / SR keep one strand"""
    txps, left, right, flip = stranded_reads(seed=91)
    absent = np.full_like(right, 4)
    got, ref = run_both(oracle, txps, left, absent, lib_type=LIB[lib], pre_merge_thresh=1.0)
    cap = got["flags"].shape[1]
    valid = np.arange(cap)[None, :] < got["n_aln"][:, None]
    assert ((((got["flags"] >> 2) & 3) == 1) | ~valid).all()
    fw = (got["flags"] & 1) == 1
    if lib == "SF":
        assert fw[valid].all()
    if lib == "SR":
        assert (~fw[valid]).all()
    assert (got["n_aln"] > 0).sum() > (1500 if lib != "U" else 4000)
