"""The GPU mapping path (k_seed_chain_w, k_dp_classify, k_dp_pair, k_dp_general, k_assign) against the oracle bit for
bit at non-default mapping options: band, k, stride, read length, scores, minScoreFraction, the ungapped shortcut, the
fragment-length model and the filters.  The workload plants indels of up to 24 bases (so an alignment needs a diagonal
far from its candidate's, where a wrong band edge shows), mates with exactly the mismatches that land on the shortcut's
bound, mates hanging over transcript ends, N in mates and transcripts, and random pairs."""
import numpy as np
import pytest

import softclip_ref as S
from salmon_b200._capi import Index, MapContext, SalmonB200Error, map_default_params
from salmon_b200.synth import revcomp, synth_txome
from test_map_gpu import bits, check_classes, check_state
from test_map_host import BANDS, SCORES, compare, fuzz_trials, planted_pairs, tie_mismatches

pytestmark = pytest.mark.gpu
CTR = ("lookups", "postings", "seeds", "kept", "label_entries", "mapped")


def workload(seed, n, L, n_genes=40, subs=(), sub_frac=0.0, frac_over=0.08, frac_random=0.05, frac_n=0.03):
    """n pairs of L-base mates: planted indels in 45 % of the mates (and exactly m substitutions, m from subs, in a
    fraction sub_frac), pairs hanging over a transcript end (edge list), mates with an N and transcripts with N (byte
    path), random pairs"""
    rng = np.random.default_rng(seed)
    txps, _ = synth_txome(seed=seed, n_genes=n_genes)
    left, right = planted_pairs(txps, rng, n, L, frag_mean=2 * L + 50, indel_frac=0.45, subs=subs, sub_frac=sub_frac)
    n_over, n_rand = int(n * frac_over), int(n * frac_random)
    rows = rng.permutation(n)
    ol, orr, _, _ = S.overhang_pairs(txps, rng, n_over, L=L)
    left[rows[:n_over]], right[rows[:n_over]] = ol, orr
    r = rows[n_over:n_over + n_rand]
    left[r] = rng.integers(0, 4, (len(r), L), dtype=np.uint8)
    right[r] = rng.integers(0, 4, (len(r), L), dtype=np.uint8)
    for m in (left, right):
        sel = np.flatnonzero(rng.random(n) < frac_n)
        m[sel, rng.integers(0, L, len(sel))] = 4
    txps = [t.copy() for t in txps]          # N placed after the reads were drawn
    for t in rng.choice(len(txps), max(1, len(txps) // 10), replace=False):
        txps[t][rng.integers(0, len(txps[t]), 2)] = 4
    return txps, np.ascontiguousarray(left), np.ascontiguousarray(right)


def oracle_for(oracle, txps, k=31):
    """-> run(mode, left, right, **over): oracle.map_reads for mode 0, the soft-clip oracle for modes 1 and 2"""
    oix, six = oracle.MapIndex(txps, k=k), S.OracleIndex(txps, k=k)

    def run(mode, left, right, **over):
        p = oracle.map_params(k=k, **over)
        return oracle.map_reads(oix, p, left, right, 0) if mode == 0 else S.oracle_map(six, p, mode, 0, left, right)
    return run


def gpu_map(idx, left, right, opts=None, cap_len=None, **over):
    p = map_default_params(**{"k": idx.k, **over})
    ctx = MapContext(idx, p, batch_cap=max(1024, left.shape[0]), max_read_len=cap_len or left.shape[1])
    for key, v in (opts or {}).items():
        ctx.set_option(key, v)
    st = ctx.map_batch(left, right)
    got = ctx.last_alignments()
    ctx.close()
    return got, st


def check(got, st, ref, cap, what, binned=True):
    try:
        compare(got, ref, cap, binned)
        for key in CTR:
            assert getattr(st, key) == ref["counters"][key], key
    except AssertionError as e:
        raise AssertionError(f"{what}: {e}") from None


def differs(a, b):
    if not np.array_equal(a["n_aln"], b["n_aln"]):
        return True
    m = np.arange(a["score"].shape[1])[None, :] < a["n_aln"][:, None]
    return not np.array_equal(a["score"][m], b["score"][m])


def npos(L, k, stride):
    """seed positions per mate (map.cu): up to 32 run k_seed_chain_w<*, 1>, more <*, 2>"""
    return (L - k) // stride + 1 + (1 if (L - k) % stride else 0)


PATHS = (("variant 1, fast_dp on", dict(variant=1, fast_dp=1)), ("variant 1, fast_dp off", dict(variant=1, fast_dp=0)),
         ("variant 0", dict(variant=0)))


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("L", [100, 200])
def test_band_sweep(oracle, L, mode):
    """--bandwidth 0 .. 15 at both read-word widths (NWR 4 and 8) and every scoring mode, every DP kernel path.  The
    planted indels reach one base past each band, so the oracle's results at every band below 15 differ from band 15's:
    a kernel that scores diagonals outside the band shows."""
    txps, left, right = workload(seed=10 + L + mode, n=1200, L=L)
    idx = Index(txps)
    orc = oracle_for(oracle, txps)
    refs = {B: orc(mode, left, right, band=B) for B in BANDS}
    bad = []
    for B in BANDS:
        if B < 15:
            assert differs(refs[B], refs[15]), B
        for name, opts in PATHS:
            if mode and opts["variant"] == 0:
                continue
            got, st = gpu_map(idx, left, right, opts, band=B, softclip=mode)
            try:
                check(got, st, refs[B], 200, f"band {B}, {name}")
            except AssertionError as e:
                bad.append(str(e))
                continue
            if opts["variant"] == 1:
                assert st.full_dp > 0, (B, name)
                if opts["fast_dp"]:
                    assert st.full_dp < st.candidates, (B, name)
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("k", [9, 15, 19, 25, 31])
def test_k_and_stride(oracle, k):
    """k x stride, each at two read lengths: 32 seed positions per mate (one round of k_seed_chain_w) and 34 (two
    rounds); the context's capacity is the read length, so both the 2- and 4-word seed instances run.  The lookups
    counter confirms the positions per mate."""
    txps, _ = synth_txome(seed=50 + k, n_genes=25)
    idx = Index(txps, k=k)
    orc = oracle_for(oracle, txps, k)
    for stride in (1, 2, 4, 7):
        L1, L2 = k + 31 * stride, k + 32 * stride + 1
        assert npos(L1, k, stride) == 32 and npos(L2, k, stride) == 34 and L2 <= 256
        for L in (L1, L2):
            rng = np.random.default_rng(k * 1000 + L)
            left, right = planted_pairs(txps, rng, 300, L, frag_mean=2 * L + 50, indel_frac=0.4)
            left[rng.integers(0, 300, 10), rng.integers(0, L, 10)] = 4
            ref = orc(0, left, right, stride=stride)
            got, st = gpu_map(idx, left, right, stride=stride)
            check(got, st, ref, 200, f"k {k}, stride {stride}, L {L}")
            assert (st.lookups > 2 * 300 * 32) == (L == L2)     # mates with N skip the lookups that cover it


@pytest.mark.parametrize("L", [156, 200, 256])
def test_long_reads_at_defaults(oracle, L):
    """reads longer than 150 bases at the default options (the 8-word DP instances): from 156 bases on, k 31 and stride 4
    give more than 32 seed positions per mate, the two-round seed instance k_seed_chain_w<4, 2>"""
    txps, left, right = workload(seed=70 + L, n=800, L=L)
    ref = oracle_for(oracle, txps)(0, left, right)
    for name, opts in PATHS:
        got, st = gpu_map(Index(txps), left, right, opts)
        check(got, st, ref, 200, f"L {L}, {name}")
        assert st.lookups > 2 * 800 * 32


def test_seed_position_limit_at_its_edge(oracle):
    """a context takes at most 64 seed positions per mate, (max_read_len - k) / stride + 2: 64 is accepted and maps
    like the oracle (63 and 64 positions per mate), 65 is refused"""
    for k, stride, edge in ((31, 1, 93), (9, 3, 197)):
        assert (edge - k) // stride + 2 == 64
        txps, _ = synth_txome(seed=80 + k, n_genes=25)
        idx = Index(txps, k=k)
        with pytest.raises(SalmonB200Error, match="at most 64 seed positions per mate"):
            MapContext(idx, map_default_params(k=k, stride=stride), batch_cap=64, max_read_len=edge + 1)
        rng = np.random.default_rng(k)
        left, right = planted_pairs(txps, rng, 300, edge, frag_mean=2 * edge + 50)
        ref = oracle_for(oracle, txps, k)(0, left, right, stride=stride)
        got, st = gpu_map(idx, left, right, stride=stride)
        check(got, st, ref, 200, (k, stride, edge))
        assert npos(edge, k, stride) in (63, 64) and st.lookups > 2 * 300 * 62


@pytest.mark.parametrize("scores", SCORES)
def test_scores_and_min_score_fraction(oracle, scores):
    """--ma / --mp / --go / --ge x --minScoreFraction, the ungapped shortcut on and off.  Where m mismatches cost exactly
    go + ge, mates with exactly m mismatches are planted: their best ungapped score is the shortcut's bound."""
    ma, mp, go, ge = scores
    m = tie_mismatches(*scores)
    txps, left, right = workload(seed=90 + ma + go, n=1000, L=100, subs=(m,) if m else (), sub_frac=0.3)
    idx = Index(txps)
    orc = oracle_for(oracle, txps)
    sc = dict(ma=ma, mp=mp, go=go, ge=ge)
    for msf in (0.3, 0.65, 0.95):
        ref = orc(0, left, right, min_score_fraction=msf, **sc)
        for fast in (1, 0):
            got, st = gpu_map(idx, left, right, dict(fast_dp=fast), min_score_fraction=msf, **sc)
            check(got, st, ref, 200, (scores, msf, fast))
            assert st.full_dp > 0 and (st.full_dp < st.candidates if fast else st.full_dp == st.candidates)
        if m:   # alignments scored exactly at the shortcut's bound: the pair's score is the sum of its mates'
            pm = np.arange(200)[None, :] < ref["n_aln"][:, None]
            assert (ref["score"][pm] == 2 * ma * 100 - (go + ge)).any()


@pytest.mark.parametrize("scores", [(2, -4, 6, -1), (1, 2, 6, 2)])
def test_fast_dp_option_respects_inexact_scores(oracle, scores):
    """scores under which the ungapped shortcut is not exact (a gap extension that pays, a mismatch above a match):
    set_option("fast_dp", 1) leaves the shortcut off, every alignment goes to the DP and the results are the oracle's"""
    txps, left, right = workload(seed=95, n=800, L=100)
    sc = dict(zip(("ma", "mp", "go", "ge"), scores))
    ref = oracle_for(oracle, txps)(0, left, right, **sc)
    got, st = gpu_map(Index(txps), left, right, dict(fast_dp=1), **sc)
    check(got, st, ref, 200, scores)
    assert st.full_dp == st.candidates > 0


def test_dp_lists_each_run(oracle):
    """the byte-code list (every mate has an N) and the edge list (no transcript is long enough for a whole band) on
    their own: every DP task goes there, and the results are the oracle's"""
    txps, left, right = workload(seed=97, n=600, L=100)
    left[:, 37] = 4
    right[:, 61] = 4
    ref = oracle_for(oracle, txps)(0, left, right)
    got, st = gpu_map(Index(txps), left, right)
    check(got, st, ref, 200, "byte list")
    assert st.full_dp == st.candidates > 0
    rng = np.random.default_rng(98)
    L = 100
    short = [rng.integers(0, 4, int(rng.integers(L + 5, L + 30)), dtype=np.uint8) for _ in range(80)]
    left = np.zeros((600, L), np.uint8)
    right = np.zeros((600, L), np.uint8)
    for i in range(600):
        t = short[int(rng.integers(len(short)))]
        a, b = t[int(rng.integers(0, len(t) - L + 1)):][:L], revcomp(t[len(t) - L - int(rng.integers(0, len(t) - L + 1)):][:L])
        left[i], right[i] = (a, b) if i % 2 else (b, a)
    rows, cols = rng.integers(0, 600, 100), rng.integers(0, L, 100)
    left[rows, cols] = (left[rows, cols] + 1) % 4                  # some mismatches
    ref = oracle_for(oracle, short)(0, left, right)
    got, st = gpu_map(Index(short), left, right, dict(fast_dp=0))
    check(got, st, ref, 200, "edge list")
    assert st.full_dp == st.candidates > 0 and st.mapped > 300


FRAG_SETTINGS = [
    dict(max_frag_len=200, fld_mean=150.0, fld_sd=10.0, score_exp=0.5),
    dict(max_frag_len=400, fld_mean=400.0, fld_sd=80.0, score_exp=2.0, min_aln_prob=0.0),
    dict(max_frag_len=2000, fld_mean=400.0, fld_sd=80.0, min_aln_prob=1e-3, consensus_frac=0.3),
    dict(consensus_frac=1.0, max_read_occ=1, chain_gap=0),
    dict(max_read_occ=2, max_occs_per_hit=1, range_bins=1),
    dict(max_occs_per_hit=3, chain_gap=30, range_bins=0, min_aln_prob=0.0),
    dict(range_bins=8, hard_filter=1, max_read_occ=255, score_exp=2.0),
    dict(max_frag_len=2000, fld_mean=150.0, fld_sd=10.0, hard_filter=1, min_aln_prob=1e-3, score_exp=0.5),
]


@pytest.mark.parametrize("over", FRAG_SETTINGS)
def test_fragment_model_and_filters_across_batches(oracle, over):
    """--fldMax / --fldMean / --fldSD / --scoreExp, the alignment-probability floor, the consensus fraction,
    --maxReadOcc, maxOccsPerHit, the chain gap, range bins and the hard filter, over three batches that cross
    numPreBurninFrags and numBurninFrags: online state bit-exact after every batch, then the class table, unique and
    total counts and effective lengths"""
    txps, left, right = workload(seed=100, n=1800, L=100)
    oix = oracle.MapIndex(txps)
    # the fragment counter passes numPreBurninFrags in the first batch and numBurninFrags in the second
    m0 = oracle.map_reads(oix, oracle.map_params(**over), left[:600], right[:600], 0)["counters"]["mapped"]
    reg = dict(num_pre_burnin=m0 // 2, num_burnin=m0 + m0 // 2)
    p = map_default_params(mini_batch=250, seed=7, **reg, **over)
    ctx = MapContext(Index(txps), p, batch_cap=600, max_read_len=100)
    on = oracle.Online(oix, oracle.map_params(**reg, **over), seed=7, mini_batch=250)
    cap = p.max_read_occ
    parts, burned = [], []
    for b in range(3):
        sl = slice(600 * b, 600 * (b + 1))
        ctx.map_batch(left[sl], right[sl])
        ref = on.batch(left[sl], right[sl])
        compare(ctx.last_alignments(), ref, cap, p.range_bins > 0)
        check_state(ctx.online_state(), on.state())
        parts.append(ref)
        burned.append(on.state()["burned_in"])
    assert burned == [0, 1, 1], burned
    res = ctx.finish()
    merged = {k: np.concatenate([q[k] for q in parts]) for k in ("n_aln", "label", "weight")}
    check_classes(res, oracle.eq_aggregate(merged, cap, p.range_bins > 0), exact_weights=False)
    fin = on.finish(res["off"], res["tids"], res["counts"])
    assert np.array_equal(res["unique_counts"], fin["unique_counts"])
    assert np.array_equal(res["total_counts"], fin["total_counts"])
    assert np.array_equal(bits(res["eff_len"]), bits(fin["eff_len"]))
    ctx.close()


@pytest.mark.parametrize("master_seed", [2, 5])
def test_fuzz_gpu_against_oracle(oracle, master_seed):
    """the randomised trials of the host fuzz test (test_map_host.fuzz_trials) through the GPU path: both kernel
    variants, random pipeline chunk sizes and a random context capacity above the read length"""
    rng = np.random.default_rng(1000 + master_seed)
    done = 0
    for t in fuzz_trials(master_seed, 70):
        over, L = t["over"], t["L"]
        k = over.get("k", 31)
        ref = oracle.map_reads(oracle.MapIndex(t["txps"], k=k), oracle.map_params(**over), t["left"], t["right"], 0)
        idx = Index(t["txps"], k=k)
        p = map_default_params(**over)
        caps = [c for c in (L, L, 160, 256) if c >= L and (c - k) // p.stride + 2 <= 64]
        for variant in (1, 0):
            opts = dict(variant=variant)
            if rng.random() < 0.5:
                opts["chunk"] = int(rng.choice([97, 300, 1024]))
            got, st = gpu_map(idx, t["left"], t["right"], opts, cap_len=int(rng.choice(caps)), **over)
            check(got, st, ref, p.max_read_occ, (master_seed, done, variant, L, over), p.range_bins > 0)
        done += 1
    assert done >= 40
