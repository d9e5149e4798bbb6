"""Workloads and helpers of the Bowtie2-mimicking presets (`--mimicBT2`, `--mimicStrictBT2`, DESIGN.md section 14):
the preset values by name, the gapless-settlement rule restated, mates planted on both sides of the lowest mate score
that can change an outcome, and a tandem-repeat transcript whose reads have more than 255 joint hits."""
import numpy as np

from salmon_b200._capi import map_default_params, map_mimic_bt2
from test_map_host import planted_pairs

PRESET_KEYS = ("max_read_occ", "consensus_frac", "allow_orphans", "min_score_fraction", "ma", "mp", "go", "ge")


def preset_over(strict, lib_type=0):
    """the preset's values for a library type as keyword overrides (names shared by sb_map_params and the oracle's
    parameters); single-end types also get salmon's single-end pre-merge threshold"""
    p = map_mimic_bt2(map_default_params(lib_type=lib_type), strict=strict)
    over = {k: getattr(p, k) for k in PRESET_KEYS}
    return dict(over, lib_type=lib_type, pre_merge_thresh=1.0) if lib_type >= 3 else over


def s_min(over, L, paired=True):
    """the lowest mate score that can change an outcome"""
    f, perfect = over["min_score_fraction"], over["ma"] * L
    return (2 * f - 1) * perfect if paired else f * perfect


def gapless(over, L, paired=True):
    """k_dp_classify settles every alignment by its best ungapped diagonal: G = ma*L - go - ge < s_min, compared the way
    assign_read compares a hit with its threshold (so G = s_min, a pair at exactly the threshold, does not settle)"""
    f, perfect = over["min_score_fraction"], over["ma"] * L
    G = perfect - over["go"] - over["ge"]
    return G < f * perfect and (not paired or G + perfect < f * (2 * perfect))


def tie_mismatches(over, L, paired=True):
    """the number of mismatches that puts an ungapped mate at s_min (rounded to the nearest)"""
    return int(round((over["ma"] * L - s_min(over, L, paired)) / (over["ma"] - over["mp"])))


def around_s_min(txps, over, L, n, seed, paired=True):
    """n pairs: a third with one mate carrying m0 - 1, m0 or m0 + 1 mismatches (m0 = tie_mismatches, so the mate scores
    on both sides of s_min while its partner is perfect), the mismatches inside the first L - 40 read bases so that a
    k-mer of the mate survives; a third with planted indels of 1 to 24 bases in either mate; a third exact."""
    rng = np.random.default_rng(seed)
    m0 = tie_mismatches(over, L, paired)
    assert 0 < m0 + 1 <= L - 40, (m0, L)
    k = n // 3
    left, right = planted_pairs(txps, rng, n - k, L, frag_mean=2 * L + 50, indel_frac=0.0)
    il, ir = planted_pairs(txps, rng, k, L, frag_mean=2 * L + 50, indel_frac=0.9)
    left, right = np.concatenate([left, il]), np.concatenate([right, ir])
    groups = np.full(n, -1)
    for i in range(k):
        m = m0 - 1 + i % 3
        q = rng.choice(L - 40, m, replace=False)
        left[i, q] = (left[i, q] + rng.integers(1, 4, m)) % 4
        groups[i] = i % 3
    return np.ascontiguousarray(left), np.ascontiguousarray(right), groups


def tandem_txome(seed, unit_len=60, copies=50, flank=200, n_plain=20):
    """a transcript of `copies` exact copies of a random unit between random flanks, plus ordinary random transcripts"""
    rng = np.random.default_rng(seed)
    unit = rng.integers(0, 4, unit_len, dtype=np.uint8)
    rep = np.concatenate([rng.integers(0, 4, flank, dtype=np.uint8), np.tile(unit, copies),
                          rng.integers(0, 4, flank, dtype=np.uint8)])
    return [rep] + [rng.integers(0, 4, int(rng.integers(800, 2000)), dtype=np.uint8) for _ in range(n_plain)]


def tandem_reads(txps, seed, n, L=100, frag=250, frac_plain=0.5):
    """pairs from inside the repeat of txps[0] (hundreds of joint hits each) and ordinary pairs from the rest"""
    from salmon_b200.synth import revcomp
    rng = np.random.default_rng(seed)
    left = np.zeros((n, L), np.uint8)
    right = np.zeros((n, L), np.uint8)
    rep = np.zeros(n, bool)
    for i in range(n):
        plain = rng.random() < frac_plain
        t = txps[int(rng.integers(1, len(txps)))] if plain else txps[0]
        lo, hi = (0, len(t) - frag) if plain else (200, len(t) - 200 - frag)
        pos = int(rng.integers(lo, hi + 1))
        a, b = t[pos:pos + L], revcomp(t[pos + frag - L:pos + frag])
        left[i], right[i] = (a, b) if rng.random() < 0.5 else (b, a)
        rep[i] = not plain
    return left, right, rep
