"""Workloads for the seed kernel's rare paths (tests/test_seed_paths_*.py), and the regime of a mate as the oracle's
per-mate report (orc_mate_info) proves it.

k_seed_chain_w (map_kernels.cuh) picks its path per mate from D, the number of distinct (transcript, orientation,
diagonal) keys among the kept seeds, and T, the number of seeds:
  R1  D <= 32                         hash mode, keys sorted in registers
  R2  33 <= D <= 128                  hash mode, shared-memory sort
  R3  D > 128, T <= 512               all seeds sorted in the shared region
  R4  D > 128, 512 < T <= 2048        all seeds sorted in the per-warp global scratch
  R5  more than 2048 postings         the 2048-seed cut (R5b: the cut falls in the second round of 32 lookups)
  R6  more than 64 survivors          the top-64 cut
  R7  a chain crosses a 32-key chunk  the carry of the chain scan (over the distinct keys in hash mode, the seeds else)
Each exists in four instances <CW, RD>: CW 4 when the context takes reads over 128 bases, RD 2 when a mate has more than
32 seed positions.  SHAPES gives one read length / stride / context pair per instance.

D is set by families of near-identical copies (one diagonal per copy) and tandem arrays (units of 8 bases or less, and
homopolymer / dinucleotide runs, chain adjacent diagonals); T by the copy count and by N bases that kill chosen
lookups."""
import numpy as np

from salmon_b200.synth import revcomp

K = 31
# name: (CW, RD), read length, stride, the context's max_read_len
SHAPES = {"cw2_rd1": ((2, 1), 100, 4, 100), "cw2_rd2": ((2, 2), 100, 2, 100),
          "cw4_rd1": ((4, 1), 200, 8, 200), "cw4_rd2": ((4, 2), 200, 4, 200)}
REGIMES = ("R1", "R2", "R3", "R4", "R5", "R5b", "R6", "R7")
FLANK, UNIT = 40, 640
FAMILIES = {"f60": 60, "f110": 110, "f150": 150}
MAX_LEN = (1 << 21) - 1            # the longest reference sb_index_build takes (22-bit diagonal field of the seed key)


def npos(L, stride, k=K):
    return (L - k) // stride + 1 + (1 if (L - k) % stride else 0)


def positions(L, stride, k=K):
    """seed positions of a mate in lookup order (the kernel's lane + 32 * round)"""
    return [min(j * stride, L - k) for j in range(npos(L, stride, k))]


def regimes(info, rd):
    """the regimes the oracle's report proves for one mate of a shape with `rd` lookup rounds"""
    D, T = info["distinct"], info["seeds"]
    out = set()
    if T == 0:
        return out
    if D <= 32:
        out.add("R1")
    elif D <= 128:
        out.add("R2")
    elif T <= 512:
        out.add("R3")
    else:
        out.add("R4")
    if info["cut_round"]:
        out.add("R5")
        if info["cut_round"] == 2:
            assert rd == 2
            out.add("R5b")
    if info["survivors"] > 64:
        out.add("R6")
    if (info["straddle_distinct"] if D <= 128 else info["straddle_seeds"]) > 0:
        out.add("R7")
    return out


def _rand(rng, n):
    return rng.integers(0, 4, n).astype(np.uint8)


def txome(seed=11):
    """background transcripts, three families of near-identical copies, tandem arrays and low-complexity runs.
    Returns (txps, sources): sources[name] = list of (tid, first, last) ranges reads are drawn from."""
    rng = np.random.default_rng(seed)
    txps, src = [], {}

    def add(name, seq, first, last):
        src.setdefault(name, []).append((len(txps), first, last))
        txps.append(np.ascontiguousarray(seq, dtype=np.uint8))

    for _ in range(30):
        add("uniq", _rand(rng, 1200), 0, 1200)
    for name, copies in FAMILIES.items():
        unit = _rand(rng, UNIT)
        for c in range(copies):
            u = unit.copy()
            if c % 3 == 2:                 # near-identical: two substitutions, so the copies' coverages differ
                for q in rng.choice(UNIT, 2, replace=False):
                    u[q] = (u[q] + 1 + rng.integers(0, 3)) % 4
            add(name, np.concatenate([_rand(rng, FLANK), u, _rand(rng, FLANK)]), FLANK, FLANK + UNIT)

    def array(name, unit, copies):
        body = np.tile(np.asarray(unit, dtype=np.uint8), copies)
        add(name, np.concatenate([_rand(rng, FLANK), body, _rand(rng, FLANK)]), FLANK, FLANK + body.shape[0])

    array("tan5", _rand(rng, 5), 80)        # 400 bases: one chain of about 80 to 110 adjacent diagonals (hash mode)
    array("tan6", _rand(rng, 6), 300)       # 1800 bases: one long chain over the seed array
    array("polyA", [0], 700)
    array("dinuc", [1, 2], 350)
    # a 40-base unit 1001 times: its k-mers of phase 0..9 have 1001 postings, of phase 10..39 exactly 1000
    array("tan40", _rand(rng, 40), 1001)
    return txps, src


def max_occs_phase(L_first, stride, L):
    """tan40 reads starting `L_first` bases into the array: (lookups with 1000 postings, lookups with 1001)"""
    ph = [(L_first + q) % 40 for q in positions(L, stride)]
    return sum(p >= 10 for p in ph), sum(p < 10 for p in ph)


def keep_only(seq, blocks, stride):
    """N every base outside the windows of the lookups in `blocks` ([lo, hi) ranges of lookup indices), so that only
    those lookups stay valid"""
    L = seq.shape[0]
    pos = positions(L, stride)
    cov = np.zeros(L, bool)
    for lo, hi in blocks:
        for j in range(lo, min(hi, len(pos))):
            cov[pos[j]:pos[j] + K] = True
    seq = seq.copy()
    seq[~cov] = 4
    return seq


def recipes(shape):
    """mate recipes of a shape: name -> (source, blocks of kept lookups or None for all)"""
    (cw, rd), L, stride, _ = SHAPES[shape]
    n = npos(L, stride)
    r = {"uniq": ("uniq", None), "f60": ("f60", None), "f110": ("f110", None), "tan5": ("tan5", None),
         "f150_t3": ("f150", [(0, 3)]), "f150_t8": ("f150", [(0, 8)]), "f150": ("f150", None),
         "tan6": ("tan6", None), "polyA": ("polyA", None), "dinuc": ("dinuc", None), "tan40": ("tan40", None),
         "f150_t1": ("f150", [(0, 1)])}
    if rd == 2:
        # every round-2 lookup and enough round-1 ones that the 16 lookups pass 2048 postings, which the round-1
        # ones alone do not (a third of the copies carry substitutions, so a lookup has a little under 150)
        c1 = 16 - (n - 32)
        assert 0 < c1 and 150 * c1 < 2048
        r["f150_cut2"] = ("f150", [(0, c1), (32, n)])
    return r


def mate(rng, txps, src, recipe, L, stride):
    name, blocks = recipe
    tid, first, last = src[name][rng.integers(0, len(src[name]))]
    a = int(rng.integers(first, last - L + 1))
    s = txps[tid][a:a + L]
    if rng.integers(0, 2):
        s = revcomp(s)
    return keep_only(s, blocks, stride) if blocks else s.copy()


def pair(rng, txps, src, rl, rr, L, stride):
    """a fragment when both recipes draw from the same source (left forward, right reverse complement, inward), else
    two independent mates"""
    if rl[0] == rr[0]:
        name = rl[0]
        tid, first, last = src[name][rng.integers(0, len(src[name]))]
        F = int(rng.integers(L + 20, min(last - first, L + 300) + 1))
        a = int(rng.integers(first, last - F + 1))
        t = txps[tid]
        left, right = t[a:a + L].copy(), revcomp(t[a + F - L:a + F])
        if rng.integers(0, 2):
            left, right = right, left
        return (keep_only(left, rl[1], stride) if rl[1] else left,
                keep_only(right, rr[1], stride) if rr[1] else right)
    return mate(rng, txps, src, rl, L, stride), mate(rng, txps, src, rr, L, stride)


def reads(shape, n, seed, txps=None, src=None):
    """n pairs of the shape.  The pair kinds repeat with a prime period (13), so reads r and r + W of one warp (W the
    kernel's warp count, a multiple of 8 and 6) are of different kinds; the kinds include both orders of mates in
    different regimes.  Returns (left, right, kinds)."""
    if txps is None:
        txps, src = txome()
    _, L, stride, _ = SHAPES[shape]
    R = recipes(shape)
    kinds = [("uniq", "uniq"), ("f60", "f60"), ("f150", "f150"), ("f150_t3", "f150"), ("f150", "f150_t3"),
             ("f150_t8", "uniq"), ("uniq", "f150_t8"), ("tan5", "f110"), ("tan6", "tan5"), ("polyA", "dinuc"),
             ("tan40", "tan40"), ("f150_t1", "f60"),
             ("f150_cut2", "f150_t3") if "f150_cut2" in R else ("dinuc", "polyA")]
    assert len(kinds) == 13
    rng = np.random.default_rng(seed)
    left = np.empty((n, L), np.uint8)
    right = np.empty((n, L), np.uint8)
    names = []
    for i in range(n):
        kl, kr = kinds[i % 13]
        left[i], right[i] = pair(rng, txps, src, R[kl], R[kr], L, stride)
        names.append((kl, kr))
    return left, right, names


def long_txome(seed=5, length=MAX_LEN):
    """one reference of `length` bases and a short one; reads on the last bases of the long one in both orientations"""
    rng = np.random.default_rng(seed)
    return [_rand(rng, length), _rand(rng, 900)]


def long_reads(txps, L, seed=6, n=64):
    rng = np.random.default_rng(seed)
    t = txps[0]
    T = t.shape[0]
    left = np.empty((n, L), np.uint8)
    right = np.empty((n, L), np.uint8)
    for i in range(n):
        e = T - int(rng.integers(0, 8))             # the fragment ends at most 7 bases before the reference's end
        F = int(rng.integers(L + 10, L + 200))
        a = e - F
        l, r = t[a:a + L].copy(), revcomp(t[e - L:e])
        if i % 2:
            l, r = r, l
        left[i], right[i] = l, r
    return left, right


def oracle_candidates(oix, p, mates):
    """the oracle's candidates of every mate: counts [m], fields [m, 64] (tid, ori, diag_c, cov) and the reports"""
    import oracle_lib as O
    m = mates.shape[0]
    out = dict(n=np.zeros(m, np.uint32), tid=np.zeros((m, 64), np.uint32), ori=np.zeros((m, 64), np.uint32),
               diag_c=np.zeros((m, 64), np.int32), cov=np.zeros((m, 64), np.uint32))
    infos = []
    for i in range(m):
        c, info = O.mate_candidates(oix, p, mates[i])
        out["n"][i] = c.shape[0]
        for k in ("tid", "ori", "diag_c", "cov"):
            out[k][i, :c.shape[0]] = c[k]
        infos.append(info)
    return out, infos


def split_cands(n, cand):
    """the product's Cand records [m, 64] with their counts as the fields oracle_candidates gives"""
    return dict(n=np.asarray(n, np.uint32) & 0x7fffffff, tid=cand["tid"], ori=cand["ori_cov"] >> 31,
                diag_c=cand["diag_c"], cov=cand["ori_cov"] & 0x7fffffff)


def check_candidates(got, ref, what=""):
    """bit for bit, mate by mate: count, then tid, orientation, diag_c and coverage of every candidate"""
    bad = np.flatnonzero(got["n"] != ref["n"])
    assert bad.size == 0, f"{what}: {bad.size} mates differ in count, first {bad[0]}: {got['n'][bad[0]]} != {ref['n'][bad[0]]}"
    live = np.arange(64)[None, :] < ref["n"][:, None]
    for k in ("tid", "ori", "diag_c", "cov"):
        diff = np.flatnonzero((np.asarray(got[k]) != ref[k]) & live) // 64
        assert diff.size == 0, f"{what}: {k} differs in {np.unique(diff).size} mates, first {diff[0]}"
