"""Orphan rescue (--recoverOrphans, DESIGN.md section 11) without a GPU: the product's bit-vector search (map_core.h,
host build) and the oracle's Sellers DP against edlib's goldens; the rule on hand-built cases; the product's per-read
path against the independent restatement (tests/oracle_rescue.c) read by read; the command line."""
import os
import subprocess

import numpy as np
import pytest

import oracle_lib as O
import rescue_ref as R

ROOT = R.ROOT


def test_search_forms_equal_edlib_goldens():
    cases, dist, end = R.golden()
    for i, (pat, win, K) in enumerate(cases):
        assert R.host_myers(pat, win, K) == (int(dist[i]), int(end[i])), ("product", i, len(pat), len(win))
        assert R.sellers(pat, win, K) == (int(dist[i]), int(end[i])), ("oracle", i, len(pat), len(win))
    assert (dist >= 0).sum() > len(cases) // 2 and (dist < 0).sum() > 10


def test_edit_limit():
    from salmon_b200._capi import map_default_params
    lib = R.host_lib()
    import ctypes as C
    p = map_default_params()
    assert lib.hrs_edit_limit(C.byref(p), 100) == 35
    assert lib.hrs_edit_limit(C.byref(p), 150) == 52
    # no alignment with more than K edits passes: K + 1 cheapest edits (ge each) already fail the threshold
    for L in R.LENGTHS:
        K = lib.hrs_edit_limit(C.byref(p), L)
        assert p.ma * L - (K + 1) * min(p.ma - p.mp, p.ge) < p.min_score_fraction * p.ma * L


def _txome(rng, lens):
    return [rng.integers(0, 4, n, dtype=np.uint8) for n in lens]


def _pair(t, pos, fl, L=100, left_fw=True):
    from salmon_b200.synth import revcomp
    frag = t[pos:pos + fl]
    a, b = frag[:L].copy(), revcomp(frag[-L:]).copy()
    return (a, b) if left_fw else (b, a)


def _run_both(txps, pairs, **over):
    """host product path and oracle restatement on the same reads; both must agree read by read"""
    from salmon_b200._capi import Index, map_default_params
    left = np.ascontiguousarray(np.stack([a for a, _ in pairs]))
    right = np.ascontiguousarray(np.stack([b for _, b in pairs]))
    p = map_default_params(recover_orphans=1, **over)
    h = R.host_map(Index(txps), p, left, right)
    o = R.oracle_map(R.OracleIndex(txps), O.map_params(**over), left, right)
    cap = p.max_read_occ
    assert np.array_equal(h["n_aln"], o["n_aln"])
    for k in ("tid", "score", "pos", "mate_pos", "flags", "flen", "prob", "weight"):
        m = np.arange(cap)[None, :] < h["n_aln"][:, None]
        assert np.array_equal(h[k][m], o[k][m]), k
    assert h["rescue"] == o["rescue"], (h["rescue"], o["rescue"])
    return h


def test_rule_on_hand_built_cases():
    rng = np.random.default_rng(3)
    txps = _txome(rng, [1500, 1500, 700])
    t = txps[0]
    kill = lambda r: R.kill_seeds(r, rng)
    # plain: the right mate unseedable, the left anchors -> one concordant pair with the true fragment length
    a, b = _pair(t, 400, 260)
    h = _run_both(txps, [(a, kill(b))])
    assert h["n_aln"][0] == 1 and (h["flags"][0, 0] >> 2) == 0 and h["flen"][0, 0] == 260 and h["rescue"] == [1, 1, 0]
    # reverse-strand fragment: the anchor is the reverse mate, the window lies upstream
    a, b = _pair(t, 800, 300, left_fw=False)
    h = _run_both(txps, [(a, kill(b))])
    assert h["n_aln"][0] == 1 and h["flen"][0, 0] == 300
    # clipping at either transcript end
    a, b = _pair(t, 0, 250)
    assert _run_both(txps, [(kill(a), b)])["n_aln"][0] == 1
    a, b = _pair(t, 1500 - 250, 250)
    assert _run_both(txps, [(a, kill(b))])["n_aln"][0] == 1
    # F smaller than the true fragment: the mate is out of reach, the orphan stays
    a, b = _pair(t, 300, 400)
    h = _run_both(txps, [(a, kill(b))], max_frag_len=350)
    assert h["rescue"][0] == 0 and h["n_aln"][0] == 1 and (h["flags"][0, 0] >> 2) == 1
    # an anchor whose own score fails: no search
    a, b = _pair(t, 500, 250)
    bad = a.copy(); bad[40:] = rng.integers(0, 4, 60, dtype=np.uint8)
    h = _run_both(txps, [(bad, kill(b))])
    assert h["rescue"][1] == 0
    # ISF: a left anchor on the reverse strand would form an incompatible pair; ISR accepts it
    a, b = _pair(t, 600, 250, left_fw=False)
    assert _run_both(txps, [(a, kill(b))], lib_type=1)["rescue"][1] == 0
    assert _run_both(txps, [(a, kill(b))], lib_type=2)["rescue"][0] == 1
    a, b = _pair(t, 600, 250, left_fw=True)
    assert _run_both(txps, [(a, kill(b))], lib_type=2)["rescue"][1] == 0
    assert _run_both(txps, [(a, kill(b))], lib_type=1)["rescue"][0] == 1


def test_dovetail():
    rng = np.random.default_rng(5)
    txps = _txome(rng, [1200])
    t = txps[0]
    from salmon_b200.synth import revcomp
    # the reverse mate starts 20 bases before the forward mate
    fw = t[500:600].copy()
    rv = revcomp(t[480:580]).copy()
    pairs = [(fw, R.kill_seeds(rv, rng))]
    assert _run_both(txps, pairs)["rescue"][0] == 0
    h = _run_both(txps, pairs, allow_dovetail=1)
    assert h["rescue"][0] == 1 and h["n_aln"][0] == 1


def test_full_candidate_list():
    """a repeat copied 70 times gives the left mate 64 orphan anchors; the right mate already holds 10 candidates of its
    own, so 54 rescued mates fit and 10 anchors find no room"""
    rng = np.random.default_rng(9)
    unit = rng.integers(0, 4, 700, dtype=np.uint8)
    a, b = _pair(unit, 200, 250)
    b = R.kill_seeds(b, rng)
    own = [np.concatenate([rng.integers(0, 4, 150, dtype=np.uint8), b, rng.integers(0, 4, 150, dtype=np.uint8)]) for _ in range(10)]
    txps = [unit.copy() for _ in range(70)] + own
    h = _run_both(txps, [(a, b)], max_read_occ=255)
    assert h["rescue"] == [1, 74, 10], h["rescue"]
    assert h["n_aln"][0] > 0 and all((h["flags"][0, :h["n_aln"][0]] >> 2) == 0)


def test_host_path_equals_oracle_on_planted_workload():
    from salmon_b200._capi import Index, map_default_params
    txps, left, right, truth = R.planted_workload(seed=5, n=1500, n_planted=250)
    for over in ({}, {"lib_type": 1}, {"lib_type": 2}, {"max_read_occ": 3}):
        p = map_default_params(recover_orphans=1, **over)
        h = R.host_map(Index(txps), p, left, right)
        o = R.oracle_map(R.OracleIndex(txps), O.map_params(**over), left, right)
        cap = p.max_read_occ
        assert np.array_equal(h["n_aln"], o["n_aln"]), over
        m = np.arange(cap)[None, :] < h["n_aln"][:, None]
        for k in ("tid", "score", "pos", "mate_pos", "flags", "flen", "prob", "weight"):
            assert np.array_equal(h[k][m], o[k][m]), (over, k)
        lm = np.arange(2 * cap)[None, :] < 2 * h["n_aln"][:, None]
        assert np.array_equal(h["label"][lm], o["label"][lm]), over
        assert h["rescue"] == o["rescue"], over
        if not over:
            assert h["rescue"][0] >= 0.9 * truth["planted"].sum()
    # off: exactly the plain path
    import hostmap_lib
    p0 = map_default_params()
    a0 = hostmap_lib.map_reads(Index(txps), p0, left, right)
    h0 = R.host_map(Index(txps), p0, left, right)
    assert np.array_equal(a0["n_aln"], h0["n_aln"]) and h0["rescue"] == [0, 0, 0]


def test_cli_parses_recover_orphans(tmp_path):
    exe = os.path.join(ROOT, "salmon_b200", "sb_salmon")
    if not os.path.exists(exe):
        pytest.skip("sb_salmon not built")
    r = subprocess.run([exe, "quant", "--recoverOrphans"], capture_output=True, text=True)   # parsed, then no -o: usage
    assert "outside the hot path" not in r.stderr and "unknown option" not in r.stderr
    assert "[--recoverOrphans]" in subprocess.run([exe], capture_output=True, text=True).stderr
