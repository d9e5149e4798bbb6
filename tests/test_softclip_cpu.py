"""Scoring modes of the DP (--softclipOverhangs = 1, --softclip = 2; DESIGN.md section 12) without a GPU: the product's
serial DP (map_core.h, host build) against the independent restatement (tests/oracle_softclip.c) and a pure-Python
Gotoh; the mode-2 identity with the default DP; mode 1's two formulations; closed forms; the product's per-read path
against the restatement read by read; the mate search's edit limit; the command line."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_lib as O
import rescue_ref as R
import softclip_ref as S

ROOT = S.ROOT


@pytest.fixture(scope="module")
def dp_world():
    txps = S.dp_txome(seed=1)
    return txps, S.OracleIndex(txps)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_serial_dp_equals_oracle(dp_world, mode):
    from salmon_b200._capi import map_default_params
    txps, oix = dp_world
    p, op = map_default_params(softclip=mode), O.map_params()
    cases = S.dp_cases(100 + mode, 3000, txps)
    differ = 0
    for i, (read, ori, t, d) in enumerate(cases):
        want = S.oracle_dp(oix, op, read, ori, t, d, mode)
        assert S.product_dp(oix, p, read, ori, t, d) == want, (mode, i, len(read), ori, t, d)
        if mode == 1:   # the second formulation: cells outside the transcript live at score 0, no gaps there
            assert S.oracle_dp(oix, op, read, ori, t, d, 1, form=1) == want, (i, len(read), ori, t, d)
        if mode:
            differ += want != S.oracle_dp(oix, op, read, ori, t, d, 0)
    if mode:
        assert differ > 300   # the cases exercise what the mode changes


def test_python_gotoh_agrees(dp_world):
    txps, oix = dp_world
    op = O.map_params()
    for mode in (0, 1, 2):
        for i, (read, ori, t, d) in enumerate(S.dp_cases(200 + mode, 120, txps, max_len=90)):
            want = S.oracle_dp(oix, op, read, ori, t, d, mode)
            got = S.gotoh(txps[t].tolist(), S.oriented(read, ori).tolist(), d, 15, 2, -4, 6, 2, mode)
            assert got == want, (mode, i)


def test_mode2_is_best_substring_of_default(dp_world):
    """score_2(read, d) = max over 0 <= a < b <= L of score_0(read[a:b], d + a), read oriented to the forward strand,
    score_0 by the CPU oracle's own DP"""
    txps, oix = dp_world
    op = O.map_params()
    for i, (read, ori, t, d) in enumerate(S.dp_cases(300, 25, txps, max_len=44)):
        fw = S.oriented(read, ori)
        L = len(fw)
        best = max(S.oracle_dp_default(oix, op, fw[a:b], 0, t, d + a) for a in range(L) for b in range(a + 1, L + 1))
        assert S.oracle_dp(oix, op, read, ori, t, d, 2) == best, (i, L)


def test_closed_forms():
    """an otherwise exact read: k bases over the transcript end score ma*(L-k) in modes 1 and 2 and less in mode 0; a
    c-base junk tail scores ma*(L-c) in mode 2 (two-letter transcript, junk from the other two letters: nothing in the
    overhang or the tail can match anywhere)"""
    from salmon_b200._capi import map_default_params
    rng = np.random.default_rng(8)
    ref = rng.integers(0, 2, 600, dtype=np.uint8)
    oix = S.OracleIndex([ref])
    op = O.map_params()
    for L in (31, 100, 150, 256):
        for k in [k for k in (1, 5, 17, 40) if k < L - 10]:
            junk = rng.integers(2, 4, k, dtype=np.uint8)
            for side in (0, 1):
                if side == 0:   # hangs over the start
                    fw = np.concatenate([junk, ref[:L - k]]); d = -k
                else:           # hangs over the end
                    fw = np.concatenate([ref[600 - (L - k):], junk]); d = 600 - (L - k)
                for ori in (0, 1):
                    from salmon_b200.synth import revcomp
                    read = revcomp(fw) if ori else fw
                    s = {m: S.product_dp(oix, map_default_params(softclip=m), read, ori, 0, d) for m in (0, 1, 2)}
                    assert s[1] == s[2] == 2 * (L - k), (L, k, side, ori, s)
                    assert s[0] < 2 * (L - k)
                    assert S.oracle_dp(oix, op, read, ori, 0, d, 1) == s[1]
        for c in (1, 4, 25, 30):
            pos = 200
            fw = np.concatenate([ref[pos:pos + L - c], rng.integers(2, 4, c, dtype=np.uint8)])
            assert S.product_dp(oix, map_default_params(softclip=2), fw, 0, 0, pos) == 2 * (L - c), (L, c)
            assert S.oracle_dp(oix, op, fw, 0, 0, pos, 2) == 2 * (L - c)


def _compare(h, o, cap, what):
    assert np.array_equal(h["n_aln"], o["n_aln"]), what
    m = np.arange(cap)[None, :] < h["n_aln"][:, None]
    for k in ("tid", "score", "pos", "mate_pos", "flags", "flen", "prob", "weight"):
        assert np.array_equal(h[k][m], o[k][m]), (what, k)
    lm = np.arange(2 * cap)[None, :] < 2 * h["n_aln"][:, None]
    assert np.array_equal(h["label"][lm], o["label"][lm]), what
    assert h["rescue"] == o["rescue"], (what, h["rescue"], o["rescue"])


@pytest.mark.parametrize("mode", [1, 2])
def test_product_path_equals_oracle(mode):
    from salmon_b200._capi import Index, map_default_params
    txps, left, right = S.workload(seed=21, n=1500, n_over=200)
    # plus orphans for the rescue to find
    ptx, pl, pr, _ = R.planted_workload(seed=5, n=600, n_planted=150)
    ix, oix = Index(txps), S.OracleIndex(txps)
    pix, poix = Index(ptx), S.OracleIndex(ptx)
    rescued = {}
    for lib_type in (0, 1, 2):
        for ro in (0, 1):
            over = dict(lib_type=lib_type)
            p = map_default_params(softclip=mode, recover_orphans=ro, **over)
            for (idx, orc, lft, rgt, nm) in ((ix, oix, left, right, "adapters"), (pix, poix, pl, pr, "orphans")):
                h = R.host_map(idx, p, lft, rgt)
                o = S.oracle_map(orc, O.map_params(**over), mode, ro, lft, rgt)
                _compare(h, o, p.max_read_occ, (mode, lib_type, ro, nm))
                rescued[(lib_type, ro, nm)] = h["rescue"][0]
    assert rescued[(0, 1, "orphans")] >= 100 and rescued[(0, 0, "orphans")] == 0
    # mode 0 through the restatement is the CPU oracle
    want = O.map_reads(O.MapIndex(txps), O.map_params(), left, right)
    got = S.oracle_map(oix, O.map_params(), 0, 0, left, right)
    assert np.array_equal(want["n_aln"], got["n_aln"])
    m = np.arange(400)[None, :] < 2 * want["n_aln"][:, None]
    assert np.array_equal(want["label"][m], got["label"][m])


def test_modes_change_the_mapping_rate():
    from salmon_b200._capi import Index, map_default_params
    from salmon_b200.synth import synth_reads, synth_txome
    rng = np.random.default_rng(4)
    txps, _ = synth_txome(seed=4, n_genes=40)
    left, right, _ = synth_reads(txps, seed=5, n=400, read_len=100)
    al, ar, _ = S.with_adapters(left, right, rng, 1.0, 25, 25)
    ix = Index(txps)
    rate = {m: float((R.host_map(ix, map_default_params(softclip=m), al, ar)["n_aln"] > 0).mean()) for m in (0, 1, 2)}
    assert rate[2] >= 0.97 and rate[0] < 0.1 and rate[1] < 0.1, rate


def test_edit_limit():
    from salmon_b200._capi import map_default_params
    lib = R.host_lib()
    for over in ({}, dict(ma=1), dict(ma=3, mp=-2, ge=4), dict(min_score_fraction=0.5)):
        for mode in (0, 1, 2):
            p = map_default_params(softclip=mode, **over)
            for L in R.LENGTHS:
                K = lib.hrs_edit_limit(C.byref(p), L)
                assert K == S.oracle_lib().orc_sc_edit_limit(C.addressof(O.map_params(**over)), mode, L)
                # K + 1 of the cheapest edits already fail the threshold; a clipped base (modes 1, 2) costs ma
                per = min(p.ma - p.mp, p.ge, p.ma) if mode else min(p.ma - p.mp, p.ge)
                assert p.ma * L - (K + 1) * per < p.min_score_fraction * p.ma * L, (over, mode, L)
    p = map_default_params(softclip=2)
    assert lib.hrs_edit_limit(C.byref(p), 100) == 35 and lib.hrs_edit_limit(C.byref(p), 150) == 52


def test_cli_and_bad_mode(tmp_path):
    from salmon_b200 import _capi
    from salmon_b200._capi import Index, MapContext, map_default_params
    with pytest.raises(_capi.SalmonB200Error, match="softclip"):
        MapContext(Index(S.dp_txome(2)[:3]), map_default_params(softclip=3), batch_cap=64, max_read_len=100)
    with pytest.raises(_capi.SalmonB200Error, match="softclip"):
        MapContext(Index(S.dp_txome(2)[:3]), map_default_params(softclip=-1), batch_cap=64, max_read_len=100)
    exe = os.path.join(ROOT, "salmon_b200", "sb_salmon")
    if not os.path.exists(exe):
        pytest.skip("sb_salmon not built")
    for flag in ("--softclip", "--softclipOverhangs"):
        r = subprocess.run([exe, "quant", flag], capture_output=True, text=True)   # parsed, then no -o: usage
        assert "unknown option" not in r.stderr and "outside the hot path" not in r.stderr
    assert "[--softclip] [--softclipOverhangs]" in subprocess.run([exe], capture_output=True, text=True).stderr
