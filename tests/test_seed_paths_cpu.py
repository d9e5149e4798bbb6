"""The seed stage's rare paths without a GPU: the workloads of seed_ref.py put mates in every regime R1-R7 of
k_seed_chain_w at each of its four <CW, RD> instances (the oracle's per-mate report proves which), and the host build
of map_core.h's mate_candidates equals the oracle's candidates mate by mate, bit for bit."""
import ctypes as C

import numpy as np
import pytest

import hostmap_lib
import oracle_lib as O
import seed_ref as S
from salmon_b200._capi import CAND_DTYPE, Index, SalmonB200Error, map_default_params
from test_map_host import compare

N_READS = 1300      # 100 pairs of each of the 13 kinds


@pytest.fixture(scope="module")
def world():
    txps, src = S.txome()
    return txps, src, Index(txps), O.MapIndex(txps)


def host_candidates(idx, p, mates):
    """map_core.h's mate_candidates on the host for every mate, and the summed {lookups, postings, seeds}"""
    lib = hostmap_lib.build()
    lib.hmc_mate_candidates.restype = C.c_uint32
    ha = idx.host_arrays()
    m, L = mates.shape
    n = np.zeros(m, np.uint32)
    cand = np.zeros((m, 64), CAND_DTYPE)
    ctr = np.zeros(3, np.uint64)
    tot = np.zeros(3, np.uint64)
    for i in range(m):
        read = np.ascontiguousarray(mates[i])
        n[i] = lib.hmc_mate_candidates(C.c_uint32(idx.n_txps), C.c_uint32(idx.k), C.c_void_p(ha["tx_off"]),
                                       C.c_void_p(ha["codes"]), C.c_void_p(ha["table"]),
                                       C.c_uint64(ha["table_capacity"]), C.c_void_p(ha["postings"]), C.byref(p),
                                       read.ctypes.data_as(C.c_void_p), C.c_uint32(L),
                                       cand[i].ctypes.data_as(C.c_void_p), ctr.ctypes.data_as(C.c_void_p))
        tot += ctr
    return S.split_cands(n, cand), dict(zip(("lookups", "postings", "seeds"), (int(x) for x in tot)))


def test_every_regime_at_every_instance(world, capsys):
    """the regime table: mates per regime R1-R7 at each <CW, RD> instance; every cell where the regime can occur is
    reached (R5b, the cut in the second lookup round, needs RD = 2)"""
    txps, src, _, oix = world
    table = {}
    for shape, ((cw, rd), L, stride, _) in S.SHAPES.items():
        left, right, kinds = S.reads(shape, N_READS, seed=1, txps=txps, src=src)
        _, infos = S.oracle_candidates(oix, O.map_params(stride=stride), np.concatenate([left, right]))
        regs = [S.regimes(i, rd) for i in infos]
        table[shape] = {g: sum(g in r for r in regs) for g in S.REGIMES}
        for g in S.REGIMES:
            assert (table[shape][g] > 0) == (g != "R5b" or rd == 2), (shape, g)
        # pairs whose mates are in different regimes, in both orders
        n = len(kinds)
        pairs = {(frozenset(regs[i]), frozenset(regs[n + i])) for i in range(n)}
        assert any((b, a) in pairs for a, b in pairs if a != b), shape
        # a k-mer with exactly max_occs_per_hit (1000) postings is looked up, one with 1001 is dropped
        tan40 = [infos[i] for i in range(2 * n) if kinds[i % n][i // n] == "tan40"]
        assert all(i["postings_all"] % 1000 == 0 for i in tan40)
        assert any(0 < i["postings_all"] // 1000 < i["lookups"] for i in tan40)
    with capsys.disabled():
        print("\nmates per regime (paired-end, %d pairs per instance)" % N_READS)
        print("%-8s" % "" + "".join("%8s" % s for s in S.SHAPES))
        for g in S.REGIMES:
            print("%-8s" % g + "".join("%8d" % table[s][g] for s in S.SHAPES))


@pytest.mark.parametrize("shape", list(S.SHAPES))
def test_host_serial_equals_oracle_per_mate(world, shape):
    """map_core.h's mate_candidates (what variant 0 runs, and the rule the warp kernel restates) against the oracle"""
    txps, src, idx, oix = world
    _, L, stride, _ = S.SHAPES[shape]
    left, right, _ = S.reads(shape, N_READS, seed=2, txps=txps, src=src)
    mates = np.concatenate([left, right])
    ref, infos = S.oracle_candidates(oix, O.map_params(stride=stride), mates)
    got, ctr = host_candidates(idx, map_default_params(stride=stride), mates)
    S.check_candidates(got, ref, shape)
    assert ctr["lookups"] == sum(i["lookups"] for i in infos)
    assert ctr["postings"] == ctr["seeds"] == sum(i["seeds"] for i in infos)
    assert (ref["n"] == 64).sum() > 0 and (ref["n"] == 0).sum() < mates.shape[0]


@pytest.mark.parametrize("shape", list(S.SHAPES))
def test_batch_counters_and_alignments(world, shape):
    txps, src, idx, oix = world
    _, L, stride, _ = S.SHAPES[shape]
    left, right, _ = S.reads(shape, N_READS, seed=3, txps=txps, src=src)
    got = hostmap_lib.map_reads(idx, map_default_params(stride=stride), left, right)
    ref = O.map_reads(oix, O.map_params(stride=stride), left, right)
    compare(got, ref, 200)
    for k in ("lookups", "postings", "seeds", "candidates", "kept", "label_entries", "mapped"):
        assert got["counters"][k] == ref["counters"][k], k
    assert 0 < ref["counters"]["mapped"] < N_READS


def test_longest_reference():
    """a reference of 2^21 - 1 bases (the longest the index takes) with reads on its last bases in both orientations:
    the diagonal field of the seed key at its top; 2^21 bases are refused"""
    txps = S.long_txome()
    idx, oix = Index(txps), O.MapIndex(txps)
    for L, stride in ((100, 4), (200, 4)):
        left, right = S.long_reads(txps, L)
        mates = np.concatenate([left, right])
        ref, _ = S.oracle_candidates(oix, O.map_params(stride=stride), mates)
        got, _ = host_candidates(idx, map_default_params(stride=stride), mates)
        S.check_candidates(got, ref, L)
        assert (ref["n"] > 0).all() and set(ref["ori"][:, 0]) == {0, 1}
        assert ref["diag_c"][:, 0].max() + L > S.MAX_LEN - 8
        a = hostmap_lib.map_reads(idx, map_default_params(stride=stride), left, right)
        b = O.map_reads(oix, O.map_params(stride=stride), left, right)
        compare(a, b, 200)
        assert (b["n_aln"] > 0).all()
    with pytest.raises(SalmonB200Error, match="2\\^21"):
        Index(S.long_txome(length=S.MAX_LEN + 1))
