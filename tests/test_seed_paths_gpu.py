"""The seed kernel's rare paths on the GPU (seed_ref.py): the candidates k_seed_chain_w leaves for every mate, read back
through MapContext.last_candidates(), equal the oracle's bit for bit at each <CW, RD> instance, in variant 0 and for
single-end reads; so do the lookup / posting / seed counters, the alignments and the class tables.  Hash-mode probe
failures (33 <= D <= 128) depend on the order of the shared-memory atomics; the bit-exact check shows the output does
not."""
import numpy as np
import pytest
import torch

import oracle_lib as O
import seed_ref as S
from salmon_b200._capi import Index, MapContext, SalmonB200Error, map_default_params
from test_map_gpu import check_classes
from test_map_host import compare

pytestmark = pytest.mark.gpu
CAP = 200


@pytest.fixture(scope="module")
def world():
    txps, src = S.txome()
    return dict(txps=txps, src=src, idx=Index(txps), oix=O.MapIndex(txps), cache={})


def seed_warps(cw):
    """warps of k_seed_chain_w: 4 blocks per SM of 8 (CW 2) or 6 (CW 4) warps; warp w maps reads w, w + W, ..."""
    return torch.cuda.get_device_properties(0).multi_processor_count * 4 * (8 if cw == 2 else 6)


def workload(world, shape):
    """reads of the shape, enough that every seed warp maps at least two, and the oracle's view of them"""
    if shape not in world["cache"]:
        (cw, rd), L, stride, _ = S.SHAPES[shape]
        n = 2 * seed_warps(cw) + 400
        left, right, kinds = S.reads(shape, n, seed=10 + len(world["cache"]), txps=world["txps"], src=world["src"])
        op = O.map_params(stride=stride)
        cl, il = S.oracle_candidates(world["oix"], op, left)
        cr, ir = S.oracle_candidates(world["oix"], op, right)
        world["cache"][shape] = dict(left=left, right=right, cl=cl, cr=cr, il=il, ir=ir,
                                     ref=O.map_reads(world["oix"], op, left, right))
    return world["cache"][shape]


def run(world, shape, left, right, variant=1, **over):
    _, L, stride, max_len = S.SHAPES[shape]
    p = map_default_params(stride=stride, **over)
    ctx = MapContext(world["idx"], p, batch_cap=left.shape[0], max_read_len=max_len)
    ctx.set_option("variant", variant)
    st = ctx.map_batch(left, right)
    got, cand = ctx.last_alignments(), ctx.last_candidates()
    res = ctx.finish()
    ctx.close()
    return st, got, cand, res


def check_all(st, got, cand, res, ref, cl, cr, what):
    S.check_candidates(S.split_cands(cand["n_l"], cand["cand_l"]), cl, f"{what} left")
    S.check_candidates(S.split_cands(cand["n_r"], cand["cand_r"]), cr, f"{what} right")
    assert (ref["n_aln"][(cand["n_l"] >> 31) == 1] == 0).all()     # flagged by the seed kernel: no joint hit, or too many
    compare(got, ref, CAP)
    for k in ("lookups", "postings", "seeds", "kept", "label_entries", "mapped"):
        assert getattr(st, k) == ref["counters"][k], (what, k)
    check_classes(res, O.eq_aggregate(ref, CAP, True), exact_weights=True)


@pytest.mark.parametrize("shape", list(S.SHAPES))
def test_candidates_equal_oracle(world, shape):
    """paired-end, the warp kernel <CW, RD> of the shape: every regime R1-R7 it can take, pairs whose mates are in
    different regimes (both orders), and consecutive reads of one warp in different regimes"""
    w = workload(world, shape)
    (cw, rd), _, _, _ = S.SHAPES[shape]
    regs = [S.regimes(i, rd) for i in w["il"] + w["ir"]]
    for g in S.REGIMES:
        assert any(g in r for r in regs) == (g != "R5b" or rd == 2), g
    n, W = w["left"].shape[0], seed_warps(cw)
    per_read = [frozenset(regs[i]) | frozenset("r" + x for x in regs[n + i]) for i in range(n)]
    assert sum(per_read[r] != per_read[r + W] for r in range(n - W)) > (n - W) // 2
    st, got, cand, res = run(world, shape, w["left"], w["right"])
    check_all(st, got, cand, res, w["ref"], w["cl"], w["cr"], shape)
    assert st.seeds == sum(i["seeds"] for i in w["il"] + w["ir"])
    assert 0 < st.mapped < n


@pytest.mark.parametrize("shape", ["cw2_rd2", "cw4_rd1"])
def test_variant0_candidates(world, shape):
    """the serial-form kernel k_seed_chain on the same reads"""
    w = workload(world, shape)
    st, got, cand, res = run(world, shape, w["left"], w["right"], variant=0)
    check_all(st, got, cand, res, w["ref"], w["cl"], w["cr"], (shape, "variant 0"))


@pytest.mark.parametrize("shape", ["cw2_rd1", "cw4_rd2"])
def test_single_end(world, shape):
    """single-end reads: the left mates of the workload, the absent second mate has no candidate"""
    w = workload(world, shape)
    _, L, stride, _ = S.SHAPES[shape]
    left = w["left"]
    ref = O.map_reads(world["oix"], O.map_params(stride=stride, lib_type=3), left, np.full_like(left, 4))
    st, got, cand, res = run(world, shape, left, None, lib_type=3)
    empty = dict(n=np.zeros(left.shape[0], np.uint32), **{k: np.zeros((left.shape[0], 64), w["cl"][k].dtype)
                                                          for k in ("tid", "ori", "diag_c", "cov")})
    check_all(st, got, cand, res, ref, w["cl"], empty, (shape, "single-end"))
    assert st.mapped > 0


@pytest.mark.parametrize("L", [100, 200])
def test_longest_reference(L):
    """a reference of 2^21 - 1 bases with pairs on its last bases in both orientations (CW 2 at L = 100, CW 4 at 200)"""
    txps = S.long_txome()
    left, right = S.long_reads(txps, L)
    oix = O.MapIndex(txps)
    op = O.map_params()
    cl, _ = S.oracle_candidates(oix, op, left)
    cr, _ = S.oracle_candidates(oix, op, right)
    ref = O.map_reads(oix, op, left, right)
    ctx = MapContext(Index(txps), map_default_params(), batch_cap=left.shape[0], max_read_len=L)
    st = ctx.map_batch(left, right)
    got, cand = ctx.last_alignments(), ctx.last_candidates()
    res = ctx.finish()
    ctx.close()
    check_all(st, got, cand, res, ref, cl, cr, L)
    assert (ref["n_aln"] > 0).all() and max(cl["diag_c"][:, 0].max(), cr["diag_c"][:, 0].max()) + L > S.MAX_LEN - 8


def test_tap_refuses_what_it_cannot_show(world):
    """the candidate buffers hold one chunk, and orphan rescue appends to them"""
    w = workload(world, "cw2_rd1")
    left, right = w["left"][:3000], w["right"][:3000]
    for opts, over in ((dict(chunk=1024), {}), ({}, dict(recover_orphans=1))):
        p = map_default_params(stride=4, **over)
        ctx = MapContext(world["idx"], p, batch_cap=3000, max_read_len=100)
        for k, v in opts.items():
            ctx.set_option(k, v)
        ctx.map_batch(left, right)
        with pytest.raises(SalmonB200Error, match="one chunk without orphan rescue"):
            ctx.last_candidates()
        ctx.close()
