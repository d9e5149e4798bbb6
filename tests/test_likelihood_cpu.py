"""salmon's fragment-likelihood options (--incompatPrior, --noSingleFragProb, --noFragLengthDist,
--noEffectiveLengthCorrection; DESIGN.md section 13) without a GPU: the command line, the product's per-read path
(map_core.h compiled for the host) against the independent restatement (tests/oracle_likelihood.c) bit for bit, the
restatement against the unchanged oracle at the defaults, and the multi-rank sum of the compatible-fragment count."""
import os
import subprocess
import sys

import numpy as np
import pytest

import hostmap_lib
import likelihood_ref as LK
import oracle_lib as O
from salmon_b200._capi import Index, map_default_params

ROOT = LK.ROOT
SB = os.path.join(ROOT, "salmon_b200", "sb_salmon")

# (options, library type): each option alone and in combination
CASES = [
    (dict(), 2),
    (dict(incompat_prior=1e-20), 2),
    (dict(incompat_prior=0.3), 1),
    (dict(incompat_prior=1e-101), 2),          # below the threshold: ignored, as 0
    (dict(no_single_frag_prob=1), 2),
    (dict(no_frag_len_dist=1, no_eff_len_correction=1), 2),
    (dict(no_eff_len_correction=1), 2),
    (dict(incompat_prior=1e-5, no_single_frag_prob=1, no_frag_len_dist=1, no_eff_len_correction=1), 2),
    (dict(incompat_prior=1e-20), 0),
]


@pytest.fixture(scope="module")
def work():
    txps, fd, left, right = LK.stranded_workload(seed=5, n=2500)
    return txps, fd, left, right, Index(txps), LK.OracleIndex(txps)


def _run(work, over, lib_type, frag_counter, single_end=False, extra=None):
    txps, fd, left, right, idx, oix = work
    o = LK.opts(**over)
    base = dict(lib_type=lib_type + (3 if single_end else 0), first_decoy=fd, num_pre_burnin=1000, num_burnin=2000)
    if single_end:
        base["pre_merge_thresh"] = 1.0
    base.update(extra or {})
    prod = map_default_params(**base, **LK.product_fields(o))
    r = np.full_like(right, 4) if single_end else right
    got = hostmap_lib.map_reads(idx, prod, left, r, frag_counter)
    want = LK.oracle_map(oix, O.map_params(**base), o, left, r, frag_counter)
    return got, want, prod


@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("frag_counter", [0, 1500, 5000])   # before the aux model, before and after burn-in
def test_serial_form_equals_restatement(work, case, frag_counter):
    over, lt = CASES[case]
    got, want, prod = _run(work, over, lt, frag_counter)
    assert LK.same(got, want, prod.max_read_occ) is None, (over, frag_counter, LK.same(got, want, prod.max_read_occ))
    for k in ("kept", "mapped", "label_entries", "candidates"):
        assert got["counters"][k] == want["counters"][k], k


@pytest.mark.parametrize("over", [dict(incompat_prior=1e-20), dict(incompat_prior=0.5, no_single_frag_prob=1), dict()])
@pytest.mark.parametrize("extra", [dict(hard_filter=1), dict(min_aln_prob=1e-3), dict(decoy_threshold=0.9)])
def test_filters_with_incompatible_hits(work, over, extra):
    """an incompatible best hit above compatible lower hits under --hardFilter, minAlnProb and the decoy threshold"""
    got, want, prod = _run(work, over, 2, 5000, extra=extra)
    assert LK.same(got, want, prod.max_read_occ) is None


@pytest.mark.parametrize("over", [dict(), dict(incompat_prior=1e-20), dict(no_single_frag_prob=1),
                                  dict(no_frag_len_dist=1, no_eff_len_correction=1)])
@pytest.mark.parametrize("frag_counter", [0, 5000])
def test_single_end_equals_restatement(work, over, frag_counter):
    got, want, prod = _run(work, over, 2, frag_counter, single_end=True)
    assert LK.same(got, want, prod.max_read_occ) is None


def test_workload_plants_what_it_should(work):
    """the prior keeps antisense-only fragments that 0 drops; ties and incompatible-best hits occur; orphans and decoys map"""
    txps, fd, left, right, idx, oix = work
    base, lo = _run(work, {}, 2, 5000)[1], _run(work, dict(incompat_prior=1e-20), 2, 5000)[1]
    assert lo["counters"]["mapped"] > base["counters"]["mapped"] + 300
    assert base["counters"]["compatible"] == base["counters"]["mapped"]
    assert lo["counters"]["compatible"] < lo["counters"]["mapped"]
    st = (lo["flags"] >> 2) & 3
    m = np.arange(lo["tid"].shape[1])[None, :] < lo["n_aln"][:, None]
    assert np.any(st[m] != 0)                                    # orphans
    M = len(txps)
    tie_reads = np.arange(len(left)) % 10 == 0
    assert np.all(lo["n_aln"][tie_reads & (base["n_aln"] > 0)] >= 1)
    # every 13th read: under the prior its best hit is the exact antisense copy of u, so with --hardFilter it moves there
    hf = _run(work, dict(incompat_prior=1e-20), 2, 5000, extra=dict(hard_filter=1))[1]
    r13 = (np.arange(len(left)) % 13 == 0) & (np.arange(len(left)) % 10 != 0) & (np.arange(len(left)) % 9 != 0)
    assert np.mean(hf["tid"][r13, 0][hf["n_aln"][r13] > 0] == M - 4) > 0.8
    hf0 = _run(work, {}, 2, 5000, extra=dict(hard_filter=1))[1]
    assert np.mean(hf0["tid"][r13, 0][hf0["n_aln"][r13] > 0] == M - 5) > 0.8


@pytest.mark.parametrize("frag_counter", [0, 1500, 5000])
@pytest.mark.parametrize("lt", [0, 1, 2])
def test_defaults_equal_unchanged_oracle(work, frag_counter, lt):
    txps, fd, left, right, idx, oix = work
    p = O.map_params(lib_type=lt, first_decoy=fd, num_pre_burnin=1000, num_burnin=2000)
    a = LK.oracle_map(oix, p, LK.opts(), left, right, frag_counter)
    b = LK.oracle_map_unchanged(oix, p, left, right, frag_counter)
    assert LK.same(a, b, p.max_read_occ) is None
    assert a["counters"]["compatible"] == a["counters"]["mapped"] == b["counters"]["mapped"]


def test_default_params_leave_the_new_fields_zero():
    p = map_default_params()
    assert (p.incompat_prior, p.no_single_frag_prob, p.no_frag_len_dist, p.no_eff_len_correction) == (0.0, 0, 0, 0)


def _cli(*args):
    return subprocess.run([SB, "quant", *args], capture_output=True, text=True, timeout=60)


@pytest.mark.parametrize("args,msg", [
    (["--incompatPrior", "-0.1"], "--incompatPrior takes a probability"),
    (["--incompatPrior", "abc"], "--incompatPrior takes a probability"),
    (["--incompatPrior", "1e-3x"], "--incompatPrior takes a probability"),
    (["--incompatPrior", "2"], "--incompatPrior takes a probability"),
    (["--noFragLengthDist"], "without also enabling --noEffectiveLengthCorrection"),
])
def test_cli_refusals(tmp_path, args, msg):
    r = _cli("-i", str(tmp_path / "none"), "-l", "ISR", "-1", "a.fq", "-2", "b.fq", "-o", str(tmp_path / "o"), *args)
    assert r.returncode != 0 and msg in r.stderr, r.stderr


@pytest.mark.parametrize("args", [["--incompatPrior", "1e-20"], ["--incompatPrior", "0"], ["--noSingleFragProb"],
                                  ["--noFragLengthDist", "--noEffectiveLengthCorrection"], ["--noEffectiveLengthCorrection"]])
def test_cli_accepts(tmp_path, args):
    """the options parse (the run then fails only at the missing index, with no device needed) and are recorded"""
    out = tmp_path / "o"
    r = _cli("-i", str(tmp_path / "none"), "-l", "ISR", "-1", "a.fq", "-2", "b.fq", "-o", str(out), *args)
    assert "unknown option" not in r.stderr and "--incompatPrior takes" not in r.stderr, r.stderr
    assert "loading the index" in r.stderr, r.stderr
    import json
    info = json.load(open(out / "cmd_info.json"))
    for a in args:
        if a.startswith("--"):
            assert a[2:] in info
    if args[0] == "--incompatPrior":
        assert info["incompatPrior"] == args[1]


def test_cli_eqclasses_mode_takes_them(tmp_path):
    """under `quant -e` the options are mapping options like the others: accepted, no effect on the optimiser"""
    r = _cli("-e", str(tmp_path / "missing.txt"), "-o", str(tmp_path / "o"), "--incompatPrior", "1e-20", "--noSingleFragProb")
    assert "unknown option" not in r.stderr


def _gloo_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from salmon_b200.dist import reduce_partials
    M, nf = 5, 8
    p = dict(mass=np.full(M, np.inf), fld_hist=np.full(nf, -3.0), fld_tot=0.0, fld_prior_hist=np.full(nf, -3.0),
             fld_prior_tot=0.0, fld_min=7, unique_counts=np.zeros(M, np.uint64), total_counts=np.zeros(M, np.uint64),
             cluster_hits=np.zeros(M, np.uint64), cluster_root=np.arange(M, dtype=np.uint32), assigned=100 + rank,
             compatible=40 + 3 * rank)
    g, _ = reduce_partials(p, dist, "cpu")
    q.put((rank, g["assigned"], g["compatible"]))
    dist.destroy_process_group()


def test_dist_sums_the_compatible_count():
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in range(world)]
    for p in procs:
        p.join(60)
    assert sorted(res) == [(0, 201, 83), (1, 201, 83)]


if __name__ == "__main__":
    sys.exit(pytest.main([__file__, "-q"]))
