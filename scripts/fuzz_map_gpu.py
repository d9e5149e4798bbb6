"""Randomised GPU parity (dev helper, needs a GPU): the CUDA mapping path (both kernel variants) against
the oracle over adversarial transcriptomes, read lengths and option settings -- the GPU twin of
tests/test_map_host.py::test_fuzz_host_logic_against_oracle.  Prints every mismatch, exits 1 if there was one.
usage: fuzz_map_gpu.py [master_seed] [trials]"""
import os
import sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import oracle_lib as oracle
from test_map_host import compare
from salmon_b200._capi import Index, MapContext, map_default_params
from salmon_b200.synth import synth_reads, synth_txome

rng = np.random.default_rng(int(sys.argv[1]) if len(sys.argv) > 1 else 1)
trials = int(sys.argv[2]) if len(sys.argv) > 2 else 60
bad = done = 0
for trial in range(trials):
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
        if max(len(t) for t in txps) < 150:
            txps.append(r.integers(0, 4, size=400, dtype=np.uint8))
    L = int(rng.choice([35, 50, 75, 100, 125, 150]))
    try:
        left, right, _ = synth_reads(txps, seed=seed + 1, n=int(rng.integers(50, 600)), read_len=L,
                                     frag_mean=float(rng.choice([max(L + 20, 120), 250])), frag_sd=float(rng.choice([5, 25])),
                                     sub_rate=float(rng.choice([0.0, 0.01, 0.05])), indel_rate=float(rng.choice([0.0, 0.003, 0.02])),
                                     random_frac=0.1)
    except Exception:  # noqa: BLE001
        continue
    over = {}
    for key, p_use, choices in (("stride", 0.5, [1, 2, 3, 4, 7]), ("max_read_occ", 0.4, [1, 2, 5, 50]),
                                ("max_occs_per_hit", 0.4, [1, 3, 16, 200]), ("range_bins", 0.4, [0, 1, 8]),
                                ("hard_filter", 0.3, [1]), ("min_score_fraction", 0.3, [0.3, 0.8, 0.95]),
                                ("consensus_frac", 0.3, [0.3, 0.9, 1.0]), ("k", 0.3, [15, 21, 25]),
                                ("band", 0.3, [3, 8, 15]), ("max_frag_len", 0.3, [200, 400])):
        if rng.random() < p_use:
            v = rng.choice(choices)
            over[key] = float(v) if isinstance(choices[0], float) else int(v)
    if rng.random() < 0.2:
        over["first_decoy"] = max(1, len(txps) - int(rng.integers(1, 4)))
    k = over.get("k", 31)
    ref = oracle.map_reads(oracle.MapIndex(txps, k=k), oracle.map_params(**over), left, right, 0)
    idx = Index(txps, k=k)
    for variant in (1, 0):
        p = map_default_params(**over)
        ctx = MapContext(idx, p, batch_cap=1024, max_read_len=int(rng.choice([L, L, 160, 256])) if L <= 160 else L)
        ctx.set_option("variant", variant)
        if rng.random() < 0.5:
            ctx.set_option("chunk", int(rng.choice([97, 300, 1024])))
        try:
            ctx.map_batch(left, right)
            compare(ctx.last_alignments(), ref, p.max_read_occ)
        except AssertionError as e:
            bad += 1
            print("MISMATCH trial", trial, "seed", seed, "variant", variant, "L", L, over, str(e)[:200], flush=True)
        ctx.close()
    done += 1
print("trials", done, "mismatches", bad)
sys.exit(1 if bad else 0)
