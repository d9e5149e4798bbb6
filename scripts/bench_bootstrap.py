"""Cost of `--bootstrapReproject` (DESIGN.md section 15): sb_bootstrap on the configs[1] table (synth_eq(seed=1),
500 000 classes, 250 000 transcripts, 20 M fragments), VBEM, with and without the reprojection, alternated three times in
one process after one optimise and a short warm-up bootstrap of each kind.  Prints one JSON line per run -- wall time of
the sb_bootstrap call (it synchronises after every replicate), ms per replicate -- with the card's name and power limit
read in the same run.
usage: bench_bootstrap.py [n_boot] [use_vbem]"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from salmon_b200 import EMContext, default_params
from salmon_b200.synth import synth_eq

n_boot = int(sys.argv[1]) if len(sys.argv) > 1 else 100
vbem = int(sys.argv[2]) if len(sys.argv) > 2 else 1
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip().splitlines()
card = gpu[0] if gpu else "unknown"
print("card:", card, flush=True)

eq, proj, eff, uniq = synth_eq(seed=1, C=500_000, M=250_000, total_count=20_000_000)
nmapped = float(eq.counts.sum())
ctx = EMContext(0)
alpha, st, ok = ctx.optimize(eq, default_params(use_vbem=vbem), proj, eff, uniq)
assert ok
print(f"table: {eq.n_classes} classes, {eq.n_txps} transcripts, {eq.nnz} entries; optimise {st.iters} iterations",
      flush=True)
modes = {"plain": default_params(use_vbem=vbem, min_iter=50, max_iter=10000),
         "reproject": default_params(use_vbem=vbem, min_iter=50, max_iter=10000, bootstrap_reproject=1)}
for p in modes.values():
    ctx.bootstrap(p, nmapped, 2, 7)                      # warm-up
for rep in range(3):
    for name, p in modes.items():
        t0 = time.perf_counter()
        boots, okb = ctx.bootstrap(p, nmapped, n_boot, 1234)
        dt = time.perf_counter() - t0
        assert okb and boots.shape == (n_boot, eq.n_txps) and np.isfinite(boots).all()
        print(json.dumps(dict(rep=rep, mode=name, use_vbem=vbem, n_boot=n_boot, seconds=round(dt, 3),
                              ms_per_replicate=round(dt / n_boot * 1e3, 3), card=card)), flush=True)
ctx.close()
