"""Cost of orphan rescue (--recoverOrphans): 2 M pairs on the synthetic index of scripts/bench_map.py, with 0 %, 2 % and
5 % of the pairs given a planted unseedable mate (substitutions spaced so that no k-mer survives), the option off and on
alternated three times in one process.  Prints pairs/s (device time of sb_map_batch), the rescue kernels' device time
(CUDA events), mate searches per second of rescue time, and the card's name and power limit.
usage: bench_rescue.py [n_genes] [n_pairs] [batch]"""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from salmon_b200._capi import Index, MapContext, map_default_params, pin
from salmon_b200.synth import flatten_txome, synth_reads_fast, synth_txome

n_genes = int(sys.argv[1]) if len(sys.argv) > 1 else 20000
n_pairs = int(sys.argv[2]) if len(sys.argv) > 2 else 2_000_000
batch = int(sys.argv[3]) if len(sys.argv) > 3 else 262144
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip().splitlines()
print("card:", gpu[0] if gpu else "unknown", flush=True)
txps, _ = synth_txome(seed=44, n_genes=n_genes)
flat = flatten_txome(txps)
left, right, _ = synth_reads_fast(txps, seed=7, n=n_pairs, flat=flat)
idx = Index(txps)
L = left.shape[1]
print(f"txome {len(txps)} transcripts, {flat[1].shape[0] / 1e6:.1f} Mb; {n_pairs} pairs of {L} bases", flush=True)
rng = np.random.default_rng(3)
r2 = right.copy()
pin(left); pin(r2)
for frac in (0.0, 0.02, 0.05):
    r2[:] = right
    sel = rng.choice(n_pairs, int(frac * n_pairs), replace=False)
    for q in range(int(rng.integers(3, 8)), L, 25):    # kill every 31-mer of the chosen mates
        r2[sel, q] = (r2[sel, q] + 1) % 4
    for rep in range(3):
        for ro in (0, 1):
            ctx = MapContext(idx, map_default_params(recover_orphans=ro), batch_cap=batch, max_read_len=L)
            ctx.map_batch(left[:batch], r2[:batch])        # warm-up
            ctx.reset()
            dev = resc = 0.0
            searches = rescued = mapped = 0
            for s in range(0, n_pairs, batch):
                st = ctx.map_batch(left[s:s + batch], r2[s:s + batch])
                dev += st.device_ms; resc += st.rescue_kernel_ms; searches += st.rescue_searches
                rescued += st.orphans_rescued; mapped += st.mapped
            print(f"orphans {frac * 100:.0f}% rep {rep} rescue {'on ' if ro else 'off'}: {n_pairs / dev * 1e3 / 1e6:.3f} M pairs/s "
                  f"(device {dev:.1f} ms), rescue kernels {resc:.2f} ms, {searches} searches"
                  f"{f' ({searches / resc * 1e3 / 1e6:.2f} M searches/s)' if resc > 0 else ''}, {rescued} rescued, "
                  f"{mapped} mapped", flush=True)
            ctx.close()
