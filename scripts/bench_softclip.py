"""Cost of the DP scoring modes (--softclipOverhangs = 1, --softclip = 2): 2 M pairs of 100 bases on the synthetic index
of scripts/bench_rescue.py, with 0 %, 10 % and 50 % of the pairs reading 20-30 bases into the adapter on both mates,
modes 0, 1 and 2 alternated three times in one process.  Prints one JSON line per run -- device time of sb_map_batch,
pairs/s, alignments the ungapped shortcut could not settle (full_dp), the mapping rate -- and the card's name and power
limit.
usage: bench_softclip.py [n_genes] [n_pairs] [batch]"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np

from salmon_b200._capi import Index, MapContext, map_default_params, pin
from salmon_b200.synth import flatten_txome, synth_reads_fast, synth_txome
from softclip_ref import with_adapters

n_genes = int(sys.argv[1]) if len(sys.argv) > 1 else 20000
n_pairs = int(sys.argv[2]) if len(sys.argv) > 2 else 2_000_000
batch = int(sys.argv[3]) if len(sys.argv) > 3 else 262144
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip().splitlines()
card = gpu[0] if gpu else "unknown"
print("card:", card, flush=True)
txps, _ = synth_txome(seed=44, n_genes=n_genes)
flat = flatten_txome(txps)
left, right, _ = synth_reads_fast(txps, seed=7, n=n_pairs, flat=flat)
idx = Index(txps)
L = left.shape[1]
print(f"txome {len(txps)} transcripts, {flat[1].shape[0] / 1e6:.1f} Mb; {n_pairs} pairs of {L} bases", flush=True)
al, ar = left.copy(), right.copy()
pin(al); pin(ar)          # registered once, refilled per adapter fraction
for frac in (0.0, 0.1, 0.5):
    al[:], ar[:] = with_adapters(left, right, np.random.default_rng(3), frac)[:2]
    for rep in range(3):
        for mode in (0, 1, 2):
            ctx = MapContext(idx, map_default_params(softclip=mode), batch_cap=batch, max_read_len=L)
            ctx.map_batch(al[:batch], ar[:batch])        # warm-up
            ctx.reset()
            dev = 0.0
            full_dp = mapped = 0
            for s in range(0, n_pairs, batch):
                st = ctx.map_batch(al[s:s + batch], ar[s:s + batch])
                dev += st.device_ms; full_dp += st.full_dp; mapped += st.mapped
            print(json.dumps(dict(adapter_frac=frac, rep=rep, softclip=mode, device_ms=round(dev, 2),
                                  pairs_per_s=round(n_pairs / dev * 1e3), full_dp=full_dp,
                                  mapping_rate=round(mapped / n_pairs, 5), card=card)), flush=True)
            ctx.close()
