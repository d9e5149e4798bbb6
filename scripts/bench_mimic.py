"""Cost of the Bowtie2-mimicking presets (DESIGN.md section 14): 2 M pairs of 100 bases on the 60 000-gene synthetic
transcriptome, the default options, --mimicBT2 and --mimicStrictBT2 alternated three times in one process; then
max_read_occ 200 against 1000 (alternated three times) on a tandem-repeat workload, where a tenth of the pairs come from
tandem repeats and have hundreds of joint hits.  Prints one JSON line per run -- device time of sb_map_batch, M pairs/s,
alignments the banded DP scored (full_dp), the mapping rate -- with the card's name and power limit read in the same run.
usage: bench_mimic.py [n_genes] [n_pairs] [batch]"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np

from mimic_ref import tandem_txome
from salmon_b200._capi import Index, MapContext, map_default_params, map_mimic_bt2, pin
from salmon_b200.synth import flatten_txome, synth_reads_fast, synth_txome

n_genes = int(sys.argv[1]) if len(sys.argv) > 1 else 60000
n_pairs = int(sys.argv[2]) if len(sys.argv) > 2 else 2_000_000
batch = int(sys.argv[3]) if len(sys.argv) > 3 else 262144
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip().splitlines()
card = gpu[0] if gpu else "unknown"
print("card:", card, flush=True)


def run(idx, left, right, p, **tags):
    L = left.shape[1]
    ctx = MapContext(idx, p, batch_cap=batch, max_read_len=L)
    ctx.map_batch(left[:batch], right[:batch])        # warm-up
    ctx.reset()
    dev = 0.0
    full_dp = mapped = 0
    for s in range(0, left.shape[0], batch):
        st = ctx.map_batch(left[s:s + batch], right[s:s + batch])
        dev += st.device_ms; full_dp += st.full_dp; mapped += st.mapped
    ctx.close()
    print(json.dumps(dict(**tags, device_ms=round(dev, 2), m_pairs_per_s=round(left.shape[0] / dev * 1e-3, 3),
                          full_dp=full_dp, mapping_rate=round(mapped / left.shape[0], 5), card=card)), flush=True)


txps, _ = synth_txome(seed=44, n_genes=n_genes)
flat = flatten_txome(txps)
left, right, _ = synth_reads_fast(txps, seed=7, n=n_pairs, flat=flat)
pin(left); pin(right)
idx = Index(txps)
print(f"txome {len(txps)} transcripts, {flat[1].shape[0] / 1e6:.1f} Mb; {n_pairs} pairs of {left.shape[1]} bases", flush=True)
modes = {"default": map_default_params(), "mimicBT2": map_mimic_bt2(map_default_params()),
         "mimicStrictBT2": map_mimic_bt2(map_default_params(), strict=True)}
for rep in range(3):
    for name, p in modes.items():
        run(idx, left, right, p, workload="synthetic", rep=rep, mode=name)
del idx, left, right

# tandem repeats: 200 repeat transcripts (60-base unit x 50) among ordinary ones; 10 % of the pairs from the repeats
rng = np.random.default_rng(11)
tx = [t for s in range(200) for t in tandem_txome(seed=1000 + s, n_plain=0)] + txps[:20000]
off, codes = flatten_txome(tx)
L, frag = 100, 250
rep_pair = rng.random(n_pairs) < 0.1
t = np.where(rep_pair, rng.integers(0, 200, n_pairs), rng.integers(200, len(tx), n_pairs))
tlen = (off[t + 1] - off[t]).astype(np.int64)
ok = tlen >= frag + 400
t, tlen, rep_pair = t[ok], tlen[ok], rep_pair[ok]
lo = np.where(rep_pair, 200, 0)
pos = lo + (rng.random(t.shape[0]) * (tlen - 2 * lo - frag + 1)).astype(np.int64)
base = off[t].astype(np.int64) + pos
a = codes[base[:, None] + np.arange(L)]
b = 3 - codes[base[:, None] + frag - 1 - np.arange(L)]
swap = rng.random(t.shape[0]) < 0.5
tl = np.ascontiguousarray(np.where(swap[:, None], b, a).astype(np.uint8))
tr = np.ascontiguousarray(np.where(swap[:, None], a, b).astype(np.uint8))
pin(tl); pin(tr)
idx = Index(tx)
print(f"tandem workload: {len(tx)} transcripts, {tl.shape[0]} pairs, {rep_pair.mean():.3f} from repeats", flush=True)
for rep in range(3):
    for cap in (200, 1000):
        run(idx, tl, tr, map_default_params(max_read_occ=cap), workload="tandem", rep=rep, max_read_occ=cap)
