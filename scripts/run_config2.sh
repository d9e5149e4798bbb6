#!/bin/bash
# BASELINE.json configs[2] as written: human-scale cDNA-only index (synth_txome seed 44, 60000 genes), 20 M synthetic 2x100 bp
# IU pairs, one GPU: `sb_salmon quant` from FASTQ files to quant.sf in ONE timed run.  Files live in /dev/shm.
set -e
N=${1:-20000000}
D=/dev/shm/sb_cfg2; mkdir -p $D/idx gpurun_out
python - <<PY
import os, sys, time, numpy as np
sys.path.insert(0, os.getcwd())
from salmon_b200._capi import Index
from salmon_b200.synth import synth_txome, synth_reads_fast, flatten_txome
t0 = time.time()
txps, _ = synth_txome(seed=44, n_genes=60000); flat = flatten_txome(txps)
names = [f"ENST{i:08d}.1" for i in range(len(txps))]
idx = Index(txps, names=names); idx.save("$D/idx/sb_index.bin")
print(f"index: {len(txps)} transcripts, {flat[1].shape[0]/1e6:.0f} Mb, {time.time()-t0:.0f} s", flush=True)
lut = np.frombuffer(b"ACGTN", dtype=np.uint8)
n, step = $N, 4_000_000
f = [open(f"$D/r_{t}.fq", "wb") for t in (1, 2)]
t0 = time.time()
for s in range(0, n, step):
    m = min(step, n - s)
    left, right, _ = synth_reads_fast(txps, seed=7 + s, n=m, read_len=100, flat=flat)
    for fh, codes in zip(f, (left, right)):
        L = codes.shape[1]
        rec = np.empty((m, 3 + L + 3 + L + 1), dtype=np.uint8)
        rec[:, 0:3] = np.frombuffer(b"@r\n", dtype=np.uint8); rec[:, 3:3 + L] = lut[codes]
        rec[:, 3 + L:6 + L] = np.frombuffer(b"\n+\n", dtype=np.uint8); rec[:, 6 + L:6 + 2 * L] = ord("I"); rec[:, 6 + 2 * L] = 10
        rec.tofile(fh)
for fh in f: fh.close()
print(f"reads: {n} pairs written in {time.time()-t0:.0f} s", flush=True)
PY
ls -la $D
python - <<PY > gpurun_out/config2_run.txt 2>&1 || true
import subprocess, time, resource
t0 = time.time()
r = subprocess.run("salmon_b200/sb_salmon quant -i $D/idx -l IU -1 $D/r_1.fq -2 $D/r_2.fq -o $D/out -p 32 --maxReadLen 128".split(),
                   stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
print(r.stdout)
ru = resource.getrusage(resource.RUSAGE_CHILDREN)
print(f"exit {r.returncode}  Elapsed wall {time.time() - t0:.2f} s  user {ru.ru_utime:.1f} s  sys {ru.ru_stime:.1f} s  Maximum resident {ru.ru_maxrss / 1024:.0f} MiB")
PY
tail -30 gpurun_out/config2_run.txt
head -3 $D/out/quant.sf; wc -l $D/out/quant.sf; cat $D/out/aux_info/meta_info.json | head -40 > gpurun_out/config2_meta_info.json
if [ -n "$GZ" ]; then
  # the same reads as .fastq.gz (the first $GZ pairs): parallel inflate (pgzip.h) against one zlib thread per file
  head -n $((GZ * 4)) $D/r_1.fq | gzip -1 > $D/g_1.fq.gz &
  head -n $((GZ * 4)) $D/r_2.fq | gzip -1 > $D/g_2.fq.gz
  wait
  ls -la $D/*.gz
  for INF in "" 1; do
    echo "== .fastq.gz, SB_READS_INFLATERS=${INF:-default}"
    SB_READS_PROFILE=1 env ${INF:+SB_READS_INFLATERS=$INF} salmon_b200/sb_salmon quant -i $D/idx -l IU -1 $D/g_1.fq.gz -2 $D/g_2.fq.gz -o $D/outg$INF -p 32 --maxReadLen 128 2>&1 | grep -E "sb_reads|sb_quant|mapping|index loaded|observed" | tee -a gpurun_out/config2_gz.txt
  done
  cmp $D/outg/quant.sf $D/outg1/quant.sf && echo "quant.sf identical for both inflate paths" | tee -a gpurun_out/config2_gz.txt
fi
rm -rf $D
