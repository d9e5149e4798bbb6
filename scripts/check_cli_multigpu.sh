#!/bin/bash
# multi-GPU C++ driver (run on a machine with N GPUs): `sb_salmon quant --gpus N` from reads vs one GPU, and
# `sb_salmon quant -e ... --numBootstraps / --numGibbsSamples --gpus N` (samples split over the GPUs) vs one GPU
N=${1:-2}
set -e
python - <<'PY'
import os, sys, gzip, numpy as np
sys.path.insert(0, os.getcwd()); sys.path.insert(0, "tests")
from salmon_b200 import _capi
from salmon_b200._capi import Index
from salmon_b200.synth import synth_txome, synth_reads_fast, synth_eq
os.makedirs("/tmp/mg", exist_ok=True)
txps, _ = synth_txome(seed=61, n_genes=2000)
left, right, truth = synth_reads_fast(txps, seed=62, n=600_000)
names = [f"ENST{i:06d}" for i in range(len(txps))]
idx = Index(txps, names=names)
os.makedirs("/tmp/mg/idx", exist_ok=True)
idx.save("/tmp/mg/idx/sb_index.bin")
lut = np.frombuffer(b"ACGTN", dtype=np.uint8)
for tag, codes in (("1", left), ("2", right)):
    n, L = codes.shape
    rec = np.empty((n, 3 + L + 3 + L + 1), dtype=np.uint8)
    rec[:, 0:3] = np.frombuffer(b"@r\n", dtype=np.uint8); rec[:, 3:3 + L] = lut[codes]
    rec[:, 3 + L:6 + L] = np.frombuffer(b"\n+\n", dtype=np.uint8); rec[:, 6 + L:6 + 2 * L] = ord("I"); rec[:, 6 + 2 * L] = 10
    rec.tofile(f"/tmp/mg/r_{tag}.fq")
eq, proj, eff, uniq = synth_eq(seed=63, C=60000, M=20000, total_count=3_000_000)
_capi.write_eq_classes("/tmp/mg/eq.txt.gz", [f"t{i}" for i in range(eq.n_txps)], eq.off, eq.tids, eq.counts, eq.weights)
PY
EXE=salmon_b200/sb_salmon
$EXE quant -i /tmp/mg/idx -l IU -1 /tmp/mg/r_1.fq -2 /tmp/mg/r_2.fq -o /tmp/mg/one --batch 65536 --maxReadLen 128 2>&1 | tail -2
$EXE quant -i /tmp/mg/idx -l IU -1 /tmp/mg/r_1.fq -2 /tmp/mg/r_2.fq -o /tmp/mg/multi --batch 65536 --maxReadLen 128 --gpus $N 2>&1 | tail -2
$EXE quant -e /tmp/mg/eq.txt.gz -o /tmp/mg/b1 --numBootstraps 8 --seed 5 2>&1 | tail -1
$EXE quant -e /tmp/mg/eq.txt.gz -o /tmp/mg/bN --numBootstraps 8 --seed 5 --gpus $N 2>&1 | tail -1
$EXE quant -e /tmp/mg/eq.txt.gz -o /tmp/mg/g1 --numGibbsSamples 48 --seed 5 2>&1 | tail -1
$EXE quant -e /tmp/mg/eq.txt.gz -o /tmp/mg/gN --numGibbsSamples 48 --seed 5 --gpus $N 2>&1 | tail -1
python - <<'PY'
import gzip, json, numpy as np
def sf(p):
    rows = open(p).read().splitlines()[1:]
    return np.array([float(r.split("\t")[4]) for r in rows]), np.array([float(r.split("\t")[3]) for r in rows])
a1, t1 = sf("/tmp/mg/one/quant.sf"); aN, tN = sf("/tmp/mg/multi/quant.sf")
m1 = json.load(open("/tmp/mg/one/aux_info/meta_info.json")); mN = json.load(open("/tmp/mg/multi/aux_info/meta_info.json"))
r = np.corrcoef(a1, aN)[0, 1]
conds = dict(mapped=m1["num_mapped"] == mN["num_mapped"], processed=m1["num_processed"] == mN["num_processed"],
             total=abs(a1.sum() - aN.sum()) < 1e-3 * a1.sum(), corr=r > 0.9995)
ok = all(conds.values())
print(conds, m1["num_processed"], mN["num_processed"], a1.sum(), aN.sum())
print(f"reads: mapped {m1['num_mapped']} vs {mN['num_mapped']} on {mN['sb_num_gpus']} GPUs, corr(NumReads) {r:.6f}, max |dTPM| {np.abs(t1 - tN).max():.3f} -> {'OK' if ok else 'FAIL'}")
def boots(p, n):
    raw = gzip.open(p + "/aux_info/bootstrap/bootstraps.gz", "rb").read()
    return np.frombuffer(raw, dtype=np.float64).reshape(n, -1)
b1, bN = boots("/tmp/mg/b1", 8), boots("/tmp/mg/bN", 8)
okb = np.array_equal(b1, bN)
print(f"bootstraps split over the GPUs bit-identical to one GPU: {okb} -> {'OK' if okb else 'FAIL'}")
g1, gN = boots("/tmp/mg/g1", 48), boots("/tmp/mg/gN", 48)
eff = np.full(g1.shape[1], 100.0)
tp = lambda g: ((g / eff) / (g / eff).sum(axis=1, keepdims=True)).mean(axis=0)
d = np.abs(tp(g1) - tp(gN)).max()
okg = d < 1e-3 and abs(gN.sum(axis=1) / g1.sum(axis=1) - 1).max() < 1e-6
print(f"Gibbs: posterior-mean TPM fraction, max |split - one GPU| = {d:.2e} (criterion 1e-3) -> {'OK' if okg else 'FAIL'}")
print("ALL", "OK" if (ok and okb and okg) else "FAIL")
PY
