"""Cost of the SAM output (`--writeMappings`): files -> classes with and without it, and the format kernels' device time.

Builds the benchmark's human-scale synthetic transcriptome (bench.py's Stage A shape: synth_txome(seed=44, n_genes=60000),
100-base pairs), writes the reads as FASTQ to a scratch directory (default /dev/shm), then runs sb_quant_files three
ways, alternating: without SAM output, with --writeMappings to a file in the scratch directory, and with
--writeMappings --writeQualities.  Prints one JSON line: pairs/s of each, SAM MB/s, and the format kernels' device ms per
batch (from a run of the SAM sink on the same reads in memory).  Needs a GPU."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from salmon_b200 import _capi  # noqa: E402
from salmon_b200.synth import synth_reads_fast, synth_txome  # noqa: E402


def write_fastq(path, m):
    lut = np.frombuffer(b"ACGTN", dtype=np.uint8)
    n, L = m.shape
    qual = b"I" * L
    with open(path, "wb", buffering=1 << 24) as f:
        seqs = lut[np.minimum(m, 4)]
        for i in range(n):
            f.write(b"@p%d sim\n%s\n+\n%s\n" % (i, seqs[i].tobytes(), qual))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=4_000_000)
    ap.add_argument("--genes", type=int, default=60_000)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--scratch", default="/dev/shm")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    d = tempfile.mkdtemp(prefix="sb_bench_sam_", dir=args.scratch)
    try:
        txps, _ = synth_txome(seed=44, n_genes=args.genes)
        left, right, _ = synth_reads_fast(txps, seed=7, n=args.pairs, read_len=100)
        p1, p2 = os.path.join(d, "r1.fq"), os.path.join(d, "r2.fq")
        write_fastq(p1, left)
        write_fastq(p2, right)
        idx = _capi.Index(txps)
        sam = os.path.join(d, "out.sam")
        runs = {"plain": {}, "sam": dict(write_mappings=sam.encode()),
                "sam_qual": dict(write_mappings=sam.encode(), write_qualities=1)}
        best = {k: None for k in runs}
        sam_bytes = 0
        for _ in range(args.repeats):
            for k, extra in runs.items():
                t0 = time.perf_counter()
                _, s = _capi.quant_files_native(idx, [p1], [p2], None, threads=32, **extra)
                dt = time.perf_counter() - t0
                best[k] = dt if best[k] is None else min(best[k], dt)
                if k == "sam":
                    sam_bytes = os.path.getsize(sam)
                if os.path.exists(sam):
                    os.remove(sam)
        # format kernels alone: the sink on in-memory batches of 262144 pairs
        B = 262_144
        mc = _capi.MapContext(idx, _capi.map_default_params(), batch_cap=B, max_read_len=100)
        sink = _capi.SamSink(idx, sam)
        mc.attach_sam(sink)
        names = [b"p%d" % i for i in range(B)]
        nb = 0
        for b0 in range(0, min(args.pairs, 8 * B) - B + 1, B):
            mc.map_batch_sam(left[b0:b0 + B], right[b0:b0 + B], names)
            nb += 1
        st = sink.stats()
        mc.attach_sam(None)
        sink.close()
        mc.close()
        res = {"gpu": gpu, "pairs": args.pairs,
               "pairs_per_s": {k: args.pairs / v for k, v in best.items()},
               "seconds": best,
               "sam_mb": sam_bytes / 1e6, "sam_mb_per_s": sam_bytes / 1e6 / best["sam"],
               "format_ms_per_batch": st["format_ms"] / max(nb, 1), "format_batches": nb, "batch": B,
               # host wall time per batch of the in-memory run: window copies, waits for a buffer, the writer's fwrite
               "copy_ms_per_batch": st["copy_ms"] / max(nb, 1), "slot_wait_ms_per_batch": st["slot_wait_ms"] / max(nb, 1),
               "write_ms_per_batch": st["write_ms"] / max(nb, 1)}
        print(json.dumps(res))
    finally:
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
