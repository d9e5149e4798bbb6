#!/bin/bash
# Host-side sanitizer runs of the reader / length-bucketing code (salmon_b200/csrc/ingest.cu, pipeline.cu), no GPU needed:
#   tsan : ThreadSanitizer, built WITHOUT OpenMP (libgomp's barriers are invisible to TSan and drown the report), so the
#          std::thread / mutex / condition-variable logic is what is checked
#   asan : AddressSanitizer + UndefinedBehaviorSanitizer + LeakSanitizer, with OpenMP, plain (memory-mapped) and gzip input
# usage: scripts/sanitize_reader/run.sh   (from the repository root)
set -e
HERE=$(cd "$(dirname "$0")" && pwd); ROOT=$(cd "$HERE/../.." && pwd); W=$(mktemp -d)
python - "$W" <<'PY'
import sys, numpy as np
rng = np.random.default_rng(3); lut = np.frombuffer(b"ACGT", dtype=np.uint8); n = 60000
def write(path, lens):
    with open(path, "wb") as f:
        for i, L in enumerate(lens):
            f.write(b"@r%d\n%s\n+\n%s\n" % (i, lut[rng.integers(0, 4, size=L)].tobytes(), b"I" * L))
l1 = np.where(rng.random(n) < 0.7, 100, rng.integers(20, 101, size=n)); l2 = np.where(rng.random(n) < 0.7, l1, rng.integers(20, 101, size=n))
write(sys.argv[1] + "/t_1.fq", l1); write(sys.argv[1] + "/t_2.fq", l2)
M, C = 300, 2000
with open(sys.argv[1] + "/eq.txt", "w") as f:
    f.write(f"{M}\n{C}\n" + "".join(f"tx{i}\n" for i in range(M)))
    for c in range(C):
        k = int(rng.integers(1, 7)); t = np.sort(rng.choice(M, size=k, replace=False)); w = rng.random(k)
        f.write(f"{k}\t" + "\t".join(map(str, t)) + "\t" + "\t".join(f"{x:.6g}" for x in w) + f"\t{int(rng.integers(1, 99))}\n")
    f.write("".join(f"tx{i}\t{100 + i}.5\n" for i in range(0, M, 2)))
with open(sys.argv[1] + "/t.fa", "w") as f:
    for i in range(200):
        s = lut[rng.integers(0, 4, size=int(rng.integers(20, 900)))].tobytes().decode() + ("A" * 30 if i % 5 == 0 else "")
        if i % 17 == 1: s = prev
        prev = s
        f.write(f">ENST{i}|g{i // 3} d\n" + "\n".join(s[j:j + 70] for j in range(0, len(s), 70)) + "\n")
PY
gzip -k "$W/t_1.fq" "$W/t_2.fq"
SRC="$HERE/driver.cpp $ROOT/salmon_b200/csrc/ingest.cu $ROOT/salmon_b200/csrc/pipeline.cu $HERE/stubs.cu"
NV="nvcc -O1 -g -std=c++17 -gencode arch=compute_90a,code=sm_90a"
$NV -Xcompiler -fsanitize=thread -Xcompiler -Wno-unknown-pragmas -o "$W/tsan" $SRC -lz -ltsan
$NV -Xcompiler -fsanitize=address -Xcompiler -fsanitize=undefined -Xcompiler -fopenmp -o "$W/asan" $SRC -lgomp -lz -lasan -lubsan
echo "== tsan"; TSAN_OPTIONS=halt_on_error=1 "$W/tsan" "$W/t_1.fq" "$W/t_2.fq"
echo "== tsan gzip (parallel inflate)"; TSAN_OPTIONS=halt_on_error=1 SB_READS_INFLATERS=4 "$W/tsan" "$W/t_1.fq.gz" "$W/t_2.fq.gz"
echo "== asan plain"; ASAN_OPTIONS=detect_leaks=1:protect_shadow_gap=0 "$W/asan" "$W/t_1.fq" "$W/t_2.fq" "$W/eq.txt" "$W/t.fa"
echo "== asan gzip"; SB_READS_INFLATERS=4 ASAN_OPTIONS=detect_leaks=1:protect_shadow_gap=0 "$W/asan" "$W/t_1.fq.gz" "$W/t_2.fq.gz"
rm -rf "$W"; echo "sanitizers clean"
