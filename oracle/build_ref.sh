#!/usr/bin/env bash
# oracle/build_ref.sh -- compile the reference's OWN translation units that build
# standalone (no cmake, no external libraries) from where they lie in a salmon source
# tree ($REF), outputs only into oracle/_ref/ (git-ignored).  tests/golden/make_ref_golden.py
# records what they return as the golden vectors the tests compare against.
#
#   src/xxhash.c   XXH64 used by TranscriptGroup::hash (src/model/TranscriptGroup.cpp:10-15)
#   src/edlib.cpp  Myers edit distance used by recoverOrphans (--recoverOrphans)
#   include/eigen3/unsupported/Eigen/SpecialFunctions  the vendored (Cephes-derived) digamma, through a 5-line shim of ours
#   include/kseq++.hpp  the vendored FASTA/FASTQ parser (klibpp), through a shim of ours that returns the sequence lines
#
# Everything else on the path needs Boost / oneTBB / pufferfish (absent): unbuildable here,
# see DESIGN.md section 2.  Reference SOURCES are never copied into the repo.
set -euo pipefail
REF=${REF:?"set REF to a salmon source tree"}
HERE="$(cd "$(dirname "$0")" && pwd)"
OUT="$HERE/_ref"
mkdir -p "$OUT"
if [ ! -d "$REF" ]; then echo "build_ref: $REF absent, nothing to do"; exit 0; fi
CC=/usr/bin/gcc; CXX=/usr/bin/g++
$CC  -O2 -fPIC -shared -I"$REF/include" -o "$OUT/libxxhash_ref.so" "$REF/src/xxhash.c"
$CXX -O2 -fPIC -shared -std=c++17 -I"$REF/include" -o "$OUT/libedlib_ref.so" "$REF/src/edlib.cpp"
$CXX -O2 -fPIC -shared -std=c++17 -I"$REF/include/eigen3" -o "$OUT/libeigen_digamma_ref.so" "$HERE/ref_shims/eigen_digamma.cpp"
$CXX -O2 -fPIC -shared -std=c++17 -I"$REF/include" -o "$OUT/libkseq_ref.so" "$HERE/ref_shims/kseq_parse.cpp" -lz
echo "build_ref: built $(ls "$OUT")"
