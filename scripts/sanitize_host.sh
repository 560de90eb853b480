#!/bin/bash
# The host library's threaded code under ThreadSanitizer and AddressSanitizer + UBSan (CPU only, no GPU needed): builds the
# host sources with the sanitizer next to tests/tools/sanitize_main.cpp and runs the self-tests. Any report fails the run.
set -e
ROOT=$(cd "$(dirname "$0")/.." && pwd)
H=$ROOT/mashmap_b200/csrc/host
OUT=${TMPDIR:-/tmp}/mm_sanitize
mkdir -p "$OUT"
for san in thread address,undefined; do
  bin=$OUT/t_$(echo $san | tr ',' '_')
  g++ -std=c++17 -O1 -g -fsanitize=$san -fno-sanitize-recover=all -fno-omit-frame-pointer -pthread -w "$ROOT/tests/tools/sanitize_main.cpp" \
      $H/skch_stats.cpp $H/skch_seqio.cpp $H/skch_index.cpp $H/skch_tail.cpp $H/skch_map.cpp $H/skch_args.cpp $H/skch_cview.cpp $H/skch_align.cpp \
      -I"$ROOT/include" -L"$ROOT/mashmap_b200" -lmashmap_nccl -lmashmap_b200 -lz -Wl,-rpath,"$ROOT/mashmap_b200" -o "$bin"
  echo "== -fsanitize=$san"
  TSAN_OPTIONS=halt_on_error=1 ASAN_OPTIONS=detect_leaks=0 "$bin"
done
echo "sanitizer runs clean"
