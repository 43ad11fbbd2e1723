#!/bin/bash
# Builds affnet_b200/lib/libaffnet_b200.so for sm_90a (H100; nvcc cross-compiles without a GPU).
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
OUT="$HERE/../lib"
mkdir -p "$OUT" "$HERE/obj"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
FLAGS="${AG_EXTRA_FLAGS:-} -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -Xptxas -v"
pids=()
for f in "$HERE"/*.cu; do
  o="$HERE/obj/$(basename "${f%.cu}").o"
  stale=0
  for d in "$f" "$HERE"/*.cuh "$HERE/../../include/affnet_b200.h"; do [ "$d" -nt "$o" ] && stale=1; done
  # verify.cu: no fused multiply-adds, so its fp64 decisions equal those of the numpy restatement (tests/oracle_ransac.py)
  extra=""; [ "$(basename "$f")" = verify.cu ] && extra="-fmad=false"
  if [ ! -f "$o" ] || [ $stale = 1 ]; then
    ( $NVCC $FLAGS $extra -c "$f" -o "$o" > "$o.log" 2>&1 || { cat "$o.log"; exit 1; } ) &
    pids+=($!)
  fi
done
fail=0
for p in "${pids[@]}"; do wait $p || fail=1; done
if [ $fail = 1 ]; then echo "build failed" >&2; rm -f "$HERE"/obj/*.o.failed; for l in "$HERE"/obj/*.o.log; do grep -l "error" "$l" >/dev/null 2>&1 && rm -f "${l%.log}"; done; exit 1; fi
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o "$OUT/libaffnet_b200.so" "$HERE"/obj/*.o -lcudart
echo "built $OUT/libaffnet_b200.so"
