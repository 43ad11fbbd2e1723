#!/bin/bash
# Developer A/B builds: scripts/build_variant.sh NAME "-DFLAG1 -DFLAG2"  ->  affnet_b200/lib/libaffnet_b200_NAME.so
# (use with AFFNET_B200_LIB=affnet_b200/lib/libaffnet_b200_NAME.so; never shipped, *.so is git-ignored)
set -e
NAME="$1"; EXTRA="$2"
HERE="$(cd "$(dirname "$0")/../affnet_b200/csrc" && pwd)"
OBJ="$HERE/obj_$NAME"; mkdir -p "$OBJ"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
FLAGS="$EXTRA -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC"
pids=()
for f in "$HERE"/*.cu; do
  # verify.cu without fused multiply-adds, as build.sh compiles it: otherwise the variant's RANSACs differ from the shipped ones
  extra=""; [ "$(basename "$f")" = verify.cu ] && extra="-fmad=false"
  ( $NVCC $FLAGS $extra -c "$f" -o "$OBJ/$(basename "${f%.cu}").o" > "$OBJ/$(basename "${f%.cu}").log" 2>&1 || { cat "$OBJ/$(basename "${f%.cu}").log"; exit 1; } ) &
  pids+=($!)
done
for p in "${pids[@]}"; do wait $p; done
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o "$HERE/../lib/libaffnet_b200_$NAME.so" "$OBJ"/*.o -lcudart
echo "built libaffnet_b200_$NAME.so"
