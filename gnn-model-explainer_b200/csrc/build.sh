#!/bin/bash
# Builds libgnnx.so (sm_90a only) in-tree: gnn-model-explainer_b200/gnnx/lib/libgnnx.so
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
ROOT="$(cd "$HERE/../.." && pwd)"
OUT="${GNNX_BUILD_OUT:-$HERE/../gnnx/lib}"   # GNNX_BUILD_OUT + GNNX_NVCC_EXTRA: A-B builds for tools/ (e.g. -DGXG_UNROLL=4)
mkdir -p "$OUT"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -I$ROOT/include -I$HERE ${GNNX_NVCC_EXTRA}"
SRCS="api node_mode graph_mode unconstrained khop explain_node explain_graph explain_stream explain_gang explain_var explain_dense forward trace denoise comm densify_graphs"
HEADERS=("$ROOT/include/gnnx.h" "$HERE"/*.cuh)
for f in $SRCS; do
  stale=0
  for dep in "$HERE/$f.cu" "${HEADERS[@]}"; do
    if [ ! -f "$OUT/$f.o" ] || [ "$dep" -nt "$OUT/$f.o" ]; then stale=1; fi
  done
  if [ $stale = 1 ]; then
    $NVCC $FLAGS -c "$HERE/$f.cu" -o "$OUT/$f.o" &
  fi
done
wait
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o "$OUT/libgnnx.so.tmp" $(for f in $SRCS; do echo "$OUT/$f.o"; done) -ldl
mv -f "$OUT/libgnnx.so.tmp" "$OUT/libgnnx.so"   # atomic: a snapshot never sees a half-written library
echo "built $OUT/libgnnx.so"
