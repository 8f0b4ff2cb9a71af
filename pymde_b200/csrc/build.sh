#!/bin/bash
# Build libmde_b200.so (sm_90a, H100) in-tree.  Usage: pymde_b200/csrc/build.sh
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
OUT="$HERE/../libmde_b200.so"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC"
mkdir -p "$HERE/_build"
pids=()
for f in mde_edges mde_tiled mde_pull mde_ell mde_project mde_project_wide mde_solver mde_graph mde_knn mde_knn_sparse mde_knn_approx mde_knn_graph; do
  ( $NVCC $FLAGS -c "$HERE/$f.cu" -o "$HERE/_build/$f.o" ) &
  pids+=($!)
done
for p in "${pids[@]}"; do wait $p; done
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o "$OUT" "$HERE/_build/mde_edges.o" "$HERE/_build/mde_tiled.o" "$HERE/_build/mde_pull.o" "$HERE/_build/mde_ell.o" "$HERE/_build/mde_project.o" "$HERE/_build/mde_project_wide.o" "$HERE/_build/mde_solver.o" "$HERE/_build/mde_graph.o" "$HERE/_build/mde_knn.o" "$HERE/_build/mde_knn_sparse.o" "$HERE/_build/mde_knn_approx.o" "$HERE/_build/mde_knn_graph.o" -lcudart
echo "built $OUT"
