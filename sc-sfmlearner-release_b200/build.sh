#!/bin/bash
# Build libscsfm.so (sm_90a only) in-tree.  nvcc cross-compiles without a GPU.  Every source is recompiled
# (in parallel, ~40 s): timestamp-based skipping proved unreliable with sub-second edits.
set -e
cd "$(dirname "$0")"
OUT=scsfm/libscsfm.so
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
mkdir -p build
OBJS=""
PIDS=""
for s in csrc/*.cu; do
  o=build/$(basename ${s%.cu}).o
  $NVCC -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC ${NVCC_EXTRA} -c $s -o $o &
  PIDS="$PIDS $!"
  OBJS="$OBJS $o"
done
for p in $PIDS; do wait $p; done
$NVCC -shared -gencode arch=compute_90a,code=sm_90a -o $OUT $OBJS -lcudart
echo "built $OUT"
