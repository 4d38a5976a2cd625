#!/bin/bash
# Build A/B variants of librsb.so (same sources, one -D switch each) for kernel experiments on the GPU box.
#   usage: build_variants.sh NAME "-DFLAG ..." [NAME2 "-D..."]...
# Output: retrieval_scaling_b200/_variants/librsb_NAME.so ; use with RSB_LIBRARY=<path> python bench.py ...
set -e
cd "$(dirname "$0")/.."
OUT=retrieval_scaling_b200/_variants
mkdir -p "$OUT"
FLAGS="-O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC --expt-relaxed-constexpr"
while [ $# -ge 2 ]; do
  NAME=$1; DEFS=$2; shift 2
  TMP=$(mktemp -d)
  # the library's source list (retrieval_scaling_b200/_build.py), so a variant links every object librsb.so has
  for s in $(python3 -c "import sys; sys.path.insert(0, 'retrieval_scaling_b200'); import _build; print(' '.join(_build.SOURCES))"); do
    nvcc $FLAGS $DEFS -c retrieval_scaling_b200/csrc/$s -o $TMP/${s%.cu}.o &
  done
  wait
  nvcc -shared -o $OUT/librsb_$NAME.so $TMP/*.o -lcudart
  rm -rf $TMP
  echo "built $OUT/librsb_$NAME.so ($DEFS)"
done
