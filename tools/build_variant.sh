#!/bin/bash
# builds a variant of libals_b200.so with extra nvcc defines into variants/<name>.so (A/B runs: ALS_B200_LIB=variants/<name>.so)
#   tools/build_variant.sh long13 -DALS_LONG_MIN_BLOCKS=13
#   VARIANT_SRC=topk tools/build_variant.sh name -DNAME=value      (recompiles that source instead of cholesky.cu)
set -e
NAME=$1; shift
ROOT=$(cd "$(dirname "$0")/.." && pwd)
OUT=$ROOT/variants; mkdir -p $OUT/obj_$NAME
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-fvisibility=hidden -ccbin /usr/bin/g++ --expt-relaxed-constexpr -I /usr/include"
SRC=${VARIANT_SRC:-cholesky}
for f in api csr gen gramian cholesky cholesky_tc cholesky_short dense cholesky_wide cholesky_xwide cg loss topk topk_tc comm; do
  if [ "$f" = "$SRC" ]; then
    /usr/local/cuda/bin/nvcc $FLAGS "$@" -Xptxas -v -c $ROOT/implicit_b200/csrc/$f.cu -o $OUT/obj_$NAME/$f.o 2>&1 | grep -E "cholesky_half_kernelILi4" -A2 | grep -E "Used|spill" | head -2
  else
    cp $ROOT/implicit_b200/csrc/_obj/$f.o $OUT/obj_$NAME/$f.o
  fi
done
/usr/local/cuda/bin/nvcc -shared -o $OUT/$NAME.so $OUT/obj_$NAME/*.o -lcudart -ldl -lpthread -ccbin /usr/bin/g++
echo built $OUT/$NAME.so
