#!/bin/bash
# Builds libmdm_b200.so (sm_90a) in-tree. Used by __graft_entry__.build().
set -e
cd "$(dirname "$0")"
SRC=ml-mdm_b200/csrc
OUT=ml-mdm_b200/mdm_b200/libmdm_b200.so
mkdir -p build
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Iinclude -I$SRC --compiler-options -fPIC"
pids=()
for f in gemm_tc kernels engine net capi diffusion attention token_attention optim; do
  [ -f $SRC/$f.cu ] || continue
  if [ ! -f build/$f.o ] || [ $SRC/$f.cu -nt build/$f.o ] || [ -n "$(find $SRC include -name '*.cuh' -newer build/$f.o -o -name '*.h' -newer build/$f.o 2>/dev/null | head -1)" ]; then
    nvcc $FLAGS -c -o build/$f.o $SRC/$f.cu &
    pids+=($!)
  fi
done
for p in "${pids[@]}"; do wait $p; done
OBJS=""
for f in gemm_tc kernels engine net capi diffusion attention token_attention optim; do [ -f build/$f.o ] && OBJS="$OBJS build/$f.o"; done
# link to a temporary name and rename: a concurrent reader or loader never sees a half-written library
nvcc -arch=sm_90a -shared -o $OUT.tmp $OBJS -lcudart
mv -f $OUT.tmp $OUT
echo "built $OUT"
