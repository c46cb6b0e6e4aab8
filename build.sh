#!/bin/bash
# Builds libplonk_b200.so (sm_90a, H100) in-tree; translation units compile in parallel.
set -e
cd "$(dirname "$0")"
SRC=${PB200_SRC:-plonk_b200/csrc}
OUT=${PB200_OUT:-plonk_b200/libplonk_b200.so}
OBJ=${PB200_OBJ:-build/obj}
mkdir -p $OBJ
NVFLAGS="-std=c++17 -O3 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC -Xcompiler -O2 $*"
pids=()
for f in capi ntt msm prover ecntt verify debugger pp; do
  nvcc $NVFLAGS -c -o $OBJ/$f.o $SRC/$f.cu &
  pids+=($!)
done
g++ -std=c++17 -O2 -fPIC -c -o $OBJ/host_field.o $SRC/host_field.cpp
g++ -std=c++17 -O2 -fPIC -c -o $OBJ/composer.o $SRC/composer.cpp
g++ -std=c++17 -O2 -fPIC -c -o $OBJ/compress.o $SRC/compress.cpp
for p in "${pids[@]}"; do wait $p; done
nvcc -shared -o "$OUT" $OBJ/capi.o $OBJ/ntt.o $OBJ/msm.o $OBJ/prover.o $OBJ/ecntt.o $OBJ/verify.o $OBJ/debugger.o $OBJ/pp.o $OBJ/host_field.o $OBJ/composer.o $OBJ/compress.o
echo "built $OUT"
