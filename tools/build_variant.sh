#!/bin/bash
# A/B builds of the library with different compile-time choices (experiments only; the product is `make`):
#   tools/build_variant.sh minb6 -DENGINE_MINB=6   ->  rapidcfd-dev_b200/lib/libb200ldu_minb6.so
# run with  B200LDU_LIB=rapidcfd-dev_b200/lib/libb200ldu_minb6.so python bench.py ...
set -e
name=$1; shift
cd "$(dirname "$0")/../rapidcfd-dev_b200/csrc"
mkdir -p build_$name
NV="/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo --extended-lambda -Xcompiler -fPIC,-fopenmp,-Wall,-Wno-unused-function -ccbin /usr/bin/g++"
for f in ldu layout comm solvers gamg fv fvmatrix fieldops lduops mules vof; do
  $NV "$@" -c -o build_$name/$f.o $f.cu &
done
wait
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../lib/libb200ldu_$name.so build_$name/*.o -Xcompiler -fopenmp -lnccl -lcudart
rm -rf build_$name
echo built ../lib/libb200ldu_$name.so
