#!/bin/bash
# builds librqb200.so (sm_90a, H100) in-tree next to the sources.  nvcc cross-compiles without a GPU.
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -Xptxas -v"
OBJS=""
for f in *.cu; do
  f=${f%.cu}
  if [ ! -f $f.o ] || [ $f.cu -nt $f.o ] || [ common.cuh -nt $f.o ] || [ tc_common.cuh -nt $f.o ] || [ wgmma.cuh -nt $f.o ] || \
     [ kernels.h -nt $f.o ] || [ ../../include/rqb200.h -nt $f.o ] || [ build.sh -nt $f.o ]; then
    echo "nvcc $f.cu"
    $NVCC $FLAGS -c $f.cu -o $f.o 2> $f.ptxas.log || { cat $f.ptxas.log; exit 1; }
    grep -E "warning|spill|Performance" $f.ptxas.log | grep -v "0 bytes spill" | head -5 || true
  fi
  OBJS="$OBJS $f.o"
done
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o librqb200.so $OBJS -lcudart
echo "built $(pwd)/librqb200.so"
