#!/bin/bash
# Builds libkfac_b200.so (sm_90a, H100) in-tree.  Used by __graft_entry__.build().
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
ARCH="-gencode arch=compute_90a,code=sm_90a"
FLAGS="$ARCH -O3 -lineinfo -std=c++17 -Xcompiler -fPIC"
OBJS=""
for f in api gemm_simt gemm_tc gemm_grouped factor eigh sytrd stedc eigh_direct precond ekfac norm reduce tied recurrent embedding_bag $EXTRA_SRCS; do
  if [ ! -f $f.o ] || [ $f.cu -nt $f.o ] || [ common.cuh -nt $f.o ] || [ tc_common.cuh -nt $f.o ] || [ tc_pipeline.cuh -nt $f.o ] || [ ../../include/kfac_b200.h -nt $f.o ] || [ eigh_direct.cuh -nt $f.o ] || [ gemm_grouped.cuh -nt $f.o ] || [ build.sh -nt $f.o ]; then
    echo "nvcc $f.cu"
    $NVCC $FLAGS ${PTXAS_V:+-Xptxas -v} -c $f.cu -o $f.o
  fi
  OBJS="$OBJS $f.o"
done
# link to a temporary name and rename: a concurrent reader never sees a half-written library
$NVCC $ARCH -shared -o libkfac_b200.so.tmp $OBJS -lcudart_static -ldl -lrt -lpthread
mv -f libkfac_b200.so.tmp libkfac_b200.so
echo "built $(pwd)/libkfac_b200.so"
