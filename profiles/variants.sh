#!/bin/bash
# Build experimental variants of the library here (no GPU needed): profiles/variants.sh NAME "-DFLAG=..." [NAME2 "flags2" ...]
# Each lands in zstd-rs_b200/variants/libb200zstd_NAME.so (git-ignored, travels with gpurun); run with B200Z_LIB=<path>.
set -e
cd "$(dirname "$0")/../zstd-rs_b200"
mkdir -p variants build/var
ARCH="-gencode arch=compute_90a,code=sm_90a"
FL="$ARCH -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -cudart static"
[ -f build/api.o ] && [ -f build/plan.o ] || make -s
while [ $# -ge 2 ]; do
  NAME=$1; DEFS=$2; shift 2
  nvcc $FL $DEFS -c csrc/kernels.cu -o build/var/kernels_$NAME.o
  nvcc $ARCH -shared -cudart static -o variants/libb200zstd_$NAME.so build/var/kernels_$NAME.o build/api.o build/plan.o -Xlinker --exclude-libs,ALL
  echo built variants/libb200zstd_$NAME.so "($DEFS)"
done
