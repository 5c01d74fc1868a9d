#!/bin/bash
# Builds libnlt_b200.so in-tree for sm_90a (H100) (nvcc cross-compiles without a GPU).  Translation units compile in parallel.
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -I../../include"
OBJS=""
PIDS=""
for f in nlt_gconv nlt_ops nlt_small nlt_tc nlt_barron nlt_ssim nlt_pwx nlt_norm nlt_tiny nlt_wop nlt_pool nlt_lpips ${NLT_EXTRA_SRCS}; do
  if [ ! -f $f.o ] || [ $f.cu -nt $f.o ] || [ nlt_common.cuh -nt $f.o ] || [ nlt_barron_core.h -nt $f.o ] || [ ../../include/nlt_b200.h -nt $f.o ] || [ build.sh -nt $f.o ]; then
    echo "nvcc $f.cu"
    if [ -n "${NLT_PTXAS_V}" ]; then
      $NVCC $FLAGS -Xptxas -v -c $f.cu -o $f.o            # verbose builds stay sequential (readable output)
    else
      ( $NVCC $FLAGS -c $f.cu -o $f.o.tmp && mv $f.o.tmp $f.o ) &
      PIDS="$PIDS $!"
    fi
  fi
  OBJS="$OBJS $f.o"
done
for p in $PIDS; do wait $p || { echo "nvcc failed" >&2; exit 1; }; done
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o libnlt_b200.so $OBJS -lcudart
echo "built $(pwd)/libnlt_b200.so"
