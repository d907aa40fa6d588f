#!/bin/bash
# Builds pb_bss_b200/libpbb.so for sm_90a (H100; cross-compiles without a GPU).
set -euo pipefail
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
ARCH="-gencode arch=compute_90a,code=sm_90a"
FLAGS="$ARCH -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Xptxas -v --expt-relaxed-constexpr ${PBB_EXTRA_FLAGS:-}"
OUT=${PBB_OUT:-../libpbb.so}
BUILD=${PBB_BUILD_DIR:-build}
mkdir -p $BUILD
# objects built with other flags (another architecture) are not reused
if [ "$(cat $BUILD/flags 2>/dev/null)" != "$FLAGS" ]; then rm -f $BUILD/*.o; echo "$FLAGS" > $BUILD/flags; fi
pids=()
for src in api_cacgmm api_linalg api_dhtv api_integration api_mask api_transform api_srmr api_bss_eval api_stoi api_sxr api_kmeans api_mm_utils api_wpe prof; do
  if [ ! -f $BUILD/$src.o ] || [ $src.cu -nt $BUILD/$src.o ] || [ -n "$(find . -maxdepth 1 -name '*.cuh' -newer $BUILD/$src.o)" ] || [ ../../include/pbb.h -nt $BUILD/$src.o ]; then
    ( $NVCC $FLAGS -c $src.cu -o $BUILD/$src.o > $BUILD/$src.log 2>&1 || { cat $BUILD/$src.log; exit 1; } ) &
    pids+=($!)
  fi
done
for p in "${pids[@]:-}"; do [ -n "$p" ] && wait $p; done
$NVCC $ARCH -shared -o $OUT $BUILD/*.o -lcudart_static -lpthread -ldl -lrt
echo "built $(realpath $OUT)"
