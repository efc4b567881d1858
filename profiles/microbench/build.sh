#!/bin/bash
# builds the microbenchmarks next to their sources (binaries are git-ignored)
set -e
cd "$(dirname "$0")/../.."
python -c "import websplat_b200 as ws; ws.build_library(force=False)"
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -I web-splat_b200/csrc -I include"
nvcc $FLAGS profiles/microbench/sort_vs_cub.cu web-splat_b200/build/radix_sort.o -o profiles/microbench/sort_vs_cub
# look-back width A/B (radix_sort.cu: WS_LB_WIDTH loads in flight per look-back step; the library ships 16)
for w in 4 8; do
  nvcc $FLAGS -lineinfo -Xcompiler -fPIC -DWS_LB_WIDTH=$w -c web-splat_b200/csrc/radix_sort.cu -o /tmp/radix_sort_w$w.o
  nvcc $FLAGS profiles/microbench/sort_vs_cub.cu /tmp/radix_sort_w$w.o -o profiles/microbench/sort_vs_cub_w$w
done
# occupancy A/B: the pass compiled for 3 resident CTAs per SM (80 registers) against the default 2
nvcc $FLAGS -lineinfo -Xcompiler -fPIC -DWS_SORT_CTAS=3 -c web-splat_b200/csrc/radix_sort.cu -o /tmp/radix_sort_c3.o
nvcc $FLAGS profiles/microbench/sort_vs_cub.cu /tmp/radix_sort_c3.o -o profiles/microbench/sort_vs_cub_c3
# ... and for 4 resident CTAs per SM (64 registers, second half of the values loaded inside the reorder)
for w in 4 16; do
  nvcc $FLAGS -lineinfo -Xcompiler -fPIC -DWS_SORT_CTAS=4 -DWS_LB_WIDTH=$w -c web-splat_b200/csrc/radix_sort.cu -o /tmp/radix_sort_c4w$w.o
  nvcc $FLAGS profiles/microbench/sort_vs_cub.cu /tmp/radix_sort_c4w$w.o -o profiles/microbench/sort_vs_cub_c4w$w
done
