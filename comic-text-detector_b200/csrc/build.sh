#!/bin/bash
# Builds libctd_b200.so for sm_90a (cross-compiles without a GPU).  One object per source, compiled in
# parallel; objects live in csrc/_obj (git-ignored).  Extra arguments go to every nvcc compile; CTD_BUILD_DIR=<dir> puts the
# objects and the library of such a variant build into <dir> instead of over the shipped ones.
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -Xcompiler -fvisibility=hidden"
OBJ=${CTD_BUILD_DIR:-_obj}
OUT=${CTD_BUILD_DIR:-..}/libctd_b200.so
mkdir -p "$OBJ"
pids=()
for f in engine pipeline conv_tc conv_ends simt postproc segrep refine_mk resize gather group region_plan region jpeg_plan jpeg jpeg_enc png png_plan png_dec; do
  [ -f $f.cu ] || [ -f $f.cpp ] || continue
  src=$f.cu; [ -f $src ] || src=$f.cpp
  extra=""
  # the crop planner restates OpenCV's double arithmetic operation for operation: no contraction into FMAs
  [ $f = region_plan ] && extra="-Xcompiler -ffp-contract=off"
  if [ ! -f "$OBJ"/$f.o ] || [ $src -nt "$OBJ"/$f.o ] || [ -n "$(find . -maxdepth 1 \( -name '*.h' -o -name '*.cuh' \) -newer "$OBJ"/$f.o)" ] \
     || [ ../../include/ctd_b200.h -nt "$OBJ"/$f.o ]; then
    $NVCC $FLAGS $extra "$@" -c $src -o "$OBJ"/$f.o &
    pids+=($!)
  fi
done
for p in "${pids[@]}"; do wait $p; done
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o "$OUT" "$OBJ"/*.o
