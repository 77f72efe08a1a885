#!/bin/bash
# Builds experiment variants of the library next to the product build:
#   tools/build_variants.sh NAME "-DATL_WIND_B=4 -DATL_WIND_MINB=5" [file.cu ...]
# -> build_variants/libatlite_b200_NAME.so (git-ignored, travels with gpurun); only the listed
# sources (default wind.cu) are recompiled with the extra flags, the other objects are reused.
set -e
NAME=$1; FLAGS=$2; shift 2
FILES=${@:-wind.cu}
cd "$(dirname "$0")/../atlite_b200/csrc"
mkdir -p ../../build_variants/obj_$NAME
OBJS=""
for f in plan wind pv heat pointwise csp host_stream indicator era5 decode; do
  if [[ " $FILES " == *" $f.cu "* ]]; then
    nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -ftz=true -prec-div=false -prec-sqrt=false \
      -Xcompiler -fPIC -Xptxas -v $FLAGS -c $f.cu -o ../../build_variants/obj_$NAME/$f.o 2> ../../build_variants/obj_$NAME/$f.ptxas.log
    OBJS="$OBJS ../../build_variants/obj_$NAME/$f.o"
  else
    OBJS="$OBJS $f.o"
  fi
done
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../../build_variants/libatlite_b200_$NAME.so $OBJS -lz
echo built build_variants/libatlite_b200_$NAME.so
