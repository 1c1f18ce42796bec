#!/bin/bash
# Build A/B variants of libgsx.so that differ only in the compile-time switches of one translation unit.
#   scripts/build_variants.sh gsx_sor.cu  base:""  tma:"-DGSX_KNN_TMA=1"  i64:"-DGSX_KNN_I32=0"
# -> 3dgsconverter_b200/lib/variants/libgsx_<name>.so (not tracked)
set -e
cd "$(dirname "$0")/../3dgsconverter_b200/csrc"
make -j8 >/dev/null
TU=$1; shift
mkdir -p ../lib/variants ../build_var
NV="/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo --fmad=false -prec-div=true -prec-sqrt=true -std=c++17 -Xcompiler -fPIC,-O2 -ccbin /usr/bin/g++"
OBJS=$(ls ../build/*.o | grep -v "/${TU%.cu}.o")
for spec in "$@"; do
  name=${spec%%:*}; flags=${spec#*:}
  $NV $flags -c -o ../build_var/${TU%.cu}_$name.o $TU
  /usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../lib/variants/libgsx_$name.so $OBJS ../build_var/${TU%.cu}_$name.o -ccbin /usr/bin/g++
  echo "built libgsx_$name.so ($flags)"
done
