#!/bin/bash
# Builds build/lib_<name>.so: the listed sources recompiled with extra macros, linked with the default objects of
# every other source.  Selected at run time with DAB_LIB_PATH.
# usage: tools/build_variant.sh name src1.cu[,src2.cu...] [-DMACRO=1 ...]
set -e
cd "$(dirname "$0")/.."
name=$1; srcs=$(echo $2 | tr ',' ' '); shift 2
make -C diskann_b200/csrc -j16 > /dev/null
mkdir -p build /tmp/dab_var/$name
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-O3 -std=c++17 -lineinfo -fmad=false -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-Wall -cudart static"
cd diskann_b200/csrc
objs=""
for o in *.o; do
  keep=1; for s in $srcs; do [ "${s%.cu}.o" = "$o" ] && keep=0; done
  [ $keep = 1 ] && objs="$objs $o"
done
for s in $srcs; do
  $NVCC $FLAGS "$@" -c -o /tmp/dab_var/$name/${s%.cu}.o $s &
done
wait
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -cudart static -o ../../build/lib_${name}.so $objs /tmp/dab_var/$name/*.o -ldl
echo "build/lib_${name}.so  ($srcs $*)"
