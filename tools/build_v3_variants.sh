#!/bin/bash
# Builds build/lib_v3_<name>.so: search_kernel_v3 (and its dispatcher) recompiled with tuning macros,
# linked with the default objects.  usage: tools/build_v3_variants.sh name:-DMACRO=1,-DOTHER=2 ...
set -e
cd "$(dirname "$0")/.."
make -C diskann_b200/csrc -j8 > /dev/null
mkdir -p build /tmp/dab_v3
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-O3 -std=c++17 -lineinfo -fmad=false -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-Wall -cudart static"
cd diskann_b200/csrc
others=$(ls *.o | grep -v -e '^search_kernel_v3.o$' -e '^search_kernel.o$')
build_one() {  # name, macros...
  name=$1; shift
  $NVCC $FLAGS "$@" -c -o /tmp/dab_v3/${name}_v3.o search_kernel_v3.cu
  $NVCC $FLAGS "$@" -c -o /tmp/dab_v3/${name}_sk.o search_kernel.cu
  $NVCC -gencode arch=compute_90a,code=sm_90a -shared -cudart static -o ../../build/lib_v3_${name}.so $others /tmp/dab_v3/${name}_v3.o /tmp/dab_v3/${name}_sk.o
  echo "build/lib_v3_${name}.so  ($*)"
}
for spec in "$@"; do
  name=${spec%%:*}; macros=${spec#*:}
  build_one $name $(echo $macros | tr ',' ' ') &
done
wait
