#!/bin/bash
# Development aid: build A/B variants of the TSDF translation unit into build_variants/ (git-ignored, shipped to the GPU box).
# usage: build_variants.sh name1:"-DFOO=1 -DBAR=2" name2:"..."   ;  run with BF_B200_LIB=build_variants/lib_<name>.so
set -e
cd "$(dirname "$0")/.."
mkdir -p build_variants
make -s -C bundlefusion_b200/csrc >/dev/null 2>&1
C=bundlefusion_b200/csrc
FLAGS="-O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-fvisibility=hidden -gencode arch=compute_90a,code=sm_90a -fmad=false -prec-div=true -prec-sqrt=true"
for spec in "$@"; do
  name="${spec%%:*}"; defs="${spec#*:}"
  nvcc $FLAGS $defs -c $C/tsdf.cu -o build_variants/tsdf_$name.o
  nvcc -shared -gencode arch=compute_90a,code=sm_90a -o build_variants/lib_$name.so build_variants/tsdf_$name.o $C/host_api.o $C/solver.o -lcudart
  echo "built build_variants/lib_$name.so  ($defs)"
done
