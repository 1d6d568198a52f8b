#!/bin/bash
# An instrumented copy of the library (-DPP_TILE_PROF): k_tile records clock64() at its phase boundaries (thread 0 of every CTA) and the
# cycles / count of the ordered-depth walks; pp_polish_resident prints the per-tile averages on stderr.  Not part of the product build.
#   tools/build_tile_prof.sh && POLYPOLISH_LIB=$PWD/build_ab/libpp_prof.so python bench.py --steps 3 --warmup 2 --no-t3 --no-cpu-baseline 2>&1 | grep "tile prof"
set -e
cd "$(dirname "$0")/.."
mkdir -p build_ab/prof
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-Wall,-Wno-unused-function,-ffp-contract=off -fmad=false -DPP_TILE_PROF"
for f in polish_kernels.cu filter_kernels.cu tok_kernels.cu fasta.cpp sam_pack.cpp filter_pack.cpp host_api.cpp synth.cpp shard.cpp; do
  nvcc $FLAGS -x cu -c polypolish_b200/csrc/$f -o build_ab/prof/${f%.*}.o &
done
wait
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o build_ab/libpp_prof.so build_ab/prof/*.o -lz -lpthread
echo build_ab/libpp_prof.so
