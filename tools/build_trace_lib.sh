#!/bin/bash
# Debug build of the library with the GEMM event timeline compiled in (TB200_GEMM_TIMELINE); used by tools/gemm_trace.py
# through TB200_LIB.  The product library never carries the timeline code.
set -e
cd "$(dirname "$0")/../tengine_b200/csrc"
mkdir -p ../../build/trace
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-fvisibility=hidden --expt-relaxed-constexpr -DTB200_GEMM_TIMELINE"
for f in engine kernels_direct gemm_tcgen05 dw_tma; do nvcc $FLAGS -c $f.cu -o ../../build/trace/$f.o; done
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../../build/trace/libtengine_b200_trace.so ../../build/trace/*.o
echo built build/trace/libtengine_b200_trace.so
