#!/bin/bash
# Debug build of the library with the GEMM event timeline compiled in (TB200_GEMM_TIMELINE); used by tools/gemm_trace.py
# through TB200_LIB.  The product library never carries the timeline code.
set -e
cd "$(dirname "$0")/../tengine_b200/csrc"
rm -rf ../../build/trace && mkdir -p ../../build/trace
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-fvisibility=hidden --expt-relaxed-constexpr -DTB200_GEMM_TIMELINE"
SRCS=$(sed -n 's/^SRCS := //p' Makefile) # every source of the product library, so that the debug build links completely
for f in $SRCS; do nvcc $FLAGS -c $f -o ../../build/trace/${f%.cu}.o & done
for j in $(jobs -p); do wait $j; done # (set -e: a failed compile stops the script)
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../../build/trace/libtengine_b200_trace.so ../../build/trace/*.o -Xlinker --no-undefined
echo built build/trace/libtengine_b200_trace.so
