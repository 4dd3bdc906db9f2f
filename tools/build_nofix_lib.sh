#!/bin/bash
# Timing experiment only: the library with the tie guard disabled (TB200_TIE_EPS = -1: no element ever takes the literal rare path,
# so ~2.4e-4 of the bytes may be off by one).  Used through TB200_LIB to measure what the rare path costs the epilogue warps
# (an epilogue warp inside it holds up its accumulator stage).  Also the mutation check of the tie tests:
#   TB200_LIB=build/nofix/libtengine_b200_nofix.so python -m pytest tests/test_gpu_requant_ties.py -m gpu
# must fail every tie-dense case of a fast epilogue (exact-epilogue, LUT and tb200k_* cases still pass).  Never shipped.
set -e
cd "$(dirname "$0")/../tengine_b200/csrc"
rm -rf ../../build/nofix && mkdir -p ../../build/nofix
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-fvisibility=hidden --expt-relaxed-constexpr -DTB200_TIE_EPS=-1.0f"
SRCS=$(sed -n 's/^SRCS := //p' Makefile) # every source of the product library, so that the build links completely
for f in $SRCS; do nvcc $FLAGS -c $f -o ../../build/nofix/${f%.cu}.o & done
for j in $(jobs -p); do wait $j; done # (set -e: a failed compile stops the script)
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../../build/nofix/libtengine_b200_nofix.so ../../build/nofix/*.o -ldl -Xlinker --no-undefined
echo built build/nofix/libtengine_b200_nofix.so
