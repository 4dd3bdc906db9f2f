#!/bin/bash
# Timing experiment only: the library with the tie guard disabled (TB200_TIE_EPS = -1: no element ever takes the literal rare path,
# so ~2.4e-4 of the bytes may be off by one).  Used through TB200_LIB to measure what the rare path costs the epilogue warps
# (an epilogue warp inside it holds up its accumulator stage).  Also the mutation check of the tie tests:
#   TB200_LIB=build/nofix/libtengine_b200_nofix.so python -m pytest tests/test_gpu_requant_ties.py -m gpu
# must fail every tie-dense case of a fast epilogue (exact-epilogue, LUT and tb200k_* cases still pass).  Never shipped.
set -e
cd "$(dirname "$0")/../tengine_b200/csrc"
mkdir -p ../../build/nofix
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-fvisibility=hidden --expt-relaxed-constexpr -DTB200_TIE_EPS=-1.0f"
for f in engine kernels_direct gemm_tcgen05 dw_tma conv_window yolo_detect conv_fp32; do nvcc $FLAGS -c $f.cu -o ../../build/nofix/$f.o & done
wait
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../../build/nofix/libtengine_b200_nofix.so ../../build/nofix/*.o -ldl
echo built build/nofix/libtengine_b200_nofix.so
