#!/bin/bash
# Experimental build of the library: scripts/build_variant.sh <suffix> <extra nvcc flags...> -> csrc/libvlfb_<suffix>.so
# (gemm_tc.cu recompiled with the flags, everything else the product's objects: run __graft_entry__.build() first).
# Select it at run time with VLFB_LIB=<path>.
set -e
sfx=$1; shift
cd "$(dirname "$0")/../video-long-term-feature-banks_b200/csrc"
mkdir -p /tmp/variant_build_$sfx
nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -I../../include "$@" -Xptxas -v -c gemm_tc.cu -o /tmp/variant_build_$sfx/gemm_tc.o 2> /tmp/variant_build_$sfx/ptxas.log
nvcc -shared -o libvlfb_$sfx.so /tmp/variant_build_$sfx/gemm_tc.o api.o gemm_simt.o gconv.o ops.o fbo.o bn.o -lcudart
grep -c "Compiling entry" /tmp/variant_build_$sfx/ptxas.log
grep -E "spill" /tmp/variant_build_$sfx/ptxas.log | sort | uniq -c | sort -rn | head -8
