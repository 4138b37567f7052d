#!/bin/bash
# Diagnostic build of the library: gemm_tc.cu with -DVLFB_TRACE (per-CTA clock64 timelines, scripts/trace_gemm.py).
# Everything else is the product's objects, so run __graft_entry__.build() first.
set -e
cd "$(dirname "$0")/../video-long-term-feature-banks_b200/csrc"
mkdir -p /tmp/trace_build
for f in api gemm_tc; do
  nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -I../../include -DVLFB_TRACE=1 -c $f.cu -o /tmp/trace_build/$f.o
done
nvcc -shared -o libvlfb_trace.so /tmp/trace_build/api.o /tmp/trace_build/gemm_tc.o gemm_simt.o ops.o fbo.o -lcudart
python - <<'PY'
import ctypes, os
l = ctypes.CDLL(os.path.abspath('libvlfb_trace.so'))
assert l.vlfb_debug_set_trace and l.vlfb_fbo_nl_fwd and l.vlfb_version() == 100
print('libvlfb_trace.so ok')
PY
