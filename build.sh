#!/usr/bin/env bash
# Build the C-ABI shared library for sm_90a (H100), in-tree.
set -euo pipefail
cd "$(dirname "$0")"
OUT=ns2vc_b200/_C
mkdir -p "$OUT"
SRC="ns2vc_b200/csrc/kernels_misc.cu ns2vc_b200/csrc/sampler.cu ns2vc_b200/csrc/gemm_simt.cu ns2vc_b200/csrc/gemm_tc.cu ns2vc_b200/csrc/attention.cu ns2vc_b200/csrc/attention_v2.cu ns2vc_b200/csrc/engine.cu ns2vc_b200/csrc/pre_kernels.cu ns2vc_b200/csrc/pre_engine.cu ns2vc_b200/csrc/frontend.cu ns2vc_b200/csrc/vocoder.cu ns2vc_b200/csrc/content.cu ns2vc_b200/csrc/stream.cu ns2vc_b200/csrc/slicer.cu ns2vc_b200/csrc/loss.cu ns2vc_b200/csrc/kernel_check.cu"
nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -shared \
     ${NVCC_EXTRA:-} -o "$OUT/libns2vc_b200.so" $SRC
echo "built $OUT/libns2vc_b200.so"
