#!/usr/bin/env bash
# Test infrastructure only (never imported by the product path).
#
# Compiles the UNMODIFIED reference CUDA extension (csrc/quant_gemv.cu, csrc/dequant.cu,
# csrc/quant_gemv_v2.cu, csrc/ops.cc) from where it lies under /root/reference into
# oracle/_ref/libvptq.so for sm_90a, bypassing the reference's CMake (which needs the legacy
# FindCUDA macros and pins the pre-C++11 ABI; see DESIGN.md "oracle/_ref").
# Outputs go ONLY to oracle/_ref/ (git-ignored build products).
# No reference source is copied into this repository.
set -euo pipefail
REF=${REF:-/root/reference}
HERE=$(cd "$(dirname "$0")" && pwd)
OUT=$HERE/_ref
mkdir -p "$OUT/obj"
if [ ! -d "$REF/csrc" ]; then echo "no reference tree at $REF; keeping prebuilt $OUT" >&2; exit 0; fi
T=$(python -c "import torch,os;print(os.path.dirname(torch.__file__))")
PYINC=$(python -c "import sysconfig;print(sysconfig.get_paths()['include'])")
NVFLAGS=(-I"$REF/csrc" -I"$REF/third_party/cutlass/include" -I"$T/include"
  -I"$T/include/torch/csrc/api/include" -I"$PYINC" -std=c++17 -O3 --use_fast_math -w
  -Xcompiler -fPIC -DTORCH_EXTENSION_NAME=libvptq
  -U__CUDA_NO_HALF_OPERATORS__ -U__CUDA_NO_HALF_CONVERSIONS__ -U__CUDA_NO_HALF2_OPERATORS__
  -U__CUDA_NO_BFLOAT16_OPERATORS__ -U__CUDA_NO_BFLOAT16_CONVERSIONS__
  -U__CUDA_NO_BFLOAT162_OPERATORS__ -U__CUDA_NO_BFLOAT162_CONVERSIONS__
  -gencode arch=compute_90a,code=sm_90a)
pids=()
for tu in quant_gemv quant_gemv_v2 dequant; do
  if [ ! -f "$OUT/obj/$tu.o" ]; then
    ( nvcc "${NVFLAGS[@]}" -c "$REF/csrc/$tu.cu" -o "$OUT/obj/$tu.o.tmp" && mv "$OUT/obj/$tu.o.tmp" "$OUT/obj/$tu.o" ) &
    pids+=($!)
  fi
done
g++ -std=c++17 -O2 -fPIC -w -DTORCH_EXTENSION_NAME=libvptq -I"$T/include" -I"$T/include/torch/csrc/api/include" \
    -I"$PYINC" -I/usr/local/cuda/include -c "$REF/csrc/ops.cc" -o "$OUT/obj/ops.o"
for p in "${pids[@]}"; do wait "$p"; done
g++ -shared -o "$OUT/libvptq.so" "$OUT/obj/ops.o" "$OUT/obj/quant_gemv.o" "$OUT/obj/quant_gemv_v2.o" "$OUT/obj/dequant.o" \
    -L"$T/lib" -ltorch -ltorch_cpu -ltorch_cuda -lc10 -lc10_cuda -ltorch_python \
    -L/usr/local/cuda/lib64 -lcudart -Wl,-rpath,"$T/lib"
echo "built $OUT/libvptq.so"
