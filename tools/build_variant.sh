#!/usr/bin/env bash
# Developer aid: libvptq_b200.so with another warps-per-CTA / batch-size configuration of the list kernel, next to
# the product library:  tools/build_variant.sh 24 3  ->  vptq_b200/libvptq_b200_w24b3.so
# (select it with VPTQ_B200_LIB=<path>; the product build is untouched)
set -euo pipefail
W=$1; B=$2
ROOT=$(cd "$(dirname "$0")/.." && pwd)
python -m vptq_b200.build >/dev/null
OBJ=$ROOT/vptq_b200/build
nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -Xcompiler -fvisibility=hidden \
     --expt-relaxed-constexpr -I"$ROOT/include" -DVPTQ_LISTS_WARPS=$W -DVPTQ_LISTS_BATCH=$B \
     -c "$ROOT/vptq_b200/csrc/gemv_lists.cu" -o "$OBJ/gemv_lists_w${W}b${B}.o"
OBJS=$(ls $OBJ/*.o | grep -v "gemv_lists")
nvcc -shared -o "$ROOT/vptq_b200/libvptq_b200_w${W}b${B}.so" $OBJS "$OBJ/gemv_lists_w${W}b${B}.o" \
     -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC -lcudart
echo "$ROOT/vptq_b200/libvptq_b200_w${W}b${B}.so"
