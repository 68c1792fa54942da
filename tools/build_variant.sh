#!/bin/bash
# tools/build_variant.sh NAME SRC [extra nvcc flags]: build rav1e_b200/variants/libb200rdo_NAME.so
# with rav1e_b200/csrc/SRC.cu compiled with the extra flags (kernel A/B experiments; load it with
# B200RDO_LIB=...).  The other objects come from the regular build (build/obj).
set -e
cd "$(dirname "$0")/.."
name=$1; src=$2; shift 2
mkdir -p build/variants rav1e_b200/variants
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -ccbin /usr/bin/g++ \
  --expt-relaxed-constexpr -Iinclude "$@" -c rav1e_b200/csrc/$src.cu -o build/variants/${src}_$name.o
objs=$(ls build/obj/*.o | grep -v "/$src.o")
nvcc -gencode arch=compute_90a,code=sm_90a -shared -ccbin /usr/bin/g++ -o rav1e_b200/variants/libb200rdo_$name.so \
  build/variants/${src}_$name.o $objs -lcudart_static -lpthread -ldl -lrt
echo rav1e_b200/variants/libb200rdo_$name.so
