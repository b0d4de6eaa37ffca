#!/bin/bash
# Builds variants/lib_<name>.so: the shipped library with mf.cu recompiled under extra -D switches
# (experiment knobs in csrc/mf.cu: GEN_CHUNK, BWD_MINB, BWD_MINB1, BWD_FAST, BWD_BULK, BWD_OPT_CT=2 for Adagrad).
# Usage: bash profiles/build_variant.sh bulk "-DBWD_BULK=1"   then, on the GPU,   bash profiles/run_variants.sh base bulk
set -e
name=$1; flags=$2
cd "$(dirname "$0")/../spotlight_b200/csrc"
make >/dev/null
mkdir -p ../../variants
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC $flags -c mf.cu -o build/mf_$name.o
objs=$(make -s print-objs)
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../../variants/lib_$name.so ${objs/build\/mf.o/build/mf_$name.o}
echo "built variants/lib_$name.so"
