#!/bin/bash
# Variant build of the product library for experiments: scripts/build_variant.sh NAME "-DFLAG=... ..."
#   -> build/NAME/libxllm_ingest_NAME.so (only sp_encode.cu is recompiled); run with XLLM_INGEST_LIB=<that path>.
set -e
cd "$(dirname "$0")/.."
NAME=$1; FLAGS=$2
make lib >/dev/null
mkdir -p build/$NAME
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
$NVCC -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Iinclude --expt-relaxed-constexpr \
  $FLAGS -c xllm_service_b200/csrc/sp_encode.cu -o build/$NAME/sp_encode.cu.o
OBJS=$(ls build/*.o | grep -v sp_encode.cu.o)
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o build/$NAME/libxllm_ingest_$NAME.so $OBJS build/$NAME/sp_encode.cu.o -lcudart -ldl
echo build/$NAME/libxllm_ingest_$NAME.so
