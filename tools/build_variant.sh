#!/bin/bash
# usage: tools/build_variant.sh <name> <extra nvcc flags...>   -> variants/libbrotli_b200_<name>.so  (A/B experiments)
set -e
cd "$(dirname "$0")/.."
name=$1; shift
mkdir -p variants
for f in bro_encoder bro_capi; do
  nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -I rust-brotli_b200/csrc -I include "$@" \
       -c rust-brotli_b200/csrc/$f.cu -o variants/${f}_$name.o &
done
wait
nvcc -shared -o variants/libbrotli_b200_$name.so variants/bro_encoder_$name.o variants/bro_capi_$name.o -lcudart
rm -f variants/*_$name.o
echo variants/libbrotli_b200_$name.so
