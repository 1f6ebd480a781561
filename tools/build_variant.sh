#!/bin/bash
# Builds a variant of the library with extra -D flags on one translation unit:
#   tools/build_variant.sh <name> <file.cu> "-DDESC_MIN_CTAS=5"
# -> openpano_b200/_variants/<name>.so (git-ignored); use with
#   PANO_B200_LIB=openpano_b200/_variants/<name>.so python tools/ab_value.py
set -e
name=$1; tu=$2; defs=$3
cd "$(dirname "$0")/../openpano_b200/csrc"
NVCC=/usr/local/cuda/bin/nvcc
ARCH="-gencode arch=compute_90a,code=sm_90a"
FLAGS="$ARCH -O3 -lineinfo -std=c++17 --fmad=false -Xcompiler -fPIC -Xcompiler -fvisibility=hidden -Xcompiler -ffp-contract=off"
mkdir -p build/var_$name ../_variants
$NVCC $FLAGS $defs -c $tu -o build/var_$name/${tu%.cu}.o
objs=""
for f in *.cu; do
  if [ "$f" == "$tu" ]; then objs="$objs build/var_$name/${f%.cu}.o"; else objs="$objs build/${f%.cu}.o"; fi
done
$NVCC $ARCH -shared -o ../_variants/$name.so $objs -lcudart_static -lpthread -ldl -lrt
echo built openpano_b200/_variants/$name.so
