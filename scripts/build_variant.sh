#!/bin/bash
# build_variant.sh NAME "EXTRA_NVCC_FLAGS": builds futuresdr_b200/variants/libb200sdr_NAME.so for A/B runs
# (select with B2S_LIB=futuresdr_b200/variants/libb200sdr_NAME.so).  *.so is git-ignored.
set -e
cd "$(dirname "$0")/../futuresdr_b200/csrc"
NAME=$1; EXTRA=$2
mkdir -p ../variants build_$NAME
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Xcompiler -ffp-contract=off -ccbin /usr/bin/g++ -I../../include -I. --expt-relaxed-constexpr $EXTRA"
OBJS=""
for f in abi fir_direct fir_tc fir_fft firdes fft apply resamp pfbarb rotator chan synth mavg ring peer; do
  /usr/local/cuda/bin/nvcc $FLAGS -c $f.cu -o build_$NAME/$f.o &
  OBJS="$OBJS build_$NAME/$f.o"
done
wait
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../variants/libb200sdr_$NAME.so $OBJS -lcudart_static -ldl -lrt -lpthread
rm -rf build_$NAME
echo built ../variants/libb200sdr_$NAME.so
