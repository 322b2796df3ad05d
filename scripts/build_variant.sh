#!/bin/bash
# build_variant.sh NAME "EXTRA_NVCC_FLAGS": builds futuresdr_b200/variants/libb200sdr_NAME.so for A/B runs
# (select with B2S_LIB=futuresdr_b200/variants/libb200sdr_NAME.so).  *.so is git-ignored.
set -e
cd "$(dirname "$0")/../futuresdr_b200/csrc"
NAME=$1; EXTRA=$2
mkdir -p ../variants
make -j8 OUT=../variants/libb200sdr_$NAME.so BUILD=build_$NAME EXTRA="$EXTRA"
rm -rf build_$NAME
echo built ../variants/libb200sdr_$NAME.so
